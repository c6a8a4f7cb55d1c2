"""One prefill rank's KV pushed to every decode rank that needs it in one re-paging scatter launch, timed against one launch per
decode rank.

Shapes (fully contiguous OperationalNHD pools with random block tables, tokens [0, 4096)):
  Llama-3-70B  80 layers, K/V, 8 KV heads x 128, bf16, pages 16 -> 64: prefill TP2 rank 0 -> decode TP4 (2 targets, heads
               partitioned), TP1 -> TP8 (8 targets, one head each), TP2 rank 0 -> TP16 (8 targets, each head to 2 of them)
  DeepSeek MLA 61 layers, one 576-wide latent head, bf16, pages 64 -> 64 and 1 -> 64, to 8 decode ranks
  fp8 -> bf16  Llama-3-70B TP2 rank 0 -> TP16 with an fp8 e4m3 prefill cache
Arms, alternating inside each round in one process, each timed with CUDA events around its launches:
  (a) scatter   one kvbm_kernels_paged_repage_scatter launch
  (b) singles   one single-target kvbm_kernels_paged_stage_repage_gather launch per target, back to back on one stream
  (c) fan-out   the paged copy's replicate fan-out (kvbm_kernels_paged_copy_v2, one source table for every destination), the read-once
                ceiling, where pages and formats allow it (MLA 64 -> 64: same page, same format, whole blocks)
Printed: one JSON line per arm with the median of the round medians and their range, the bytes the hand-off needs (every source
byte some target takes, read once, plus every destination byte written) and that over the time as GB/s, the card's name and power
limit read in this run; then the same as a markdown table.  Sampled destination blocks of (a) are compared with
tests/scatter_oracle.py in every run.  Needs a GPU; there is no fallback."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from dynamo_b200 import kernels as K  # noqa: E402
from dynamo_b200.physical import tp_pp_scatter_plan  # noqa: E402
from tests.scatter_oracle import repage_scatter  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--iters", type=int, default=10, help="launches per arm per round")
p.add_argument("--rounds", type=int, default=5)
p.add_argument("--only", default=None, help="comma-separated case names")
p.add_argument("--tokens", type=int, default=4096)
a = p.parse_args(None if __name__ == "__main__" else [])   # imported: the defaults
if not torch.cuda.is_available():
    sys.exit("scatter_bench.py needs a GPU")
dev = torch.device("cuda:0")
torch.cuda.set_device(0)
stream = torch.cuda.current_stream()
sp = int(stream.cuda_stream)
NHD = int(K.KvBlockLayout.OperationalNHD)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "not read")
    return {"name": name, "power_limit": limit}


class Pool:
    """A fully contiguous NHD pool of nb blocks [nl, no, page * nh * row] of random bytes."""

    def __init__(self, nb, nl, no, page, nh, row, seed):
        self.nb, self.nl, self.no, self.page, self.nh, self.row = nb, nl, no, page, nh, row
        self.region = page * nh * row
        self.block = nl * no * self.region
        g = torch.Generator(device=dev).manual_seed(seed)
        self.buf = torch.randint(0, 256, (nb * self.block,), dtype=torch.uint8, device=dev, generator=g)
        base = self.buf.data_ptr()
        self.layer_base = torch.tensor([base + l * no * self.region for l in range(nl)], dtype=torch.int64, device=dev)
        self.desc = K.PagedLayout(self.layer_base.data_ptr(), self.block, self.region, self.region, nl, no, nb)

    def side(self, ids):
        return K.PermuteSide(self.desc, ids.data_ptr(), NHD)

    def host_block(self, b):
        return self.buf[b * self.block:(b + 1) * self.block].cpu().numpy()


# name: (num_kv_heads, layers, outer, head_dim, src_tp, dst_tp, Ps, Pd, cast)
CASES = {
    "llama70b_tp2_to_tp4_rank0": (8, 80, 2, 128, 2, 4, 16, 64, 0),
    "llama70b_tp1_to_tp8": (8, 80, 2, 128, 1, 8, 16, 64, 0),
    "llama70b_tp2_to_tp16_rank0": (8, 80, 2, 128, 2, 16, 16, 64, 0),
    "mla_x8_64_to_64": (1, 61, 1, 576, 1, 8, 64, 64, 0),
    "mla_x8_1_to_64": (1, 61, 1, 576, 1, 8, 1, 64, 0),
    "llama70b_tp2_to_tp16_rank0_fp8_to_bf16": (8, 80, 2, 128, 2, 16, 16, 64, int(K.CastMode.FP8E4M3_TO_BF16)),
}


def run(name, H, nl, no, hd, src_tp, dst_tp, ps, pd, cast):
    se, de = (1, 2) if cast else (2, 2)
    s_row, d_row = hd * se, hd * de
    tb, te = 0, a.tokens
    plan = tp_pp_scatter_plan(H, nl, src_tp, 1, dst_tp, 1, 0)
    ranks = sorted({w.dst_rank for w in plan})
    src_nh, dst_nh = max(1, H // src_tp), max(1, H // dst_tp)
    ns, nd = -(-te // ps), -(-te // pd)
    src = Pool(ns + 4, nl, no, ps, src_nh, s_row, 1)
    dsts = [Pool(nd + 4, nl, no, pd, dst_nh, d_row, 2 + i) for i in range(len(ranks))]
    rng = np.random.default_rng(3)
    sids = rng.permutation(src.nb)[:ns].astype(np.int32)
    dids = [rng.permutation(d.nb)[:nd].astype(np.int32) for d in dsts]
    sids_t = torch.from_numpy(sids).to(dev)
    dids_t = [torch.from_numpy(x).to(dev) for x in dids]
    windows = [(ranks.index(w.dst_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
               for w in plan]
    targets = [K.ScatterTarget(dsts[t].side(dids_t[t]), dst_nh, sb, db, k, sl, dl, c, None) for t, sl, dl, c, sb, db, k in windows]
    covered = len({h for w in windows for h in range(w[4], w[4] + w[6])})
    moved = (te - tb) * nl * no * (covered * s_row + sum(w[6] for w in windows) * d_row)

    def k_scatter():
        K.check(K.paged_repage_scatter(src.side(sids_t), src_nh, ps, targets, pd, tb, te, 0, nl, s_row, cast, stream=sp), "scatter")

    def k_singles():
        for t, sl, dl, c, sb, db, k in windows:
            one = [K.StageSource(K.PermuteSource(src.side(sids_t), src_nh, sb, db, k), sl, dl, c)]
            K.check(K.paged_stage_repage_gather(one, ps, dsts[t].side(dids_t[t]), dst_nh, pd, tb, te, dl, dl + c, s_row, cast, stream=sp), "single")

    arms = {"scatter": k_scatter, "singles": k_singles}
    if ps == pd and not cast and src_nh == dst_nh and len({w[4:] for w in windows}) == 1:
        ws = torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device=dev)
        fan = [K.PagedDst(d.desc, sids_t.data_ptr(), x.data_ptr(), 0, 0) for d, x in zip(dsts, dids_t)]
        opts = K.PagedCopyOpts(sync_workspace=ws.data_ptr())

        def k_fanout():
            K.check(K.paged_copy(src.desc, fan, ns, 0, nl, 0, opts, sp), "fan-out")
        arms["fanout"] = k_fanout

    # (a) against the oracle on sampled destination blocks of the first and last target, from destinations of known bytes
    for d in dsts:
        d.buf.fill_(0x5A)
    k_scatter()
    torch.cuda.synchronize()
    before = np.full(dsts[0].block, 0x5A, dtype=np.uint8)
    for w in sorted({0, len(windows) - 1}):
        t = windows[w][0]
        for j in sorted({0, nd - 1}):
            lo, hi = max(tb, j * pd), min(te, (j + 1) * pd)
            s_blocks = [src.host_block(b) for b in sids[lo // ps:-(-hi // ps)]]
            pools = [np.stack([before])]
            repage_scatter((s_blocks, NHD, src_nh, nl), [(0, [0], NHD, dst_nh, nl, windows[w][1:])], pools, no, ps, pd, s_row, lo, hi, cast)
            assert np.array_equal(dsts[t].host_block(dids[t][j]), pools[0][0]), (name, "target", w, "block", j)

    def events(fn):
        ts = []
        for _ in range(a.iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            fn()
            e1.record(stream)
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return statistics.median(ts)

    for fn in arms.values():
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    rounds = {k: [] for k in arms}
    for _ in range(a.rounds):              # the arms alternate within every round
        for k, fn in arms.items():
            rounds[k].append(events(fn))
    torch.cuda.synchronize()
    info = card()
    rows = []
    for k in arms:
        ms = statistics.median(rounds[k])
        rows.append({"case": name, "targets": len(windows), "pairs": sum(w[6] for w in windows), "covered_heads": covered, "src_page": ps,
                     "dst_page": pd, "cast": "fp8-to-bf16" if cast else "none", "tokens": te - tb, "arm": k, "ms": round(ms, 4),
                     "ms_range": [round(min(rounds[k]), 4), round(max(rounds[k]), 4)], "GBps": round(moved / ms / 1e6, 1), "bytes": moved,
                     "timed_as": "CUDA events, median of %d alternated rounds of median-of-%d" % (a.rounds, a.iters), "card": info})
        print(json.dumps(rows[-1]), flush=True)
    del src, dsts
    torch.cuda.empty_cache()
    return rows


def main():
    rows = []
    for name, args in CASES.items():
        if not a.only or name in a.only.split(","):
            rows += run(name, *args)
    info = card()
    print(f"\n{info['name']}, power limit {info['power_limit']}; ms = median of {a.rounds} round medians (min-max over rounds); "
          "GB/s = source bytes read once + destination bytes written, over the time\n")
    print("| case | targets | pairs | MiB | scatter ms | GB/s | n singles ms | GB/s | fan-out ms | GB/s |")
    print("|---|---:|---:|---:|---:|---:|---:|---:|---:|---:|")
    for name in dict.fromkeys(r["case"] for r in rows):
        g = {r["arm"]: r for r in rows if r["case"] == name}
        cell = lambda r: f"{r['ms']:.3f} ({r['ms_range'][0]:.3f}-{r['ms_range'][1]:.3f}) | {r['GBps']:.0f}" if r else "not run | -"  # noqa: E731
        s = g["scatter"]
        print(f"| {name} | {s['targets']} | {s['pairs']} | {s['bytes'] / 2**20:.0f} | {cell(s)} | {cell(g['singles'])} | {cell(g.get('fanout'))} |")


if __name__ == "__main__":
    main()

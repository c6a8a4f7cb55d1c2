"""A batch of sequences in one re-paging launch, timed against the same sequences one launch each.

Llama-3-8B KV geometry (32 layers, K/V, 8 heads x 128) on fully contiguous NHD pools with random block tables, bf16 -> bf16 and
fp8 -> bf16, pages Ps:Pd of 16:64, 1:16 and 16:16, every sequence starting inside a block (a prefix-cache hit).  Batches of
8 x 2048, 32 x 512 and 128 x 128 tokens and one mixed batch.  Arms, alternating inside each of five rounds in one process:
  (a) batch    one kvbm_kernels_paged_stage_repage_gather_batch launch / one TransferManager.execute_repage_batch call
  (b) singles  n kvbm_kernels_paged_stage_repage_gather launches back to back on one stream / n execute_stage_repage_gather calls
  (c) ceiling  one single-sequence launch / call of the same total tokens
each through the kernel ABI, timed with CUDA events, and through the manager, timed with a host clock that ends when the (last)
notification's wait returns.  (b) and (c) are one full-window source, so they run kvbm_paged_repage_kernel; a batch always runs
the gather kernel.  Printed: one JSON line per arm with the median of the round medians and their range, bytes read + written
from the shapes, and the card's name and power limit read in this run; then the same as a markdown table.  Sampled destination
blocks of (a) are compared with tests/stage_repage_oracle.py in every run.  Needs a GPU; there is no fallback."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from dynamo_b200 import kernels as K  # noqa: E402
from dynamo_b200.physical import LayoutConfig, ShardWindow, StorageKind, TransferManager, TransferOptions  # noqa: E402
from tests.stage_repage_oracle import stage_repage_gather  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--iters", type=int, default=10, help="launches per arm per round")
p.add_argument("--rounds", type=int, default=5)
p.add_argument("--only", default=None, help="comma-separated batch names (8x2048, 32x512, 128x128, mixed)")
p.add_argument("--pages", default="16:64,1:16,16:16")
p.add_argument("--casts", default="none,fp8-to-bf16")
a = p.parse_args()
if not torch.cuda.is_available():
    sys.exit("repage_batch_bench.py needs a GPU")
dev = torch.device("cuda:0")
torch.cuda.set_device(0)
stream = torch.cuda.current_stream()
sp = int(stream.cuda_stream)
NL, NO, NH, HD = 32, 2, 8, 128
NHD = int(K.KvBlockLayout.OperationalNHD)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "not read")
    return {"name": name, "power_limit": limit}


def batches():
    rng = np.random.default_rng(7)
    mixed = [int(x) for x in rng.choice([1, 17, 128, 300, 512, 1000, 2048, 4000], 48)]
    out = {"8x2048": [2048] * 8, "32x512": [512] * 32, "128x128": [128] * 128, "mixed": mixed}
    return {k: v for k, v in out.items() if not a.only or k in a.only.split(",")}


class Pool:
    """A fully contiguous pool of nb blocks [NL, NO, page * NH * HD * elem] of random bytes."""

    def __init__(self, nb, page, elem, seed):
        self.nb, self.page, self.elem = nb, page, elem
        self.region = page * NH * HD * elem
        self.block = NL * NO * self.region
        g = torch.Generator(device=dev).manual_seed(seed)
        self.buf = torch.randint(0, 256, (nb * self.block,), dtype=torch.uint8, device=dev, generator=g)
        base = self.buf.data_ptr()
        self.layer_base = torch.tensor([base + l * NO * self.region for l in range(NL)], dtype=torch.int64, device=dev)
        self.desc = K.PagedLayout(self.layer_base.data_ptr(), self.block, self.region, self.region, NL, NO, nb)

    def side(self, ids):
        return K.PermuteSide(self.desc, ids.data_ptr(), NHD)

    def host_block(self, b):
        return self.buf[b * self.block:(b + 1) * self.block].cpu().numpy()

    def register(self, mgr):
        cfg = LayoutConfig(self.nb, NL, NO, self.page, NH * HD, dtype_width_bytes=self.elem, num_heads=NH, allow_fp8=self.elem == 1)
        h = mgr.register_fully_contiguous(cfg, self.buf.data_ptr(), self.buf.numel(), StorageKind.Device, 0)
        mgr.set_kv_block_layout(h, K.KvBlockLayout.OperationalNHD)
        return h


def blocks(tb, te, page):
    return -(-te // page) - tb // page


def run(name, lengths, ps, pd, cast):
    se, de = (1, 2) if cast else (2, 2)
    s_row = HD * se
    big = max(ps, pd)
    seqs = [(5 + (11 * i) % (big - 1 if big > 6 else 1), 0) for i in range(len(lengths))]     # starts inside a block of the larger page
    seqs = [(tb, tb + n) for (tb, _), n in zip(seqs, lengths)]
    total = sum(lengths)
    whole = (5, 5 + total)                                                                     # the ceiling's one sequence
    n_s, n_d = [blocks(*q, ps) for q in seqs], [blocks(*q, pd) for q in seqs]
    src = Pool(max(sum(n_s), blocks(*whole, ps)) + 8, ps, se, 1)
    dst = Pool(max(sum(n_d), blocks(*whole, pd)) + 8, pd, de, 2)
    rng = np.random.default_rng(3)
    s_perm, d_perm = rng.permutation(src.nb).astype(np.int64), rng.permutation(dst.nb).astype(np.int64)
    cut = lambda perm, counts: np.split(perm[:sum(counts)], np.cumsum(counts)[:-1])  # noqa: E731
    sids, dids = cut(s_perm, n_s), cut(d_perm, n_d)
    w_sids, w_dids = s_perm[:blocks(*whole, ps)], d_perm[:blocks(*whole, pd)]
    i32 = lambda x: torch.from_numpy(np.ascontiguousarray(x, dtype=np.int32)).to(dev)  # noqa: E731
    units_np, ns, nd = K.repage_batch_units(seqs, ps, pd)
    units = torch.from_numpy(units_np.view(np.int32)).to(dev)
    cat_s, cat_d = i32(np.concatenate(sids)), i32(np.concatenate(dids))
    one_s, one_d = [i32(x) for x in sids], [i32(x) for x in dids]
    ws_t, wd_t = i32(w_sids), i32(w_dids)
    stage = lambda ids: [K.StageSource(K.PermuteSource(src.side(ids), NH, 0, 0, NH), 0, 0, NL)]  # noqa: E731
    moved = total * NL * NO * NH * HD * (se + de)

    def k_batch():
        K.check(K.paged_stage_repage_gather_batch(stage(cat_s), ps, dst.side(cat_d), NH, pd, seqs, units.data_ptr(), len(units_np), 0, NL,
                                                  s_row, cast, stream=sp), "batch")

    def k_singles():
        for (tb, te), s, d in zip(seqs, one_s, one_d):
            K.check(K.paged_stage_repage_gather(stage(s), ps, dst.side(d), NH, pd, tb, te, 0, NL, s_row, cast, stream=sp), "single")

    def k_ceiling():
        K.check(K.paged_stage_repage_gather(stage(ws_t), ps, dst.side(wd_t), NH, pd, whole[0], whole[1], 0, NL, s_row, cast, stream=sp), "one")

    mgr = TransferManager(device=0, worker_id=21)
    hs, hd_ = src.register(mgr), dst.register(mgr)
    plan = [ShardWindow(0, 0, 0, NL, 0, 0, NH)]
    opts = TransferOptions(cast_mode=K.CastMode(cast))
    reqs = [(range(tb, te), {0: s}, d) for (tb, te), s, d in zip(seqs, sids, dids)]

    def m_batch():
        mgr.execute_repage_batch({0: hs}, hd_, reqs, plan, opts).wait(60.0)

    def m_singles():
        notes = [mgr.execute_stage_repage_gather({0: (hs, src_ids[0])}, hd_, d, plan, t, opts) for t, src_ids, d in reqs]
        for n in notes:
            n.wait(60.0)

    def m_ceiling():
        mgr.execute_stage_repage_gather({0: (hs, w_sids)}, hd_, w_dids, plan, range(*whole), opts).wait(60.0)

    # (a) against the oracle on sampled destination blocks, from a destination of known bytes
    dst.buf.fill_(0x5A)
    k_batch()
    torch.cuda.synchronize()
    before = np.full(dst.block, 0x5A, dtype=np.uint8)
    windows = [(0, 0, 0, NL, 0, 0, NH)]
    for i in sorted({0, len(seqs) // 2, len(seqs) - 1}):
        tb, te = seqs[i]
        for j in sorted({0, n_d[i] - 1}):
            lo, hi = max(tb, (tb // pd + j) * pd), min(te, (tb // pd + j + 1) * pd)
            s_blocks = [src.host_block(b) for b in sids[i][lo // ps - tb // ps:-(-hi // ps) - tb // ps]]
            want = stage_repage_gather([(s_blocks, NHD, NH, NL)], windows, [before], NHD, NH, NL, NO, ps, pd, s_row, lo, hi, cast)[0]
            assert np.array_equal(dst.host_block(dids[i][j]), want), (name, ps, pd, cast, "sequence", i, "block", j)

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

    def host(fn):
        ts = []
        for _ in range(a.iters):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        return statistics.median(ts)

    arms = {"kernel_batch": (k_batch, events), "kernel_singles": (k_singles, events), "kernel_ceiling": (k_ceiling, events),
            "manager_batch": (m_batch, host), "manager_singles": (m_singles, host), "manager_ceiling": (m_ceiling, host)}
    for fn, _ in arms.values():
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    rounds = {k: [] for k in arms}
    for _ in range(a.rounds):              # the arms alternate within every round
        for k, (fn, clock) in arms.items():
            rounds[k].append(clock(fn))
    torch.cuda.synchronize()
    mgr.close()
    info = card()
    rows = []
    for k in arms:
        ms = statistics.median(rounds[k])
        rows.append({"batch": name, "sequences": len(seqs), "tokens": total, "src_page": ps, "dst_page": pd, "cast": "fp8-to-bf16" if cast else "none",
                     "arm": k, "ms": round(ms, 4), "ms_range": [round(min(rounds[k]), 4), round(max(rounds[k]), 4)],
                     "GBps": round(moved / ms / 1e6, 1), "bytes": moved, "units": len(units_np),
                     "timed_as": ("CUDA events" if k.startswith("kernel") else "host clock to the notification's wait") +
                                 ", median of %d alternated rounds of median-of-%d" % (a.rounds, a.iters), "card": info})
        print(json.dumps(rows[-1]), flush=True)
    del src, dst
    torch.cuda.empty_cache()
    return rows


def main():
    rows = []
    for cast_name in a.casts.split(","):
        cast = int(K.CastMode.FP8E4M3_TO_BF16) if cast_name == "fp8-to-bf16" else 0
        for pages in a.pages.split(","):
            ps, pd = (int(x) for x in pages.split(":"))
            for name, lengths in batches().items():
                rows += run(name, lengths, ps, pd, cast)
    info = card()
    print(f"\n{info['name']}, power limit {info['power_limit']}; ms = median of {a.rounds} round medians (min-max over rounds)\n")
    print("| cast | Ps:Pd | batch | MiB | kernel: batch | n singles | ceiling | manager: batch | n singles | ceiling |")
    print("|---|---|---|---:|---:|---:|---:|---:|---:|---:|")
    key = lambda r: (r["cast"], r["src_page"], r["dst_page"], r["batch"])  # noqa: E731
    for k in dict.fromkeys(key(r) for r in rows):
        g = {r["arm"]: r for r in rows if key(r) == k}
        cell = lambda r: f"{r['ms']:.3f} ({r['ms_range'][0]:.3f}-{r['ms_range'][1]:.3f})"  # noqa: E731
        first = g["kernel_batch"]
        print(f"| {k[0]} | {k[1]}:{k[2]} | {k[3]} ({first['sequences']} seq, {first['tokens']} tok) | {first['bytes'] / 2**20:.0f} | " +
              " | ".join(cell(g[x]) for x in ("kernel_batch", "kernel_singles", "kernel_ceiling", "manager_batch", "manager_singles",
                                              "manager_ceiling")) + " |")


main()

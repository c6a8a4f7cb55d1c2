"""A prefill batch's sequences pushed to every decode rank in one batch re-paging scatter launch, timed against one scatter launch
per sequence.

Shapes: scatter_bench.py's Llama-3-70B prefill TP2 rank 0 -> decode TP16 and TP1 -> TP8 (80 layers, K/V, 8 KV heads x 128, pages
16 -> 64), bf16 and fp8 e4m3 -> bf16; fully contiguous OperationalNHD pools with random block tables.
Batches: 8 x 2048, 32 x 512 and 128 x 128 tokens, and a mixed batch of 12 sequences of 1 to 4000 tokens; every sequence starts
inside a 64-token block (its own prefix-cache hit).
Arms, alternated inside each of --rounds rounds in one process, each timed with CUDA events around its launches (median of --iters):
  batch       one kvbm_kernels_paged_repage_scatter_batch launch
  singles     one kvbm_kernels_paged_repage_scatter launch per sequence, back to back on one stream
  one_range   one kvbm_kernels_paged_repage_scatter of the batch's total tokens as one range (the ceiling: no per-sequence edges)
  mgr_batch   TransferManager.execute_repage_scatter_batch, host call to completion (host clock around call and wait)
  mgr_singles one TransferManager.execute_repage_scatter per sequence, then a wait for the last
Streamed tail (bf16 shapes; --no-tail skips it): a producer stream emulates the prefill with a --layer-us busy kernel per layer and
then the layer's ready flag, on the same GPU.  The streamed batch (spinning, default grid) and n streamed scatters (spinning, default
grid, back to back on one stream) are enqueued before the producer; the time from the producer's last flag to the end of the
transfer is the exposed tail.
Sampled destination blocks of the batch are compared with tests/scatter_oracle.py in every run, and every arm's whole destination
pools with the batch's.  One JSON line per arm with the card's name and power limit read in this run, then a markdown table.
Needs a GPU; there is no fallback."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
import scatter_bench as SB  # noqa: E402
import transform_stream_bench as TB  # noqa: E402
from dynamo_b200 import kernels as K  # noqa: E402
from dynamo_b200.physical import LayoutConfig, ScatterWindow, StorageKind, TransferManager, TransferOptions, tp_pp_scatter_plan  # noqa: E402
from tests.scatter_oracle import repage_scatter  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--iters", type=int, default=5, help="launches per arm per round")
p.add_argument("--rounds", type=int, default=5)
p.add_argument("--only", default=None, help="comma-separated shape names")
p.add_argument("--batches", default=None, help="comma-separated batch names")
p.add_argument("--layer-us", type=float, default=100.0, help="busy time of one emulated prefill layer (streamed tail)")
p.add_argument("--no-tail", action="store_true")
a = p.parse_args()
dev = SB.dev
NHD = SB.NHD
SHAPES = ["llama70b_tp2_to_tp16_rank0", "llama70b_tp1_to_tp8", "llama70b_tp2_to_tp16_rank0_fp8_to_bf16"]
SB.CASES["llama70b_tp1_to_tp8_fp8_to_bf16"] = SB.CASES["llama70b_tp1_to_tp8"][:-1] + (int(K.CastMode.FP8E4M3_TO_BF16),)
SHAPES.append("llama70b_tp1_to_tp8_fp8_to_bf16")


def _batch(n, length):
    return [(1 + 7 * i, 1 + 7 * i + length) for i in range(n)]


def _mixed():
    rng = np.random.default_rng(7)
    lens = [1, 4000] + [int(x) for x in rng.integers(1, 4001, 10)]
    return [(int(tb), int(tb) + n) for tb, n in zip(rng.integers(1, 64, len(lens)) | 1, lens)]


BATCHES = {"8x2048": _batch(8, 2048), "32x512": _batch(32, 512), "128x128": _batch(128, 128), "mixed": _mixed()}


def tlen(tb, te, page):
    return 0 if tb == te else -(-te // page) - tb // page


def run(name, batch, H, nl, no, hd, src_tp, dst_tp, ps, pd, cast):
    seqs = BATCHES[batch]
    se, de = (1, 2) if cast else (2, 2)
    s_row, d_row = hd * se, hd * de
    plan = tp_pp_scatter_plan(H, nl, src_tp, 1, dst_tp, 1, 0)
    ranks = sorted({w.dst_rank for w in plan})
    src_nh, dst_nh = max(1, H // src_tp), max(1, H // dst_tp)
    total = sum(te - tb for tb, te in seqs)
    ns, nd = sum(tlen(tb, te, ps) for tb, te in seqs), sum(tlen(tb, te, pd) for tb, te in seqs)
    src = SB.Pool(max(ns, -(-total // ps)) + 4, nl, no, ps, src_nh, s_row, 1)
    dsts = [SB.Pool(max(nd, -(-total // pd)) + 4, nl, no, pd, dst_nh, d_row, 2 + i) for i in range(len(ranks))]
    init = [d.buf.clone() for d in dsts]
    rng = np.random.default_rng(3)
    sids = rng.permutation(src.nb)[:ns].astype(np.int32)
    dids = [rng.permutation(d.nb)[:nd].astype(np.int32) for d in dsts]
    one_s = rng.permutation(src.nb)[:-(-total // ps)].astype(np.int32)
    one_d = [rng.permutation(d.nb)[:-(-total // pd)].astype(np.int32) for d in dsts]
    as_t = lambda x: torch.from_numpy(x).to(dev)  # noqa: E731
    sids_t, dids_t, one_s_t, one_d_t = as_t(sids), [as_t(x) for x in dids], as_t(one_s), [as_t(x) for x in one_d]
    units, _, _ = K.repage_batch_units(seqs, ps, pd)
    units_t = as_t(np.ascontiguousarray(units).view(np.int32).reshape(-1))
    windows = [(ranks.index(w.dst_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
               for w in plan]

    def targets(ids):
        return [K.ScatterTarget(dsts[t].side(ids[t]), dst_nh, sb, db, k, sl, dl, c, None) for t, sl, dl, c, sb, db, k in windows]

    stream = torch.cuda.current_stream()
    sp = int(stream.cuda_stream)
    offs, so, do = [], 0, 0   # per sequence: its slices of the concatenated tables
    for tb, te in seqs:
        offs.append((so, do, tlen(tb, te, ps), tlen(tb, te, pd)))
        so, do = so + offs[-1][2], do + offs[-1][3]
    single_args = [(sids_t[o[0]:o[0] + o[2]], targets([d[o[1]:o[1] + o[3]] for d in dids_t]), tb, te) for (tb, te), o in zip(seqs, offs) if o[2]]
    tg_batch, tg_one = targets(dids_t), targets(one_d_t)

    def k_batch():
        K.check(K.paged_repage_scatter_batch(src.side(sids_t), src_nh, ps, tg_batch, pd, seqs, units_t.data_ptr(), len(units), 0, nl, s_row, cast,
                                             stream=sp), "batch")

    def k_singles():
        for s_t, tg, tb, te in single_args:
            K.check(K.paged_repage_scatter(src.side(s_t), src_nh, ps, tg, pd, tb, te, 0, nl, s_row, cast, stream=sp), "single")

    def k_one():
        K.check(K.paged_repage_scatter(src.side(one_s_t), src_nh, ps, tg_one, pd, 0, total, 0, nl, s_row, cast, stream=sp), "one range")

    mgr = TransferManager(device=0, worker_id=61)
    reg = lambda pool, nh, w: mgr.register_fully_contiguous(  # noqa: E731
        LayoutConfig(pool.nb, nl, no, pool.page, nh * hd, dtype_width_bytes=w, num_heads=nh, allow_fp8=w == 1), pool.buf.data_ptr(),
        pool.buf.numel(),
        StorageKind.Device, 0)
    sh = reg(src, src_nh, se)
    dhs = [reg(d, dst_nh, de) for d in dsts]
    for h in [sh] + dhs:
        mgr.set_kv_block_layout(h, K.KvBlockLayout.OperationalNHD)
    mplan = [ScatterWindow(*w) for w in windows]
    reqs = [(range(tb, te), sids[o[0]:o[0] + o[2]].astype(np.int64), [d[o[1]:o[1] + o[3]].astype(np.int64) for d in dids])
            for (tb, te), o in zip(seqs, offs)]
    opts = TransferOptions(cast_mode=cast)

    def m_batch():
        mgr.execute_repage_scatter_batch(sh, dhs, reqs, mplan, opts).wait(60.0)

    def m_singles():
        note = None
        for tokens, s, d in reqs:
            note = mgr.execute_repage_scatter(sh, s, dhs, d, mplan, tokens, opts)
        note.wait(60.0)

    # the batch against the oracle on sampled blocks (first and last sequence, first and last target), then as the reference
    k_batch()
    torch.cuda.synchronize()
    for i in sorted({0, len(seqs) - 1}):
        tb, te = seqs[i]
        so, do, a_n, b_n = offs[i]
        for w in sorted({0, len(windows) - 1}):
            t = windows[w][0]
            for j in sorted({0, b_n - 1}):
                first = (tb // pd + j) * pd
                lo, hi = max(tb, first), min(te, first + pd)
                s_blocks = [src.host_block(int(b)) for b in sids[so + lo // ps - tb // ps:so + -(-hi // ps) - tb // ps]]
                blk = int(dids[t][do + j])   # a Python int: block offsets pass 2^31 bytes
                pools = [np.stack([init[t][blk * dsts[t].block:(blk + 1) * dsts[t].block].cpu().numpy()])]
                repage_scatter((s_blocks, NHD, src_nh, nl), [(0, [0], NHD, dst_nh, nl, windows[w][1:])], pools, no, ps, pd, s_row, lo, hi, cast)
                assert np.array_equal(dsts[t].host_block(blk), pools[0][0]), (name, batch, "seq", i, "target", w, "block", j)
    reference = [d.buf.clone() for d in dsts]

    def check(arm):
        torch.cuda.synchronize()
        for d, ref, x in zip(dsts, reference, init):
            assert torch.equal(d.buf, ref), f"{name} {batch} {arm}: destination pools differ from the batch's"
            d.buf.copy_(x)
        torch.cuda.synchronize()

    def reset():
        torch.cuda.synchronize()
        for d, x in zip(dsts, init):
            d.buf.copy_(x)
        torch.cuda.synchronize()

    arms = {"batch": k_batch, "singles": k_singles, "one_range": k_one, "mgr_batch": m_batch, "mgr_singles": m_singles}
    for k, fn in arms.items():   # warm-up; every arm but the one-range ceiling (its own tables) leaves the batch's bytes
        fn()
        check(k) if k != "one_range" else reset()

    def timed(k, fn):
        ts = []
        for _ in range(a.iters):
            if k.startswith("mgr"):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                ts.append((time.perf_counter() - t0) * 1e3)
            else:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                fn()
                e1.record(stream)
                e1.synchronize()
                ts.append(e0.elapsed_time(e1))
        return statistics.median(ts)

    rounds = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, fn in arms.items():
            rounds[k].append(timed(k, fn))
    info = SB.card()
    moved = total * nl * no * (len({h for w in windows for h in range(w[4], w[4] + w[6])}) * s_row + sum(w[6] for w in windows) * d_row)
    base = {"bench": "scatter_batch", "case": name, "batch": batch, "seqs": len(seqs), "tokens": total, "targets": len(windows),
            "cast": "fp8-to-bf16" if cast else "none", "bytes": moved, "rounds": a.rounds, "iters": a.iters, "gpu": info["name"],
            "power_limit": info["power_limit"]}
    rows = []
    for k in arms:
        ms = statistics.median(rounds[k])
        rows.append({**base, "arm": k, "ms": round(ms, 4), "ms_range": [round(min(rounds[k]), 4), round(max(rounds[k]), 4)],
                     "GBps": round(moved / ms / 1e6, 1)})
        print(json.dumps(rows[-1]), flush=True)

    if not a.no_tail and not cast:
        reset()   # the one-range arm wrote blocks of its own tables
        ready = torch.zeros(nl, dtype=torch.int32, device=dev)
        completion = torch.zeros(1, dtype=torch.int32, device=dev)
        wss = [torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device=dev) for _ in range(len(single_args) + 1)]
        epoch = [0]
        sstream = torch.cuda.Stream()
        ssp = int(sstream.cuda_stream)

        def desc(ws):
            st = K.PermuteStream()
            st.layer_ready_flags[0] = ready.data_ptr()
            st.epoch = epoch[0]
            st.sync_workspace = ws.data_ptr()
            st.gate_mode = K.GATE_SPIN
            st.completion_flag = completion.data_ptr()
            st.completion_value = epoch[0]
            return st

        def s_batch():
            K.check(K.paged_repage_scatter_batch_streamed(src.side(sids_t), src_nh, ps, tg_batch, pd, seqs, units_t.data_ptr(), len(units), 0, nl,
                                                          s_row, cast, None, desc(wss[0]), ssp), "streamed batch")

        def s_singles():
            for i, (s_t, tg, tb, te) in enumerate(single_args):
                K.check(K.paged_repage_scatter_streamed(src.side(s_t), src_nh, ps, tg, pd, tb, te, 0, nl, s_row, cast, None, desc(wss[1 + i]),
                                                        ssp), "streamed single")

        prod = torch.cuda.Stream()
        cycles = TB.layer_cycles(a.layer_us)
        with torch.cuda.stream(prod):
            torch.cuda._sleep(100)
            K.check(K.set_flags(ready.data_ptr(), 0, 1, 0, int(prod.cuda_stream)), "set_flags")
        torch.cuda.synchronize()
        tails = {"streamed_batch": s_batch, "n_streamed_singles": s_singles}
        times = {k: [] for k in tails}
        for it in range(a.iters + 2):
            for k, fn in tails.items():
                epoch[0] += 1
                torch.cuda.synchronize()
                last, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                fn()
                TB.emulate_prefill(prod, [ready.data_ptr()], nl, epoch[0], cycles)
                last.record(prod)
                end.record(sstream)
                end.synchronize()
                if it >= 2:
                    times[k].append(last.elapsed_time(end) * 1e3)
                if it == 0:
                    check(k)
        for k in tails:
            rows.append({**base, "arm": k, "mode": "tail", "exposed_tail_us": round(statistics.median(times[k]), 1),
                         "tail_range_us": [round(min(times[k]), 1), round(max(times[k]), 1)], "layer_us": a.layer_us})
            print(json.dumps(rows[-1]), flush=True)
    mgr.close()
    del src, dsts
    torch.cuda.empty_cache()
    return rows


def main():
    rows = []
    for nm in SHAPES:
        if a.only and nm not in a.only.split(","):
            continue
        for b in BATCHES:
            if not a.batches or b in a.batches.split(","):
                rows += run(nm, b, *SB.CASES[nm])
    info = SB.card()
    print(f"\n{info['name']}, power limit {info['power_limit']}; ms = median of {a.rounds} round medians (min-max over rounds)\n")
    print("| shape | batch | batch ms | n singles ms | one range ms | mgr batch ms | mgr n singles ms | streamed batch tail us | n streamed tail us |")
    print("|---|---|---:|---:|---:|---:|---:|---:|---:|")
    for nm, b in dict.fromkeys((r["case"], r["batch"]) for r in rows):
        g = {r["arm"]: r for r in rows if r["case"] == nm and r["batch"] == b}
        ms = lambda k: f"{g[k]['ms']:.3f} ({g[k]['ms_range'][0]:.3f}-{g[k]['ms_range'][1]:.3f})"  # noqa: E731
        tail = lambda k: f"{g[k]['exposed_tail_us']:.0f} ({g[k]['tail_range_us'][0]:.0f}-{g[k]['tail_range_us'][1]:.0f})" if k in g else "-"  # noqa: E731
        print(f"| {nm} | {b} | {ms('batch')} | {ms('singles')} | {ms('one_range')} | {ms('mgr_batch')} | {ms('mgr_singles')} | "
              f"{tail('streamed_batch')} | {tail('n_streamed_singles')} |")


if __name__ == "__main__":
    main()

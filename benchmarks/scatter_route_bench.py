"""A prefill batch whose sequences belong to different decode workers, pushed in one routed re-paging scatter launch, timed against one
batch scatter per worker and one scatter per sequence.

Shapes (every pool on one GPU, fully contiguous OperationalNHD, random block tables, every sequence starting inside a block):
  llama70b_tp4_to_4x_tp4        Llama-3-70B (80 layers, K/V, 8 KV heads x 128) prefill TP4 rank 0 -> 4 decode workers at TP4: 4 targets
  llama70b_tp2_to_4x_tp4        prefill TP2 rank 0 -> 4 decode workers at TP4: 8 targets, bf16, and fp8 e4m3 -> bf16
  mla_to_8_dp                   DeepSeek MLA (61 layers, 1 x 576) to 8 decode DP ranks, each owning whole sequences: 8 targets
Pages 16 -> 64 (64 -> 64 for MLA).  Batches 32 x 512, 128 x 128 and a mixed batch of 12 sequences of 1 to 4000 tokens; each sequence
is routed to one worker (round robin over a shuffled order).
Arms, alternated inside each of --rounds rounds in one process, CUDA events around each arm's launches (median of --iters):
  routed        one kvbm_kernels_paged_repage_scatter_routed launch
  per_worker    one kvbm_kernels_paged_repage_scatter_batch per worker over its sequences and targets, back to back on one stream
  singles       one kvbm_kernels_paged_repage_scatter per sequence to its worker's targets
  routed_all    the routed launch with every mask all ones ...
  batch_all     ... against kvbm_kernels_paged_repage_scatter_batch with every sequence to every target: the cost of routing itself
  mgr_routed    TransferManager.execute_repage_scatter_routed, host clock around call and wait
  mgr_per_worker one TransferManager.execute_repage_scatter_batch per worker, then a wait for the last
Streamed tail (--no-tail skips it): a producer stream emulates the prefill with a --layer-us busy kernel per layer and then the
layer's ready flag, on the same GPU.  The routed streamed launch and one streamed batch per worker (back to back on ONE stream) are
enqueued before the producer, in the spinning form at its default grid and in the stream-wait form; the time from the producer's
last flag to the end of the transfer is the exposed tail.
Every arm's whole destination pools are compared with the routed launch's (the all-ones pair with each other), and sampled
destination blocks of the routed launch with tests/scatter_oracle.py.  One JSON line per arm with the card's name and power limit
read in this run, then a markdown table.  Needs a GPU; there is no fallback."""
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
from dynamo_b200.physical import (LayoutConfig, ScatterWindow, StorageKind, TransferManager, TransferOptions, tile_scatter_plan,  # noqa: E402
                                  tp_pp_scatter_plan)
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
FP8 = int(K.CastMode.FP8E4M3_TO_BF16)
# name: (num_kv_heads, layers, outer, head_dim, src_tp, dst_tp, workers, Ps, Pd, cast)
SHAPES = {
    "llama70b_tp4_to_4x_tp4": (8, 80, 2, 128, 4, 4, 4, 16, 64, 0),
    "llama70b_tp2_to_4x_tp4": (8, 80, 2, 128, 2, 4, 4, 16, 64, 0),
    "llama70b_tp2_to_4x_tp4_fp8_to_bf16": (8, 80, 2, 128, 2, 4, 4, 16, 64, FP8),
    "mla_to_8_dp": (1, 61, 1, 576, 1, 1, 8, 64, 64, 0),
}


def _batch(n, length):
    return [(1 + 7 * i, 1 + 7 * i + length) for i in range(n)]


def _mixed():
    rng = np.random.default_rng(7)
    lens = [1, 4000] + [int(x) for x in rng.integers(1, 4001, 10)]
    return [(int(tb), int(tb) + n) for tb, n in zip(rng.integers(1, 64, len(lens)) | 1, lens)]


BATCHES = {"32x512": _batch(32, 512), "128x128": _batch(128, 128), "mixed": _mixed()}


def tlen(tb, te, page):
    return 0 if tb == te else -(-te // page) - tb // page


def run(name, batch, H, nl, no, hd, src_tp, dst_tp, W, ps, pd, cast):
    ranges = BATCHES[batch]
    rng = np.random.default_rng(3)
    order = rng.permutation(len(ranges))
    worker = [0] * len(ranges)
    for k, i in enumerate(order):
        worker[i] = k % W
    se, de = (1, 2) if cast else (2, 2)
    s_row, d_row = hd * se, hd * de
    one = tp_pp_scatter_plan(H, nl, src_tp, 1, dst_tp, 1, 0)
    ranks = sorted({w.dst_rank for w in one})
    one = [ScatterWindow(ranks.index(w.dst_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin,
                         w.head_count) for w in one]
    R = len(ranks)
    plan = tile_scatter_plan(one, W, R)
    src_nh, dst_nh = max(1, H // src_tp), max(1, H // dst_tp)
    total = sum(te - tb for tb, te in ranges)
    ns, nd = sum(tlen(tb, te, ps) for tb, te in ranges), sum(tlen(tb, te, pd) for tb, te in ranges)
    src = SB.Pool(ns + 4, nl, no, ps, src_nh, s_row, 1)
    dsts = [SB.Pool(nd + 4, nl, no, pd, dst_nh, d_row, 2 + i) for i in range(W * R)]
    init = [d.buf.clone() for d in dsts]
    sids = rng.permutation(src.nb)[:ns].astype(np.int32)
    dids = [rng.permutation(d.nb)[:nd].astype(np.int32) for d in dsts]
    as_t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    sids_t, dids_t = as_t(sids), [as_t(x) for x in dids]
    masks = [sum(1 << j for j, w in enumerate(plan) if w.dst_rank // R == worker[i]) for i in range(len(ranges))]
    every = (1 << len(plan)) - 1
    seqs = [(tb, te, m) for (tb, te), m in zip(ranges, masks)]
    seqs_all = [(tb, te, every) for tb, te in ranges]
    units = K.repage_route_units(seqs, ps, pd)[0]
    units_t = as_t(units.view(np.int32).reshape(-1))
    units_all_t = as_t(K.repage_route_units(seqs_all, ps, pd)[0].view(np.int32).reshape(-1))
    bunits = K.repage_batch_units(ranges, ps, pd)[0]
    bunits_t = as_t(bunits.view(np.int32).reshape(-1))

    def targets(ids, windows):
        return [K.ScatterTarget(dsts[w.dst_rank].side(ids[w.dst_rank]), dst_nh, w.src_head_begin, w.dst_head_begin, w.head_count,
                                w.src_layer_begin, w.dst_layer_begin, w.layer_count, None) for w in windows]

    offs, so, do = [], 0, 0   # per sequence: its slices of the concatenated tables
    for tb, te in ranges:
        offs.append((so, do, tlen(tb, te, ps), tlen(tb, te, pd)))
        so, do = so + offs[-1][2], do + offs[-1][3]
    # per worker: its sequences' concatenated tables, unit table and targets
    per_w = []
    for k in range(W):
        idx = [i for i in range(len(ranges)) if worker[i] == k and offs[i][2]]
        s_ids = np.concatenate([sids[offs[i][0]:offs[i][0] + offs[i][2]] for i in idx]) if idx else np.zeros(1, np.int32)
        d_ids = [np.concatenate([d[offs[i][1]:offs[i][1] + offs[i][3]] for i in idx]) if idx else np.zeros(1, np.int32) for d in dids]
        wr = [ranges[i] for i in idx]
        u = K.repage_batch_units(wr, ps, pd)[0] if idx else np.zeros((1, 4), np.uint32)
        dt = [as_t(x) for x in d_ids]
        per_w.append((as_t(s_ids), dt, wr, as_t(u.view(np.int32).reshape(-1)), len(wr) and len(u),
                      targets(dt, [w for w in plan if w.dst_rank // R == k]), idx))
    tg_all = targets(dids_t, plan)
    stream = torch.cuda.current_stream()
    sp = int(stream.cuda_stream)
    single_args = [(sids_t[o[0]:o[0] + o[2]], targets([d[o[1]:o[1] + o[3]] for d in dids_t], [w for w in plan if w.dst_rank // R == worker[i]]),
                    tb, te) for i, ((tb, te), o) in enumerate(zip(ranges, offs)) if o[2]]

    def k_routed():
        K.check(K.paged_repage_scatter_routed(src.side(sids_t), src_nh, ps, tg_all, pd, seqs, units_t.data_ptr(), len(units), 0, nl, s_row, cast,
                                              stream=sp), "routed")

    def k_per_worker():
        for s_t, _, wr, u_t, nu, tg, _ in per_w:
            if nu:
                K.check(K.paged_repage_scatter_batch(src.side(s_t), src_nh, ps, tg, pd, wr, u_t.data_ptr(), nu, 0, nl, s_row, cast, stream=sp),
                        "per-worker batch")

    def k_singles():
        for s_t, tg, tb, te in single_args:
            K.check(K.paged_repage_scatter(src.side(s_t), src_nh, ps, tg, pd, tb, te, 0, nl, s_row, cast, stream=sp), "single")

    def k_routed_all():
        K.check(K.paged_repage_scatter_routed(src.side(sids_t), src_nh, ps, tg_all, pd, seqs_all, units_all_t.data_ptr(), len(units), 0, nl,
                                              s_row, cast, stream=sp), "routed all ones")

    def k_batch_all():
        K.check(K.paged_repage_scatter_batch(src.side(sids_t), src_nh, ps, tg_all, pd, ranges, bunits_t.data_ptr(), len(bunits), 0, nl, s_row,
                                             cast, stream=sp), "batch everywhere")

    mgr = TransferManager(device=0, worker_id=63)
    reg = lambda pool, nh, w: mgr.register_fully_contiguous(  # noqa: E731
        LayoutConfig(pool.nb, nl, no, pool.page, nh * hd, dtype_width_bytes=w, num_heads=nh, allow_fp8=w == 1), pool.buf.data_ptr(),
        pool.buf.numel(), StorageKind.Device, 0)
    sh = reg(src, src_nh, se)
    dhs = [reg(d, dst_nh, de) for d in dsts]
    for h in [sh] + dhs:
        mgr.set_kv_block_layout(h, K.KvBlockLayout.OperationalNHD)
    reqs = []
    for i, ((tb, te), o) in enumerate(zip(ranges, offs)):
        mine = range(worker[i] * R, (worker[i] + 1) * R)
        reqs.append((range(tb, te), sids[o[0]:o[0] + o[2]].astype(np.int64), {d: dids[d][o[1]:o[1] + o[3]].astype(np.int64) for d in mine}))
    wreqs = [[(t, s, [dd[d] for d in range(k * R, (k + 1) * R)]) for i, (t, s, dd) in enumerate(reqs) if worker[i] == k] for k in range(W)]
    opts = TransferOptions(cast_mode=cast)

    def m_routed():
        mgr.execute_repage_scatter_routed(sh, dhs, reqs, plan, opts).wait(60.0)

    def m_per_worker():
        note = None
        for k in range(W):
            if wreqs[k]:
                note = mgr.execute_repage_scatter_batch(sh, dhs[k * R:(k + 1) * R], wreqs[k], one, opts)
        note.wait(60.0)

    # the routed launch against the oracle on sampled blocks (first and last sequence, first and last of its windows)
    k_routed()
    torch.cuda.synchronize()
    for i in sorted({0, len(ranges) - 1}):
        tb, te = ranges[i]
        so, do, a_n, b_n = offs[i]
        mine = [w for w in plan if w.dst_rank // R == worker[i]]
        for w in sorted({0, len(mine) - 1}):
            win = mine[w]
            t = win.dst_rank
            for j in sorted({0, b_n - 1}):
                first = (tb // pd + j) * pd
                lo, hi = max(tb, first), min(te, first + pd)
                s_blocks = [src.host_block(int(b)) for b in sids[so + lo // ps - tb // ps:so + -(-hi // ps) - tb // ps]]
                blk = int(dids[t][do + j])
                pools = [np.stack([init[t][blk * dsts[t].block:(blk + 1) * dsts[t].block].cpu().numpy()])]
                wt = (win.src_layer_begin, win.dst_layer_begin, win.layer_count, win.src_head_begin, win.dst_head_begin, win.head_count)
                repage_scatter((s_blocks, NHD, src_nh, nl), [(0, [0], NHD, dst_nh, nl, wt)], pools, no, ps, pd, s_row, lo, hi, cast)
                assert np.array_equal(dsts[t].host_block(blk), pools[0][0]), (name, batch, "seq", i, "window", w, "block", j)
    weights = torch.randint(-(1 << 62), 1 << 62, (dsts[0].block // 4,), dtype=torch.int64, device=dev, generator=torch.Generator(device=dev).manual_seed(5))

    def fingerprint():
        """Per destination block, a weighted sum of its 32-bit words: whole pools compared without a second copy of them."""
        return [torch.cat([(c.view(torch.int32).view(-1, d.block // 4).to(torch.int64) * weights).sum(dim=1)
                           for c in d.buf.split(64 * d.block)]) for d in dsts]

    reference = fingerprint()
    for d, x in zip(dsts, init):
        d.buf.copy_(x)
    k_routed_all()
    torch.cuda.synchronize()
    reference_all = fingerprint()
    for d, x in zip(dsts, init):
        d.buf.copy_(x)

    def check(arm):
        torch.cuda.synchronize()
        ref = reference_all if arm.endswith("_all") else reference
        assert all(torch.equal(f, r) for f, r in zip(fingerprint(), ref)), f"{name} {batch} {arm}: destination pools differ"
        for d, x in zip(dsts, init):
            d.buf.copy_(x)
        torch.cuda.synchronize()

    arms = {"routed": k_routed, "per_worker": k_per_worker, "singles": k_singles, "routed_all": k_routed_all, "batch_all": k_batch_all,
            "mgr_routed": m_routed, "mgr_per_worker": m_per_worker}
    for _ in range(2):   # warm-up, and every arm's bytes
        for k, fn in arms.items():
            fn()
            check(k)

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
    covered = len({h for w in one for h in range(w.src_head_begin, w.src_head_begin + w.head_count)})
    moved = total * nl * no * (covered * s_row + sum(w.head_count for w in one) * d_row)
    base = {"bench": "scatter_route", "case": name, "batch": batch, "seqs": len(ranges), "tokens": total, "workers": W, "targets": len(plan),
            "cast": "fp8-to-bf16" if cast else "none", "bytes": moved, "rounds": a.rounds, "iters": a.iters, "gpu": info["name"],
            "power_limit": info["power_limit"]}
    rows = []
    for k in arms:
        ms = statistics.median(rounds[k])
        rows.append({**base, "arm": k, "ms": round(ms, 4), "ms_range": [round(min(rounds[k]), 4), round(max(rounds[k]), 4)]})
        print(json.dumps(rows[-1]), flush=True)

    if not a.no_tail:
        for d, x in zip(dsts, init):   # the timed rounds leave the all-ones arms' bytes
            d.buf.copy_(x)
        ready = torch.zeros(nl, dtype=torch.int32, device=dev)
        completion = torch.zeros(1, dtype=torch.int32, device=dev)
        wss = [torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device=dev) for _ in range(W + 1)]
        epoch = [0]
        sstream = torch.cuda.Stream()
        ssp = int(sstream.cuda_stream)

        def desc(ws, gate):
            st = K.PermuteStream()
            st.layer_ready_flags[0] = ready.data_ptr()
            st.epoch = epoch[0]
            st.sync_workspace = ws.data_ptr()
            st.gate_mode = gate
            st.completion_flag = completion.data_ptr()
            st.completion_value = epoch[0]
            return st

        def s_routed(gate):
            K.check(K.paged_repage_scatter_routed_streamed(src.side(sids_t), src_nh, ps, tg_all, pd, seqs, units_t.data_ptr(), len(units), 0, nl,
                                                           s_row, cast, None, desc(wss[0], gate), ssp), "streamed routed")

        def s_per_worker(gate):
            for k, (s_t, _, wr, u_t, nu, tg, _) in enumerate(per_w):
                if nu:
                    K.check(K.paged_repage_scatter_batch_streamed(src.side(s_t), src_nh, ps, tg, pd, wr, u_t.data_ptr(), nu, 0, nl, s_row, cast,
                                                                  None, desc(wss[1 + k], gate), ssp), "streamed per-worker batch")

        prod = torch.cuda.Stream()
        cycles = TB.layer_cycles(a.layer_us)
        with torch.cuda.stream(prod):
            torch.cuda._sleep(100)
            K.check(K.set_flags(ready.data_ptr(), 0, 1, 0, int(prod.cuda_stream)), "set_flags")
        torch.cuda.synchronize()
        tails = {"streamed_routed_spin": (s_routed, K.GATE_SPIN), "streamed_per_worker_spin": (s_per_worker, K.GATE_SPIN),
                 "streamed_routed_wait": (s_routed, K.GATE_STREAM_WAIT), "streamed_per_worker_wait": (s_per_worker, K.GATE_STREAM_WAIT)}
        times = {k: [] for k in tails}
        for it in range(a.iters + 2):
            for k, (fn, gate) in tails.items():
                epoch[0] += 1
                torch.cuda.synchronize()
                last, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                fn(gate)
                TB.emulate_prefill(prod, [ready.data_ptr()], nl, epoch[0], cycles)
                last.record(prod)
                end.record(sstream)
                end.synchronize()
                assert completion.item() == epoch[0], f"{k}: the gate timed out"
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
    for nm, shape in SHAPES.items():
        if a.only and nm not in a.only.split(","):
            continue
        for b in BATCHES:
            if not a.batches or b in a.batches.split(","):
                rows += run(nm, b, *shape)
    info = SB.card()
    print(f"\n{info['name']}, power limit {info['power_limit']}; ms = median of {a.rounds} round medians (min-max over rounds)\n")
    print("| shape | batch | routed ms | per worker ms | n singles ms | routed all-ones ms | batch everywhere ms | mgr routed ms | "
          "mgr per worker ms | tail routed spin us | tail per worker spin us | tail routed wait us | tail per worker wait us |")
    print("|---|---|" + "---:|" * 11)
    for nm, b in dict.fromkeys((r["case"], r["batch"]) for r in rows):
        g = {r["arm"]: r for r in rows if r["case"] == nm and r["batch"] == b}
        ms = lambda k: f"{g[k]['ms']:.3f} ({g[k]['ms_range'][0]:.3f}-{g[k]['ms_range'][1]:.3f})"  # noqa: E731
        tail = lambda k: f"{g[k]['exposed_tail_us']:.0f} ({g[k]['tail_range_us'][0]:.0f}-{g[k]['tail_range_us'][1]:.0f})" if k in g else "-"  # noqa: E731
        print(f"| {nm} | {b} | {ms('routed')} | {ms('per_worker')} | {ms('singles')} | {ms('routed_all')} | {ms('batch_all')} | "
              f"{ms('mgr_routed')} | {ms('mgr_per_worker')} | {tail('streamed_routed_spin')} | {tail('streamed_per_worker_spin')} | "
              f"{tail('streamed_routed_wait')} | {tail('streamed_per_worker_wait')} |")


if __name__ == "__main__":
    main()

"""The re-paging scatter streamed layer by layer behind the prefill's ready flags (kvbm_kernels_paged_repage_scatter_streamed),
timed against the unstreamed scatter and against today's only streamed push: one streamed single-target re-paging gather
(kvbm_kernels_paged_stage_repage_gather_streamed) per decode rank, back to back on one stream.

Shapes: scatter_bench.py's Llama-3-70B TP2 rank 0 -> TP16 and TP1 -> TP8 (pages 16 -> 64), DeepSeek MLA to 8 decode ranks
(pages 64 -> 64) and the fp8 -> bf16 TP2 rank 0 -> TP16; tokens [0, 4096), fully contiguous OperationalNHD pools.
gate: every ready flag is set before the launch.  Arms alternate within each of --iters rounds, timed with CUDA events (median):
      the unstreamed scatter, the spinning form at max_ctas 16 / 32 / the default (half the SMs), and the stream-wait form.
tail: a producer stream emulates the prefill as transform_stream_bench.py does (per layer a --layer-us busy kernel, then the
      layer's ready flag).  Streamed arms are enqueued before the producer; the unstreamed scatter waits for the last flag.  Each
      arm's time runs from an event after the last flag to the end of the transfer (the exposed tail), median of --iters.  Arms:
      the unstreamed scatter, both streamed forms (spinning at the default grid), and n streamed gathers (spinning, default grid).
The unstreamed scatter's sampled destination blocks are compared with tests/scatter_oracle.py, and every arm's whole destination
pools with the unstreamed scatter's, in every run.  One JSON line per arm, with the card's name and power limit."""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
import scatter_bench as SB  # noqa: E402
import transform_stream_bench as TB  # noqa: E402
from dynamo_b200 import kernels as K  # noqa: E402
from dynamo_b200.physical import tp_pp_scatter_plan  # noqa: E402
from tests.scatter_oracle import repage_scatter  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--iters", type=int, default=10)
p.add_argument("--tokens", type=int, default=4096)
p.add_argument("--mode", choices=["gate", "tail", "both"], default="both")
p.add_argument("--layer-us", type=float, default=100.0, help="busy time of one emulated prefill layer (tail mode)")
p.add_argument("--only", default=None, help="comma-separated case names")
a = p.parse_args()
SHAPES = ["llama70b_tp2_to_tp16_rank0", "llama70b_tp1_to_tp8", "mla_x8_64_to_64", "llama70b_tp2_to_tp16_rank0_fp8_to_bf16"]
NHD = SB.NHD


def run(name, H, nl, no, hd, src_tp, dst_tp, ps, pd, cast):
    dev = SB.dev
    se, de = (1, 2) if cast else (2, 2)
    s_row, d_row = hd * se, hd * de
    tb, te = 0, a.tokens
    plan = tp_pp_scatter_plan(H, nl, src_tp, 1, dst_tp, 1, 0)
    ranks = sorted({w.dst_rank for w in plan})
    src_nh, dst_nh = max(1, H // src_tp), max(1, H // dst_tp)
    ns, nd = -(-te // ps), -(-te // pd)
    src = SB.Pool(ns + 4, nl, no, ps, src_nh, s_row, 1)
    dsts = [SB.Pool(nd + 4, nl, no, pd, dst_nh, d_row, 2 + i) for i in range(len(ranks))]
    init = [d.buf.clone() for d in dsts]
    rng = np.random.default_rng(3)
    sids = rng.permutation(src.nb)[:ns].astype(np.int32)
    dids = [rng.permutation(d.nb)[:nd].astype(np.int32) for d in dsts]
    sids_t = torch.from_numpy(sids).to(dev)
    dids_t = [torch.from_numpy(x).to(dev) for x in dids]
    windows = [(ranks.index(w.dst_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
               for w in plan]
    targets = [K.ScatterTarget(dsts[t].side(dids_t[t]), dst_nh, sb, db, k, sl, dl, c, None) for t, sl, dl, c, sb, db, k in windows]
    ready = torch.zeros(nl, dtype=torch.int32, device=dev)
    completion = torch.zeros(1, dtype=torch.int32, device=dev)
    wss = [torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device=dev) for _ in range(len(windows) + 1)]
    stream = torch.cuda.Stream()
    sp = int(stream.cuda_stream)
    epoch = [0]

    def desc(mode, ctas, ws):
        st = K.PermuteStream()
        st.layer_ready_flags[0] = ready.data_ptr()
        st.epoch = epoch[0]
        st.sync_workspace = ws.data_ptr()
        st.gate_mode = mode
        st.max_ctas = ctas
        st.completion_flag = completion.data_ptr()
        st.completion_value = epoch[0]
        return st

    def unstreamed(_mode=None, _ctas=0):
        K.check(K.paged_repage_scatter(src.side(sids_t), src_nh, ps, targets, pd, tb, te, 0, nl, s_row, cast, stream=sp), "scatter")

    def streamed(mode, ctas):
        K.check(K.paged_repage_scatter_streamed(src.side(sids_t), src_nh, ps, targets, pd, tb, te, 0, nl, s_row, cast, None,
                                                desc(mode, ctas, wss[0]), sp), "streamed scatter")

    def gathers(mode, ctas):
        for i, (t, sl, dl, c, sb, db, k) in enumerate(windows):
            one = [K.StageSource(K.PermuteSource(src.side(sids_t), src_nh, sb, db, k), sl, dl, c)]
            K.check(K.paged_stage_repage_gather_streamed(one, ps, dsts[t].side(dids_t[t]), dst_nh, pd, tb, te, dl, dl + c, s_row, cast, None,
                                                         desc(mode, ctas, wss[1 + i]), sp), "streamed gather")

    # the unstreamed scatter against the oracle on sampled blocks of the first and last target, then its pools as the reference
    unstreamed()
    torch.cuda.synchronize()
    for w in sorted({0, len(windows) - 1}):
        t = windows[w][0]
        for j in sorted({0, nd - 1}):
            lo, hi = max(tb, j * pd), min(te, (j + 1) * pd)
            s_blocks = [src.host_block(b) for b in sids[lo // ps:-(-hi // ps)]]
            pools = [np.stack([init[t][dids[t][j] * dsts[t].block:(dids[t][j] + 1) * dsts[t].block].cpu().numpy()])]
            repage_scatter((s_blocks, NHD, src_nh, nl), [(0, [0], NHD, dst_nh, nl, windows[w][1:])], pools, no, ps, pd, s_row, lo, hi, cast)
            assert np.array_equal(dsts[t].host_block(dids[t][j]), pools[0][0]), (name, "target", w, "block", j)
    reference = [d.buf.clone() for d in dsts]

    def check(arm, streamed_arm):
        torch.cuda.synchronize()
        if streamed_arm:
            assert completion.item() & 0xFFFFFFFF == epoch[0], f"{name} {arm}: completion word {completion.item() & 0xFFFFFFFF:#x}"
        for d, ref, x in zip(dsts, reference, init):
            assert torch.equal(d.buf, ref), f"{name} {arm}: destination pools differ from the unstreamed scatter's"
            d.buf.copy_(x)
        torch.cuda.synchronize()

    info = SB.card()
    base = {"bench": "scatter_stream", "case": name, "targets": len(windows), "pairs": sum(w[6] for w in windows), "src_page": ps,
            "dst_page": pd, "cast": "fp8-to-bf16" if cast else "none", "tokens": te - tb, "layers": nl, "iters": a.iters,
            "gpu": info["name"], "power_limit": info["power_limit"]}
    # name: (launch, gate mode or None, max_ctas)
    arms = {"unstreamed": (unstreamed, None, 0), "spin_ctas_16": (streamed, K.GATE_SPIN, 16), "spin_ctas_32": (streamed, K.GATE_SPIN, 32),
            "spin_ctas_default": (streamed, K.GATE_SPIN, 0), "stream_wait": (streamed, K.GATE_STREAM_WAIT, 0),
            "n_streamed_gathers": (gathers, K.GATE_SPIN, 0)}

    if a.mode in ("gate", "both"):
        gate_arms = [k for k in arms if k != "n_streamed_gathers"]
        times = {k: [] for k in gate_arms}
        for it in range(a.iters + 2):
            epoch[0] += 1
            ready.fill_(epoch[0])
            torch.cuda.synchronize()
            for k in gate_arms:
                fn, mode, ctas = arms[k]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                fn(mode, ctas)
                e1.record(stream)
                e1.synchronize()
                if it >= 2:
                    times[k].append(e0.elapsed_time(e1) * 1e3)
                if it == 0:
                    check(k, mode is not None)
        un = statistics.median(times["unstreamed"])
        for k in gate_arms:
            us = statistics.median(times[k])
            print(json.dumps({**base, "mode": "gate", "arm": k, "median_us": round(us, 1), "x_unstreamed": round(us / un, 2)}), flush=True)

    if a.mode in ("tail", "both"):
        prod = torch.cuda.Stream()
        cycles = TB.layer_cycles(a.layer_us)
        with torch.cuda.stream(prod):   # the producer's kernels load before anything spins
            torch.cuda._sleep(100)
            K.check(K.set_flags(ready.data_ptr(), 0, 1, epoch[0], int(prod.cuda_stream)), "set_flags")
        torch.cuda.synchronize()
        tail_arms = ["unstreamed", "spin_ctas_default", "stream_wait", "n_streamed_gathers"]
        times = {k: [] for k in tail_arms}
        for it in range(a.iters + 2):
            for k in tail_arms:
                fn, mode, ctas = arms[k]
                epoch[0] += 1
                torch.cuda.synchronize()
                last, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                if mode is not None:
                    fn(mode, ctas)              # enqueued before the prefill starts
                TB.emulate_prefill(prod, [ready.data_ptr()], nl, epoch[0], cycles)
                last.record(prod)
                if mode is None:
                    stream.wait_event(last)
                    fn()
                end.record(stream)
                end.synchronize()
                if it >= 2:
                    times[k].append(last.elapsed_time(end) * 1e3)
                if it == 0:
                    check(k, mode is not None)
        for k in tail_arms:
            print(json.dumps({**base, "mode": "tail", "arm": k, "exposed_tail_us": round(statistics.median(times[k]), 1),
                              "layer_us": a.layer_us}), flush=True)
    del src, dsts
    torch.cuda.empty_cache()


for nm in SHAPES:
    if not a.only or nm in a.only.split(","):
        run(nm, *SB.CASES[nm])

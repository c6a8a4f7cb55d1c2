"""A decode step whose new sequences were served by different prefill workers, pulled in one routed re-paging gather launch, timed
against one batch gather per worker and one gather per sequence.

Shapes (every pool on one GPU, fully contiguous OperationalNHD, random block tables, every sequence starting inside a block):
  llama70b_4x_tp4_to_tp2   Llama-3-70B (80 layers, K/V, 8 KV heads x 128), decode TP2 rank 0 from 4 prefill workers at TP4: 8 sources
  llama70b_2x_tp8_to_tp1   decode TP1 from 2 prefill workers at TP8: 16 sources
  mla_8x_dp                DeepSeek MLA (61 layers, 1 x 576) from 8 prefill DP workers, every window writing the one latent head
Pages 16 -> 64 (64 -> 64 for MLA).  Batches 32 x 512, 128 x 128 and a mixed batch of 12 sequences of 1 to 4000 tokens; each sequence
is served by one worker (round robin over a shuffled order).
Arms, alternated inside each of --rounds rounds in one process, CUDA events around each arm's launches (median of --iters):
  routed        one kvbm_kernels_paged_stage_repage_gather_routed launch
  per_worker    one kvbm_kernels_paged_stage_repage_gather_batch per worker over its sequences and windows, back to back on one stream
  singles       one kvbm_kernels_paged_stage_repage_gather per sequence over its worker's windows
  routed_all    the routed launch over worker 0's windows alone (disjoint heads) with every mask all ones ...
  batch_all     ... against kvbm_kernels_paged_stage_repage_gather_batch on the same plan and tables: the cost of routing itself
  mgr_routed    TransferManager.execute_repage_batch_routed, host clock around call and wait
  mgr_per_worker one TransferManager.execute_repage_batch per worker, then a wait for the last
Streamed tail (--no-tail skips it): a producer stream emulates every prefill worker's forward pass with a --layer-us busy kernel per
layer and then every source's ready flag for that layer, on the same GPU.  The routed streamed launch and one streamed batch per
worker (back to back on ONE stream) are enqueued right after the producer, while its first layers run, in the spinning form at its
default grid and in the stream-wait form; the time from the producer's last flag to the end of the transfer is the exposed tail.
Every arm's whole destination pool is compared with the routed launch's (the all-ones pair with each other), and sampled
destination blocks of the routed launch with tests/stage_repage_oracle.py.  One JSON line per arm with the card's name and power
limit read in this run, then a markdown table.  Needs a GPU; there is no fallback."""
import argparse
import json
import os
import statistics
import sys
import time

# a stream-wait launch holds the hardware queue its stream maps to, and the manager adds streams of its own: one queue per stream
# keeps the producer from queueing behind the transfer's waits (NOTES item 7)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
import numpy as np  # noqa: E402
import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
import scatter_bench as SB  # noqa: E402
import transform_stream_bench as TB  # noqa: E402
from dynamo_b200 import kernels as K  # noqa: E402
from dynamo_b200.physical import (LayoutConfig, ShardWindow, StorageKind, TransferManager, tile_reshard_plan,  # noqa: E402
                                  tp_pp_reshard_plan)
from tests.stage_repage_oracle import stage_repage_gather  # noqa: E402

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
# name: (num_kv_heads, layers, outer, head_dim, src_tp, dst_tp, workers, Ps, Pd)
SHAPES = {
    "llama70b_4x_tp4_to_tp2": (8, 80, 2, 128, 4, 2, 4, 16, 64),
    "llama70b_2x_tp8_to_tp1": (8, 80, 2, 128, 8, 1, 2, 16, 64),
    "mla_8x_dp": (1, 61, 1, 576, 1, 1, 8, 64, 64),
}


def _batch(n, length):
    return [(1 + 7 * i, 1 + 7 * i + length) for i in range(n)]


def _mixed():
    rng = np.random.default_rng(7)
    lens = [1, 4000] + [int(x) for x in rng.integers(1, 4001, 10)]
    return [(int(tb), int(tb) + n) for tb, n in zip(rng.integers(1, 64, len(lens)) | 1, lens)]


BATCHES = {"32x512": _batch(32, 512), "128x128": _batch(128, 128), "mixed": _mixed()}
STREAMS = (torch.cuda.Stream(), torch.cuda.Stream())   # the streamed transfer's and the producer's, the same for every shape


def tlen(tb, te, page):
    return 0 if tb == te else -(-te // page) - tb // page


def run(name, batch, H, nl, no, hd, src_tp, dst_tp, W, ps, pd):
    ranges = BATCHES[batch]
    rng = np.random.default_rng(3)
    worker = [0] * len(ranges)
    for k, i in enumerate(rng.permutation(len(ranges))):
        worker[i] = k % W
    row = hd * 2
    one = tp_pp_reshard_plan(H, nl, src_tp, 1, dst_tp, 1, 0)
    ranks = sorted({w.src_rank for w in one})
    one = [ShardWindow(ranks.index(w.src_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin,
                       w.head_count) for w in one]
    R = len(ranks)
    plan = tile_reshard_plan(one, W, R)
    src_nh, dst_nh = max(1, H // src_tp), max(1, H // dst_tp)
    total = sum(te - tb for tb, te in ranges)
    offs, so, do = [], 0, 0   # per sequence: its slices of the concatenated tables
    for tb, te in ranges:
        offs.append((so, do, tlen(tb, te, ps), tlen(tb, te, pd)))
        so, do = so + offs[-1][2], do + offs[-1][3]
    ns, nd = so, do
    # worker 0's pools hold every sequence's blocks (the all-ones arms read them all); the others only their own sequences'
    srcs = [SB.Pool((ns if r < R else sum(o[2] for i, o in enumerate(offs) if worker[i] == r // R)) + 2, nl, no, ps, src_nh, row, 1 + r)
            for r in range(W * R)]
    dst = SB.Pool(nd + 4, nl, no, pd, dst_nh, row, 100)
    init = dst.buf.clone()
    sids = []   # per pool: the batch-layout table, 0 at positions of sequences its worker did not serve
    for r, pool in enumerate(srcs):
        ids, perm, used = np.zeros(ns, np.int32), rng.permutation(pool.nb), 0
        for i, o in enumerate(offs):
            if worker[i] == r // R or r < R:
                ids[o[0]:o[0] + o[2]] = perm[used:used + o[2]]
                used += o[2]
        sids.append(ids)
    dids = rng.permutation(dst.nb)[:nd].astype(np.int32)
    as_t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    sids_t, dids_t = [as_t(x) for x in sids], as_t(dids)
    masks = [sum(1 << j for j, w in enumerate(plan) if w.src_rank // R == worker[i]) for i in range(len(ranges))]
    seqs = [(tb, te, m) for (tb, te), m in zip(ranges, masks)]
    seqs_all = [(tb, te, (1 << len(one)) - 1) for tb, te in ranges]
    units = K.repage_route_units(seqs, ps, pd)[0]
    units_t = as_t(units.view(np.int32).reshape(-1))
    units_all_t = as_t(K.repage_route_units(seqs_all, ps, pd)[0].view(np.int32).reshape(-1))
    bunits = K.repage_batch_units(ranges, ps, pd)[0]
    bunits_t = as_t(bunits.view(np.int32).reshape(-1))

    def sources(ids, windows):
        return [K.StageSource(K.PermuteSource(srcs[w.src_rank].side(ids[w.src_rank]), src_nh, w.src_head_begin, w.dst_head_begin,
                                              w.head_count), w.src_layer_begin, w.dst_layer_begin, w.layer_count) for w in windows]

    per_w = []   # per worker: its sequences' concatenated tables, unit table and windows
    for k in range(W):
        idx = [i for i in range(len(ranges)) if worker[i] == k and offs[i][2]]
        cat = lambda t, a_, n_: np.concatenate([t[offs[i][a_]:offs[i][a_] + offs[i][n_]] for i in idx]) if idx else np.zeros(1, np.int32)  # noqa: E731
        s_t = {r: as_t(cat(sids[r], 0, 2)) for r in range(k * R, (k + 1) * R)}
        wr = [ranges[i] for i in idx]
        u = K.repage_batch_units(wr, ps, pd)[0] if idx else np.zeros((1, 4), np.uint32)
        per_w.append((s_t, as_t(cat(dids, 1, 3)), wr, as_t(u.view(np.int32).reshape(-1)), len(u) if idx else 0,
                      [w for w in plan if w.src_rank // R == k], idx))
    src_all = sources(sids_t, plan)
    stream = torch.cuda.current_stream()
    sp = int(stream.cuda_stream)
    single_args = []
    for i, ((tb, te), o) in enumerate(zip(ranges, offs)):
        if o[2]:
            ids = {r: sids_t[r][o[0]:o[0] + o[2]] for r in range(worker[i] * R, (worker[i] + 1) * R)}
            single_args.append((sources(ids, [w for w in plan if w.src_rank // R == worker[i]]), dids_t[o[1]:o[1] + o[3]], tb, te))

    def k_routed():
        K.check(K.paged_stage_repage_gather_routed(src_all, ps, dst.side(dids_t), dst_nh, pd, seqs, units_t.data_ptr(), len(units), 0, nl, row,
                                                   stream=sp), "routed")

    def k_per_worker():
        for s_t, d_t, wr, u_t, nu, wins, _ in per_w:
            if nu:
                K.check(K.paged_stage_repage_gather_batch(sources(s_t, wins), ps, dst.side(d_t), dst_nh, pd, wr, u_t.data_ptr(), nu, 0, nl, row,
                                                          stream=sp), "per-worker batch")

    def k_singles():
        for s, d_t, tb, te in single_args:
            K.check(K.paged_stage_repage_gather(s, ps, dst.side(d_t), dst_nh, pd, tb, te, 0, nl, row, stream=sp), "single")

    def k_routed_all():
        K.check(K.paged_stage_repage_gather_routed(sources(sids_t, one), ps, dst.side(dids_t), dst_nh, pd, seqs_all, units_all_t.data_ptr(),
                                                   len(units), 0, nl, row, stream=sp), "routed all ones")

    def k_batch_all():
        K.check(K.paged_stage_repage_gather_batch(sources(sids_t, one), ps, dst.side(dids_t), dst_nh, pd, ranges, bunits_t.data_ptr(),
                                                  len(bunits), 0, nl, row, stream=sp), "batch of worker 0")

    mgr = TransferManager(device=0, worker_id=67)
    reg = lambda pool, nh: mgr.register_fully_contiguous(  # noqa: E731
        LayoutConfig(pool.nb, nl, no, pool.page, nh * hd, dtype_width_bytes=2, num_heads=nh), pool.buf.data_ptr(), pool.buf.numel(),
        StorageKind.Device, 0)
    shs = {r: reg(x, src_nh) for r, x in enumerate(srcs)}
    dh = reg(dst, dst_nh)
    for h in list(shs.values()) + [dh]:
        mgr.set_kv_block_layout(h, K.KvBlockLayout.OperationalNHD)
    reqs = []
    for i, ((tb, te), o) in enumerate(zip(ranges, offs)):
        mine = range(worker[i] * R, (worker[i] + 1) * R)
        reqs.append((range(tb, te), {r: sids[r][o[0]:o[0] + o[2]].astype(np.int64) for r in mine}, dids[o[1]:o[1] + o[3]].astype(np.int64)))
    wreqs = [[(t, {r - k * R: x for r, x in s.items()}, d) for i, (t, s, d) in enumerate(reqs) if worker[i] == k] for k in range(W)]

    def m_routed():
        mgr.execute_repage_batch_routed(shs, dh, reqs, plan).wait(60.0)

    def m_per_worker():
        note = None
        for k in range(W):
            if wreqs[k]:
                note = mgr.execute_repage_batch({r: shs[k * R + r] for r in range(R)}, dh, wreqs[k], one)
        note.wait(60.0)

    # the routed launch against the oracle on sampled blocks: the first destination block of the first and the last sequence
    k_routed()
    torch.cuda.synchronize()
    for i in sorted({0, len(ranges) - 1}):
        tb, te = ranges[i]
        so, do, a_n, b_n = offs[i]
        lo, hi = tb, min(te, (tb // pd + 1) * pd)
        mine = [w for w in plan if w.src_rank // R == worker[i]]
        blocks = {w.src_rank: [srcs[w.src_rank].host_block(int(b)) for b in sids[w.src_rank][so:so + tlen(lo, hi, ps)]] for w in mine}
        order = sorted(blocks)
        wins = [(order.index(w.src_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
                for w in mine]
        blk = int(dids[do])
        want = stage_repage_gather([(blocks[r], NHD, src_nh, nl) for r in order], wins, [init[blk * dst.block:(blk + 1) * dst.block].cpu().numpy()],
                                   NHD, dst_nh, nl, no, ps, pd, row, lo, hi)
        assert np.array_equal(dst.host_block(blk), want[0]), (name, batch, "seq", i)
    weights = torch.randint(-(1 << 62), 1 << 62, (dst.block // 4,), dtype=torch.int64, device=dev, generator=torch.Generator(device=dev).manual_seed(5))

    def fingerprint():
        """Per destination block, a weighted sum of its 32-bit words: the whole pool compared without a second copy of it."""
        return torch.cat([(c.view(torch.int32).view(-1, dst.block // 4).to(torch.int64) * weights).sum(dim=1) for c in dst.buf.split(64 * dst.block)])

    reference = fingerprint()
    dst.buf.copy_(init)
    k_routed_all()
    torch.cuda.synchronize()
    reference_all = fingerprint()
    dst.buf.copy_(init)

    def check(arm):
        torch.cuda.synchronize()
        assert torch.equal(fingerprint(), reference_all if arm.endswith("_all") else reference), f"{name} {batch} {arm}: destination differs"
        dst.buf.copy_(init)
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
    moved = total * nl * no * sum(w.head_count for w in one) * row * 2   # read once and written once per routed window head
    base = {"bench": "gather_route", "case": name, "batch": batch, "seqs": len(ranges), "tokens": total, "workers": W, "sources": len(plan),
            "bytes": moved, "rounds": a.rounds, "iters": a.iters, "gpu": info["name"], "power_limit": info["power_limit"]}
    rows = []
    for k in arms:
        rows.append({**base, "arm": k, "ms": round(statistics.median(rounds[k]), 4), "ms_range": [round(min(rounds[k]), 4), round(max(rounds[k]), 4)]})
        print(json.dumps(rows[-1]), flush=True)

    if not a.no_tail:
        dst.buf.copy_(init)
        ready = [torch.zeros(nl, dtype=torch.int32, device=dev) for _ in srcs]
        completion = torch.zeros(1, dtype=torch.int32, device=dev)
        wss = [torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device=dev) for _ in range(W + 1)]
        epoch = [0]
        sstream, prod = STREAMS
        ssp = int(sstream.cuda_stream)

        def desc(ws, gate, windows):
            st = K.PermuteStream()
            for j, w in enumerate(windows):
                st.layer_ready_flags[j] = ready[w.src_rank].data_ptr()
            st.epoch = epoch[0]
            st.sync_workspace = ws.data_ptr()
            st.gate_mode = gate
            st.completion_flag = completion.data_ptr()
            st.completion_value = epoch[0]
            return st

        def s_routed(gate):
            K.check(K.paged_stage_repage_gather_routed_streamed(src_all, ps, dst.side(dids_t), dst_nh, pd, seqs, units_t.data_ptr(), len(units), 0,
                                                                nl, row, 0, None, desc(wss[0], gate, plan), ssp), "streamed routed")

        def s_per_worker(gate):
            for k, (s_t, d_t, wr, u_t, nu, wins, _) in enumerate(per_w):
                if nu:
                    K.check(K.paged_stage_repage_gather_batch_streamed(sources(s_t, wins), ps, dst.side(d_t), dst_nh, pd, wr, u_t.data_ptr(), nu, 0,
                                                                       nl, row, 0, None, desc(wss[1 + k], gate, wins), ssp), "streamed batch")

        cycles = TB.layer_cycles(a.layer_us)
        with torch.cuda.stream(prod):
            torch.cuda._sleep(100)
            K.check(K.set_flags(ready[0].data_ptr(), 0, 1, 0, int(prod.cuda_stream)), "set_flags")
        torch.cuda.synchronize()
        tails = {"streamed_routed_spin": (s_routed, K.GATE_SPIN), "streamed_per_worker_spin": (s_per_worker, K.GATE_SPIN),
                 "streamed_routed_wait": (s_routed, K.GATE_STREAM_WAIT), "streamed_per_worker_wait": (s_per_worker, K.GATE_STREAM_WAIT)}
        times = {k: [] for k in tails}
        for it in range(a.iters + 2):
            for k, (fn, gate) in tails.items():
                epoch[0] += 1
                torch.cuda.synchronize()
                last, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                # the producer first: a stream-wait launch enqueues a wait per (layer, source), up to 1280 here, and a host thread
                # that fills the stream's queue with them blocks until the GPU drains it, so it could not enqueue the producer after
                TB.emulate_prefill(prod, [x.data_ptr() for x in ready], nl, epoch[0], cycles)
                fn(gate)
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
    del srcs, dst
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
    print("| shape | batch | routed ms | per worker ms | n singles ms | routed all-ones ms | batch (worker 0) ms | mgr routed ms | "
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

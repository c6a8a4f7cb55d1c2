"""Layout-transforming hand-off, timed: kvbm_kernels_paged_permute (layouts + block tables, no pointer tables) against the flow the
reference's K2 needs (host builds nb*nl*no chunk pointers + nb universal pointers, uploads them, launches
kvbm_kernels_launch_universal_from_block -- tensor_kernels.rs:177-215) and against the plain paged copy of the same bytes.
Llama-3-70B KV geometry by default.  Prints one JSON line; roofline = bytes read + written / the HBM peak bench.py uses
(the measured copy peak, else the H100 data sheet's)."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import bench  # noqa: E402
from dynamo_b200 import kernels as K  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--blocks", type=int, default=64)
p.add_argument("--pool", type=int, default=96)
p.add_argument("--layers", type=int, default=80)
p.add_argument("--heads", type=int, default=8)
p.add_argument("--head-dim", type=int, default=128)
p.add_argument("--page", type=int, default=16)
p.add_argument("--iters", type=int, default=20)
p.add_argument("--peer", type=int, default=-1, help="put one pool on this GPU (the launch stays on GPU 0); -1 = same GPU")
p.add_argument("--peer-side", choices=["dst", "src"], default="dst", help="dst: universal pool on the peer (push); src: engine pool on the peer (pull)")
p.add_argument("--cast", choices=["none", "fp8-to-bf16", "bf16-to-fp8"], default="none",
               help="time the transform with the fused cast against the paged copy's cast and the two-pass workaround instead")
p.add_argument("--scaled", action="store_true",
               help="with --cast: also time the same launches with per-(layer, K/V) fp8 KV-cache scales, alternating with the unscaled arms")
p.add_argument("--reshard", default=None, metavar="SRC_TP:DST_TP",
               help="time one decode rank's assembly of its heads from the source ranks' pools (TP re-shard) instead; --cast composes")
p.add_argument("--pp", default=None, metavar="SRC_PP:SRC_TP:DST_TP",
               help="time decode rank 0's assembly of its layers and heads from a PP x TP prefill group (one pool per source rank, "
                    "holding its stage's layers) instead; --cast composes")
a = p.parse_args()
nl, no, nt, nh, hd, elem = a.layers, 2, a.page, a.heads, a.head_dim, 2
row, region = hd * elem, nt * nh * hd * elem
nb, n = a.pool, a.blocks
dev = torch.device("cuda:0")
torch.cuda.set_device(0)
ddev = torch.device(f"cuda:{a.peer}") if a.peer >= 0 and a.peer_side == "dst" else dev
sdev = torch.device(f"cuda:{a.peer}") if a.peer >= 0 and a.peer_side == "src" else dev
if a.peer >= 0:
    import ctypes
    rt = ctypes.CDLL("libcudart.so")
    rt.cudaDeviceEnablePeerAccess(a.peer, 0)
peak, peak_src = bench.peaks()

# engine pool: layer-separate, block-is-second-dim (vLLM), NHD inside a region; universal pool: fully contiguous
op = [torch.randint(0, 256, (no * nb * region,), dtype=torch.uint8, device=sdev) for _ in range(nl)]
torch.cuda.synchronize(sdev)
uni = torch.zeros(nb * nl * no * region, dtype=torch.uint8, device=ddev)
op_base = torch.tensor([t.data_ptr() for t in op], dtype=torch.int64, device=dev)
op_desc = K.PagedLayout(op_base.data_ptr(), region, nb * region, region, nl, no, nb)
bs = nl * no * region
uni_base = torch.tensor([uni.data_ptr() + l * no * region for l in range(nl)], dtype=torch.int64, device=dev)
uni_desc = K.PagedLayout(uni_base.data_ptr(), bs, region, region, nl, no, nb)
rng = np.random.default_rng(0)
sid, did = rng.permutation(nb)[:n].astype(np.int32), rng.permutation(nb)[:n].astype(np.int32)
sid_d, did_d = torch.from_numpy(sid).to(dev), torch.from_numpy(did).to(dev)
stream = torch.cuda.current_stream()
sp = int(stream.cuda_stream)
moved = n * bs


def timed(fn, iters=a.iters, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def pool_pair(e):
    """An engine pool (as `op`) and a universal pool (as `uni`) of e-byte elements: (engine layers, universal tensor, engine
    descriptor, universal descriptor, the layer-base tables the descriptors point to)."""
    reg = nt * nh * hd * e
    eng = [torch.randint(0, 256, (no * nb * reg,), dtype=torch.uint8, device=sdev) for _ in range(nl)]
    un = torch.zeros(nb * nl * no * reg, dtype=torch.uint8, device=ddev)
    torch.cuda.synchronize(sdev)
    eb = torch.tensor([t.data_ptr() for t in eng], dtype=torch.int64, device=dev)
    ub = torch.tensor([un.data_ptr() + l * no * reg for l in range(nl)], dtype=torch.int64, device=dev)
    return eng, un, K.PagedLayout(eb.data_ptr(), reg, nb * reg, reg, nl, no, nb), K.PagedLayout(ub.data_ptr(), nl * no * reg, reg, reg, nl, no, nb), (eb, ub)


def cast_bench():
    """(a) the fused permute + cast, engine -> universal and back; (b) the paged copy's fused cast of the same bytes (the floor
    for 3 bytes per element); (c) the cheapest two-pass workaround: the permute in fp8 through a staging pool plus the paged
    copy's cast, ordered so that the permute moves the narrow dtype (5 bytes per element)."""
    up = a.cast == "fp8-to-bf16"
    mode = K.CastMode.FP8E4M3_TO_BF16 if up else K.CastMode.BF16_TO_FP8E4M3
    _eng8, uni8, eng8_desc, uni8_desc, _bases = pool_pair(1)  # the tensors stay alive while the descriptors are used
    # source / destination descriptors of the engine -> universal direction; the fp8 pool of the other side is the staging pool
    es, us, ed, ud = (eng8_desc, uni8_desc, op_desc, uni_desc) if up else (op_desc, uni_desc, eng8_desc, uni8_desc)
    out = uni if up else uni8
    src_row = hd * (1 if up else 2)
    side = lambda desc, ids, kv: K.PermuteSide(desc, ids.data_ptr(), kv)  # noqa: E731

    def fused_to():
        K.check(K.paged_permute_cast(side(es, sid_d, 4), side(ud, did_d, 1), n, 0, nl, nh, nt, src_row, mode, stream=sp))

    def fused_from():
        K.check(K.paged_permute_cast(side(us, did_d, 1), side(ed, sid_d, 4), n, 0, nl, nh, nt, src_row, mode, stream=sp))

    def cast_copy():
        K.check(K.paged_copy(es, [K.PagedDst(ud, sid_d.data_ptr(), did_d.data_ptr(), 0, 0)], n, 0, nl, int(mode), None, sp))

    def two_pass():
        if up:   # permute fp8 into the fp8 universal pool, then cast it into the bf16 one
            K.check(K.paged_permute(side(eng8_desc, sid_d, 4), side(uni8_desc, did_d, 1), n, 0, nl, nh, nt, hd, stream=sp))
            K.check(K.paged_copy(uni8_desc, [K.PagedDst(uni_desc, did_d.data_ptr(), did_d.data_ptr(), 0, 0)], n, 0, nl, int(mode), None, sp))
        else:    # cast into the fp8 engine pool, then permute fp8 into the fp8 universal pool
            K.check(K.paged_copy(op_desc, [K.PagedDst(eng8_desc, sid_d.data_ptr(), sid_d.data_ptr(), 0, 0)], n, 0, nl, int(mode), None, sp))
            K.check(K.paged_permute(side(eng8_desc, sid_d, 4), side(uni8_desc, did_d, 1), n, 0, nl, nh, nt, hd, stream=sp))

    fused_to()
    torch.cuda.synchronize()
    fused_out = out.clone()
    out.zero_()
    torch.cuda.synchronize(ddev)
    two_pass()
    torch.cuda.synchronize()
    same = bool(torch.equal(fused_out, out))
    elems = n * nl * no * nt * nh * hd
    res = {"geometry": {"blocks": n, "layers": nl, "outer": no, "page": nt, "heads": nh, "head_dim": hd, "cast": a.cast,
                        "MiB_fp8": elems / 2**20, "MiB_bf16": 2 * elems / 2**20},
           "peer": a.peer, "peer_side": a.peer_side if a.peer >= 0 else None, "fused_equals_two_pass": same,
           "hbm_peak_GBps": peak, "hbm_peak_source": peak_src}
    arms = [("fused_permute_cast_to_universal", fused_to, 3), ("fused_permute_cast_from_universal", fused_from, 3),
            ("paged_copy_cast", cast_copy, 3), ("two_pass_fp8_permute_and_cast_copy", two_pass, 5)]
    if a.scaled:
        arms = scaled_arms(arms, res, mode, side, es, us, ed, ud, src_row, out, _eng8 if up else op)
    for name, fn, per_elem in arms:
        # --scaled: the median of three runs, the arms alternating so that scaled and unscaled see the same card state
        ms = statistics.median(times[name]) if a.scaled else timed(fn)
        moved_rw = per_elem * elems
        res[name] = {"ms": round(ms, 4), "bytes_read_plus_write": moved_rw, "GBps_read_plus_write": round(moved_rw / ms / 1e6, 1),
                     "frac_of_hbm_peak": round(moved_rw / ms / 1e6 / peak, 3)}
    print(json.dumps(res))


times = {}


def scaled_arms(arms, res, mode, side, es, us, ed, ud, src_row, out, eng):
    """The scaled twins of the fused permute + cast (both directions) and of the paged copy's cast, distinct scales per (layer,
    K/V); checks two sampled blocks of each against tests/scaled_cast_oracle.py and times every arm three times, alternating."""
    from tests.scaled_cast_oracle import cast_bytes_scaled, kv_layout_permute_cast_scaled
    h = (np.random.default_rng(1).uniform(0.01, 4.0, nl * no) * (1 + np.arange(nl * no) * 1e-3)).astype(np.float32)
    sc = torch.from_numpy(h).to(dev)

    def fused_to_s():
        K.check(K.paged_permute_heads(side(es, sid_d, 4), side(ud, did_d, 1), n, 0, nl, nh, 0, nh, 0, nh, nt, src_row, mode, stream=sp,
                                      cast_scales=sc))

    def fused_from_s():
        K.check(K.paged_permute_heads(side(us, did_d, 1), side(ed, sid_d, 4), n, 0, nl, nh, 0, nh, 0, nh, nt, src_row, mode, stream=sp,
                                      cast_scales=sc))

    def cast_copy_s():
        K.check(K.paged_copy(es, [K.PagedDst(ud, sid_d.data_ptr(), did_d.data_ptr(), 0, 0)], n, 0, nl, int(mode),
                             K.PagedCopyOpts(cast_scales=sc.data_ptr()), sp))

    src_block = lambda b: np.concatenate([eng[l].view(no, nb, -1)[o, b].cpu().numpy() for l in range(nl) for o in range(no)])  # noqa: E731
    ok = True
    for fn in (fused_to_s, cast_copy_s):
        out.zero_()
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
        for i in (0, n - 1):
            blk = src_block(int(sid[i]))
            got = out.view(nb, -1)[int(did[i])].cpu().numpy()
            if fn is fused_to_s:
                want = kv_layout_permute_cast_scaled(blk, 4, 1, nl, no, nt, nh, src_row, int(mode), h)
            else:   # region (l, o) of the universal block, cast with its own scale
                want = np.concatenate([cast_bytes_scaled(r, int(mode), float(h[k])) for k, r in enumerate(np.split(blk, nl * no))])
            ok = ok and bool(np.array_equal(got, want))
    res["scaled_equals_oracle"] = ok
    res["card"] = card()
    res["scales"] = "distinct per (layer, outer), uniform in [0.01, 4)"
    named = {"fused_permute_cast_to_universal": fused_to_s, "fused_permute_cast_from_universal": fused_from_s, "paged_copy_cast": cast_copy_s}
    out_arms = []
    for name, fn, per in arms:
        out_arms.append((name, fn, per))
        if name in named:
            out_arms.append((name + "_scaled", named[name], per))
    for _ in range(3):
        for name, fn, _per in out_arms:
            times.setdefault(name, []).append(timed(fn))
    return out_arms


def card():
    """The name and power limit of GPU 0, read now: they belong beside every time this run prints."""
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "not read")
    return {"name": name, "power_limit": limit}


def reshard_bench():
    """Decode rank 0 of a SRC_TP -> DST_TP re-shard: every launch of its plan (kvbm_kernels_paged_permute_heads, engine pools
    OperationalNHD layer-separate on both sides, --cast fused in), per hand-off, median over three runs.  Compared with the plain
    paged copy (its cast with --cast) of the same destination bytes and with the full-head permute (every head of a TP1 pool,
    NHD -> NHD) per byte.  reshard_one_launch runs the same plan as one kvbm_kernels_paged_permute_gather launch on the same
    pools and stream; one_launch_equals_per_entry compares the whole destination pool after either arm."""
    from dynamo_b200.physical import tp_reshard_plan
    from oracle import oracle as O
    from tests.reshard_oracle import reshard_block
    src_tp, dst_tp = (int(x) for x in a.reshard.split(":"))
    mode = {"none": K.CastMode.NONE, "fp8-to-bf16": K.CastMode.FP8E4M3_TO_BF16, "bf16-to-fp8": K.CastMode.BF16_TO_FP8E4M3}[a.cast]
    se, de = {"none": (2, 2), "fp8-to-bf16": (1, 2), "bf16-to-fp8": (2, 1)}[a.cast]
    snh, dnh = max(1, nh // src_tp), max(1, nh // dst_tp)
    plan = tp_reshard_plan(nh, src_tp, dst_tp, 0)

    def engine(heads, e, device):
        reg = nt * heads * hd * e
        layers = [torch.randint(0, 256, (no * nb * reg,), dtype=torch.uint8, device=device) for _ in range(nl)]
        base = torch.tensor([t.data_ptr() for t in layers], dtype=torch.int64, device=dev)
        return layers, base, K.PagedLayout(base.data_ptr(), reg, nb * reg, reg, nl, no, nb)

    srcs = {w.src_rank: engine(snh, se, sdev) for w in plan}
    dst = engine(dnh, de, ddev)
    side = lambda desc, ids: K.PermuteSide(desc, ids.data_ptr(), int(K.KvBlockLayout.OperationalNHD))  # noqa: E731

    def assemble():
        for w in plan:
            K.check(K.paged_permute_heads(side(srcs[w.src_rank][2], sid_d), side(dst[2], did_d), n, 0, nl, snh, w.src_head_begin, dnh,
                                          w.dst_head_begin, w.head_count, nt, hd * se, int(mode), stream=sp))

    assemble()
    torch.cuda.synchronize()
    def block(pool, b):   # the [layer][outer] regions of block b of a block-is-second-dim pool
        return np.concatenate([pool[0][l].view(no, nb, -1)[o, b].cpu().numpy() for l in range(nl) for o in range(no)])

    same = sum(w.head_count for w in plan) == dnh   # the plan writes every destination head, so the old bytes do not matter
    for i in (0, n - 1):   # sampled blocks against the oracle
        want = np.zeros(nl * no * nt * dnh * hd * de, dtype=np.uint8)
        for w in plan:
            want = reshard_block(block(srcs[w.src_rank], int(sid[i])), want, O.KV_OPERATIONAL_NHD, O.KV_OPERATIONAL_NHD, nl, no, nt, snh,
                                 dnh, hd * se, int(mode), w.src_head_begin, w.dst_head_begin, w.head_count)
        same = same and bool(np.array_equal(block(dst, int(did[i])), want))
    gather_srcs = [K.PermuteSource(side(srcs[w.src_rank][2], sid_d), snh, w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan]

    def one_launch():   # the same plan as one kvbm_kernels_paged_permute_gather launch
        K.check(K.paged_permute_gather(gather_srcs, side(dst[2], did_d), dnh, n, 0, nl, nt, hd * se, int(mode), stream=sp))

    def dst_after(fn):   # the whole destination pool after fn, from the same pre-filled pool
        for t in dst[0]:
            t.fill_(0x5A)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
        return [t.clone() for t in dst[0]]

    one_equal = all(torch.equal(x, y) for x, y in zip(dst_after(assemble), dst_after(one_launch)))
    plain_src = engine(dnh, se, sdev)   # the same destination bytes as one paged copy (its cast with --cast)

    def plain():
        K.check(K.paged_copy(plain_src[2], [K.PagedDst(dst[2], sid_d.data_ptr(), did_d.data_ptr(), 0, 0)], n, 0, nl, int(mode), None, sp))

    full_src, full_dst = engine(nh, se, sdev), engine(nh, de, ddev)

    def full_permute():
        K.check(K.paged_permute_heads(side(full_src[2], sid_d), side(full_dst[2], did_d), n, 0, nl, nh, 0, nh, 0, nh, nt, hd * se, int(mode),
                                      stream=sp))

    elems = n * nl * no * nt * dnh * hd
    res = {"geometry": {"blocks": n, "layers": nl, "outer": no, "page": nt, "heads": nh, "head_dim": hd, "cast": a.cast,
                        "src_tp": src_tp, "dst_tp": dst_tp, "src_heads_per_rank": snh, "dst_heads_per_rank": dnh},
           "plan": [[w.src_rank, w.src_head_begin, w.dst_head_begin, w.head_count] for w in plan],
           "window_widths": [w.head_count for w in plan], "launches": len(plan), "reshard_equals_oracle": same,
           "peer": a.peer, "peer_side": a.peer_side if a.peer >= 0 else None, "hbm_peak_GBps": peak, "hbm_peak_source": peak_src,
           "one_launch_equals_per_entry": one_equal, "card": card()}
    for name, fn, count in (("reshard_assembly", assemble, elems), ("reshard_one_launch", one_launch, elems),
                            ("plain_paged_copy_same_bytes", plain, elems),
                            ("full_head_permute_tp1", full_permute, n * nl * no * nt * nh * hd)):
        ms = statistics.median([timed(fn) for _ in range(3)])
        rw = count * (se + de)
        res[name] = {"ms": round(ms, 4), "bytes_read_plus_write": rw, "GBps_read_plus_write": round(rw / ms / 1e6, 1),
                     "frac_of_hbm_peak": round(rw / ms / 1e6 / peak, 3)}
    print(json.dumps(res))


def pp_bench():
    """Decode rank 0 (PP1) of a SRC_PP x SRC_TP -> DST_TP re-shard, engine pools OperationalNHD layer-separate on both sides, each
    source pool holding only its stage's nl / SRC_PP layers.  Arms, alternated within each of five rounds (median of --iters per
    arm and round): (1) stage_gather_one_launch, kvbm_kernels_paged_stage_gather over the plan; (2) per_stage_gathers, one
    kvbm_kernels_paged_permute_gather per stage over that stage's layer range, its sources described by nl-entry layer_base
    tables whose entries in the stage's range point at the pool's layers (the workaround without the staged gather, open to
    operational formats only); (3) gather_from_full_layer_sources, the same bytes gathered from sources that hold every layer
    (the ceiling); (4) plain_paged_copy_same_bytes.  stage_equals_per_stage compares the whole destination pool after arms 1
    and 2.  gate_overhead: the streamed form with every flag already released, both gate modes, against arm 1."""
    from dynamo_b200.physical import tp_pp_reshard_plan, tp_reshard_plan
    src_pp, src_tp, dst_tp = (int(x) for x in a.pp.split(":"))
    mode = {"none": K.CastMode.NONE, "fp8-to-bf16": K.CastMode.FP8E4M3_TO_BF16, "bf16-to-fp8": K.CastMode.BF16_TO_FP8E4M3}[a.cast]
    se, de = {"none": (2, 2), "fp8-to-bf16": (1, 2), "bf16-to-fp8": (2, 1)}[a.cast]
    snh, dnh, snl = max(1, nh // src_tp), max(1, nh // dst_tp), nl // src_pp
    plan = tp_pp_reshard_plan(nh, nl, src_tp, src_pp, dst_tp, 1, 0)
    keep = []

    def engine(heads, e, layers, table=None):
        reg = nt * heads * hd * e
        ts = [torch.randint(0, 256, (no * nb * reg,), dtype=torch.uint8, device=dev) for _ in range(layers)]
        ptrs = table(ts) if table else [t.data_ptr() for t in ts]
        base = torch.tensor(ptrs, dtype=torch.int64, device=dev)
        keep.append(base)
        return ts, K.PagedLayout(base.data_ptr(), reg, nb * reg, reg, len(ptrs), no, nb)

    side = lambda desc, ids: K.PermuteSide(desc, ids.data_ptr(), int(K.KvBlockLayout.OperationalNHD))  # noqa: E731
    srcs = {w.src_rank: engine(snh, se, snl) for w in plan}
    dst = engine(dnh, de, nl)
    row = hd * se
    staged = [K.StageSource(K.PermuteSource(side(srcs[w.src_rank][1], sid_d), snh, w.src_head_begin, w.dst_head_begin, w.head_count),
                            w.src_layer_begin, w.dst_layer_begin, w.layer_count) for w in plan]

    def stage_one():
        K.check(K.paged_stage_gather(staged, side(dst[1], did_d), dnh, n, 0, nl, nt, row, int(mode), stream=sp))

    # arm 2: per stage, each source seen through an nl-entry layer_base table shifted to the stage's destination layers
    stages = sorted({(w.dst_layer_begin, w.layer_count) for w in plan})
    per_stage = []
    for d0, c in stages:
        ws = [w for w in plan if w.dst_layer_begin == d0]
        shifted = {}
        for w in ws:
            ts = srcs[w.src_rank][0]
            ptrs = [ts[min(max(l - d0 + w.src_layer_begin, 0), snl - 1)].data_ptr() for l in range(nl)]
            base = torch.tensor(ptrs, dtype=torch.int64, device=dev)
            keep.append(base)
            shifted[w.src_rank] = K.PagedLayout(base.data_ptr(), nt * snh * hd * se, nb * nt * snh * hd * se, nt * snh * hd * se, nl, no, nb)
        per_stage.append((d0, d0 + c, [K.PermuteSource(side(shifted[w.src_rank], sid_d), snh, w.src_head_begin, w.dst_head_begin, w.head_count)
                                       for w in ws]))

    def stage_each():
        for lb, le, ps in per_stage:
            K.check(K.paged_permute_gather(ps, side(dst[1], did_d), dnh, n, lb, le, nt, row, int(mode), stream=sp))

    tp_plan = tp_reshard_plan(nh, src_tp, dst_tp, 0)
    full = {w.src_rank: engine(snh, se, nl) for w in tp_plan}
    full_srcs = [K.PermuteSource(side(full[w.src_rank][1], sid_d), snh, w.src_head_begin, w.dst_head_begin, w.head_count) for w in tp_plan]

    def ceiling():
        K.check(K.paged_permute_gather(full_srcs, side(dst[1], did_d), dnh, n, 0, nl, nt, row, int(mode), stream=sp))

    plain_src = engine(dnh, se, nl)

    def plain():
        K.check(K.paged_copy(plain_src[1], [K.PagedDst(dst[1], sid_d.data_ptr(), did_d.data_ptr(), 0, 0)], n, 0, nl, int(mode), None, sp))

    def dst_after(fn):
        for t in dst[0]:
            t.fill_(0x5A)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
        return [t.clone() for t in dst[0]]

    same = all(torch.equal(x, y) for x, y in zip(dst_after(stage_one), dst_after(stage_each)))
    flags = {r: torch.ones(snl, dtype=torch.int32, device=dev) for r in srcs}
    ws_words = torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device=dev)

    def streamed(gate):
        st = K.PermuteStream()
        for j, w in enumerate(plan):
            st.layer_ready_flags[j] = flags[w.src_rank].data_ptr()
        st.epoch, st.sync_workspace, st.gate_mode = 1, ws_words.data_ptr(), gate
        return lambda: K.check(K.paged_stage_gather_streamed(staged, side(dst[1], did_d), dnh, n, 0, nl, nt, row, int(mode), None, st, sp))

    arms = [("stage_gather_one_launch", stage_one), ("per_stage_gathers", stage_each), ("gather_from_full_layer_sources", ceiling),
            ("plain_paged_copy_same_bytes", plain), ("streamed_spin_flags_released", streamed(K.GATE_SPIN)),
            ("streamed_stream_wait_flags_released", streamed(K.GATE_STREAM_WAIT))]
    rounds = {name: [] for name, _ in arms}
    for _ in range(5):
        for name, fn in arms:
            rounds[name].append(timed(fn))
    elems = n * nl * no * nt * dnh * hd
    rw = elems * (se + de)
    res = {"geometry": {"blocks": n, "layers": nl, "outer": no, "page": nt, "heads": nh, "head_dim": hd, "cast": a.cast, "src_pp": src_pp,
                        "src_tp": src_tp, "dst_tp": dst_tp, "layers_per_source": snl},
           "plan": [[w.src_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count]
                    for w in plan],
           "stage_equals_per_stage": same, "hbm_peak_GBps": peak, "hbm_peak_source": peak_src, "card": card(),
           "bytes_read_plus_write": rw}
    for name, _ in arms:
        ms = statistics.median(rounds[name])
        res[name] = {"ms": round(ms, 4), "ms_min": round(min(rounds[name]), 4), "ms_max": round(max(rounds[name]), 4),
                     "GBps_read_plus_write": round(rw / ms / 1e6, 1), "frac_of_hbm_peak": round(rw / ms / 1e6 / peak, 3)}
    print(json.dumps(res))


if a.pp:
    pp_bench()
    sys.exit(0)
if a.reshard:
    reshard_bench()
    sys.exit(0)
if a.cast != "none":
    cast_bench()
    sys.exit(0)


def paged():
    K.check(K.paged_permute(K.PermuteSide(op_desc, sid_d.data_ptr(), 4), K.PermuteSide(uni_desc, did_d.data_ptr(), 1), n, 0, nl, nh, nt, row, stream=sp))


def paged_back():
    K.check(K.paged_permute(K.PermuteSide(uni_desc, did_d.data_ptr(), 1), K.PermuteSide(op_desc, sid_d.data_ptr(), 4), n, 0, nl, nh, nt, row, stream=sp))


chunk_tab = torch.empty(n * nl * no, dtype=torch.int64).pin_memory()
uni_tab = torch.empty(n, dtype=torch.int64).pin_memory()
chunk_dev, uni_dev = torch.empty(n * nl * no, dtype=torch.int64, device=dev), torch.empty(n, dtype=torch.int64, device=dev)
op_ptrs = np.array([t.data_ptr() for t in op], dtype=np.int64)


def legacy_kernel_only():
    K.check(K.universal_from_block(uni_dev.data_ptr(), chunk_dev.data_ptr(), n, nh, nl, no, nt, hd, K.TensorDataType.BF16, K.BlockLayout.NHD, sp))


def legacy_flow():
    """what a caller of the reference's K2 does per transfer: build both pointer tables on the host (vectorised here; the
    reference loops in Rust), upload them, launch, and -- like executor/cuda.rs:324 -- wait for the upload before returning."""
    ct = chunk_tab.numpy().reshape(n, nl, no)
    ct[:] = op_ptrs[None, :, None] + (np.arange(no, dtype=np.int64)[None, None, :] * nb + sid.astype(np.int64)[:, None, None]) * region
    uni_tab.numpy()[:] = uni.data_ptr() + did.astype(np.int64) * bs
    chunk_dev.copy_(chunk_tab, non_blocking=True)
    uni_dev.copy_(uni_tab, non_blocking=True)
    legacy_kernel_only()


def plain_copy():
    dd = [K.PagedDst(uni_desc, sid_d.data_ptr(), did_d.data_ptr(), 0, 0)]
    K.check(K.paged_copy(op_desc, dd, n, 0, nl, 0, None, sp))


legacy_flow()
torch.cuda.synchronize()
a_ref = uni.clone()
uni.zero_()
torch.cuda.synchronize(ddev)      # the zero fill runs on the pool's own device: order it before the launch on GPU 0
paged()
torch.cuda.synchronize()
same = bool(torch.equal(a_ref, uni))


def wall(fn, iters=a.iters):
    ts = []
    for _ in range(iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


res = {"geometry": {"blocks": n, "layers": nl, "outer": no, "page": nt, "heads": nh, "head_dim": hd, "elem": elem, "MiB_moved": moved / 2**20},
       "peer": a.peer, "peer_side": a.peer_side if a.peer >= 0 else None, "paged_equals_legacy": same,
       "hbm_peak_GBps": peak, "hbm_peak_source": peak_src}
for name, fn in (("paged_permute_to_universal", paged), ("paged_permute_from_universal", paged_back), ("legacy_k2_kernel_only", legacy_kernel_only),
                 ("plain_paged_copy", plain_copy)):
    ms = timed(fn)
    res[name] = {"ms": round(ms, 4), "GBps_read_plus_write": round(2 * moved / ms / 1e6, 1), "frac_of_hbm_peak": round(2 * moved / ms / 1e6 / peak, 3)}
res["wall_ms_host_to_done"] = {"paged_permute": round(wall(paged), 4), "legacy_k2_flow_tables_h2d_launch": round(wall(legacy_flow), 4)}
print(json.dumps(res))

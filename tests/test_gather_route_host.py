"""CPU checks of the routed re-paging gather (each sequence of a decode step pulled from the prefill workers that served it, in one
launch): the exported symbols, the C layout of kvbm_repage_route_seq, the plan helper, the kernel entries' argument checks that
return before any CUDA call, the manager's rejections on a host-only manager in their order, and the 40 instantiations in the
built library.  The GPU cases are in tests/test_gpu_gather_route.py."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import (ErrorCode, KvbmError, LayoutConfig, ShardWindow, StorageKind, TransferManager, TransferOptions,
                                  tile_reshard_plan, tp_pp_reshard_plan)

KV = K.KvBlockLayout
INVAL = K.CUDA_ERROR_INVALID_VALUE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO, ROW = 2, 128


def test_routed_gather_symbols_are_exported_and_listed():
    for name in ("kvbm_kernels_paged_stage_repage_gather_routed", "kvbm_kernels_paged_stage_repage_gather_routed_streamed"):
        assert name in K.EXPORTED_SYMBOLS and callable(getattr(K.lib(), name))
    assert "kvbm_manager_execute_repage_batch_routed" in P.EXPORTED_SYMBOLS
    assert callable(P.lib().kvbm_manager_execute_repage_batch_routed)


def test_the_route_seq_mirror_matches_the_c_struct():
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("needs a C compiler")
    names = ["token_begin", "token_end", "src_ids", "n_src", "dst_ids", "n_dst", "src_mask"]
    assert [f[0] for f in P._CRepageRouteSeq._fields_] == names
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "kvbm_physical.h"', "int main(void) {"]
    lines += [f'  printf("%zu\\n", offsetof(kvbm_repage_route_seq, {f}));' for f in names]
    lines += ['  printf("%zu\\n", sizeof(kvbm_repage_route_seq));', "  return 0;", "}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "s.c"), os.path.join(d, "s")
        with open(src, "w") as f:
            f.write("\n".join(lines))
        subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", "-o", exe, src], check=True)
        got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert got[:-1] == [getattr(P._CRepageRouteSeq, f).offset for f in names]
    assert got[-1] == C.sizeof(P._CRepageRouteSeq)


def test_tile_reshard_plan():
    one = tp_pp_reshard_plan(8, 4, 4, 1, 2, 1, 0)       # decode TP2 rank 0 from one TP4 prefill worker: ranks 0 and 1
    ranks = 4
    plan = tile_reshard_plan(one, 3, ranks)
    assert len(plan) == 3 * len(one)
    for w in range(3):
        for a, b in zip(one, plan[w * len(one):(w + 1) * len(one)]):
            assert b.src_rank == a.src_rank + w * ranks
            assert (b.src_layer_begin, b.dst_layer_begin, b.layer_count, b.src_head_begin, b.dst_head_begin, b.head_count) == (
                a.src_layer_begin, a.dst_layer_begin, a.layer_count, a.src_head_begin, a.dst_head_begin, a.head_count)
    with pytest.raises(ValueError):
        tile_reshard_plan(one, 2, 1)
    with pytest.raises(ValueError):
        tile_reshard_plan(one, 0, ranks)


# ---------------------------------------------------------------------------------------------------------------------
# the kernel entries' argument checks (descriptors no check dereferences)
# ---------------------------------------------------------------------------------------------------------------------
def _side(nh, nl, page, no=NO, ids=0x2000, base=0x1000):
    reg = page * nh * ROW
    return K.PermuteSide(K.PagedLayout(base, reg, 8 * reg, reg, nl, no, 8), ids, int(KV.OperationalNHD))


def _s(nh, nl, sb, db, k, sl, dl, c, page=16, **kw):
    return K.StageSource(K.PermuteSource(_side(nh, nl, page, **kw), nh, sb, db, k), sl, dl, c)


# two workers of one prefill rank each, both writing destination heads 0-1 of layers 0..4: overlapping windows of one stage
TWO = [_s(2, 4, 0, 0, 2, 0, 0, 4, ids=0x2100), _s(2, 4, 0, 0, 2, 0, 0, 4, ids=0x2200, base=0x1100)]
SEQS = [(0, 64, 0b01), (70, 130, 0b10)]


def _rg(srcs=TWO, seqs=SEQS, ps=16, pd=64, lb=0, le=4, cast=0, scales=None, units=None, streamed=None):
    if units is None:
        u = K.repage_route_units(seqs, ps, pd)
        units = (0x7000, len(u[0]) if u is not None else 0)
    d = _side(2, 4, pd)
    if streamed is not None:
        return K.paged_stage_repage_gather_routed_streamed(srcs, ps, d, 2, pd, seqs, *units, lb, le, ROW, cast, scales, streamed)
    return K.paged_stage_repage_gather_routed(srcs, ps, d, 2, pd, seqs, *units, lb, le, ROW, cast, scales)


def test_routed_gather_argument_checks_before_any_cuda_call():
    # nothing to move signals (nothing to signal here): no sequences, only empty ranges, an empty layer range
    assert _rg(seqs=[]) == 0 and _rg(seqs=[(9, 9, 1), (70, 70, 2)]) == 0 and _rg(lb=3, le=3) == 0
    # the routing: a mask of 0, a bit at num_srcs (2) or above, also on an empty sequence
    assert _rg(seqs=[(0, 64, 1), (70, 130, 0)]) == INVAL
    assert _rg(seqs=[(0, 64, 0b101), (70, 130, 1)]) == INVAL
    assert _rg(seqs=[(0, 64, 1 << 31)]) == INVAL
    assert _rg(seqs=[(0, 64, 1), (9, 9, 0)]) == INVAL
    assert _rg(seqs=[(0, 64, 1), (9, 9, 4)]) == INVAL
    # two overlapping windows of one stage in one mask, also when no other sequence routes them together
    assert _rg(seqs=[(0, 64, 0b11)]) == INVAL
    assert _rg(seqs=[(0, 64, 0b01), (70, 130, 0b11)]) == INVAL
    # (windows never routed together are accepted: these descriptors name no memory, so an accepted call would launch; the GPU
    # cases run such plans, and the manager's host case below reaches the strategy with one)
    # sixteen sources take bits 0..15, not bit 16
    sixteen = [_s(2, 4, 0, 0, 2, 0, 0, 4, ids=0x3000 + 0x100 * i, base=0x4000 + 0x100 * i) for i in range(16)]
    assert _rg(srcs=sixteen, seqs=[(0, 64, 1 << 16)]) == INVAL
    # 256 head-map entries counted over every window, overlapping ones included: three windows of 128 heads, each sequence routed
    # to one of them, still take 384 entries
    wide = [K.StageSource(K.PermuteSource(_side(128, 4, 16, ids=0x3000 + 0x100 * i), 128, 0, 0, 128), 0, 0, 4) for i in range(3)]
    seqs = [(0, 64, 1), (64, 128, 2), (128, 192, 4)]
    u = K.repage_route_units(seqs, 16, 64)
    assert K.paged_stage_repage_gather_routed(wide, 16, _side(128, 4, 64), 128, 64, seqs, 0x7000, len(u[0]), 0, 4, ROW) == INVAL
    # the batch's own rules: a reversed range, a unit count other than the helper's, a null unit table, a null seqs
    assert _rg(seqs=[(0, 64, 1), (9, 8, 1)], units=(0x7000, 2)) == INVAL
    assert _rg(units=(0x7000, 4)) == INVAL and _rg(units=(0, 2)) == INVAL
    arr = (K.StageSource * 2)(*TWO)
    assert K.lib().kvbm_kernels_paged_stage_repage_gather_routed(arr, 2, 16, C.byref(_side(2, 4, 64)), 2, 64, None, 2, 0x7000, 2, 0, 4, ROW, 0,
                                                                None, None, 0, None, 0, None) == INVAL
    # the gather's rules
    assert _rg(lb=3, le=2) == INVAL and _rg(le=5) == INVAL
    assert _rg(srcs=[]) == INVAL and _rg(srcs=[TWO[0]] * 17, seqs=[(0, 64, 1)]) == INVAL
    assert _rg(cast=3) == INVAL and _rg(scales=0x5000) == INVAL
    assert _rg(srcs=[_s(2, 4, 0, 0, 2, 0, 0, 2)], seqs=[(0, 64, 1)]) == INVAL       # layers 2..4 uncovered
    # the streamed entry: a null descriptor; ready flags only for the routed sources
    u = K.repage_route_units(SEQS, 16, 64)
    assert K.paged_stage_repage_gather_routed_streamed(TWO, 16, _side(2, 4, 64), 2, 64, SEQS, 0x7000, len(u[0]), 0, 4, ROW, 0, None, None) == INVAL
    assert _rg(streamed=K.PermuteStream()) == INVAL
    st = K.PermuteStream()
    st.layer_ready_flags[0] = 0x9000
    st.gate_mode = K.GATE_SPIN
    assert _rg(seqs=[(0, 64, 0b01)], streamed=st) == INVAL                           # no workspace for the spinning form
    st.gate_mode = 99
    assert _rg(seqs=[(0, 64, 0b01)], streamed=st) == INVAL
    st.gate_mode = K.GATE_SPIN
    st.sync_workspace = 0x9100
    assert _rg(seqs=[(0, 64, 0b10)], streamed=st) == INVAL                           # routed source 1 has no flags
    st.gate_mode = 99                                                                 # flags for source 0 alone pass the flag rule
    assert _rg(seqs=[(0, 64, 0b01)], streamed=st) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_repage_batch_routed on host memory: its rejections in order, with codes and texts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def host_pools():
    """a, b, c: sources, 4 layers, 2 heads, 16-token pages; d: the destination, 4 layers, 2 heads, 64; e: like d."""
    mgr = TransferManager(device=-1, worker_id=19)
    bufs, hs = [], []
    for nl, nh, page in ((4, 2, 16), (4, 2, 16), (4, 2, 16), (4, 2, 64), (4, 2, 64)):
        cfg = LayoutConfig(8, nl, 2, page, nh * 64, dtype_width_bytes=2, num_heads=nh)
        b = np.zeros(cfg.required_bytes(), dtype=np.uint8)
        h = mgr.register_fully_contiguous(cfg, b.ctypes.data, b.size, StorageKind.System, 0)
        mgr.set_kv_block_layout(h, KV.OperationalNHD)
        bufs.append(b)
        hs.append(h)
    yield mgr, hs
    mgr.close()


def _err(fn):
    with pytest.raises(KvbmError) as e:
        fn()
    return e.value


# two workers (sources 0 and 1) writing the destination's heads 0-1 over every layer; source 2 writes nothing
PLAN = [ShardWindow(0, 0, 0, 4, 0, 0, 2), ShardWindow(1, 0, 0, 4, 0, 0, 2)]
CUDA_ONLY = "direct CUDA strategy only"


def _c_call(mgr, hs, seqs, plan=PLAN, num_srcs=2, ls=None, dst=3):
    """The C entry with explicit masks and NULL lists: seqs are (tb, te, {src: ids}, dst_ids, mask)."""
    keep = []
    cs = (P._CRepageRouteSeq * max(1, len(seqs)))()
    for c, (tb, te, ids, dids, mask) in zip(cs, seqs):
        arrs = {r: (C.c_size_t * max(1, len(x)))(*x) for r, x in ids.items()}
        sp = (C.c_void_p * max(1, num_srcs))(*[C.addressof(arrs[r]) if r in arrs else None for r in range(num_srcs)])
        d = (C.c_size_t * max(1, len(dids)))(*dids)
        keep += [arrs, sp, d]
        n_src = len(next(iter(ids.values()))) if ids else 0
        c.token_begin, c.token_end, c.src_ids, c.n_src, c.dst_ids, c.n_dst, c.src_mask = tb, te, C.addressof(sp), n_src, C.addressof(d), len(dids), mask
    ws = (P._CShardWindow * len(plan))(*[P._CShardWindow(w.src_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin,
                                                          w.dst_head_begin, w.head_count) for w in plan])
    srcs = (C.c_uint64 * max(1, num_srcs))(*[hs[i] if i < 3 else 10_000 + i for i in range(num_srcs)])
    o, tok = TransferOptions()._c(), C.c_uint64()
    rc = P.lib().kvbm_manager_execute_repage_batch_routed(mgr._h, num_srcs, srcs, hs[dst] if dst < len(hs) else dst, cs, len(seqs), ws, len(plan),
                                                         ls, C.byref(o), C.byref(tok))
    return rc, P.lib().kvbm_last_error().decode()


def test_the_routing_rejections_in_order(host_pools):
    mgr, hs = host_pools
    S0 = (0, 64, {0: [0, 1, 2, 3]}, [5], 0b01)
    S1 = (64, 128, {1: [4, 5, 6, 7]}, [6], 0b10)
    zero = (64, 128, {}, [6], 0)
    # with ls, its shape first
    ls = P._CLayerStream(None, 2, None)
    rc, msg = _c_call(mgr, hs, [S0, zero], ls=C.byref(ls))
    assert rc == ErrorCode.ERR and "ready flags" in msg
    # then the windows' checks: a window naming a missing source, before the routing
    rc, msg = _c_call(mgr, hs, [S0, zero], plan=PLAN + [ShardWindow(2, 0, 0, 4, 0, 0, 2)])
    assert rc == ErrorCode.RANGE and "names source 2" in msg
    # partly overlapping layer windows stay rejected
    rc, msg = _c_call(mgr, hs, [S0], plan=[ShardWindow(0, 0, 0, 4, 0, 0, 2), ShardWindow(1, 0, 1, 3, 0, 0, 2)])
    assert rc == ErrorCode.OVERLAP and "partly overlap" in msg
    # then a null sequence list
    o, tok = TransferOptions()._c(), C.c_uint64()
    srcs = (C.c_uint64 * 2)(hs[0], hs[1])
    ws = (P._CShardWindow * 2)(*[P._CShardWindow(w.src_rank, 0, 0, 4, 0, 0, 2) for w in PLAN])
    assert P.lib().kvbm_manager_execute_repage_batch_routed(mgr._h, 2, srcs, hs[3], None, 2, ws, 2, None, C.byref(o), C.byref(tok)) == ErrorCode.ERR
    assert "null sequence list" in P.lib().kvbm_last_error().decode()
    # then more than 32 sources
    rc, msg = _c_call(mgr, hs, [S0, zero], num_srcs=33)
    assert rc == ErrorCode.UNSUPPORTED and "at most 32 sources" in msg
    # then, sequence by sequence, the routing
    rc, msg = _c_call(mgr, hs, [S0, zero])
    assert rc == ErrorCode.RANGE and "sequence 1 is routed to no source" in msg
    rc, msg = _c_call(mgr, hs, [S0, (64, 128, {}, [6], 0b100)])
    assert rc == ErrorCode.RANGE and "sequence 1 is routed past the 2 sources" in msg
    rc, msg = _c_call(mgr, hs, [S0, (64, 128, {2: [4, 5, 6, 7]}, [6], 0b100)], num_srcs=3)
    assert rc == ErrorCode.RANGE and "sequence 1 is routed to a source no window reads" in msg
    rc, msg = _c_call(mgr, hs, [S0, (64, 128, {0: [4, 5, 6, 7], 1: [4, 5, 6, 7]}, [6], 0b11)])
    assert rc == ErrorCode.OVERLAP and msg.endswith("windows 0 and 1 overlap in the destination")
    staged = [ShardWindow(0, 0, 0, 2, 0, 0, 2), ShardWindow(1, 0, 2, 2, 0, 0, 2)]
    rc, msg = _c_call(mgr, hs, [(0, 64, {0: [0, 1, 2, 3], 1: [0, 1, 2, 3]}, [5], 0b11), S0], plan=staged)
    assert rc == ErrorCode.RANGE and "destination layer 2 of the layer range is in no window's layers" in msg
    # the routing of a later sequence comes before the request checks of an earlier one
    rc, msg = _c_call(mgr, hs, [(0, 64, {0: [0, 1, 2]}, [5], 0b01), zero])
    assert rc == ErrorCode.RANGE and "routed to no source" in msg
    # then the single call's checks, sequence by sequence: the id counts, then the strategy of a non-empty sequence
    rc, msg = _c_call(mgr, hs, [(0, 64, {0: [0, 1, 2]}, [5], 0b01), S1])
    assert rc == ErrorCode.LENGTH_MISMATCH
    rc, msg = _c_call(mgr, hs, [S0, S1])
    assert rc == ErrorCode.UNSUPPORTED and CUDA_ONLY in msg
    # a routed source's ids are range-checked, an unrouted one's (NULL here) are not read
    rc, msg = _c_call(mgr, hs, [(0, 64, {0: [0, 1, 2, 9]}, [5], 0b01)])
    assert rc == ErrorCode.RANGE and "out of range for source" in msg
    rc, msg = _c_call(mgr, hs, [(0, 64, {0: [0, 1, 2, 3]}, [5], 0b01)])
    assert rc == ErrorCode.UNSUPPORTED and CUDA_ONLY in msg
    # a routed source whose list is NULL is a null list
    rc, msg = _c_call(mgr, hs, [(0, 64, {0: [0, 1, 2, 3]}, [5], 0b11)], plan=staged)
    assert rc == ErrorCode.ERR and "null block id list" in msg
    rc, msg = _c_call(mgr, hs, [(0, 64, {0: [0, 1, 2, 3]}, [5], 0b10)])
    assert rc == ErrorCode.ERR and "null block id list" in msg


def test_overlapping_windows_never_routed_together_pass_the_window_checks(host_pools):
    """The batch entry rejects the same plan as overlapping; the routed one gets as far as the strategy."""
    mgr, hs = host_pools
    seqs = [(range(0, 64), {0: [0, 1, 2, 3]}, [5]), (range(64, 128), {1: [4, 5, 6, 7]}, [6])]
    e = _err(lambda: mgr.execute_repage_batch({0: hs[0], 1: hs[1]}, hs[3], [(t, {0: a, 1: a}, d) for t, a, d in
                                                                           [(s[0], list(s[1].values())[0], s[2]) for s in seqs]], PLAN))
    assert e.code == ErrorCode.OVERLAP
    e = _err(lambda: mgr.execute_repage_batch_routed({0: hs[0], 1: hs[1]}, hs[3], seqs, PLAN))
    assert e.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in e.msg


def test_nothing_to_move_returns_at_once(host_pools):
    mgr, hs = host_pools
    srcs = {0: hs[0], 1: hs[1]}
    assert mgr.execute_repage_batch_routed(srcs, hs[3], [], PLAN) is not None
    assert mgr.execute_repage_batch_routed(srcs, hs[3], [(range(9, 9), {0: []}, []), (range(70, 70), {1: []}, [])], PLAN) is not None


# ---------------------------------------------------------------------------------------------------------------------
# the instantiations in the built library
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s, pp) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True)) for pp in (True, False)}
NEW = ("kvbm_paged_repage_fanin_kernel", "kvbm_gated_repage_fanin_kernel")
TAKEN = ("batch", "route", "scatter", "push_seqs", "_stage_")
MATRIX_FAMILIES = ("kvbm_paged_permute_kernel", "kvbm_paged_gather_kernel", "kvbm_gated_gather_kernel", "kvbm_paged_repage_kernel",
                   "kvbm_paged_repage_gather_kernel", "kvbm_gated_repage_gather_kernel", "kvbm_permute_table_kernel", "kvbm_permute_kernel")


def test_the_fanin_instantiations_are_what_the_library_contains():
    """40 kernels: the 20 walks of with_repage_kernel for each of the two families; tests/test_gpu_gather_route.py reaches each.
    No new name contains a substring other tests filter the library's kernels by, nor equals a family they count."""
    so = os.path.join(ROOT, "dynamo_b200", "libkvbm_kernels.so")
    tool = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
    if not os.path.exists(so) or tool is None:
        pytest.skip("needs the built libkvbm_kernels.so and cuobjdump")
    txt = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    found = set()
    for name in re.findall(r"Function : (\S+)", txt):
        m = re.search(r"(kvbm_[a-z0-9_]+?_kernel)I((?:L[ib]\d+E)+)E", name)
        if m and "fanin" in m.group(1):
            assert m.group(1) in NEW
            c, p, s, pp = (int(v) if t == "i" else v == "1" for t, v in re.findall(r"L([ib])(\d+)E", m.group(2)))
            found.add((m.group(1), c, p, s, pp))
    assert len(WALKS) == 20 and found == {(k,) + w for k in NEW for w in WALKS}
    assert not any(s in k for k in NEW for s in TAKEN)
    assert not set(NEW) & set(MATRIX_FAMILIES)

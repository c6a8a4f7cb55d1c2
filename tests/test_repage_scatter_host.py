"""CPU checks of the re-paging scatter (one prefill rank's KV to every decode rank that needs it): the exported symbols and ctypes
struct sizes, the scatter plan as the exact inverse of the gather plans, the kernel entry's argument checks that return before any
CUDA call, the manager's rejections on a host-only manager with the first rejection pinned for requests that fail two checks, and
the instantiations in the built library.  The accepted neighbours of the kernel's rejections (16 targets, 256 pairs, one pool in
two disjoint targets, stages that split across decode stages) launch on the GPU in tests/test_gpu_repage_scatter.py: an accepted
call here would launch on descriptors no kernel may dereference."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import (ErrorCode, KvbmError, LayoutConfig, ScatterWindow, StorageKind, TransferManager, TransferOptions,
                                  tp_pp_reshard_plan, tp_pp_scatter_plan)

KV = K.KvBlockLayout
INVAL = K.CUDA_ERROR_INVALID_VALUE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_scatter_symbols_are_exported_and_listed():
    assert "kvbm_kernels_paged_repage_scatter" in K.EXPORTED_SYMBOLS and callable(K.lib().kvbm_kernels_paged_repage_scatter)
    for name in ("kvbm_tp_pp_scatter_plan", "kvbm_manager_execute_repage_scatter"):
        assert name in P.EXPORTED_SYMBOLS and callable(getattr(P.lib(), name))


def test_struct_sizes():
    """kvbm_scatter_target: a 56-byte side, seven u32 and a pointer at 88; kvbm_scatter_window: seven size_t."""
    assert C.sizeof(K.PermuteSide) == 56
    assert K.ScatterTarget.done_flag.offset == 88 and C.sizeof(K.ScatterTarget) == 96
    assert C.sizeof(P._CScatterWindow) == 7 * C.sizeof(C.c_size_t)


# ---------------------------------------------------------------------------------------------------------------------
# the plan: the inverse of the gather plans
# ---------------------------------------------------------------------------------------------------------------------
TPS = (1, 2, 4, 8, 16)


def _union_both(H, L, stp, spp, dtp, dpp, sparts=None, dparts=None):
    pull, push = set(), set()
    for d in range(dtp * dpp):
        for w in tp_pp_reshard_plan(H, L, stp, spp, dtp, dpp, d, sparts, dparts):
            pull.add((w.src_rank, d, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count))
    for s in range(stp * spp):
        plan = tp_pp_scatter_plan(H, L, stp, spp, dtp, dpp, s, sparts, dparts)
        keys = [(w.dst_rank, w.dst_layer_begin, w.dst_head_begin) for w in plan]
        assert keys == sorted(keys)
        for w in plan:
            push.add((s, w.dst_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count))
    return pull, push


@pytest.mark.parametrize("H", [1, 2, 4, 8, 16, 64])
def test_the_scatter_plans_are_the_gather_plans_inverted(H):
    for stp in TPS:
        for dtp in TPS:
            pull, push = _union_both(H, 4, stp, 1, dtp, 1)
            assert push == pull and pull


@pytest.mark.parametrize("spp,dpp,sparts,dparts", [(2, 3, None, None), (3, 2, [3, 3, 6], None), (2, 4, [5, 7], [2, 4, 3, 3]),
                                                    (4, 1, [1, 2, 4, 5], None), (1, 3, None, [1, 1, 10])])
def test_pp_splits_invert_too(spp, dpp, sparts, dparts):
    for H, stp, dtp in ((8, 2, 4), (4, 4, 1), (2, 1, 8), (1, 2, 2)):
        pull, push = _union_both(H, 12, stp, spp, dtp, dpp, sparts, dparts)
        assert push == pull and pull


def test_scatter_plan_shapes_and_errors():
    # H = 8, TP2 -> TP16: rank 0's heads 0..3, each to the two decode ranks that hold it
    plan = tp_pp_scatter_plan(8, 4, 2, 1, 16, 1, 0)
    assert [(w.dst_rank, w.src_head_begin, w.head_count) for w in plan] == [(d, d // 2, 1) for d in range(8)]
    # MLA: one head on every decode rank
    assert [w.dst_rank for w in tp_pp_scatter_plan(1, 61, 1, 1, 8, 1, 0)] == list(range(8))
    with pytest.raises(KvbmError) as e:
        tp_pp_scatter_plan(8, 4, 2, 1, 4, 1, 2)
    assert e.value.code == ErrorCode.RANGE and "src_rank 2" in e.value.msg
    with pytest.raises(KvbmError) as e:
        tp_pp_scatter_plan(6, 4, 4, 1, 2, 1, 0)
    assert e.value.code == ErrorCode.CONFIG
    with pytest.raises(KvbmError) as e:
        tp_pp_scatter_plan(8, 5, 2, 2, 2, 1, 0)
    assert e.value.code == ErrorCode.CONFIG
    n = C.c_size_t()
    assert P.lib().kvbm_tp_pp_scatter_plan(8, 4, 1, 1, None, 8, 1, None, 0, None, 0, C.byref(n)) == 0 and n.value == 8
    out = (P._CScatterWindow * 7)()
    assert P.lib().kvbm_tp_pp_scatter_plan(8, 4, 1, 1, None, 8, 1, None, 0, out, 7, C.byref(n)) == ErrorCode.ERR


# ---------------------------------------------------------------------------------------------------------------------
# the kernel entry's argument checks (descriptors no check dereferences)
# ---------------------------------------------------------------------------------------------------------------------
NO, ROW = 2, 128


def _side(nh, nl, page, no=NO, ids=0x2000, base=0x1000, region=None):
    reg = region if region is not None else page * nh * ROW
    return K.PermuteSide(K.PagedLayout(base, reg, 8 * reg, reg, nl, no, 8), ids, int(KV.OperationalNHD))


def _t(nh, nl, sb, db, k, sl, dl, c, page=64, **kw):
    return K.ScatterTarget(_side(nh, nl, page, **kw), nh, sb, db, k, sl, dl, c, None)


def _sc(targets, src_nh=4, src_nl=6, ps=16, pd=64, tb=0, te=64, lb=0, le=6, cast=0, scales=None, src=None):
    return K.paged_repage_scatter(src or _side(src_nh, src_nl, ps), src_nh, ps, targets, pd, tb, te, lb, le, ROW, cast, scales)


# stage 0: source layers 0..4 to two decode ranks (heads 0-1 and 2-3); stage 1: layers 4..6 to a third
OK = [_t(2, 4, 0, 0, 2, 0, 0, 4, ids=0x2100), _t(2, 4, 2, 0, 2, 0, 0, 4, ids=0x2200, base=0x1100), _t(2, 2, 0, 0, 2, 4, 0, 2, base=0x1200)]


def test_scatter_argument_checks_before_any_cuda_call():
    assert _sc(OK, tb=9, te=9) == 0 and _sc(OK, lb=3, le=3) == 0          # empty ranges signal (nothing to signal here)
    assert _sc(OK, tb=9, te=8) == INVAL
    assert _sc(OK, lb=4, le=3) == INVAL
    assert _sc([]) == INVAL
    assert _sc([OK[0]] * 17) == INVAL
    assert _sc(OK, cast=3) == INVAL                                       # an unknown cast
    assert K.paged_repage_scatter(_side(4, 6, 16), 4, 16, OK, 64, 0, 64, 0, 6, ROW, 0, 0x5000) == INVAL   # scales without a cast
    # pages where neither divides the other; a zero page
    assert _sc([_t(2, 4, 0, 0, 2, 0, 0, 4, page=24), _t(2, 4, 2, 0, 2, 0, 0, 4, page=24, ids=9), _t(2, 2, 0, 0, 2, 4, 0, 2, page=24)],
               pd=24) == INVAL
    assert _sc(OK, ps=0, src=_side(4, 6, 16)) == INVAL
    # rows and strides: a source region that is not its page * heads * row, a row that is not whole 16 B vectors
    assert _sc(OK, src=_side(4, 6, 32)) == INVAL
    assert K.paged_repage_scatter(_side(4, 6, 16), 4, 16, OK, 64, 0, 64, 0, 6, 120, 0, None) == INVAL
    # a layer range past the source's layers; a destination region or outer_dim other than its own
    assert _sc(OK, le=7) == INVAL
    assert _sc(OK[:2] + [_t(2, 2, 0, 0, 2, 4, 0, 2, page=32)]) == INVAL
    assert _sc(OK[:2] + [_t(2, 2, 0, 0, 2, 4, 0, 2, no=1)]) == INVAL
    # empty or out-of-range head windows
    assert _sc(OK[:2] + [_t(2, 2, 0, 0, 0, 4, 0, 2)]) == INVAL
    assert _sc(OK[:2] + [_t(2, 2, 3, 0, 2, 4, 0, 2)]) == INVAL            # past the source's 4 heads
    assert _sc(OK[:2] + [_t(2, 2, 0, 1, 2, 4, 0, 2)]) == INVAL            # past the destination's 2
    # empty or out-of-range layer windows
    assert _sc(OK[:2] + [_t(2, 2, 0, 0, 2, 4, 0, 0)]) == INVAL
    assert _sc(OK[:2] + [_t(2, 2, 0, 0, 2, 5, 0, 2)]) == INVAL            # past the source's 6 layers
    assert _sc(OK[:2] + [_t(2, 2, 0, 0, 2, 4, 1, 2)]) == INVAL            # past the destination's 2
    # two stages whose source layer windows overlap partly; a source layer no stage covers
    assert _sc(OK[:2] + [_t(2, 2, 0, 0, 2, 3, 0, 2)]) == INVAL
    assert _sc(OK[:2]) == INVAL
    assert _sc(OK[:2], lb=2, le=5) == INVAL
    # two targets on one pool and table whose destination rectangles overlap (another table, or disjoint heads, pass the check)
    assert _sc([OK[0], _t(2, 4, 2, 1, 1, 0, 0, 4, ids=0x2100), OK[1], OK[2]]) == INVAL
    assert _sc([OK[0], _t(2, 4, 2, 1, 1, 0, 3, 1, ids=0x2100)] + OK[1:]) == INVAL


def test_scatter_pair_limit():
    """257 (target, head) pairs over all stages, each stage within the limit: rejected; the 256 of the limit case launch on the GPU."""
    src = _side(200, 2, 16)
    big = [K.ScatterTarget(_side(200, 2, 64, ids=0x100 * (i + 1)), 200, 0, 0, 129 if i == 0 else 128, i, 0, 1, None) for i in range(2)]
    assert K.paged_repage_scatter(src, 200, 16, big, 64, 0, 64, 0, 2, ROW, 0, None) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_repage_scatter on host memory: its rejections, with codes and texts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def host_pools():
    """a: the source, 6 layers, 4 heads, 16-token pages; b, c: 4 layers, 2 heads, 64; d: 2 layers, 2 heads, 64; e: 2 layers,
    2 heads, 32-token pages."""
    mgr = TransferManager(device=-1, worker_id=14)
    no, hd = 2, 64
    bufs, hs = [], []
    for nl, nh, page in ((6, 4, 16), (4, 2, 64), (4, 2, 64), (2, 2, 64), (2, 2, 32)):
        cfg = LayoutConfig(8, nl, no, page, nh * hd, dtype_width_bytes=2, num_heads=nh)
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


# stage 0: source layers 0..4, heads 0-1 to b and 2-3 to c; stage 1: layers 4..6, heads 0-1 to d
PLAN = [ScatterWindow(0, 0, 0, 4, 0, 0, 2), ScatterWindow(1, 0, 0, 4, 2, 0, 2), ScatterWindow(2, 4, 0, 2, 0, 0, 2)]
CUDA_ONLY = "direct CUDA strategy only"


def _go(mgr, hs, plan, o=None, tokens=range(0, 64), n_src=4, dsts=(1, 2, 3), dst_ids=None):
    ids = dst_ids if dst_ids is not None else [[5]] * len(dsts)
    return mgr.execute_repage_scatter(hs[0], list(range(n_src)), [hs[i] if i < len(hs) else 999 for i in dsts], ids, plan, tokens, o)


def test_manager_repage_scatter_rejections(host_pools):
    mgr, hs = host_pools
    go = lambda *a, **kw: _go(mgr, hs, *a, **kw)  # noqa: E731
    # a well-formed request passes every check down to the strategy: per-destination flags are honoured, the range is the source's
    for o in (None, TransferOptions(layer_range=range(2, 5)), TransferOptions(per_dst_done_flags=[0, 0, 0])):
        e = _err(lambda: go(PLAN, o))
        assert e.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in e.msg
    e = _err(lambda: go([]))
    assert e.code == ErrorCode.ERR and "at least one destination" in e.msg
    e = _err(lambda: go(PLAN, TransferOptions(head_window=(0, 0, 1))))
    assert e.code == ErrorCode.ERR and "head_count must be 0" in e.msg
    e = _err(lambda: go([ScatterWindow(0, 0, 0, 1, 0, 0, 1)] * 17))
    assert e.code == ErrorCode.UNSUPPORTED and "at most 16" in e.msg
    e = _err(lambda: go(PLAN[:2] + [ScatterWindow(3, 4, 0, 2, 0, 0, 2)]))
    assert e.code == ErrorCode.RANGE and "names destination 3" in e.msg
    e = _err(lambda: go(PLAN[:2] + [ScatterWindow(2, 4, 0, 2, 0, 0, 0)]))
    assert e.code == ErrorCode.RANGE and "no heads" in e.msg
    e = _err(lambda: go(PLAN[:2] + [ScatterWindow(2, 4, 0, 0, 0, 0, 2)]))
    assert e.code == ErrorCode.RANGE and "no layers" in e.msg
    e = _err(lambda: go(PLAN[:2] + [ScatterWindow(2, 3, 0, 2, 0, 0, 2)]))
    assert e.code == ErrorCode.OVERLAP and "partly overlap" in e.msg
    e = _err(lambda: go(PLAN + [ScatterWindow(0, 0, 0, 4, 3, 1, 1)]))
    assert e.code == ErrorCode.OVERLAP and "overlap in destination 0" in e.msg
    e = _err(lambda: go(PLAN, dsts=(1, 1, 3)))
    assert e.code == ErrorCode.OVERLAP and "one layout" in e.msg
    e = _err(lambda: go(PLAN, dsts=(1, 2, 9)))
    assert e.code == ErrorCode.HANDLE
    e = _err(lambda: go(PLAN[:2] + [ScatterWindow(2, 4, 0, 3, 0, 0, 2)]))             # past a's 6 layers
    assert e.code == ErrorCode.RANGE and "source's num_layers" in e.msg
    e = _err(lambda: go(PLAN[:2] + [ScatterWindow(2, 4, 1, 2, 0, 0, 2)]))             # past d's 2 layers
    assert e.code == ErrorCode.RANGE and "destination's num_layers" in e.msg
    e = _err(lambda: go(PLAN[:2]))                                                    # source layers 4..6 uncovered
    assert e.code == ErrorCode.RANGE and "source layer 4" in e.msg
    e = _err(lambda: go([ScatterWindow(0, 0, 0, 4, 3, 0, 2)] + PLAN[1:]))             # past a's 4 heads: the pair's check
    assert e.code == ErrorCode.RANGE and "Head window" in e.msg
    e = _err(lambda: go(PLAN, dsts=(1, 2, 4)))                                        # e's 32-token pages
    assert e.code == ErrorCode.INCOMPATIBLE and "one page size" in e.msg
    for o in (TransferOptions(layer_done_flags=0x100), TransferOptions(layer_ready_flags=0x100), TransferOptions(multicast=1)):
        e = _err(lambda: go(PLAN, o))
        assert e.code == ErrorCode.UNSUPPORTED and "layer streaming" in e.msg
    e = _err(lambda: go(PLAN, tokens=range(70, 64)))
    assert e.code == ErrorCode.RANGE and "Token range" in e.msg
    e = _err(lambda: go(PLAN, TransferOptions(layer_range=range(0, 7))))
    assert e.code == ErrorCode.RANGE and "exceeds num_layers 6" in e.msg
    e = _err(lambda: go(PLAN, n_src=3))
    assert e.code == ErrorCode.LENGTH_MISMATCH and "span 4 source and 1 destination blocks" in e.msg
    e = _err(lambda: go(PLAN, tokens=range(0, 128), n_src=8, dst_ids=[[5, 6], [5, 5], [5, 6]]))
    assert e.code == ErrorCode.DUPLICATE_DST
    e = _err(lambda: go(PLAN, dst_ids=[[5], [8], [5]]))
    assert e.code == ErrorCode.RANGE and "out of range for destination" in e.msg
    # an empty token or layer range moves nothing
    assert go(PLAN, tokens=range(9, 9), n_src=0, dst_ids=[[], [], []]) is not None
    assert go(PLAN, TransferOptions(layer_range=range(4, 4))) is not None


def test_manager_repage_scatter_first_rejection(host_pools):
    """Requests that fail two checks report the earlier one, in the documented order."""
    mgr, hs = host_pools
    go = lambda *a, **kw: _go(mgr, hs, *a, **kw)  # noqa: E731
    # 1. the windows before the handles
    e = _err(lambda: go(PLAN + [ScatterWindow(0, 0, 0, 4, 3, 1, 1)], dsts=(1, 2, 9)))
    assert e.code == ErrorCode.OVERLAP
    # 2. the handles before the layer windows
    e = _err(lambda: go(PLAN[:2], dsts=(1, 2, 9)))
    assert e.code == ErrorCode.HANDLE
    # 3. the layer windows before the pairs (an uncovered layer and a head window past a's heads)
    e = _err(lambda: go([ScatterWindow(0, 0, 0, 4, 3, 0, 2), PLAN[1]]))
    assert e.code == ErrorCode.RANGE and "source layer 4" in e.msg
    # 4. the pair before the one page size
    e = _err(lambda: go(PLAN[:2] + [ScatterWindow(2, 4, 0, 2, 3, 0, 2)], dsts=(1, 2, 4)))
    assert e.code == ErrorCode.RANGE and "Head window" in e.msg
    # 5. the one page size before the token range
    e = _err(lambda: go(PLAN, tokens=range(70, 64), dsts=(1, 2, 4)))
    assert e.code == ErrorCode.INCOMPATIBLE and "one page size" in e.msg
    # 6. the token range before the layer range
    e = _err(lambda: go(PLAN, TransferOptions(layer_range=range(0, 7)), tokens=range(70, 64)))
    assert e.code == ErrorCode.RANGE and "Token range" in e.msg
    # 7. the source's layer range before the id counts
    e = _err(lambda: go(PLAN, TransferOptions(layer_range=range(0, 7)), n_src=3))
    assert e.code == ErrorCode.RANGE and "exceeds num_layers 6" in e.msg
    # 8. the id counts before the strategy
    e = _err(lambda: go(PLAN, n_src=3))
    assert e.code == ErrorCode.LENGTH_MISMATCH


# ---------------------------------------------------------------------------------------------------------------------
# the instantiations in the built library
# ---------------------------------------------------------------------------------------------------------------------
EXPECTED = {(c, p, s, pp) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True)) for pp in (True, False)}


def test_the_scatter_instantiations_are_what_the_library_contains():
    """20 kernels: the walks of with_walk_kernel x the small page's split; tests/test_gpu_repage_scatter.py reaches each."""
    assert len(EXPECTED) == 20
    so = os.path.join(ROOT, "dynamo_b200", "libkvbm_kernels.so")
    tool = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
    if not os.path.exists(so) or tool is None:
        pytest.skip("needs the built libkvbm_kernels.so and cuobjdump")
    txt = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    found = set()
    for name in re.findall(r"Function : (\S+)", txt):
        m = re.search(r"(kvbm_[a-z0-9_]+?_kernel)I((?:L[ib]\d+E)+)E", name)
        if m and "scatter" in m.group(1):
            assert m.group(1) == "kvbm_paged_repage_scatter_kernel"
            c, p, s, pp = (int(v) if t == "i" else v == "1" for t, v in re.findall(r"L([ib])(\d+)E", m.group(2)))
            found.add((c, p, s, pp))
    assert found == EXPECTED

"""CPU checks of the staged re-paging gather (a PP x TP re-shard across engines with different page sizes): the exported
symbols, the oracle against the re-paging gather's and the staged gather's oracles, the kernel entry's argument checks that
return before any CUDA call, the instantiations in the built library, and the manager's rejections on a host-only manager with
the first rejection pinned for requests that fail two checks."""

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, KvbmError, LayoutConfig, ShardWindow, StorageKind, TransferManager, TransferOptions
from tests.cast_oracle import dst_row_bytes
from tests.repage_gather_oracle import repage_gather
from tests.stage_oracle import stage_block
from tests.stage_repage_oracle import stage_repage_gather

KV = K.KvBlockLayout
INVAL = K.CUDA_ERROR_INVALID_VALUE
KINDS = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]


def test_stage_repage_symbols_are_exported_and_listed():
    for name in ("kvbm_kernels_paged_stage_repage_gather", "kvbm_kernels_paged_stage_repage_gather_streamed"):
        assert name in K.EXPORTED_SYMBOLS and callable(getattr(K.lib(), name))
    assert "kvbm_manager_execute_stage_repage_gather" in P.EXPORTED_SYMBOLS
    assert callable(P.lib().kvbm_manager_execute_stage_repage_gather)


# ---------------------------------------------------------------------------------------------------------------------
# the oracle against its neighbours
# ---------------------------------------------------------------------------------------------------------------------
def _blocks(rng, n, nl, no, page, nh, row):
    return [rng.integers(0, 256, nl * no * page * nh * row, dtype=np.uint8) for _ in range(n)]


@pytest.mark.parametrize("cast", [0, 1, 2])
@pytest.mark.parametrize("ps,pd,tb,te", [(16, 64, 5, 120), (64, 16, 70, 128), (1, 16, 3, 29), (12, 48, 13, 90)])
def test_an_identity_plan_is_the_repage_gather(ps, pd, tb, te, cast):
    rng = np.random.default_rng(ps + pd + cast)
    nl, no, hd = 3, 2, 16
    se = 1 if cast == 1 else 2
    row = hd * se
    n_s, n_d = -(-te // ps) - tb // ps, -(-te // pd) - tb // pd
    srcs = [(_blocks(rng, n_s, nl, no, ps, 2, row), int(KINDS[s]), 2) for s in range(2)]
    dst = _blocks(rng, n_d, nl, no, pd, 3, dst_row_bytes(row, cast))
    heads = [(0, 0, 0, 2), (1, 1, 2, 1)]
    scales = rng.uniform(0.5, 2, nl * no).astype(np.float32) if cast else None
    want = repage_gather(srcs, heads, dst, int(KV.OperationalNHD), 3, nl, no, ps, pd, row, tb, te, cast, scales, range(1, 3))
    got = stage_repage_gather([(b, kv, nh, nl) for b, kv, nh in srcs], [(s, 0, 0, nl, sb, db, k) for s, sb, db, k in heads], dst,
                              int(KV.OperationalNHD), 3, nl, no, ps, pd, row, tb, te, cast, scales, range(1, 3))
    assert all(np.array_equal(a, b) for a, b in zip(got, want))


@pytest.mark.parametrize("cast", [0, 2])
def test_one_page_over_whole_blocks_is_the_staged_gather(cast):
    """PP2 x TP2 -> TP1 with 3-layer sources into a 6-layer destination, equal pages, whole blocks."""
    rng = np.random.default_rng(cast)
    no, page, hd, n = 2, 8, 16, 3
    row = hd * 2
    d_row = dst_row_bytes(row, cast)
    windows = [(0, 0, 0, 3, 0, 0, 2), (1, 0, 0, 3, 0, 2, 2), (2, 0, 3, 3, 0, 0, 2), (3, 0, 3, 3, 0, 2, 2)]
    kvs = [KV.OperationalHND, KV.UniversalPP, KV.OperationalNHD, KV.UniversalTP]
    srcs = [(_blocks(rng, n, 3, no, page, 2, row), int(kvs[s]), 2, 3) for s in range(4)]
    dst = _blocks(rng, n, 6, no, page, 4, d_row)
    scales = rng.uniform(0.5, 2, 6 * no).astype(np.float32) if cast else None
    got = stage_repage_gather(srcs, windows, dst, int(KV.OperationalHND), 4, 6, no, page, page, row, 0, n * page, cast, scales, range(1, 5))
    for i in range(n):
        blk = dst[i]
        for s, sl, dl, c, sb, db, k in windows:
            blk = stage_block(srcs[s][0][i], blk, srcs[s][1], int(KV.OperationalHND), 3, 6, no, page, 2, 4, row, cast,
                              (sl, dl, c, sb, db, k), layers=range(1, 5), scales=scales)
        assert np.array_equal(got[i], blk)


# ---------------------------------------------------------------------------------------------------------------------
# the kernel entry's argument checks (descriptors no check dereferences)
# ---------------------------------------------------------------------------------------------------------------------
NO, ROW = 2, 128


def _side(nh, nl, page, no=NO, ids=0x2000, base=0x1000):
    reg = page * nh * ROW
    return K.PermuteSide(K.PagedLayout(base, reg, 8 * reg, reg, nl, no, 8), ids, int(KV.OperationalNHD))


def _ss(nh, nl, hb, db, k, sl, dl, c, page=16, **kw):
    return K.StageSource(K.PermuteSource(_side(nh, nl, page, **kw), nh, hb, db, k), sl, dl, c)


def _srg(srcs, dst_nh=4, dst_nl=8, ps=16, pd=64, tb=0, te=64, lb=0, le=8):
    return K.paged_stage_repage_gather(srcs, ps, _side(dst_nh, dst_nl, pd), dst_nh, pd, tb, te, lb, le, ROW)


def test_stage_repage_argument_checks_before_any_cuda_call():
    # PP2 x TP2 -> TP1 over 8 layers: stage 0 is layers 0..4 of two 4-layer sources, stage 1 layers 4..8 of two more
    ok = [_ss(2, 4, 0, 0, 2, 0, 0, 4), _ss(2, 4, 0, 2, 2, 0, 0, 4), _ss(2, 4, 0, 0, 2, 0, 4, 4), _ss(2, 4, 0, 2, 2, 0, 4, 4)]
    assert _srg(ok, tb=9, te=9) == 0 and _srg(ok, lb=3, le=3) == 0     # empty ranges signal (nothing to signal here)
    assert _srg(ok, tb=9, te=8) == INVAL
    assert _srg([]) == INVAL
    assert _srg([ok[0]] * 17) == INVAL
    # pages where neither divides the other
    assert _srg([_ss(2, 4, 0, 0, 2, 0, 0, 4, page=24), _ss(2, 4, 0, 2, 2, 0, 0, 4, page=24), _ss(2, 4, 0, 0, 2, 0, 4, 4, page=24),
                 _ss(2, 4, 0, 2, 2, 0, 4, 4, page=24)], ps=24) == INVAL
    # a partial layer overlap
    assert _srg([_ss(2, 4, 0, 0, 2, 0, 0, 4), _ss(2, 4, 0, 2, 2, 0, 0, 4), _ss(2, 4, 0, 0, 2, 0, 3, 4), _ss(2, 4, 0, 2, 2, 0, 4, 4)]) == INVAL
    # an uncovered layer: layers 4..8 in no window
    assert _srg(ok[:2]) == INVAL
    assert _srg(ok[:2], lb=2, le=5) == INVAL
    # windows past the source's layers and past the destination's; a window without layers
    assert _srg(ok[:3] + [_ss(2, 4, 0, 2, 2, 1, 4, 4)]) == INVAL
    assert _srg(ok[:3] + [_ss(2, 8, 0, 2, 2, 0, 5, 4)]) == INVAL
    assert _srg([_ss(2, 4, 0, 0, 2, 0, 0, 0)] + ok[1:]) == INVAL
    # head overlap within a stage (across stages the same heads are the point)
    assert _srg([ok[0], _ss(2, 4, 0, 1, 2, 0, 0, 4), ok[2], ok[3]]) == INVAL
    # 257 covered heads summed over stages, each stage within the limit
    big = [_ss(300, 4, 0, 0, 129, 0, 0, 4), _ss(300, 4, 0, 0, 128, 0, 4, 4)]
    assert K.paged_stage_repage_gather(big, 16, _side(300, 8, 64), 300, 64, 0, 64, 0, 8, ROW) == INVAL
    # a source region that is not its own page * heads * row, and a differing outer_dim
    assert _srg(ok[:3] + [_ss(2, 4, 0, 2, 2, 0, 4, 4, page=32)]) == INVAL
    assert _srg(ok[:3] + [_ss(2, 4, 0, 2, 2, 0, 4, 4, no=1)]) == INVAL
    # the streamed entry: the gate's rules, each on an otherwise well-formed call
    stream = lambda st: K.paged_stage_repage_gather_streamed(ok, 16, _side(4, 8, 64), 4, 64, 0, 64, 0, 8, ROW, 0, None, st)  # noqa: E731
    assert stream(None) == INVAL
    st = K.PermuteStream()
    for j in range(4):
        st.layer_ready_flags[j] = 0x3000 + 64 * j
    st.gate_mode = 7
    assert stream(st) == INVAL
    st.gate_mode = K.GATE_SPIN                      # the spinning form without a workspace
    assert stream(st) == INVAL
    st.sync_workspace = 0x4000
    st.layer_ready_flags[3] = 0                      # a used source without ready flags
    assert stream(st) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_stage_repage_gather on host memory: its rejections, with codes and texts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def host_pools():
    """a, b: 3 layers, 2 heads, 16-token pages; c: 5 layers, 2 heads, 16; d: the destination, 8 layers, 4 heads, 64-token pages;
    e: 5 layers, 2 heads, 8-token pages; f: 5 layers, 2 heads, 24-token pages."""
    mgr = TransferManager(device=-1, worker_id=13)
    no, hd = 2, 64
    bufs, hs = [], []
    for nl, nh, page in ((3, 2, 16), (3, 2, 16), (5, 2, 16), (8, 4, 64), (5, 2, 8), (5, 2, 24)):
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


# stage 0: layers 0..3 of a and b (heads 0-1 and 2-3); stage 1: layers 0..5 of c as destination layers 3..8, both head pairs
PLAN = [ShardWindow(0, 0, 0, 3, 0, 0, 2), ShardWindow(1, 0, 0, 3, 0, 2, 2), ShardWindow(2, 0, 3, 5, 0, 0, 2), ShardWindow(2, 0, 3, 5, 0, 2, 2)]
CUDA_ONLY = "direct CUDA strategy only"


def _go(mgr, hs, plan, o=None, tokens=range(0, 64), n_src=4, third=2, dst_ids=(5,), **kw):
    a, b, c, d, e, f = hs
    third_h = (a, b, c, d, e, f)[third]
    src = {0: (a, list(range(n_src))), 1: (b, list(range(1, n_src + 1))), 2: (third_h, list(range(2, n_src + 2)))}
    return mgr.execute_stage_repage_gather(src, d, list(dst_ids), plan, tokens, o, **kw)


def test_manager_stage_repage_rejections(host_pools):
    mgr, hs = host_pools
    go = lambda *a, **kw: _go(mgr, hs, *a, **kw)  # noqa: E731
    # a well-formed request passes every check down to the strategy: the layer counts differ, the range is the destination's
    for o in (None, TransferOptions(layer_range=range(2, 6))):
        e = _err(lambda: go(PLAN, o))
        assert e.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in e.msg
    e = _err(lambda: go([PLAN[0], ShardWindow(1, 0, 0, 3, 0, 1, 2)] + PLAN[2:]))
    assert e.code == ErrorCode.OVERLAP and "overlap in the destination" in e.msg
    e = _err(lambda: go(PLAN[:2] + [ShardWindow(2, 0, 2, 5, 0, 0, 2), PLAN[3]]))
    assert e.code == ErrorCode.OVERLAP and "partly overlap" in e.msg
    e = _err(lambda: go(PLAN[:2] + [ShardWindow(2, 0, 3, 0, 0, 0, 2)]))
    assert e.code == ErrorCode.RANGE and "no layers" in e.msg
    e = _err(lambda: go([ShardWindow(0, 0, 0, 1, 0, 0, 1)] * 17))
    assert e.code == ErrorCode.UNSUPPORTED and "at most 16" in e.msg
    e = _err(lambda: go(PLAN[:2] + [ShardWindow(2, 1, 3, 5, 0, 0, 2), PLAN[3]]))          # past c's 5 layers
    assert e.code == ErrorCode.RANGE and "source's num_layers" in e.msg
    e = _err(lambda: go(PLAN[:2] + [ShardWindow(2, 0, 4, 5, 0, 0, 2), ShardWindow(2, 0, 4, 5, 0, 2, 2)]))   # past the destination's 8
    assert e.code == ErrorCode.RANGE and "destination's num_layers" in e.msg
    e = _err(lambda: go(PLAN[:2]))                                                         # layers 3..8 uncovered
    assert e.code == ErrorCode.RANGE and "destination layer 3" in e.msg
    e = _err(lambda: go([ShardWindow(0, 0, 0, 3, 1, 0, 2)] + PLAN[1:]))                   # past a's heads: the pair's check
    assert e.code == ErrorCode.RANGE and "Head window" in e.msg
    e = _err(lambda: go(PLAN, third=4))                                                    # e's 8-token pages
    assert e.code == ErrorCode.INCOMPATIBLE and "one page size" in e.msg
    e = _err(lambda: go(PLAN, tokens=range(70, 64)))
    assert e.code == ErrorCode.RANGE and "Token range" in e.msg
    e = _err(lambda: go(PLAN, TransferOptions(layer_range=range(0, 9))))
    assert e.code == ErrorCode.RANGE and "exceeds num_layers 8" in e.msg
    e = _err(lambda: go(PLAN, n_src=3))
    assert e.code == ErrorCode.LENGTH_MISMATCH and "span 4 source and 1 destination blocks" in e.msg
    e = _err(lambda: go(PLAN, ready_flags={0: 0, 1: 0, 2: 0}))
    assert e.code == ErrorCode.ERR and "no layer ready flags" in e.msg
    # an empty token or layer range moves nothing
    assert go(PLAN, tokens=range(9, 9), n_src=0, dst_ids=()) is not None
    assert go(PLAN, TransferOptions(layer_range=range(4, 4))) is not None


def test_manager_stage_repage_first_rejection(host_pools):
    """Requests that fail two checks report the earlier one, in the documented order."""
    mgr, hs = host_pools
    go = lambda *a, **kw: _go(mgr, hs, *a, **kw)  # noqa: E731
    overlap = [PLAN[0], ShardWindow(1, 0, 0, 3, 0, 1, 2)] + PLAN[2:]
    # 1. the layer stream's shape before the windows
    e = _err(lambda: go(overlap, ready_flags={0: 0, 1: 0, 2: 0}))
    assert e.code == ErrorCode.ERR and "no layer ready flags" in e.msg
    # 2. the windows before the stage layers (a window also past a's layers)
    e = _err(lambda: go([ShardWindow(0, 1, 0, 3, 0, 0, 2), ShardWindow(1, 0, 0, 3, 0, 1, 2)] + PLAN[2:]))
    assert e.code == ErrorCode.OVERLAP
    # 3. the stage layers before the pairs (an uncovered layer and a head window past a's heads)
    e = _err(lambda: go([ShardWindow(0, 0, 0, 3, 1, 0, 2), PLAN[1]]))
    assert e.code == ErrorCode.RANGE and "destination layer 3" in e.msg
    # 4. the pair before the one page size, in window order
    e = _err(lambda: go(PLAN[:2] + [ShardWindow(2, 0, 3, 5, 1, 0, 2), PLAN[3]], third=4))
    assert e.code == ErrorCode.RANGE and "Head window" in e.msg
    e = _err(lambda: go(PLAN, third=5))                                                    # f's 24-token pages: neither divides 64
    assert e.code == ErrorCode.INCOMPATIBLE and "divide" in e.msg
    # 5. the one page size before the token range
    e = _err(lambda: go(PLAN, tokens=range(70, 64), third=4))
    assert e.code == ErrorCode.INCOMPATIBLE and "one page size" in e.msg
    # 6. the token range before the layer range
    e = _err(lambda: go(PLAN, TransferOptions(layer_range=range(0, 9)), tokens=range(70, 64)))
    assert e.code == ErrorCode.RANGE and "Token range" in e.msg
    # 7. the destination's layer range before the id counts
    e = _err(lambda: go(PLAN, TransferOptions(layer_range=range(0, 9)), n_src=3))
    assert e.code == ErrorCode.RANGE and "exceeds num_layers 8" in e.msg
    # 8. the id counts before the strategy
    e = _err(lambda: go(PLAN, n_src=3))
    assert e.code == ErrorCode.LENGTH_MISMATCH

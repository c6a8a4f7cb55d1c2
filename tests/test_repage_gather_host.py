"""CPU checks of re-paging with the gather's head windows (kvbm_kernels_paged_repage_gather, kvbm_manager_execute_repage_gather):
the oracle against the re-paging and re-shard oracles it is built from, the exported symbols, the kernel's argument checks that
return before any CUDA call, and the manager's rejection table on a host-only manager, where every check runs before the missing
device is reported."""
import ctypes as C
import itertools

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, HeadWindow, KvbmError, StorageKind, TransferOptions, tp_reshard_plan
from tests.repage_gather_oracle import repage_gather, split_heads
from tests.repage_oracle import repage, table_slice
from tests.reshard_oracle import rank_heads, reshard_block
from tests.test_repage_host import host_mgr  # noqa: F401  (the host-only manager fixture)

KV = K.KvBlockLayout
ALL = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]
INVAL = K.CUDA_ERROR_INVALID_VALUE


def _blocks(rng, count, nl, no, page, nh, row):
    return [rng.integers(0, 256, nl * no * page * nh * row, dtype=np.uint8) for _ in range(count)]


# ---------------------------------------------------------------------------------------------------------------------
# the oracle against the two it is built from
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ps,pd,tb,te", [(16, 64, 5, 120), (64, 16, 7, 100), (1, 16, 3, 40), (48, 16, 17, 90)])
def test_one_full_window_is_the_plain_repage(ps, pd, tb, te):
    nl, no, nh, row = 2, 2, 3, 16
    rng = np.random.default_rng(ps + pd)
    src = _blocks(rng, -(-te // ps) - tb // ps, nl, no, ps, nh, row)
    old = _blocks(rng, -(-te // pd) - tb // pd, nl, no, pd, nh, row)
    for skv, dkv in [(KV.OperationalNHD, KV.UniversalPP), (KV.UniversalTP, KV.OperationalHND)]:
        want = repage(src, old, int(skv), int(dkv), nl, no, nh, ps, pd, row, tb, te, layers=range(1, 2))
        got = repage_gather([(src, int(skv), nh)], [(0, 0, 0, nh)], old, int(dkv), nh, nl, no, ps, pd, row, tb, te, layers=range(1, 2))
        assert all(np.array_equal(a, b) for a, b in zip(got, want))


def test_equal_pages_over_whole_blocks_is_reshard_block_per_block():
    nl, no, page, row, dnh = 2, 2, 4, 16, 5
    rng = np.random.default_rng(3)
    nb = 3
    srcs = [(_blocks(rng, nb, nl, no, page, 4, row), int(KV.OperationalNHD), 4), (_blocks(rng, nb, nl, no, page, 2, row), int(KV.UniversalPP), 2)]
    windows = [(0, 1, 0, 2), (1, 0, 3, 2)]             # destination head 2 is covered by neither
    old = _blocks(rng, nb, nl, no, page, dnh, row)
    got = repage_gather(srcs, windows, old, int(KV.OperationalHND), dnh, nl, no, page, page, row, 0, nb * page)
    for i in range(nb):
        blk = old[i]
        for s, sb, db, k in windows:
            blocks, kv, nh = srcs[s]
            blk = reshard_block(blocks[i], blk, kv, int(KV.OperationalHND), nl, no, page, nh, dnh, row, 0, sb, db, k)
        assert np.array_equal(got[i], blk)


PAGE_PAIRS = [(a, b) for a, b in itertools.product([1, 16, 48, 64], repeat=2) if a % b == 0 or b % a == 0]


@pytest.mark.parametrize("ps,pd", PAGE_PAIRS, ids=lambda p: str(p))
@pytest.mark.parametrize("src_kv,dst_kv", list(itertools.product(ALL, ALL)), ids=lambda k: k.name)
def test_tp_split_and_reassembly_is_the_plain_repage(src_kv, dst_kv, ps, pd):
    """A TP1 sequence split at page Ps into TP2 / 4 / 8 ranks and reassembled at page Pd through tp_reshard_plan's windows is the
    plain re-page of the TP1 sequence."""
    H, nl, no, row = 8, 1, 2, 16
    tb, te = 5, 2 * max(ps, pd) + 3
    rng = np.random.default_rng(ps * 131 + pd + 7 * int(src_kv) + int(dst_kv))
    full = _blocks(rng, -(-te // ps) - tb // ps, nl, no, ps, H, row)       # TP1, in UniversalTP
    old = _blocks(rng, -(-te // pd) - tb // pd, nl, no, pd, H, row)
    want = repage(full, old, int(KV.UniversalTP), int(dst_kv), nl, no, H, ps, pd, row, tb, te)
    for tp in (2, 4, 8):
        sources = [(split_heads(full, int(KV.UniversalTP), nl, no, ps, H, row, rank_heads(H, tp, r), int(src_kv)), int(src_kv), H // tp)
                   for r in range(tp)]
        windows = [(w.src_rank, w.src_head_begin, w.dst_head_begin, w.head_count) for w in tp_reshard_plan(H, tp, 1, 0)]
        got = repage_gather(sources, windows, old, int(dst_kv), H, nl, no, ps, pd, row, tb, te)
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), tp


# ---------------------------------------------------------------------------------------------------------------------
# the kernel's argument checks (host descriptors nothing dereferences)
# ---------------------------------------------------------------------------------------------------------------------
def test_repage_gather_symbols_are_exported_and_listed():
    assert "kvbm_kernels_paged_repage_gather" in K.EXPORTED_SYMBOLS
    assert "kvbm_manager_execute_repage_gather" in P.EXPORTED_SYMBOLS
    assert callable(K.lib().kvbm_kernels_paged_repage_gather) and callable(P.lib().kvbm_manager_execute_repage_gather)


NL, NO, ROW = 2, 2, 128


def _side(page, nh, kv=KV.OperationalNHD, row=ROW, nl=NL, no=NO, ids=0x2000, base=0x1000, region=None):
    reg = page * nh * row if region is None else region
    return K.PermuteSide(K.PagedLayout(base, reg, 8 * reg, reg, nl, no, 8), ids, int(kv))


def _src(page=16, nh=2, sb=0, db=0, k=2, **kw):
    return K.PermuteSource(_side(page, nh, **kw), nh, sb, db, k)


def _rg(srcs, ps=16, dst=None, dnh=4, pd=64, tb=0, te=32, lb=0, le=NL, row=ROW, cast=0, scales=None):
    dst = _side(pd, dnh) if dst is None else dst
    return K.paged_repage_gather(srcs, ps, dst, dnh, pd, tb, te, lb, le, row, cast, cast_scales=scales)


def test_repage_gather_argument_checks_before_any_cuda_call():
    two = [_src(db=0), _src(db=2)]
    # ranges, cast mode, scales without a cast
    assert _rg(two, tb=5, te=4) == INVAL
    assert _rg(two, lb=1, le=0) == INVAL
    assert _rg(two, lb=-1) == INVAL
    assert _rg(two, cast=3) == INVAL
    assert _rg(two, scales=0x4000) == INVAL
    # source count: none, more than 16
    assert _rg([]) == INVAL
    assert _rg([_src(db=i % 4, k=1) for i in range(17)]) == INVAL
    # an empty token or layer range moves nothing (no flags: nothing to launch)
    assert _rg(two, tb=7, te=7) == 0 and _rg(two, lb=1, le=1) == 0
    # null destination, tables and bases
    L = K.lib()
    arr = (K.PermuteSource * 2)(*two)
    assert L.kvbm_kernels_paged_repage_gather(arr, 2, 16, None, 4, 64, 0, 32, 0, NL, ROW, 0, None, None, 0, None, 0, None) == INVAL
    assert _rg(two, dst=_side(64, 4, ids=0)) == INVAL
    assert _rg([_src(ids=0), _src(db=2)]) == INVAL
    assert _rg([_src(), _src(db=2, base=0)]) == INVAL
    # windows: no heads, past either side's heads, overlapping in the destination, more than 256 covered heads
    assert _rg([_src(k=0), _src(db=2)]) == INVAL
    assert _rg([_src(sb=1, k=2), _src(db=2)]) == INVAL
    assert _rg([_src(), _src(db=3)]) == INVAL
    assert _rg([_src(), _src(db=1)]) == INVAL
    wide = [_src(nh=160, k=160, db=0, region=16 * 160 * ROW), _src(nh=160, k=160, db=160, region=16 * 160 * ROW)]
    assert _rg(wide, dnh=320, dst=_side(64, 320)) == INVAL
    # pages: zero, neither dividing the other
    assert _rg([_src(page=1, region=2 * ROW * 16), _src(page=1, db=2, region=2 * ROW * 16)], ps=0) == INVAL
    assert _rg([_src(page=48), _src(page=48, db=2)], ps=48) == INVAL
    assert _rg(two, pd=0, dst=_side(64, 4)) == INVAL
    # geometry: layers / outer dims differ, a layer range past num_layers
    assert _rg([_src(nl=NL + 1), _src(db=2)]) == INVAL
    assert _rg([_src(), _src(db=2, no=1)]) == INVAL
    assert _rg(two, le=NL + 1) == INVAL
    # region = page * heads * row on each side, at that side's page and head count
    assert _rg(two, dst=_side(32, 4)) == INVAL
    assert _rg(two, dst=_side(64, 3)) == INVAL
    assert _rg([_src(), _src(db=2, region=16 * 2 * ROW + 16)]) == INVAL
    assert _rg([_src(row=64), _src(row=64, db=2)], dst=_side(64, 4, row=64), row=64, cast=int(K.CastMode.FP8E4M3_TO_BF16)) == INVAL
    # rows: 8 B, past 64 KiB, an odd bf16 row under the down cast
    assert _rg([_src(row=8), _src(row=8, db=2)], dst=_side(64, 4, row=8), row=8) == INVAL
    assert _rg([_src(row=ROW + 8), _src(row=ROW + 8, db=2)], dst=_side(64, 4, row=ROW + 8), row=ROW + 8) == INVAL
    odd = ROW + 1
    assert _rg([_src(row=odd), _src(row=odd, db=2)], dst=_side(64, 4, row=odd // 2), row=odd, cast=int(K.CastMode.BF16_TO_FP8E4M3)) == INVAL
    # unnamed formats, on a source or the destination
    for kv in (KV.Unknown, KV.Custom):
        assert _rg([_src(), _src(db=2, kv=kv)]) == INVAL
        assert _rg(two, dst=_side(64, 4, kv=kv)) == INVAL
    # the range's last big block must end below 2^32 tokens
    assert _rg(two, tb=2**32 - 70, te=2**32 - 1) == INVAL


def test_repage_gather_caps_one_full_window_at_256_heads():
    """One window over every head of both sides runs the plain re-page's kernel, which kvbm_kernels_paged_repage launches with
    no head limit; through the gather entry it still covers at most 256 heads."""
    nh = K.GATHER_MAX_HEADS + 1
    assert _rg([_src(nh=nh, k=nh, region=16 * nh * ROW)], dnh=nh, dst=_side(64, nh)) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_repage_gather on a host-only manager: every rejection, then the missing device
# ---------------------------------------------------------------------------------------------------------------------
def _err(fn):
    with pytest.raises(KvbmError) as e:
        fn()
    return e.value


def test_manager_repage_gather_rejections(host_mgr):  # noqa: F811
    mgr, reg = host_mgr
    # TP2 at page 16 (2 heads per rank) -> TP1 at page 64 (4 heads); tokens 5..40: 3 source blocks, 1 destination block
    s0, s1, d = reg(16, nh=2), reg(16, nh=2), reg(64, nh=4)
    plan = tp_reshard_plan(4, 2, 1, 0)
    ok = dict(sources={0: (s0, [0, 1, 2]), 1: (s1, [3, 4, 5])}, dst=d, dst_block_ids=[3], plan=plan, tokens=range(5, 40))

    def call(**kw):
        a = dict(ok)
        a.update(kw)
        return lambda: mgr.execute_repage_gather(a["sources"], a["dst"], a["dst_block_ids"], a["plan"], a["tokens"], a.get("options"))

    # the gather's window checks, with its codes and texts
    e = _err(call(plan=[]))
    assert e.code == ErrorCode.ERR and "at least one source and one window" in e.msg
    e = _err(call(options=TransferOptions(head_window=(0, 0, 2))))
    assert e.code == ErrorCode.ERR and "options.head_count must be 0" in e.msg
    e = _err(call(plan=[HeadWindow(0, 0, 0, 1)] * 17))
    assert e.code == ErrorCode.UNSUPPORTED and "at most 16 windows" in e.msg
    e = _err(call(plan=[HeadWindow(0, 0, 0, 0)]))
    assert e.code == ErrorCode.RANGE and "has no heads" in e.msg
    e = _err(call(plan=[HeadWindow(0, 0, 0, 2), HeadWindow(1, 0, 1, 2)]))
    assert e.code == ErrorCode.OVERLAP and "overlap in the destination" in e.msg
    hs = (C.c_uint64 * 1)(s0)
    ws = (P._CHeadWindow * 1)(P._CHeadWindow(1, 0, 0, 2))
    rc = P.lib().kvbm_manager_execute_repage_gather(mgr._h, 1, hs, None, 0, d, None, 0, 0, 0, ws, 1, C.byref(P._COptions()), None)
    assert rc == ErrorCode.RANGE and b"names source 1 of 1" in P.lib().kvbm_last_error()
    # HANDLE
    assert _err(call(dst=0xDEAD)).code == ErrorCode.HANDLE
    assert _err(call(sources={0: (0xDEAD, [0, 1, 2]), 1: (s1, [3, 4, 5])})).code == ErrorCode.HANDLE
    # execute_repage's pair checks, with its texts
    for o in (TransferOptions(layer_ready_flags=0x1000), TransferOptions(multicast=1), TransferOptions(bounce_buffer=(d, [0]))):
        e = _err(call(options=o))
        assert e.code == ErrorCode.UNSUPPORTED and "re-paging transfer takes no" in e.msg
    e = _err(call(sources={0: (s0, [0, 1, 2]), 1: (reg(16, nh=2, kv=None), [3, 4, 5])}))
    assert e.code == ErrorCode.UNSUPPORTED and "named KV block layouts" in e.msg
    e = _err(call(dst=reg(64, nh=4, hd=128, elem=1)))
    assert e.code == ErrorCode.INCOMPATIBLE and "equal num_heads, head_dim and dtype" in e.msg
    e = _err(call(dst=reg(64, nh=2, hd=128)))
    assert e.code == ErrorCode.INCOMPATIBLE and "Head row" in e.msg
    e = _err(call(dst=reg(24, nh=4), dst_block_ids=[0]))
    assert e.code == ErrorCode.INCOMPATIBLE and "divide" in e.msg
    e = _err(call(dst=reg(64, nh=4, nl=3)))
    assert e.code == ErrorCode.INCOMPATIBLE and "layer counts" in e.msg
    e = _err(call(dst=reg(64, nh=4, fc=False), options=TransferOptions(dst_kv_layout=int(KV.UniversalTP))))
    assert e.code == ErrorCode.INCOMPATIBLE and "fully contiguous" in e.msg
    # the window inside both sides' heads
    e = _err(call(plan=[HeadWindow(0, 1, 0, 2)]))
    assert e.code == ErrorCode.RANGE and "Head window" in e.msg
    e = _err(call(plan=[HeadWindow(0, 0, 3, 2)]))
    assert e.code == ErrorCode.RANGE and "Head window" in e.msg
    # new: sources with different page sizes
    e = _err(call(sources={0: (s0, [0, 1, 2]), 1: (reg(32, nh=2), [3, 4, 5])}))
    assert e.code == ErrorCode.INCOMPATIBLE and "one page size" in e.msg
    # ranges, with execute_repage's texts
    assert _err(call(tokens=range(9, 5))).code == ErrorCode.RANGE
    e = _err(call(options=TransferOptions(layer_range=range(0, 3))))
    assert e.code == ErrorCode.RANGE and "Layer range" in e.msg
    e = _err(call(options=TransferOptions(cast_scales=np.ones(4, np.float32))))
    assert e.code == ErrorCode.ERR and "need a cast_mode" in e.msg
    # new: id counts other than the range implies for Ps / Pd
    e = _err(call(sources={0: (s0, [0, 1]), 1: (s1, [3, 4])}))
    assert e.code == ErrorCode.LENGTH_MISMATCH and "3 source and 1 destination" in e.msg
    assert _err(call(dst_block_ids=[3, 4])).code == ErrorCode.LENGTH_MISMATCH
    assert _err(call(sources={0: (s0, [0, 1, 2]), 1: (s1, [3, 4])})).code == ErrorCode.LENGTH_MISMATCH
    # ids, per source against the destination's
    e = _err(call(sources={0: (s0, [0, 1, 2]), 1: (s1, [3, 4, 8])}))
    assert e.code == ErrorCode.RANGE and "for source" in e.msg
    e = _err(call(dst_block_ids=[8]))
    assert e.code == ErrorCode.RANGE and "for destination" in e.msg
    # empty token / layer ranges: nothing to move, accepted before the strategy
    assert mgr.execute_repage_gather({0: (s0, []), 1: (s1, [])}, d, [], plan, range(7, 7)).is_complete()
    assert mgr.execute_repage_gather(ok["sources"], d, [3], plan, range(5, 40), TransferOptions(layer_range=range(1, 1))).is_complete()
    # strategy: host pools take Memcpy, which has no re-paging launch
    h0, h1, hd = reg(16, nh=2, storage=StorageKind.System), reg(16, nh=2, storage=StorageKind.System), reg(64, nh=4, storage=StorageKind.System)
    e = _err(call(sources={0: (h0, [0, 1, 2]), 1: (h1, [3, 4, 5])}, dst=hd))
    assert e.code == ErrorCode.UNSUPPORTED and "direct CUDA strategy" in e.msg
    # CUDA: a host-only manager, after every other check
    e = _err(call())
    assert e.code == ErrorCode.CUDA and "without a CUDA device" in e.msg
    assert mgr.bytes_moved() == 0 and mgr.h2d_bytes() == 0


def test_manager_repage_gather_keeps_execute_repage_rejecting_windows(host_mgr):  # noqa: F811
    """execute_repage itself still rejects a head window, and still requires equal head counts."""
    mgr, reg = host_mgr
    s, d = reg(16, nh=2), reg(64, nh=4)
    e = _err(lambda: mgr.execute_repage(s, [0, 1, 2], d, [3], range(5, 40)))
    assert e.code == ErrorCode.INCOMPATIBLE and "equal num_heads" in e.msg


def test_manager_repage_gather_null_id_lists(host_mgr):  # noqa: F811
    mgr, reg = host_mgr
    s0, d = reg(16, nh=2), reg(64, nh=4)
    hs = (C.c_uint64 * 1)(s0)
    ws = (P._CHeadWindow * 1)(P._CHeadWindow(0, 0, 0, 2))
    tok = C.c_uint64()
    rc = P.lib().kvbm_manager_execute_repage_gather(mgr._h, 1, hs, None, 1, d, None, 1, 0, 16, ws, 1, C.byref(P._COptions()), C.byref(tok))
    assert rc == ErrorCode.ERR and b"null block id list" in P.lib().kvbm_last_error()
    PP = C.POINTER(C.c_size_t)
    ids = (PP * 1)(None)
    did = (C.c_size_t * 1)(3)
    rc = P.lib().kvbm_manager_execute_repage_gather(mgr._h, 1, hs, ids, 1, d, did, 1, 0, 16, ws, 1, C.byref(P._COptions()), C.byref(tok))
    assert rc == ErrorCode.ERR and b"null block id list" in P.lib().kvbm_last_error()
    assert P.lib().kvbm_manager_execute_repage_gather(None, 0, None, None, 0, 0, None, 0, 0, 0, None, 0, None, None) == ErrorCode.ERR


def test_table_slices_of_a_tp_group():
    """Every source of a TP group takes the same slice of its own table: the positions are the same, the ids its own."""
    tabs = [list(range(100 * r, 100 * r + 10)) for r in range(4)]
    assert [table_slice(t, 5, 40, 16) for t in tabs] == [[0, 1, 2], [100, 101, 102], [200, 201, 202], [300, 301, 302]]

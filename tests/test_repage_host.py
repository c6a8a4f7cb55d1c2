"""CPU checks of re-paging (kvbm_kernels_paged_repage, kvbm_manager_execute_repage): the oracle against a hand-derived case, the
exported symbols, the kernel's argument checks that return before any CUDA call, and the manager's rejection table on a host-only
manager, where every check runs before the missing device is reported."""
import ctypes as C

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, KvbmError, LayoutConfig, StorageKind, TransferManager, TransferOptions
from oracle import oracle as O
from tests.repage_oracle import repage, table_slice

KV = K.KvBlockLayout
INVAL = K.CUDA_ERROR_INVALID_VALUE


# ---------------------------------------------------------------------------------------------------------------------
# the oracle, pinned by a case derived by hand
# ---------------------------------------------------------------------------------------------------------------------
def _stamp(p, l, o, h, row):
    """The bytes token p of (layer l, outer o, head h) carries: its position, then its (l, o, h)."""
    b = np.zeros(row, dtype=np.uint8)
    b[0], b[1], b[2], b[3], b[4] = p & 0xFF, p >> 8, l, o, h
    b[5:] = (p * 7 + l * 3 + o * 5 + h) & 0xFF
    return b


@pytest.mark.parametrize("src_page,dst_page,src_kv,dst_kv", [(3, 6, KV.OperationalNHD, KV.OperationalHND),
                                                               (8, 2, KV.UniversalTP, KV.OperationalNHD),
                                                               (4, 4, KV.OperationalHND, KV.UniversalPP),
                                                               (1, 5, KV.UniversalPP, KV.UniversalTP)])
def test_oracle_matches_a_hand_derived_case(src_page, dst_page, src_kv, dst_kv):
    nl, no, nh, row = 2, 2, 3, 16
    tb, te = 5, 17
    order = {KV.UniversalTP: "hlot", KV.UniversalPP: "lhot", KV.OperationalHND: "loht", KV.OperationalNHD: "loth"}

    def block(kv, page, first_token, fill=None):
        size = {"h": nh, "l": nl, "o": no, "t": page}
        shape = [size[c] for c in order[kv]] + [row]
        a = np.full(shape, 0xEE, dtype=np.uint8) if fill is not None else np.zeros(shape, dtype=np.uint8)
        if fill is None:
            for idx in np.ndindex(*shape[:4]):
                d = dict(zip(order[kv], idx))
                a[idx] = _stamp(first_token + d["t"], d["l"], d["o"], d["h"], row)
        return a

    s_first, d_first = tb // src_page, -(-te // dst_page)
    src = [block(src_kv, src_page, (s_first + i) * src_page).reshape(-1) for i in range(-(-te // src_page) - s_first)]
    dst_old = [block(dst_kv, dst_page, 0, fill=True).reshape(-1) for _ in range(d_first - tb // dst_page)]
    got = repage(src, dst_old, int(src_kv), int(dst_kv), nl, no, nh, src_page, dst_page, row, tb, te)
    for i, blk in enumerate(got):
        shape = [{"h": nh, "l": nl, "o": no, "t": dst_page}[c] for c in order[dst_kv]] + [row]
        a = blk.reshape(shape)
        for idx in np.ndindex(*shape[:4]):
            d = dict(zip(order[dst_kv], idx))
            p = (tb // dst_page + i) * dst_page + d["t"]
            want = _stamp(p, d["l"], d["o"], d["h"], row) if tb <= p < te else np.full(row, 0xEE, dtype=np.uint8)
            assert np.array_equal(a[idx], want), (i, d, p)


def test_oracle_layer_range_and_table_slice():
    assert table_slice(list(range(100, 110)), 5, 17, 4) == [101, 102, 103, 104]
    assert table_slice(list(range(100, 110)), 16, 17, 16) == [101]
    assert table_slice(list(range(100, 110)), 7, 7, 4) == []
    nl, no, nh, row = 3, 1, 1, 16
    src = [np.arange(nl * no * 4 * nh * row, dtype=np.uint8)]
    old = [np.full(nl * no * 4 * nh * row, 0x11, dtype=np.uint8)]
    out = repage(src, old, 4, 4, nl, no, nh, 4, 4, row, 0, 4, layers=range(1, 2))[0].reshape(nl, no, 4, nh, row)
    assert np.array_equal(out[1], src[0].reshape(nl, no, 4, nh, row)[1])
    assert (out[0] == 0x11).all() and (out[2] == 0x11).all()


# ---------------------------------------------------------------------------------------------------------------------
# the kernel's argument checks (host descriptors nothing dereferences)
# ---------------------------------------------------------------------------------------------------------------------
def test_repage_symbols_are_exported_and_listed():
    assert "kvbm_kernels_paged_repage" in K.EXPORTED_SYMBOLS
    assert "kvbm_manager_execute_repage" in P.EXPORTED_SYMBOLS
    assert callable(K.lib().kvbm_kernels_paged_repage) and callable(P.lib().kvbm_manager_execute_repage)


NL, NO, NH, ROW = 2, 2, 4, 128


def _side(page, kv=KV.OperationalNHD, nh=NH, row=ROW, nl=NL, no=NO, ids=0x2000, base=0x1000, region=None):
    reg = page * nh * row if region is None else region
    return K.PermuteSide(K.PagedLayout(base, reg, 8 * reg, reg, nl, no, 8), ids, int(kv))


def _rp(src, ps, dst, pd, tb=0, te=32, lb=0, le=NL, nh=NH, row=ROW, cast=0, scales=None):
    return K.paged_repage(src, ps, dst, pd, tb, te, lb, le, nh, row, cast, cast_scales=scales)


def test_repage_argument_checks_before_any_cuda_call():
    s16, d64 = _side(16), _side(64)
    # ranges, cast mode, scales without a cast
    assert _rp(s16, 16, d64, 64, tb=5, te=4) == INVAL
    assert _rp(s16, 16, d64, 64, lb=1, le=0) == INVAL
    assert _rp(s16, 16, d64, 64, lb=-1) == INVAL
    assert _rp(s16, 16, d64, 64, cast=3) == INVAL
    assert _rp(s16, 16, d64, 64, scales=0x4000) == INVAL
    # an empty token or layer range moves nothing (no flags: nothing to launch)
    assert _rp(s16, 16, d64, 64, tb=7, te=7) == 0 and _rp(s16, 16, d64, 64, lb=1, le=1) == 0
    # null sides, tables and bases
    L = K.lib()
    assert L.kvbm_kernels_paged_repage(None, 16, C.byref(d64), 64, 0, 32, 0, NL, NH, ROW, 0, None, None, 0, None, 0, None) == INVAL
    assert _rp(_side(16, ids=0), 16, d64, 64) == INVAL
    assert _rp(s16, 16, _side(64, base=0), 64) == INVAL
    # page sizes: zero, neither dividing the other
    assert _rp(_side(1, region=NH * ROW * 16), 0, d64, 64) == INVAL
    assert _rp(_side(48), 48, d64, 64) == INVAL
    # geometry: layers / outer dims differ, a layer range past num_layers, no heads
    assert _rp(_side(16, nl=NL + 1), 16, d64, 64) == INVAL
    assert _rp(_side(16, no=1), 16, d64, 64) == INVAL
    assert _rp(s16, 16, d64, 64, le=NL + 1) == INVAL
    assert _rp(s16, 16, d64, 64, nh=0) == INVAL
    # region = page * heads * row on each side (the cast's destination row doubles)
    assert _rp(s16, 16, _side(32), 64) == INVAL
    assert _rp(_side(16, region=16 * NH * ROW + 16), 16, d64, 64) == INVAL
    assert _rp(_side(16, row=64), 16, _side(64, row=64), 64, row=64, cast=int(K.CastMode.FP8E4M3_TO_BF16)) == INVAL
    # rows: 8 B, past 64 KiB, an odd bf16 row under the down cast
    assert _rp(_side(16, row=8), 16, _side(64, row=8), 64, row=8) == INVAL
    assert _rp(_side(16, row=ROW + 8), 16, _side(64, row=ROW + 8), 64, row=ROW + 8) == INVAL
    assert _rp(_side(16, row=ROW + 1), 16, _side(64, row=(ROW + 1) // 2), 64, row=ROW + 1, cast=int(K.CastMode.BF16_TO_FP8E4M3)) == INVAL
    # unnamed formats, strides that are not whole 16 B vectors
    for kv in (KV.Unknown, KV.Custom):
        assert _rp(_side(16, kv=kv), 16, d64, 64) == INVAL
        assert _rp(s16, 16, _side(64, kv=kv), 64) == INVAL
    # the range's last big block must end below 2^32 tokens
    assert _rp(s16, 16, d64, 64, tb=2**32 - 70, te=2**32 - 1) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_repage on a host-only manager: every rejection, then the missing device
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def host_mgr():
    mgr = TransferManager(device=-1, worker_id=21)
    bufs = []

    def reg(page, nh=4, hd=64, elem=2, storage=StorageKind.Device, kv=KV.OperationalNHD, fc=True, num_heads=None, nb=8, nl=2):
        cfg = LayoutConfig(nb, nl, 2, page, nh * hd, dtype_width_bytes=elem, num_heads=nh if num_heads is None else num_heads,
                           allow_fp8=(elem == 1))
        b = np.zeros(cfg.required_bytes() + 64, dtype=np.uint8)
        base = (b.ctypes.data + 63) // 64 * 64
        bufs.append(b)
        if fc:
            h = mgr.register_fully_contiguous(cfg, base, cfg.required_bytes(), storage, 0)
        else:
            per = nb * 2 * page * nh * hd * elem
            ls = [np.zeros(per + 64, dtype=np.uint8) for _ in range(nl)]
            bufs.extend(ls)
            h = mgr.register_layer_separate(cfg, [(x.ctypes.data + 63) // 64 * 64 for x in ls], [per] * nl,
                                            P.BlockDimension.BlockIsSecondDim, storage, 0)
        if kv is not None and (num_heads is None or num_heads):
            mgr.set_kv_block_layout(h, kv)
        return h

    yield mgr, reg
    mgr.close()


def _err(fn):
    with pytest.raises(KvbmError) as e:
        fn()
    return e.value


def test_manager_repage_rejections(host_mgr):
    mgr, reg = host_mgr
    s16, d64 = reg(16), reg(64)
    ok = dict(src=s16, src_block_ids=[0, 1, 2], dst=d64, dst_block_ids=[3], tokens=range(5, 40))

    def call(**kw):
        a = dict(ok)
        a.update(kw)
        return lambda: mgr.execute_repage(a["src"], a["src_block_ids"], a["dst"], a["dst_block_ids"], a["tokens"], a.get("options"))

    # HANDLE
    assert _err(call(src=0xDEAD)).code == ErrorCode.HANDLE
    assert _err(call(dst=0xDEAD)).code == ErrorCode.HANDLE
    # UNSUPPORTED: rejected options, unnamed formats
    for o in (TransferOptions(head_window=(0, 0, 2)), TransferOptions(layer_ready_flags=0x1000), TransferOptions(layer_done_flags=0x1000),
              TransferOptions(multicast=1), TransferOptions(per_dst_done_flags=[0x1000]), TransferOptions(per_dst_layer_done_flags=[0x1000]),
              TransferOptions(bounce_buffer=(d64, [0]))):
        e = _err(call(options=o))
        assert e.code == ErrorCode.UNSUPPORTED and "re-paging transfer takes no" in e.msg
    e = _err(call(src=reg(16, kv=None)))
    assert e.code == ErrorCode.UNSUPPORTED and "named KV block layouts" in e.msg
    e = _err(call(options=TransferOptions(dst_kv_layout=int(KV.Custom))))
    assert e.code == ErrorCode.UNSUPPORTED and "dst=Custom" in e.msg
    # CONFIG: num_heads missing or not dividing inner_dim
    assert _err(call(src=reg(16, num_heads=0, kv=None), options=TransferOptions(src_kv_layout=int(KV.OperationalNHD)))).code == ErrorCode.CONFIG
    assert _err(call(dst=reg(64, num_heads=3, kv=None), options=TransferOptions(dst_kv_layout=int(KV.OperationalNHD)))).code == ErrorCode.CONFIG
    # INCOMPATIBLE: layers, head row, heads, dtype, cast dtype, pages that do not divide, universal on a layer-separate pool
    assert _err(call(dst=reg(64, nl=3))).code == ErrorCode.INCOMPATIBLE
    assert _err(call(dst=reg(64, hd=128, nh=2))).code == ErrorCode.INCOMPATIBLE
    e = _err(call(dst=reg(64, nh=8)))
    assert e.code == ErrorCode.INCOMPATIBLE and "equal num_heads" in e.msg
    assert _err(call(dst=reg(64, hd=128, elem=1))).code == ErrorCode.INCOMPATIBLE
    e = _err(call(options=TransferOptions(cast_mode=int(K.CastMode.FP8E4M3_TO_BF16))))
    assert e.code == ErrorCode.INCOMPATIBLE and "Head row" in e.msg
    e = _err(call(dst=reg(64, hd=128), options=TransferOptions(cast_mode=int(K.CastMode.FP8E4M3_TO_BF16))))
    assert e.code == ErrorCode.INCOMPATIBLE and "fp8->bf16" in e.msg
    e = _err(call(dst=reg(24), dst_block_ids=[0]))
    assert e.code == ErrorCode.INCOMPATIBLE and "divide" in e.msg
    e = _err(call(dst=reg(64, fc=False), options=TransferOptions(dst_kv_layout=int(KV.UniversalTP))))
    assert e.code == ErrorCode.INCOMPATIBLE and "fully contiguous" in e.msg
    # the walk's row rule (as the permuting path: UNSUPPORTED)
    e = _err(call(src=reg(16, hd=4), dst=reg(64, hd=4)))
    assert e.code == ErrorCode.UNSUPPORTED and "multiple of 16" in e.msg
    # RANGE: reversed tokens, past 2^31, layer range, cast scales too few
    assert _err(call(tokens=range(9, 5))).code == ErrorCode.RANGE
    assert _err(call(tokens=range(0, 2**31 + 1))).code == ErrorCode.RANGE
    e = _err(call(options=TransferOptions(layer_range=range(0, 3))))
    assert e.code == ErrorCode.RANGE and "Layer range" in e.msg
    f8 = reg(64, hd=64, elem=1)
    e = _err(call(dst=f8, options=TransferOptions(cast_mode=int(K.CastMode.BF16_TO_FP8E4M3), cast_scales=np.ones(3, np.float32))))
    assert e.code == ErrorCode.RANGE and "cast_scales" in e.msg
    e = _err(call(options=TransferOptions(cast_scales=np.ones(4, np.float32))))
    assert e.code == ErrorCode.ERR and "need a cast_mode" in e.msg
    # LENGTH_MISMATCH: counts other than the range implies (tokens 5..40: 3 blocks of 16, 1 of 64)
    e = _err(call(src_block_ids=[0, 1]))
    assert e.code == ErrorCode.LENGTH_MISMATCH and "3 source and 1 destination" in e.msg
    assert _err(call(dst_block_ids=[3, 4])).code == ErrorCode.LENGTH_MISMATCH
    assert _err(call(tokens=range(5, 5))).code == ErrorCode.LENGTH_MISMATCH
    # ids: duplicates in the destination, overlap within one pool, out of range
    s1, d1 = reg(1, nb=64), reg(16)
    e = _err(call(src=s1, src_block_ids=list(range(17)), dst=d1, dst_block_ids=[2, 2], tokens=range(15, 32)))
    assert e.code == ErrorCode.DUPLICATE_DST
    e = _err(call(src=s16, src_block_ids=[0, 1], dst=s16, dst_block_ids=[1, 5], tokens=range(0, 32)))
    assert e.code == ErrorCode.OVERLAP
    e = _err(call(src_block_ids=[0, 1, 8]))
    assert e.code == ErrorCode.RANGE and "for source" in e.msg
    e = _err(call(dst_block_ids=[8]))
    assert e.code == ErrorCode.RANGE and "for destination" in e.msg
    # empty token / layer ranges: nothing to move, accepted before the strategy
    assert mgr.execute_repage(s16, [], d64, [], range(7, 7)).is_complete()
    assert mgr.execute_repage(s16, [0, 1, 2], d64, [3], range(5, 40), TransferOptions(layer_range=range(1, 1))).is_complete()
    # strategy: host pools take Memcpy, which has no re-paging launch
    h16, h64 = reg(16, storage=StorageKind.System), reg(64, storage=StorageKind.System)
    e = _err(call(src=h16, dst=h64))
    assert e.code == ErrorCode.UNSUPPORTED and "direct CUDA strategy" in e.msg
    # CUDA: a host-only manager, after every other check
    e = _err(call())
    assert e.code == ErrorCode.CUDA and "without a CUDA device" in e.msg
    assert _err(call(tokens=range(0, 1), src_block_ids=[0], dst_block_ids=[3])).code == ErrorCode.CUDA
    assert mgr.bytes_moved() == 0 and mgr.h2d_bytes() == 0


def test_manager_repage_null_id_lists(host_mgr):
    mgr, reg = host_mgr
    s16, d64 = reg(16), reg(64)
    tok = C.c_uint64()
    rc = P.lib().kvbm_manager_execute_repage(mgr._h, s16, None, 1, d64, None, 1, 0, 16, C.byref(P._COptions()), C.byref(tok))
    assert rc == ErrorCode.ERR and b"null block id list" in P.lib().kvbm_last_error()
    assert P.lib().kvbm_manager_execute_repage(None, s16, None, 0, d64, None, 0, 0, 0, None, None) == ErrorCode.ERR

"""GPU parity of the layout transform with the fused fp8 e4m3 <-> bf16 cast (kvbm_kernels_paged_permute_cast, and TransferManager
transfers that change both the KvBlockLayout and the dtype) against the oracle composition in tests/cast_oracle.py, and
against the paged copy's fused cast of the same blocks.  Whole destination buffers are compared, so bytes that must not
move are checked too."""
import itertools

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import ErrorCode, KvbmError, LayoutConfig, StorageKind, TransferManager, TransferOptions
from oracle import oracle as O
from tests.cast_oracle import kv_layout_permute_cast
from tests.gpu_util import DevicePool, ids_dev, randomize, stream_ptr
from tests.test_gpu_permute import _host, _Pool

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
ALL = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]
UNIVERSAL = (KV.UniversalTP, KV.UniversalPP)
CASTS = [CM.FP8E4M3_TO_BF16, CM.BF16_TO_FP8E4M3]
ELEMS = {CM.NONE: (2, 2), CM.FP8E4M3_TO_BF16: (1, 2), CM.BF16_TO_FP8E4M3: (2, 1)}   # (source, destination) element bytes


def _expected(src, ref, sids, dids, src_kv, dst_kv, nl, no, nt, nh, src_row, cast, layers=None):
    """ref (a host twin of the destination before the transfer) after the transfer, per the oracle."""
    for s, d in zip(sids, dids):
        blk = O.read_logical_block(src, s)
        old = O.read_logical_block(ref, d)
        O.write_logical_block(ref, d, kv_layout_permute_cast(blk, int(src_kv), int(dst_kv), nl, no, nt, nh, src_row, int(cast),
                                                             layers=layers, dst_old=old))


def _run(src, dst, sids, dids, src_kv, dst_kv, nl, nh, nt, src_row, cast, lb=0, le=None, done=0, epoch=0, completion=0, value=0):
    S, D = DevicePool(src), DevicePool(dst)
    si, di = ids_dev(sids), ids_dev(dids)
    rc = K.paged_permute_cast(K.PermuteSide(S.desc, si.data_ptr(), int(src_kv)), K.PermuteSide(D.desc, di.data_ptr(), int(dst_kv)),
                              len(sids), lb, nl if le is None else le, nh, nt, src_row, int(cast), done_flag=done, epoch=epoch,
                              completion_flag=completion, completion_value=value, stream=stream_ptr())
    torch.cuda.synchronize()
    if rc == 0:
        D.download()
    return rc


def _pools(sk, dk, nb_src, nb_dst, nl, no, nt, nh, hd, cast, fill=0x5A):
    se, de = ELEMS[cast]
    return (_host(sk, nb_src, nl, no, nt, nh, hd, se), _host(dk, nb_dst, nl, no, nt, nh, hd, de, fill),
            _host(dk, nb_dst, nl, no, nt, nh, hd, de, fill))


def _check(src, dst, ref, sids, dids, src_kv, dst_kv, geom, cast, layers=None):
    nl, no, nt, nh, hd = geom
    _expected(src, ref, sids, dids, src_kv, dst_kv, nl, no, nt, nh, hd * ELEMS[cast][0], cast, layers)
    for got, want in zip(dst.buffers, ref.buffers):          # moved blocks AND every untouched byte
        assert np.array_equal(got, want)


@pytest.mark.parametrize("cast", CASTS, ids=lambda c: c.name)
@pytest.mark.parametrize("src_kv,dst_kv", list(itertools.product(ALL, ALL)), ids=lambda k: k.name)
@pytest.mark.parametrize("kinds", [("FC", "FC"), ("LWf", "LWs"), ("LWs", "FC")], ids=lambda k: "-".join(k))
def test_every_pair_of_layouts_both_casts(src_kv, dst_kv, kinds, cast):
    geom = nl, no, nt, nh, hd = 3, 2, 16, 4, 32
    sk = "FC" if src_kv in UNIVERSAL else kinds[0]
    dk = "FC" if dst_kv in UNIVERSAL else kinds[1]
    src, dst, ref = _pools(sk, dk, 7, 9, *geom, cast, fill=0xAB)
    randomize(src, 11 * int(src_kv) + int(dst_kv) + 100 * int(cast))
    sids, dids = [5, 0, 3, 6], [8, 2, 4, 0]
    assert _run(src, dst, sids, dids, src_kv, dst_kv, nl, nh, nt, hd * ELEMS[cast][0], cast) == 0
    _check(src, dst, ref, sids, dids, src_kv, dst_kv, geom, cast)


@pytest.mark.parametrize("geom", [(1, 1, 1, 1, 16), (2, 2, 5, 3, 16), (2, 1, 16, 8, 64), (4, 2, 3, 40, 64), (2, 2, 16, 8, 80),
                                  (2, 2, 5, 4, 96), (2, 1, 33, 2, 128), (1, 2, 5, 40, 128), (2, 1, 16, 1, 576), (1, 1, 33, 3, 576)],
                         ids=lambda g: "nl%d-no%d-nt%d-nh%d-hd%d" % g)
@pytest.mark.parametrize("src_kv,dst_kv", [(KV.OperationalNHD, KV.UniversalTP), (KV.UniversalTP, KV.OperationalHND),
                                           (KV.OperationalHND, KV.OperationalNHD), (KV.UniversalPP, KV.UniversalTP)], ids=lambda k: k.name)
@pytest.mark.parametrize("cast", CASTS, ids=lambda c: c.name)
def test_row_sizes_head_counts_and_odd_pages(geom, src_kv, dst_kv, cast):
    """head_dim 16 (a 16 B fp8 row, one vector) ... 576 (MLA); 64 / 128 take the shift-and-mask walk, 80 / 96 / 576 the
    multiply-high; one head (one warp) ... 40 heads (warps loop); page sizes 1, 3, 5, 33."""
    nl, no, nt, nh, hd = geom
    sk = "FC" if src_kv in UNIVERSAL else "LWs"
    dk = "FC" if dst_kv in UNIVERSAL else "LWf"
    src, dst, ref = _pools(sk, dk, 5, 5, *geom, cast)
    randomize(src, 3 + int(cast))
    sids, dids = [4, 1, 2], [0, 3, 1]
    assert _run(src, dst, sids, dids, src_kv, dst_kv, nl, nh, nt, hd * ELEMS[cast][0], cast) == 0
    _check(src, dst, ref, sids, dids, src_kv, dst_kv, geom, cast)


def _paged_copy_cast_then_permute(src, sids, dids, src_kv, dst_kv, geom, cast, fill):
    """The two-pass form: the paged copy's fused cast into a staging pool of the source's format, then the plain permute."""
    nl, no, nt, nh, hd = geom
    de = ELEMS[cast][1]
    stage = _host("FC", src.num_blocks, nl, no, nt, nh, hd, de)
    dst = _host("FC" if dst_kv in UNIVERSAL else "LWs", 4, nl, no, nt, nh, hd, de, fill)
    S, T, D = DevicePool(src), DevicePool(stage), DevicePool(dst)
    si, di = ids_dev(sids), ids_dev(dids)
    K.check(K.paged_copy(S.desc, [K.PagedDst(T.desc, si.data_ptr(), si.data_ptr(), 0, 0)], len(sids), 0, nl, int(cast), None, stream_ptr()))
    K.check(K.paged_permute(K.PermuteSide(T.desc, si.data_ptr(), int(src_kv)), K.PermuteSide(D.desc, di.data_ptr(), int(dst_kv)),
                            len(sids), 0, nl, nh, nt, hd * de, stream=stream_ptr()))
    torch.cuda.synchronize()
    D.download()
    return dst


@pytest.mark.parametrize("src_kv,dst_kv", [(KV.OperationalNHD, KV.UniversalTP), (KV.UniversalPP, KV.OperationalHND)], ids=lambda k: k.name)
def test_every_fp8_code_and_every_bf16_pattern(src_kv, dst_kv):
    """Sources holding all 256 fp8 codes (NaN 0x7f / 0xff, +-0, subnormals) and all 65 536 bf16 patterns (NaN, +-inf, overflow
    past 448, subnormals): the fused launch equals the oracle and the paged copy's fused cast of the same blocks, byte for byte."""
    sk = "FC" if src_kv in UNIVERSAL else "LWs"
    dk = "FC" if dst_kv in UNIVERSAL else "LWs"
    for cast, geom in ((CM.FP8E4M3_TO_BF16, (2, 2, 4, 2, 16)), (CM.BF16_TO_FP8E4M3, (2, 2, 32, 8, 64))):
        nl, no, nt, nh, hd = geom
        se, _ = ELEMS[cast]
        src, dst, ref = _pools(sk, dk, 3, 4, *geom, cast, fill=0x3C)
        per_block = nl * no * nt * nh * hd
        rng = np.random.default_rng(7)
        for b in range(3):   # every code / pattern in every block, in a different order each time
            if cast == CM.FP8E4M3_TO_BF16:
                vals = rng.permutation(np.arange(per_block) % 256).astype(np.uint8)
            else:
                vals = rng.permutation(np.arange(per_block, dtype=np.uint32)).astype(np.uint16).view(np.uint8)
            O.write_logical_block(src, b, vals)
        sids, dids = [2, 0, 1], [1, 3, 0]
        assert _run(src, dst, sids, dids, src_kv, dst_kv, nl, nh, nt, hd * se, cast) == 0
        _check(src, dst, ref, sids, dids, src_kv, dst_kv, geom, cast)
        two_pass = _paged_copy_cast_then_permute(src, sids, dids, src_kv, dst_kv, geom, cast, 0x3C)
        for a, b in zip(dst.buffers, two_pass.buffers):
            assert np.array_equal(a, b), cast.name


def test_layer_ranges_signals_and_argument_checks():
    geom = nl, no, nt, nh, hd = 4, 2, 16, 4, 64
    for cast in CASTS:
        se, de = ELEMS[cast]
        src = _host("LWf", 6, nl, no, nt, nh, hd, se)
        randomize(src, 9)
        for lb, le in ((0, 1), (1, 3), (3, 4), (2, 2)):
            dst, ref = _host("FC", 6, nl, no, nt, nh, hd, de, 0x33), _host("FC", 6, nl, no, nt, nh, hd, de, 0x33)
            assert _run(src, dst, [1, 2], [5, 0], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, hd * se, cast, lb, le) == 0
            if le > lb:
                _expected(src, ref, [1, 2], [5, 0], KV.OperationalNHD, KV.UniversalTP, nl, no, nt, nh, hd * se, cast, layers=range(lb, le))
            assert np.array_equal(dst.buffers[0], ref.buffers[0])
        # done flag and completion word: written after the data, also for an empty transfer
        flags = torch.zeros(4, dtype=torch.int32, device="cuda:0")
        dst = _host("FC", 6, nl, no, nt, nh, hd, de)
        assert _run(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalPP, nl, nh, nt, hd * se, cast, done=flags.data_ptr(), epoch=7,
                    completion=flags.data_ptr() + 4, value=8) == 0
        assert _run(src, dst, [], [], KV.OperationalNHD, KV.UniversalPP, nl, nh, nt, hd * se, cast, done=flags.data_ptr() + 8, epoch=9,
                    completion=flags.data_ptr() + 12, value=10) == 0
        assert flags.cpu().tolist() == [7, 8, 9, 10]
        # contract violations are cudaErrorInvalidValue, nothing is launched
        inval = K.CUDA_ERROR_INVALID_VALUE
        row = hd * se
        assert _run(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, row, 3) == inval          # unknown cast mode
        assert _run(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, row, -1) == inval
        assert _run(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, row, CM.NONE) == inval    # regions do not fit
        other = CM.BF16_TO_FP8E4M3 if cast == CM.FP8E4M3_TO_BF16 else CM.FP8E4M3_TO_BF16
        assert _run(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, row, other) == inval      # ... the other cast
        assert _run(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh * 2, nt, row, cast) == inval   # region != nt*nh*row
        assert _run(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, row, cast, 0, nl + 1) == inval
        other_nl = _host("FC", 6, nl + 1, no, nt, nh, hd, de)
        assert _run(src, other_nl, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, row, cast) == inval  # layer counts differ
    # fp8 rows shorter than 16 B or not a multiple of 16 (the regions fit, the walk cannot split the fp8 row)
    inval = K.CUDA_ERROR_INVALID_VALUE
    for hd, nt in ((8, 16), (24, 16), (40, 2)):
        for cast in CASTS:
            se, de = ELEMS[cast]
            src, dst = _host("FC", 2, 1, 1, nt, 2, hd, se), _host("FC", 2, 1, 1, nt, 2, hd, de)
            assert _run(src, dst, [0], [1], KV.UniversalTP, KV.UniversalPP, 1, 2, nt, hd * se, cast) == inval, (hd, cast)
    src, dst = _host("FC", 2, 1, 1, 16, 2, 32, 2), _host("FC", 2, 1, 1, 16, 2, 32, 1)
    assert _run(src, dst, [0], [1], KV.UniversalTP, KV.UniversalPP, 1, 2, 16, 63, CM.BF16_TO_FP8E4M3) == inval     # odd bf16 row


def test_cast_none_is_the_plain_permute():
    nl, no, nt, nh, hd = 3, 2, 16, 8, 80
    src = _host("LWs", 6, nl, no, nt, nh, hd, 2)
    randomize(src, 4)
    a, b = _host("FC", 6, nl, no, nt, nh, hd, 2, 0x77), _host("FC", 6, nl, no, nt, nh, hd, 2, 0x77)
    assert _run(src, a, [0, 5, 2], [3, 1, 4], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, hd * 2, CM.NONE) == 0
    S, B = DevicePool(src), DevicePool(b)
    si, di = ids_dev([0, 5, 2]), ids_dev([3, 1, 4])
    K.check(K.paged_permute(K.PermuteSide(S.desc, si.data_ptr(), int(KV.OperationalNHD)), K.PermuteSide(B.desc, di.data_ptr(), int(KV.UniversalTP)),
                            3, 0, nl, nh, nt, hd * 2, stream=stream_ptr()))
    torch.cuda.synchronize()
    B.download()
    assert np.array_equal(a.buffers[0], b.buffers[0]) and bool((a.buffers[0] != 0x77).any())


# ---------------------------------------------------------------------------------------------------------------------
# through the TransferManager
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=5)
    yield m
    torch.cuda.synchronize()
    m.close()


def test_manager_fuses_the_cast_into_the_permuting_launch(mgr):
    nl, no, nt, nh, hd = 4, 2, 16, 8, 128
    g8, g16 = (nl, no, nt, nh, hd, 1), (nl, no, nt, nh, hd, 2)
    op = _Pool(mgr, "LWs", 12, *g8, kv=KV.OperationalNHD)          # an fp8 engine pool (vLLM layout)
    uni = _Pool(mgr, "FC", 10, *g16, kv=KV.UniversalTP, fill=0x11)  # a bf16 universal tier
    ref = _host("FC", 10, *g16, fill=0x11)
    randomize(op.twin, 77)
    op.upload()
    sids, dids = [3, 11, 0, 7], [9, 1, 4, 2]
    launches0 = K.launch_count()
    mgr.execute_transfer(op.h, sids, uni.h, dids, TransferOptions(cast_mode=CM.FP8E4M3_TO_BF16)).wait(20.0)
    assert K.launch_count() - launches0 == 2                        # the permuting kernel + the completion signal
    uni.download()
    _expected(op.twin, ref, sids, dids, KV.OperationalNHD, KV.UniversalTP, nl, no, nt, nh, hd, CM.FP8E4M3_TO_BF16)
    assert np.array_equal(uni.twin.buffers[0], ref.buffers[0])
    # back down into a compact fp8 pool of a different operational format: bf16 UniversalTP -> fp8 OperationalHND
    hnd = _Pool(mgr, "LWf", 8, *g8, kv=KV.OperationalHND, fill=0x22)
    ref2 = _host("LWf", 8, *g8, fill=0x22)
    flag = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    launches0 = K.launch_count()
    mgr.execute_transfer(uni.h, dids, hnd.h, [0, 1, 2, 3], TransferOptions(cast_mode=CM.BF16_TO_FP8E4M3, done_flag=flag.data_ptr(),
                                                                         epoch=5)).wait(20.0)
    assert K.launch_count() - launches0 == 2
    assert int(flag.item()) == 5
    hnd.download()
    _expected(uni.twin, ref2, dids, [0, 1, 2, 3], KV.UniversalTP, KV.OperationalHND, nl, no, nt, nh, 2 * hd, CM.BF16_TO_FP8E4M3)
    for a, b in zip(hnd.twin.buffers, ref2.buffers):
        assert np.array_equal(a, b)


def test_manager_rejections_with_the_cast(mgr):
    nl, no, nt, nh, hd = 3, 2, 16, 4, 64
    g8, g16 = (nl, no, nt, nh, hd, 1), (nl, no, nt, nh, hd, 2)
    a = _Pool(mgr, "LWs", 6, *g8, kv=KV.OperationalNHD)
    b = _Pool(mgr, "FC", 6, *g16, kv=KV.UniversalTP)
    c = _Pool(mgr, "FC", 6, *g16, kv=KV.UniversalTP)
    up = CM.FP8E4M3_TO_BF16

    def err(fn):
        with pytest.raises(KvbmError) as e:
            fn()
        return e.value

    e = err(lambda: mgr.execute_fanout(a.h, [b.h, c.h], [[0], [1]], [[1], [2]], options=TransferOptions(cast_mode=up)))
    assert e.code == ErrorCode.UNSUPPORTED and "one destination" in e.msg
    ready = torch.zeros(nl, dtype=torch.int32, device="cuda:0")
    e = err(lambda: mgr.execute_transfer(a.h, [0], b.h, [1], TransferOptions(cast_mode=up, layer_ready_flags=ready.data_ptr(), epoch=1)))
    assert e.code == ErrorCode.UNSUPPORTED and "layer streaming" in e.msg
    e = err(lambda: mgr.execute_transfer(a.h, [0], b.h, [1], TransferOptions(cast_mode=up, multicast=1)))
    assert e.code == ErrorCode.UNSUPPORTED and "layer streaming / multicast" in e.msg
    unknown = _Pool(mgr, "FC", 6, *g16, kv=None)
    e = err(lambda: mgr.execute_transfer(a.h, [0], unknown.h, [1], TransferOptions(cast_mode=up)))
    assert e.code == ErrorCode.UNSUPPORTED and "Layout transformation not supported" in e.msg
    e = err(lambda: mgr.execute_transfer(a.h, [0], b.h, [1], TransferOptions(cast_mode=up, dst_kv_layout=int(KV.Custom))))
    assert e.code == ErrorCode.UNSUPPORTED and "Layout transformation not supported" in e.msg
    # host pools take the Memcpy strategy, which has neither the cast nor the transform
    h8, h16 = _host("FC", 6, *g8), _host("FC", 6, *g16)
    hs = mgr.register_fully_contiguous(LayoutConfig(6, nl, no, nt, nh * hd, dtype_width_bytes=1, num_heads=nh, allow_fp8=True),
                                       h8.buffers[0].ctypes.data, h8.buffers[0].size, StorageKind.System, 0)
    hd16 = mgr.register_fully_contiguous(LayoutConfig(6, nl, no, nt, nh * hd, dtype_width_bytes=2, num_heads=nh),
                                         h16.buffers[0].ctypes.data, h16.buffers[0].size, StorageKind.System, 0)
    mgr.set_kv_block_layout(hs, KV.OperationalNHD)
    mgr.set_kv_block_layout(hd16, KV.UniversalTP)
    e = err(lambda: mgr.execute_transfer(hs, [0], hd16, [1], TransferOptions(cast_mode=up)))
    assert e.code == ErrorCode.UNSUPPORTED and "CUDA strategies" in e.msg
    # the fp8 row must be whole 16 B vectors: head_dim 8 is a valid bf16 transform (16 B rows) but not a cast one
    s8 = _Pool(mgr, "FC", 4, 1, 1, 16, 2, 8, 1, kv=KV.UniversalTP)
    d16 = _Pool(mgr, "FC", 4, 1, 1, 16, 2, 8, 2, kv=KV.UniversalPP)
    e = err(lambda: mgr.execute_transfer(s8.h, [0], d16.h, [1], TransferOptions(cast_mode=up)))
    assert e.code == ErrorCode.UNSUPPORTED and "fused cast: head_dim must be a multiple of 16" in e.msg
    # a cast with the widths the other way round is still check_compat's error
    e = err(lambda: mgr.execute_transfer(a.h, [0], b.h, [1], TransferOptions(cast_mode=CM.BF16_TO_FP8E4M3)))
    assert e.code == ErrorCode.INCOMPATIBLE


def test_full_size_fp8_round_trip_through_a_bf16_universal_tier(mgr):
    """Llama-3-70B KV geometry (80 layers, 8 KV heads x 128, 16-token pages), 64 of 72 blocks: fp8 engine pool -> bf16 universal
    -> fp8 engine pool.  The round trip is the identity except for fp8 0xff (NaN with the sign bit set): the up-cast maps both
    NaN codes to the bf16 NaN 0x7fc0, which comes back as 0x7f."""
    nl, no, nt, nh, hd = 80, 2, 16, 8, 128
    nb, n = 72, 64
    g8, g16 = (nl, no, nt, nh, hd, 1), (nl, no, nt, nh, hd, 2)
    op = _Pool(mgr, "LWs", nb, *g8, kv=KV.OperationalNHD)
    uni = _Pool(mgr, "FC", nb, *g16, kv=KV.UniversalTP)
    back = _Pool(mgr, "LWs", nb, *g8, kv=KV.OperationalNHD)
    gen = torch.Generator(device="cuda:0").manual_seed(1)
    for t in op.mem:
        t.copy_(torch.randint(0, 256, t.shape, dtype=torch.uint8, device="cuda:0", generator=gen))
    torch.cuda.synchronize()        # the manager's streams are non-blocking: they do not wait for torch's fill
    rng = np.random.default_rng(2)
    s, u, d = (list(map(int, rng.permutation(nb)[:n])) for _ in range(3))
    mgr.execute_transfer(op.h, s, uni.h, u, TransferOptions(cast_mode=CM.FP8E4M3_TO_BF16)).wait(30.0)
    mgr.execute_transfer(uni.h, u, back.h, d, TransferOptions(cast_mode=CM.BF16_TO_FP8E4M3)).wait(30.0)
    torch.cuda.synchronize()
    region = nt * nh * hd
    for l in range(nl):             # block-is-second-dim: [outer][block][region] per layer
        src_l, dst_l = op.mem[l].view(no, nb, region)[:, s, :], back.mem[l].view(no, nb, region)[:, d, :]
        assert torch.equal(dst_l, torch.where(src_l == 0xFF, torch.full_like(src_l, 0x7F), src_l)), l
    op.download()
    uni.download()
    for i in (0, n - 1):
        want = kv_layout_permute_cast(O.read_logical_block(op.twin, s[i]), int(KV.OperationalNHD), int(KV.UniversalTP), nl, no, nt, nh, hd,
                                      int(CM.FP8E4M3_TO_BF16))
        assert np.array_equal(O.read_logical_block(uni.twin, u[i]), want)


@pytest.mark.multigpu
def test_fp8_pool_pulled_over_nvlink_into_a_bf16_universal_pool():
    """Decode-side launch: the prefill GPU's fp8 operational pool is read over NVLink and lands as bf16 universal blocks."""
    nl, no, nt, nh, hd = 4, 2, 16, 8, 128
    mgr = TransferManager(device=1, worker_id=6)
    mgr.enable_peer_access(0)
    src = _Pool(mgr, "LWs", 16, nl, no, nt, nh, hd, 1, kv=KV.OperationalNHD, device=0)
    dst = _Pool(mgr, "FC", 16, nl, no, nt, nh, hd, 2, kv=KV.UniversalTP, device=1, fill=0x44)
    ref = _host("FC", 16, nl, no, nt, nh, hd, 2, fill=0x44)
    randomize(src.twin, 8)
    src.upload()
    torch.cuda.synchronize(0)
    sids, dids = [15, 2, 9, 4, 0], [1, 14, 3, 8, 6]
    mgr.execute_transfer(src.h, sids, dst.h, dids, TransferOptions(cast_mode=CM.FP8E4M3_TO_BF16)).wait(20.0)
    torch.cuda.synchronize(1)
    dst.download()
    _expected(src.twin, ref, sids, dids, KV.OperationalNHD, KV.UniversalTP, nl, no, nt, nh, hd, CM.FP8E4M3_TO_BF16)
    assert np.array_equal(dst.twin.buffers[0], ref.buffers[0])
    mgr.close()

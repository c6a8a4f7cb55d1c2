"""GPU parity of the TP re-shard: kvbm_kernels_paged_permute_heads and TransferManager transfers with a head window, against the
oracle in tests/reshard_oracle.py.  Destinations are pre-filled with a pattern and compared whole, so the bytes outside each
window are checked untouched."""
import itertools

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import ErrorCode, KvbmError, LayoutConfig, StorageKind, TransferManager, TransferOptions, tp_reshard_plan
from oracle import oracle as O
from tests.gpu_util import DevicePool, ids_dev, randomize, stream_ptr
from tests.reshard_oracle import rank_heads, reshard_block
from tests.test_gpu_permute import _host, _Pool

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
ALL = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]
UNIVERSAL = (KV.UniversalTP, KV.UniversalPP)
CASTS = [CM.FP8E4M3_TO_BF16, CM.BF16_TO_FP8E4M3]
ELEMS = {CM.NONE: (2, 2), CM.FP8E4M3_TO_BF16: (1, 2), CM.BF16_TO_FP8E4M3: (2, 1)}   # (source, destination) element bytes
# (src_nh, dst_nh, src_head_begin, dst_head_begin, head_count): begin != 0 on either side, one head, partial, full width,
# and windows of 1 ... 8 heads (narrower than 8 take the packed CTA mapping)
WINDOWS = [(4, 2, 2, 0, 2), (2, 4, 0, 2, 2), (4, 4, 1, 2, 2), (4, 1, 3, 0, 1), (8, 8, 2, 5, 3), (3, 5, 0, 0, 3), (16, 8, 8, 0, 8),
           (8, 12, 0, 1, 8), (2, 2, 0, 0, 2)]


def _expected(src, ref, sids, dids, src_kv, dst_kv, geom, win, cast=CM.NONE, layers=None):
    nl, no, nt, hd = geom
    snh, dnh, sb, db, k = win
    for s, d in zip(sids, dids):
        O.write_logical_block(ref, d, reshard_block(O.read_logical_block(src, s), O.read_logical_block(ref, d), int(src_kv), int(dst_kv),
                                                    nl, no, nt, snh, dnh, hd * ELEMS[cast][0], int(cast), sb, db, k, layers=layers))


def _run(src, dst, sids, dids, src_kv, dst_kv, geom, win, cast=CM.NONE, lb=0, le=None, done=0, epoch=0, completion=0, value=0, row=None):
    nl, no, nt, hd = geom
    snh, dnh, sb, db, k = win
    S, D = DevicePool(src), DevicePool(dst)
    si, di = ids_dev(sids), ids_dev(dids)
    rc = K.paged_permute_heads(K.PermuteSide(S.desc, si.data_ptr(), int(src_kv)), K.PermuteSide(D.desc, di.data_ptr(), int(dst_kv)),
                               len(sids), lb, nl if le is None else le, snh, sb, dnh, db, k, nt, hd * ELEMS[cast][0] if row is None else row,
                               int(cast), done_flag=done, epoch=epoch, completion_flag=completion, completion_value=value, stream=stream_ptr())
    torch.cuda.synchronize()
    if rc == 0:
        D.download()
    return rc


def _pools(sk, dk, nb_src, nb_dst, geom, win, cast=CM.NONE, fill=0x5A):
    nl, no, nt, hd = geom
    se, de = ELEMS[cast]
    return (_host(sk, nb_src, nl, no, nt, win[0], hd, se), _host(dk, nb_dst, nl, no, nt, win[1], hd, de, fill),
            _host(dk, nb_dst, nl, no, nt, win[1], hd, de, fill))


def _check(dst, ref):
    for got, want in zip(dst.buffers, ref.buffers):          # the window AND every byte outside it
        assert np.array_equal(got, want)


@pytest.mark.parametrize("win", WINDOWS, ids=lambda w: "s%d-d%d-sb%d-db%d-k%d" % w)
@pytest.mark.parametrize("src_kv,dst_kv", list(itertools.product(ALL, ALL)), ids=lambda k: k.name)
@pytest.mark.parametrize("kinds", [("FC", "FC"), ("LWf", "LWs"), ("LWs", "FC")], ids=lambda k: "-".join(k))
def test_every_pair_of_layouts_and_windows(src_kv, dst_kv, kinds, win):
    geom = (3, 2, 16, 32)
    sk = "FC" if src_kv in UNIVERSAL else kinds[0]
    dk = "FC" if dst_kv in UNIVERSAL else kinds[1]
    src, dst, ref = _pools(sk, dk, 7, 9, geom, win, fill=0xAB)
    randomize(src, 11 * int(src_kv) + int(dst_kv) + sum(win))
    sids, dids = [5, 0, 3, 6], [8, 2, 4, 0]
    assert _run(src, dst, sids, dids, src_kv, dst_kv, geom, win) == 0
    _expected(src, ref, sids, dids, src_kv, dst_kv, geom, win)
    _check(dst, ref)


@pytest.mark.parametrize("cast", CASTS, ids=lambda c: c.name)
@pytest.mark.parametrize("src_kv,dst_kv", list(itertools.product(ALL, ALL)), ids=lambda k: k.name)
def test_every_pair_of_layouts_both_casts(src_kv, dst_kv, cast):
    geom = (3, 2, 16, 32)
    sk = "FC" if src_kv in UNIVERSAL else "LWs"
    dk = "FC" if dst_kv in UNIVERSAL else "LWf"
    for win in ((4, 2, 1, 1, 1), (2, 4, 0, 2, 2)):
        src, dst, ref = _pools(sk, dk, 5, 6, geom, win, cast, fill=0x3C)
        randomize(src, int(src_kv) + 5 * int(dst_kv) + int(cast))
        sids, dids = [4, 1, 2], [0, 5, 3]
        assert _run(src, dst, sids, dids, src_kv, dst_kv, geom, win, cast) == 0
        _expected(src, ref, sids, dids, src_kv, dst_kv, geom, win, cast)
        _check(dst, ref)


@pytest.mark.parametrize("hd,nt,win", [(16, 5, (4, 2, 1, 0, 2)), (64, 16, (8, 4, 4, 0, 4)), (80, 16, (8, 2, 3, 1, 1)), (96, 3, (2, 8, 1, 6, 1)),
                                        (128, 16, (8, 4, 0, 1, 3)), (576, 16, (1, 1, 0, 0, 1)), (576, 7, (2, 1, 1, 0, 1))],
                         ids=lambda x: str(x))
@pytest.mark.parametrize("cast", [CM.NONE] + CASTS, ids=lambda c: c.name)
def test_head_dims_mla_and_layer_ranges(hd, nt, win, cast):
    """head_dim 16 ... 576 (MLA's single latent head): 64 / 128 take the shift-and-mask walk, 80 / 96 / 576 the multiply-high."""
    nl, no = 4, 2
    geom = (nl, no, nt, hd)
    for layers in (None, range(1, 3), range(3, 4)):
        src, dst, ref = _pools("LWs", "FC", 4, 4, geom, win, cast, fill=0x66)
        randomize(src, hd + nt)
        lb, le = (0, nl) if layers is None else (layers.start, layers.stop)
        assert _run(src, dst, [3, 0], [1, 2], KV.OperationalNHD, KV.UniversalPP, geom, win, cast, lb, le) == 0
        _expected(src, ref, [3, 0], [1, 2], KV.OperationalNHD, KV.UniversalPP, geom, win, cast, layers)
        _check(dst, ref)


def test_signals_empty_transfers_and_argument_checks():
    geom = nl, no, nt, hd = 4, 2, 16, 64
    win = (4, 2, 2, 0, 2)
    src, dst, _ = _pools("LWf", "FC", 6, 6, geom, win)
    randomize(src, 9)
    flags = torch.zeros(4, dtype=torch.int32, device="cuda:0")
    assert _run(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalPP, geom, win, done=flags.data_ptr(), epoch=7,
                completion=flags.data_ptr() + 4, value=8) == 0
    assert _run(src, dst, [], [], KV.OperationalNHD, KV.UniversalPP, geom, win, done=flags.data_ptr() + 8, epoch=9,
                completion=flags.data_ptr() + 12, value=10) == 0
    assert flags.cpu().tolist() == [7, 8, 9, 10]
    inval = K.CUDA_ERROR_INVALID_VALUE
    run = lambda w, **kw: _run(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, geom, w, **kw)  # noqa: E731
    assert run(win) == 0
    assert run((4, 2, 2, 0, 0)) == inval            # head_count 0
    assert run((4, 2, 3, 0, 2)) == inval            # past the source's heads
    assert run((4, 2, 2, 1, 2)) == inval            # past the destination's heads
    assert run((4, 2, 2**32 - 1, 0, 2)) == inval    # begin + count wraps in 32 bits
    assert run((8, 2, 0, 0, 2)) == inval            # source region != nt * its num_heads * row
    assert run((4, 4, 0, 0, 2)) == inval            # destination region likewise
    assert run(win, cast=3, row=hd * 2) == inval    # unknown cast mode
    assert run(win, row=hd * 2 + 16) == inval       # the cast / row rules of paged_permute_cast
    assert run(win, lb=0, le=nl + 1) == inval
    assert _run(src, dst, [0], [1], KV.Custom, KV.UniversalTP, geom, win) == inval


def test_full_window_is_paged_permute_cast():
    geom = nl, no, nt, hd = 3, 2, 16, 80
    for cast in [CM.NONE] + CASTS:
        win = (8, 8, 0, 0, 8)
        src, a, b = _pools("LWs", "FC", 6, 6, geom, win, cast, fill=0x77)
        randomize(src, 4)
        assert _run(src, a, [0, 5, 2], [3, 1, 4], KV.OperationalNHD, KV.UniversalTP, geom, win, cast) == 0
        S, B = DevicePool(src), DevicePool(b)
        si, di = ids_dev([0, 5, 2]), ids_dev([3, 1, 4])
        K.check(K.paged_permute_cast(K.PermuteSide(S.desc, si.data_ptr(), int(KV.OperationalNHD)), K.PermuteSide(B.desc, di.data_ptr(), int(KV.UniversalTP)),
                                     3, 0, nl, 8, nt, hd * ELEMS[cast][0], int(cast), stream=stream_ptr()))
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


def test_manager_windowed_transfers(mgr):
    nl, no, nt, hd = 4, 2, 16, 128
    # equal formats, different head counts: NHD engine pools of 2 (TP4) and 4 (TP2) heads of an 8-head model
    a = _Pool(mgr, "LWs", 10, nl, no, nt, 2, hd, 2, kv=KV.OperationalNHD)
    b = _Pool(mgr, "LWs", 8, nl, no, nt, 4, hd, 2, kv=KV.OperationalNHD, fill=0x21)
    ref = _host("LWs", 8, nl, no, nt, 4, hd, 2, fill=0x21)
    randomize(a.twin, 31)
    a.upload()
    sids, dids = [9, 0, 4], [2, 7, 5]
    flag = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    launches0 = K.launch_count()
    mgr.execute_transfer(a.h, sids, b.h, dids, TransferOptions(head_window=(0, 2, 2), done_flag=flag.data_ptr(), epoch=3)).wait(20.0)
    assert K.launch_count() - launches0 == 2                        # the permuting kernel + the completion signal
    assert int(flag.item()) == 3
    b.download()
    _expected(a.twin, ref, sids, dids, KV.OperationalNHD, KV.OperationalNHD, (nl, no, nt, hd), (2, 4, 0, 2, 2))
    for x, y in zip(b.twin.buffers, ref.buffers):
        assert np.array_equal(x, y)
    # a format change, a layer range and the cast compose with the window: fp8 NHD (2 heads) -> bf16 UniversalTP (4 heads)
    a8 = _Pool(mgr, "LWs", 10, nl, no, nt, 2, hd, 1, kv=KV.OperationalNHD)
    u = _Pool(mgr, "FC", 6, nl, no, nt, 4, hd, 2, kv=KV.UniversalTP, fill=0x44)
    ref_u = _host("FC", 6, nl, no, nt, 4, hd, 2, fill=0x44)
    randomize(a8.twin, 32)
    a8.upload()
    mgr.execute_transfer(a8.h, [1, 2], u.h, [5, 0], TransferOptions(head_window=(1, 3, 1), cast_mode=CM.FP8E4M3_TO_BF16,
                                                                   layer_range=range(1, 3))).wait(20.0)
    u.download()
    _expected(a8.twin, ref_u, [1, 2], [5, 0], KV.OperationalNHD, KV.UniversalTP, (nl, no, nt, hd), (2, 4, 1, 3, 1), CM.FP8E4M3_TO_BF16,
              layers=range(1, 3))
    assert np.array_equal(u.twin.buffers[0], ref_u.buffers[0])
    # a window over every head of both sides is the plain transfer: one paged-copy launch
    c = _Pool(mgr, "LWs", 8, nl, no, nt, 4, hd, 2, kv=KV.OperationalNHD)
    launches0 = K.launch_count()
    mgr.execute_transfer(b.h, [0, 1], c.h, [1, 0], TransferOptions(head_window=(0, 0, 4))).wait(20.0)
    assert K.launch_count() - launches0 == 1
    c.download()
    assert np.array_equal(O.read_logical_block(c.twin, 1), O.read_logical_block(b.twin, 0))


def test_manager_windowed_rejections(mgr):
    nl, no, nt, hd = 3, 2, 16, 64
    a = _Pool(mgr, "LWs", 6, nl, no, nt, 2, hd, 2, kv=KV.OperationalNHD)
    b = _Pool(mgr, "LWs", 6, nl, no, nt, 4, hd, 2, kv=KV.OperationalNHD)
    c = _Pool(mgr, "LWs", 6, nl, no, nt, 4, hd, 2, kv=KV.OperationalNHD)
    W = lambda sb, db, k, **kw: TransferOptions(head_window=(sb, db, k), **kw)  # noqa: E731

    def err(fn):
        with pytest.raises(KvbmError) as e:
            fn()
        return e.value

    e = err(lambda: mgr.execute_transfer(a.h, [0], b.h, [1], W(1, 0, 2)))
    assert e.code == ErrorCode.RANGE and "Head window" in e.msg
    e = err(lambda: mgr.execute_transfer(a.h, [0], b.h, [1], W(0, 3, 2)))
    assert e.code == ErrorCode.RANGE
    e = err(lambda: mgr.execute_fanout(a.h, [b.h, c.h], [[0], [1]], [[1], [2]], options=W(0, 0, 2)))
    assert e.code == ErrorCode.UNSUPPORTED and "one destination" in e.msg
    ready = torch.zeros(nl, dtype=torch.int32, device="cuda:0")
    e = err(lambda: mgr.execute_transfer(a.h, [0], b.h, [1], W(0, 0, 2, layer_ready_flags=ready.data_ptr(), epoch=1)))
    assert e.code == ErrorCode.UNSUPPORTED and "layer streaming / multicast" in e.msg
    e = err(lambda: mgr.execute_transfer(a.h, [0], b.h, [1], W(0, 0, 2, multicast=1)))
    assert e.code == ErrorCode.UNSUPPORTED and "layer streaming / multicast" in e.msg
    unknown = _Pool(mgr, "LWs", 6, nl, no, nt, 4, hd, 2, kv=None)
    e = err(lambda: mgr.execute_transfer(a.h, [0], unknown.h, [1], W(0, 0, 2)))
    assert e.code == ErrorCode.UNSUPPORTED and "Layout transformation not supported" in e.msg
    unknown2 = _Pool(mgr, "LWs", 6, nl, no, nt, 2, hd, 2, kv=None)
    e = err(lambda: mgr.execute_transfer(unknown2.h, [0], unknown.h, [1], W(0, 0, 2)))    # Unknown -> Unknown, too
    assert e.code == ErrorCode.UNSUPPORTED and "Layout transformation not supported" in e.msg
    e = err(lambda: mgr.execute_transfer(a.h, [0], b.h, [1], W(0, 0, 2, dst_kv_layout=int(KV.Custom))))
    assert e.code == ErrorCode.UNSUPPORTED and "Layout transformation not supported" in e.msg
    e = err(lambda: mgr.execute_transfer(a.h, [0], b.h, [1], W(0, 0, 2, dst_kv_layout=int(KV.UniversalTP))))
    assert e.code == ErrorCode.INCOMPATIBLE and "fully contiguous" in e.msg
    # the heads themselves must match: head_dim 64 vs 32 (same region size, 4 vs 8 heads)
    d32 = _Pool(mgr, "LWs", 6, nl, no, nt, 8, 32, 2, kv=KV.OperationalNHD)
    e = err(lambda: mgr.execute_transfer(b.h, [0], d32.h, [1], W(0, 0, 2)))
    assert e.code == ErrorCode.INCOMPATIBLE and "Head row size mismatch" in e.msg
    other_pages = _Pool(mgr, "LWs", 6, nl, no, 8, 8, hd, 2, kv=KV.OperationalNHD)   # 8-token pages, 8 heads: same region size
    e = err(lambda: mgr.execute_transfer(b.h, [0], other_pages.h, [1], W(0, 0, 2)))
    assert e.code == ErrorCode.INCOMPATIBLE and "equal head_dim, page_size and dtype" in e.msg
    other_layers = _Pool(mgr, "LWs", 6, nl + 1, no, nt, 4, hd, 2, kv=KV.OperationalNHD)
    e = err(lambda: mgr.execute_transfer(a.h, [0], other_layers.h, [1], W(0, 0, 2)))
    assert e.code == ErrorCode.INCOMPATIBLE and "incompatible layer counts" in e.msg
    # no num_heads in a config
    cfg = LayoutConfig(6, nl, no, nt, 2 * hd, dtype_width_bytes=2)
    t = torch.zeros(cfg.required_bytes(), dtype=torch.uint8, device="cuda:0")
    nh0 = mgr.register_fully_contiguous(cfg, t.data_ptr(), t.numel(), StorageKind.Device, 0)
    e = err(lambda: mgr.execute_transfer(nh0, [0], b.h, [1], W(0, 0, 2)))
    assert e.code == ErrorCode.CONFIG and "num_heads" in e.msg
    # host pools take the Memcpy strategy, which has no permuting launch
    h2, h4 = _host("FC", 6, nl, no, nt, 2, hd, 2), _host("FC", 6, nl, no, nt, 4, hd, 2)
    hs = mgr.register_fully_contiguous(LayoutConfig(6, nl, no, nt, 2 * hd, num_heads=2), h2.buffers[0].ctypes.data, h2.buffers[0].size,
                                       StorageKind.System, 0)
    hd4 = mgr.register_fully_contiguous(LayoutConfig(6, nl, no, nt, 4 * hd, num_heads=4), h4.buffers[0].ctypes.data, h4.buffers[0].size,
                                        StorageKind.System, 0)
    mgr.set_kv_block_layout(hs, KV.OperationalNHD)
    mgr.set_kv_block_layout(hd4, KV.OperationalNHD)
    e = err(lambda: mgr.execute_transfer(hs, [0], hd4, [1], W(0, 0, 2)))
    assert e.code == ErrorCode.UNSUPPORTED and "CUDA strategies" in e.msg
    # the row rule of the transform: head_dim 4 in bf16 is an 8-byte row
    s4 = _Pool(mgr, "FC", 4, 1, 1, 16, 2, 4, 2, kv=KV.OperationalNHD)
    d4 = _Pool(mgr, "FC", 4, 1, 1, 16, 4, 4, 2, kv=KV.OperationalNHD)
    e = err(lambda: mgr.execute_transfer(s4.h, [0], d4.h, [1], W(0, 0, 2)))
    assert e.code == ErrorCode.UNSUPPORTED and "multiple of 16 bytes" in e.msg
    # a plan with one done_flag for several entries is refused before anything runs
    with pytest.raises(ValueError):
        mgr.execute_reshard({0: (a.h, [0]), 1: (a.h, [1])}, b.h, [2], tp_reshard_plan(8, 4, 2, 0), TransferOptions(done_flag=t.data_ptr()))


# ---------------------------------------------------------------------------------------------------------------------
# full-size Llama-3-70B: 80 layers, 8 KV heads x 128, 16-token pages, engine pools OperationalNHD layer-separate
# ---------------------------------------------------------------------------------------------------------------------
NL, NO, NT, H, HD = 80, 2, 16, 8, 128
NB = 20


def _layer_view(pool, l, nh, elem):
    """[outer, block, token, head, row] view of layer l of a block-is-second-dim NHD pool."""
    return pool.mem[l].view(NO, NB, NT, nh, HD * elem)


def _tp_pools(mgr, tp, elem=2, fill=0):
    nh = max(1, H // tp)
    return [_Pool(mgr, "LWs", NB, NL, NO, NT, nh, HD, elem, kv=KV.OperationalNHD, fill=fill) for _ in range(tp)]


def _shard_from(mgr, orig, tp, elem=2):
    """TP shards of a TP1 pool, cut with torch (independently of the transfer path)."""
    pools = _tp_pools(mgr, tp, elem)
    for r, p in enumerate(pools):
        hs = rank_heads(H, tp, r)
        for l in range(NL):
            _layer_view(p, l, len(hs), elem).copy_(_layer_view(orig, l, H, elem)[:, :, :, hs.start:hs.stop])
    torch.cuda.synchronize()
    return pools


def _reshard(mgr, src_pools, sids, dst_pools, dids, src_tp, dst_tp, cast=CM.NONE):
    notes = []
    for r, dp in enumerate(dst_pools):
        plan = tp_reshard_plan(H, src_tp, dst_tp, r)
        notes += mgr.execute_reshard({s: (p.h, sids) for s, p in enumerate(src_pools)}, dp.h, dids, plan, TransferOptions(cast_mode=cast))
    for n in notes:
        n.wait(60.0)
    torch.cuda.synchronize()


def _orig(mgr, elem=2, seed=1):
    orig = _Pool(mgr, "LWs", NB, NL, NO, NT, H, HD, elem, kv=KV.OperationalNHD)
    gen = torch.Generator(device="cuda:0").manual_seed(seed)
    for t in orig.mem:
        t.copy_(torch.randint(0, 256, t.shape, dtype=torch.uint8, device="cuda:0", generator=gen))
    torch.cuda.synchronize()        # the manager's streams are non-blocking: they do not wait for torch's fill
    return orig


@pytest.mark.parametrize("src_tp,dst_tp", [(4, 2), (2, 8), (8, 1)], ids=lambda t: str(t))
def test_full_size_llama_reshard_reassembles_the_tp1_blocks(mgr, src_tp, dst_tp):
    orig = _orig(mgr)
    src = _shard_from(mgr, orig, src_tp)
    dst = _tp_pools(mgr, dst_tp, fill=0x5A)
    rng = np.random.default_rng(src_tp * 10 + dst_tp)
    n = 16
    sids, dids = list(map(int, rng.permutation(NB)[:n])), list(map(int, rng.permutation(NB)[:n]))
    _reshard(mgr, src, sids, dst, dids, src_tp, dst_tp)
    untouched = [b for b in range(NB) if b not in dids]
    for r, p in enumerate(dst):
        hs = rank_heads(H, dst_tp, r)
        for l in range(NL):
            got, want = _layer_view(p, l, len(hs), 2), _layer_view(orig, l, H, 2)
            assert torch.equal(got[:, dids], want[:, sids][:, :, :, hs.start:hs.stop]), (r, l)
            assert bool((got[:, untouched] == 0x5A).all()), (r, l)


def test_full_size_llama_tp4_to_tp8_to_tp4_is_the_identity(mgr):
    orig = _orig(mgr, seed=2)
    tp4 = _shard_from(mgr, orig, 4)
    del orig
    tp8, back = _tp_pools(mgr, 8), _tp_pools(mgr, 4)
    rng = np.random.default_rng(3)
    s, m, d = (list(map(int, rng.permutation(NB)[:16])) for _ in range(3))
    _reshard(mgr, tp4, s, tp8, m, 4, 8)
    _reshard(mgr, tp8, m, back, d, 8, 4)
    for a, b in zip(tp4, back):
        for l in range(NL):
            assert torch.equal(_layer_view(a, l, 2, 2)[:, s], _layer_view(b, l, 2, 2)[:, d]), l


def test_full_size_llama_fp8_tp4_to_bf16_tp2(mgr):
    orig = _orig(mgr, elem=1, seed=4)
    src = _shard_from(mgr, orig, 4, elem=1)
    dst = _tp_pools(mgr, 2, elem=2, fill=0x13)
    sids, dids = [3, 17, 0, 9], [12, 1, 19, 6]
    _reshard(mgr, src, sids, dst, dids, 4, 2, CM.FP8E4M3_TO_BF16)
    for p in src + dst:
        p.download()
    for r, p in enumerate(dst):
        for i in (0, 3):                                  # sampled blocks against the oracle (5 MiB numpy transposes each)
            want = np.full(NL * NO * NT * 4 * HD * 2, 0x13, dtype=np.uint8)
            for w in tp_reshard_plan(H, 4, 2, r):
                want = reshard_block(O.read_logical_block(src[w.src_rank].twin, sids[i]), want, int(KV.OperationalNHD), int(KV.OperationalNHD),
                                     NL, NO, NT, 2, 4, HD, int(CM.FP8E4M3_TO_BF16), w.src_head_begin, w.dst_head_begin, w.head_count)
            assert np.array_equal(O.read_logical_block(p.twin, dids[i]), want), (r, i)


@pytest.mark.multigpu
def test_decode_gpu_pulls_its_heads_from_two_prefill_gpus():
    """TP4 -> TP2 over NVLink: decode rank 0 on GPU 1 reads heads from prefill ranks 0 and 1 (GPUs 0 and 2 when there are three,
    else both on GPU 0) and assembles its 4-head UniversalTP blocks."""
    nl, no, nt, hd = 4, 2, 16, 128
    devs = [0, 2] if torch.cuda.device_count() >= 3 else [0, 0]
    mgr = TransferManager(device=1, worker_id=6)
    for d in set(devs):
        mgr.enable_peer_access(d)
    src = [_Pool(mgr, "LWs", 8, nl, no, nt, 2, hd, 2, kv=KV.OperationalNHD, device=d) for d in devs]
    dst = _Pool(mgr, "FC", 8, nl, no, nt, 4, hd, 2, kv=KV.UniversalTP, device=1, fill=0x44)
    ref = _host("FC", 8, nl, no, nt, 4, hd, 2, fill=0x44)
    for i, p in enumerate(src):
        randomize(p.twin, 40 + i)
        p.upload()
    sids, dids = [7, 2, 5], [1, 6, 3]
    plan = tp_reshard_plan(8, 4, 2, 0)
    for n in mgr.execute_reshard({r: (p.h, sids) for r, p in enumerate(src)}, dst.h, dids, plan):
        n.wait(20.0)
    torch.cuda.synchronize(1)
    dst.download()
    for w in plan:
        _expected(src[w.src_rank].twin, ref, sids, dids, KV.OperationalNHD, KV.UniversalTP, (nl, no, nt, hd),
                  (2, 4, w.src_head_begin, w.dst_head_begin, w.head_count))
    assert np.array_equal(dst.twin.buffers[0], ref.buffers[0])
    mgr.close()

"""GPU parity of the scaled fp8 <-> bf16 cast (an engine's per-layer fp8 KV-cache scales) on every cast path: the paged copy
(kvbm_paged_copy_opts.cast_scales), the layout transform and TP re-shard (kvbm_kernels_paged_permute_heads_scaled), the gather
(kvbm_kernels_paged_permute_gather_scaled) and the TransferManager entries, bit for bit against tests/scaled_cast_oracle.py.
Scales are distinct per (layer, outer), so a wrong index shows up."""
import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import ErrorCode, HeadWindow, KvbmError, TransferManager, TransferOptions, tp_reshard_plan
from oracle import oracle as O
from tests.gpu_util import DevicePool, ids_dev, paged_dst, randomize, stream_ptr
from tests.scaled_cast_oracle import bf16_to_e4m3_scaled, cast_bytes_scaled, e4m3_to_bf16_scaled, reshard_block_scaled
from tests.test_gpu_permute import _host, _Pool

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
ALL = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]
UNIVERSAL = (KV.UniversalTP, KV.UniversalPP)
CASTS = [CM.FP8E4M3_TO_BF16, CM.BF16_TO_FP8E4M3]
ELEMS = {CM.FP8E4M3_TO_BF16: (1, 2), CM.BF16_TO_FP8E4M3: (2, 1)}   # (source, destination) element bytes
TABLE_SCALES = [1.0, 0.25, 0.0173, 3.9, 2.0**-12, 600.0]           # tests/golden/make_scaled_cast_tables.py


def _scales(nl, no, seed=0):
    """Distinct calibrated-looking scales per (layer, outer), as a float32 CUDA tensor and its host copy."""
    rng = np.random.default_rng(seed)
    host = (rng.uniform(0.004, 4.0, nl * no) * (1 + np.arange(nl * no) * 1e-3)).astype(np.float32)
    assert len(set(host.tolist())) == nl * no
    return torch.from_numpy(host).to("cuda:0"), host


def _expected_copy(src, ref, sids, dids, cast, scales, layers):
    for s, d in zip(sids, dids):
        for l in layers:
            for o in range(src.outer_dim):
                ref.region_bytes(d, l, o)[:] = cast_bytes_scaled(src.region_bytes(s, l, o), int(cast), float(scales[l * src.outer_dim + o]))


def _paged(kind, cast, nl=4, no=2, nt=16, inner=256, layers=None, ndst=1, replicate=False, scales=None, seed=0, **opt):
    """A scaled paged copy of 5 blocks to `ndst` destinations; returns (destinations, their oracle twins)."""
    se, de = ELEMS[cast]
    src = _host(kind, 8, nl, no, nt, 1, inner, se)
    randomize(src, 100 + seed)
    S = DevicePool(src)
    t, h = _scales(nl, no, seed) if scales is None else scales
    lb, le = (0, nl) if layers is None else (layers.start, layers.stop)
    perm = lambda sd: [int(x) for x in np.random.default_rng(sd).permutation(8)[:5]]  # noqa: E731
    sids = [[7, 2, 0, 5, 3]] * ndst if replicate else [perm(seed + d) for d in range(ndst)]
    dids = [perm(50 + seed + d) for d in range(ndst)]
    dsts, refs, pools, keep = [], [], [], []
    shared = ids_dev(sids[0])
    for d in range(ndst):
        dst, ref = _host(kind, 8, nl, no, nt, 1, inner, de, fill=0x5C), _host(kind, 8, nl, no, nt, 1, inner, de, fill=0x5C)
        P = DevicePool(dst)
        si = shared if replicate else ids_dev(sids[d])
        di = ids_dev(dids[d])
        keep += [si, di]
        pools.append(P)
        dsts.append(paged_dst(P, si, di))
        _expected_copy(src, ref, sids[d], dids[d], cast, h, range(lb, le))
        refs.append((dst, ref))
    o = K.PagedCopyOpts(cast_scales=t.data_ptr(), **opt)
    K.check(K.paged_copy(S.desc, dsts, 5, lb, le, int(cast), o, stream_ptr()), "paged_copy scaled")
    torch.cuda.synchronize()
    for P in pools:
        P.download()
    return refs


def _check_pairs(refs):
    for dst, ref in refs:
        for got, want in zip(dst.buffers, ref.buffers):
            assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------------------------------
# paged copy
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layers", [None, range(1, 3)], ids=["all_layers", "layers_1_3"])
@pytest.mark.parametrize("kind", ["FC", "LWs", "LWf"])
@pytest.mark.parametrize("cast", CASTS, ids=lambda c: c.name)
def test_paged_copy_scaled(cast, kind, layers):
    _check_pairs(_paged(kind, cast, layers=layers, seed=int(cast) * 10 + len(kind)))


@pytest.mark.parametrize("cast", CASTS, ids=lambda c: c.name)
def test_paged_copy_scaled_fanout_and_replicate(cast):
    _check_pairs(_paged("LWs", cast, ndst=2, seed=3))
    _check_pairs(_paged("FC", cast, ndst=2, replicate=True, seed=4))


@pytest.mark.parametrize("cast", CASTS, ids=lambda c: c.name)
def test_paged_copy_scaled_force_simt_and_odd_tiles(cast):
    _check_pairs(_paged("LWs", cast, seed=5, force_simt=1))
    _check_pairs(_paged("FC", cast, seed=6, tile_bytes=96 * ELEMS[cast][0]))   # several tiles per region, TMA and SIMT mixed


@pytest.mark.parametrize("gate_mode", [K.GATE_SPIN, K.GATE_STREAM_WAIT], ids=["spin", "stream_wait"])
@pytest.mark.parametrize("cast", CASTS, ids=lambda c: c.name)
def test_paged_copy_scaled_gated(cast, gate_mode):
    """Both gate modes, released flags: the stream-wait form launches once per layer and must index by the absolute layer."""
    nl = 4
    ready = torch.full((nl,), 1, dtype=torch.int32, device="cuda:0")
    ws = torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device="cuda:0")
    _check_pairs(_paged("LWs", cast, nl=nl, layers=range(1, 4), seed=7, layer_ready_flags=ready.data_ptr(), sync_workspace=ws.data_ptr(),
                        epoch=1, gate_mode=gate_mode))


def test_every_fp8_code_and_bf16_pattern_at_the_table_scales():
    """All 256 codes and all 65 536 patterns, one (layer, outer) per table scale; the oracle is pinned to torch on the CPU."""
    nl, no = 3, 2
    t = torch.tensor(TABLE_SCALES, dtype=torch.float32, device="cuda:0")
    for cast, inner, pattern in ((CM.FP8E4M3_TO_BF16, 16, np.arange(256, dtype=np.uint8)),
                                 (CM.BF16_TO_FP8E4M3, 4096, np.arange(65536, dtype=np.uint16).view(np.uint8))):
        se, de = ELEMS[cast]
        src = _host("FC", 2, nl, no, 16, 1, inner, se)
        for l in range(nl):
            for o in range(no):
                src.region_bytes(0, l, o)[:] = pattern
        dst = _host("FC", 2, nl, no, 16, 1, inner, de)
        S, D = DevicePool(src), DevicePool(dst)
        a, b = ids_dev([0]), ids_dev([1])
        K.check(K.paged_copy(S.desc, [paged_dst(D, a, b)], 1, 0, nl, int(cast), K.PagedCopyOpts(cast_scales=t.data_ptr()), stream_ptr()))
        torch.cuda.synchronize()
        D.download()
        for l in range(nl):
            for o in range(no):
                s = TABLE_SCALES[l * no + o]
                want = e4m3_to_bf16_scaled(pattern, s).view(np.uint8) if cast == CM.FP8E4M3_TO_BF16 else bf16_to_e4m3_scaled(pattern.view(np.uint16), s)
                assert np.array_equal(dst.region_bytes(1, l, o), want), (cast.name, s)


def test_all_ones_equals_the_unscaled_launch():
    for cast in CASTS:
        ones = torch.ones(8, dtype=torch.float32, device="cuda:0")
        refs = _paged("LWs", cast, scales=(ones, np.ones(8, np.float32)), seed=8)
        se, de = ELEMS[cast]
        src = _host("LWs", 8, 4, 2, 16, 1, 256, se)
        randomize(src, 108)
        dst = _host("LWs", 8, 4, 2, 16, 1, 256, de, fill=0x5C)
        S, D = DevicePool(src), DevicePool(dst)
        sids, dids = [int(x) for x in np.random.default_rng(8).permutation(8)[:5]], [int(x) for x in np.random.default_rng(58).permutation(8)[:5]]
        a, b = ids_dev(sids), ids_dev(dids)
        K.check(K.paged_copy(S.desc, [paged_dst(D, a, b)], 5, 0, 4, int(cast), None, stream_ptr()))
        torch.cuda.synchronize()
        D.download()
        for got, want in zip(refs[0][0].buffers, dst.buffers):
            assert np.array_equal(got, want)


def test_round_trip_equals_the_oracle_composition():
    """bf16 -> fp8 at s, then fp8 -> bf16 at s: what an engine reads back from a scaled fp8 tier."""
    nl, no = 3, 2
    t, h = _scales(nl, no, 9)
    src = _host("FC", 4, nl, no, 16, 1, 128, 2)
    randomize(src, 9)
    mid, back = _host("FC", 4, nl, no, 16, 1, 128, 1), _host("FC", 4, nl, no, 16, 1, 128, 2)
    S, M, B = DevicePool(src), DevicePool(mid), DevicePool(back)
    ids = ids_dev([0, 1, 2, 3])
    o = K.PagedCopyOpts(cast_scales=t.data_ptr())
    K.check(K.paged_copy(S.desc, [paged_dst(M, ids, ids)], 4, 0, nl, int(CM.BF16_TO_FP8E4M3), o, stream_ptr()))
    K.check(K.paged_copy(M.desc, [paged_dst(B, ids, ids)], 4, 0, nl, int(CM.FP8E4M3_TO_BF16), o, stream_ptr()))
    torch.cuda.synchronize()
    B.download()
    for b in range(4):
        for l in range(nl):
            for o_ in range(no):
                s = float(h[l * no + o_])
                want = e4m3_to_bf16_scaled(bf16_to_e4m3_scaled(src.region_bytes(b, l, o_).view(np.uint16), s), s).view(np.uint8)
                assert np.array_equal(back.region_bytes(b, l, o_), want)


def test_a_transposed_scale_index_would_be_caught():
    """The expected bytes under scales[o * nl + l] differ from the kernel's: the tests above would see a transposed index."""
    nl, no = 4, 2
    t, h = _scales(nl, no, 11)
    refs = _paged("LWs", CM.FP8E4M3_TO_BF16, nl=nl, no=no, scales=(t, h), seed=11)
    _check_pairs(refs)
    transposed = h.reshape(nl, no).T.reshape(-1).copy()
    src = _host("LWs", 8, nl, no, 16, 1, 256, 1)
    randomize(src, 111)
    wrong = cast_bytes_scaled(src.region_bytes(0, 1, 0), int(CM.FP8E4M3_TO_BF16), float(transposed[1 * no + 0]))
    right = cast_bytes_scaled(src.region_bytes(0, 1, 0), int(CM.FP8E4M3_TO_BF16), float(h[1 * no + 0]))
    assert not np.array_equal(wrong, right)


def test_paged_copy_rejects_scales_without_a_cast():
    t, _ = _scales(2, 2)
    src = _host("FC", 2, 2, 2, 16, 1, 64, 2)
    S, D = DevicePool(src), DevicePool(_host("FC", 2, 2, 2, 16, 1, 64, 2))
    a = ids_dev([0])
    rc = K.paged_copy(S.desc, [paged_dst(D, a, a)], 1, 0, 2, int(CM.NONE), K.PagedCopyOpts(cast_scales=t.data_ptr()), stream_ptr())
    assert rc == K.CUDA_ERROR_INVALID_VALUE


# ---------------------------------------------------------------------------------------------------------------------
# layout transform / TP re-shard
# ---------------------------------------------------------------------------------------------------------------------
def _permute(src_kv, dst_kv, kind, cast, window, nl=3, no=2, nt=16, hd=32, layers=None, scales=None, seed=0):
    snh, dnh, sb, db, k = window
    se, de = ELEMS[cast]
    sk = "FC" if src_kv in UNIVERSAL else kind
    dk = "FC" if dst_kv in UNIVERSAL else kind
    src = _host(sk, 6, nl, no, nt, snh, hd, se)
    randomize(src, seed)
    dst, ref = _host(dk, 6, nl, no, nt, dnh, hd, de, fill=0x3A), _host(dk, 6, nl, no, nt, dnh, hd, de, fill=0x3A)
    S, D = DevicePool(src), DevicePool(dst)
    sids, dids = [4, 0, 5], [1, 5, 2]
    si, di = ids_dev(sids), ids_dev(dids)
    t, h = _scales(nl, no, seed) if scales is None else scales
    lb, le = (0, nl) if layers is None else (layers.start, layers.stop)
    K.check(K.paged_permute_heads(K.PermuteSide(S.desc, si.data_ptr(), int(src_kv)), K.PermuteSide(D.desc, di.data_ptr(), int(dst_kv)), 3, lb,
                                  le, snh, sb, dnh, db, k, nt, hd * se, int(cast), stream=stream_ptr(), cast_scales=t))
    torch.cuda.synchronize()
    D.download()
    for s, d in zip(sids, dids):
        O.write_logical_block(ref, d, reshard_block_scaled(O.read_logical_block(src, s), O.read_logical_block(ref, d), int(src_kv), int(dst_kv),
                                                           nl, no, nt, snh, dnh, hd * se, int(cast), h, sb, db, k, layers=layers))
    return dst, ref


@pytest.mark.parametrize("kind", ["FC", "LWs"])
@pytest.mark.parametrize("cast", CASTS, ids=lambda c: c.name)
@pytest.mark.parametrize("dst_kv", ALL, ids=lambda k: k.name)
@pytest.mark.parametrize("src_kv", ALL, ids=lambda k: k.name)
def test_scaled_permute_every_format_pair(src_kv, dst_kv, cast, kind):
    seed = 16 * int(src_kv) + 4 * int(dst_kv) + int(cast)
    for window, layers, hd in (((3, 3, 0, 0, 3), None, 32), ((4, 3, 1, 1, 2), range(1, 3), 80)):
        dst, ref = _permute(src_kv, dst_kv, kind, cast, window, hd=hd, layers=layers, seed=seed)
        _check_pairs([(dst, ref)])


def test_scaled_permute_all_ones_equals_unscaled():
    for cast in CASTS:
        se, de = ELEMS[cast]
        ones = (torch.ones(6, dtype=torch.float32, device="cuda:0"), np.ones(6, np.float32))
        dst, _ = _permute(KV.OperationalNHD, KV.UniversalTP, "LWs", cast, (4, 4, 0, 0, 4), scales=ones, seed=21)
        src = _host("LWs", 6, 3, 2, 16, 4, 32, se)
        randomize(src, 21)
        plain = _host("FC", 6, 3, 2, 16, 4, 32, de, fill=0x3A)
        S, D = DevicePool(src), DevicePool(plain)
        si, di = ids_dev([4, 0, 5]), ids_dev([1, 5, 2])
        K.check(K.paged_permute_heads(K.PermuteSide(S.desc, si.data_ptr(), int(KV.OperationalNHD)),
                                      K.PermuteSide(D.desc, di.data_ptr(), int(KV.UniversalTP)), 3, 0, 3, 4, 0, 4, 0, 4, 16, 32 * se, int(cast),
                                      stream=stream_ptr()))
        torch.cuda.synchronize()
        D.download()
        assert np.array_equal(dst.buffers[0], plain.buffers[0])


def test_scaled_entries_reject_scales_without_a_cast():
    t, _ = _scales(2, 2)
    side = K.PermuteSide(K.PagedLayout(0x1000, 4096, 2048, 2048, 2, 2, 4), 0x2000, int(KV.OperationalNHD))
    assert K.paged_permute_heads(side, side, 1, 0, 2, 1, 0, 1, 0, 1, 16, 128, 0, cast_scales=t) == K.CUDA_ERROR_INVALID_VALUE
    src = K.PermuteSource(side, 1, 0, 0, 1)
    assert K.paged_permute_gather([src], side, 1, 1, 0, 2, 16, 128, 0, cast_scales=t) == K.CUDA_ERROR_INVALID_VALUE


# ---------------------------------------------------------------------------------------------------------------------
# gather
# ---------------------------------------------------------------------------------------------------------------------
def test_scaled_gather_tp8_to_tp1():
    nl, no, nt, hd = 3, 2, 16, 64
    t, h = _scales(nl, no, 31)
    for cast in CASTS:
        se, de = ELEMS[cast]
        srcs = []
        for r in range(8):
            host = _host("LWs", 4, nl, no, nt, 1, hd, se)
            randomize(host, 300 + r)
            srcs.append((host, DevicePool(host), ids_dev([3, 0])))
        plan = tp_reshard_plan(8, 8, 1, 0)
        dst, ref = _host("FC", 4, nl, no, nt, 8, hd, de, fill=0x21), _host("FC", 4, nl, no, nt, 8, hd, de, fill=0x21)
        D = DevicePool(dst)
        di = ids_dev([1, 2])
        ps = [K.PermuteSource(K.PermuteSide(srcs[w.src_rank][1].desc, srcs[w.src_rank][2].data_ptr(), int(KV.OperationalNHD)), 1,
                              w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan]
        K.check(K.paged_permute_gather(ps, K.PermuteSide(D.desc, di.data_ptr(), int(KV.UniversalTP)), 8, 2, 0, nl, nt, hd * se, int(cast),
                                       stream=stream_ptr(), cast_scales=t))
        torch.cuda.synchronize()
        D.download()
        for i, d in enumerate([1, 2]):
            blk = O.read_logical_block(ref, d)
            for w in plan:
                blk = reshard_block_scaled(O.read_logical_block(srcs[w.src_rank][0], [3, 0][i]), blk, int(KV.OperationalNHD), int(KV.UniversalTP),
                                           nl, no, nt, 1, 8, hd * se, int(cast), h, w.src_head_begin, w.dst_head_begin, w.head_count)
            O.write_logical_block(ref, d, blk)
        _check_pairs([(dst, ref)])


# ---------------------------------------------------------------------------------------------------------------------
# TransferManager
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=17)
    yield m
    torch.cuda.synchronize()
    m.close()


def _expected_pool_copy(src, ref, sids, dids, cast, scales, nl, no):
    for s, d in zip(sids, dids):
        for l in range(nl):
            for o in range(no):
                ref.region_bytes(d, l, o)[:] = cast_bytes_scaled(src.region_bytes(s, l, o), int(cast), float(scales[l * no + o]))


def test_manager_transfer_fanout_reshard_and_gather(mgr):
    nl, no, nt, nh, hd = 3, 2, 16, 4, 64
    t, h = _scales(nl, no, 41)
    cast = CM.FP8E4M3_TO_BF16
    a = _Pool(mgr, "LWs", 8, nl, no, nt, nh, hd, 1, kv=KV.OperationalNHD)
    randomize(a.twin, 41)
    a.upload()
    sids, dids = [5, 1, 6], [0, 7, 3]
    # execute_transfer: a plain scaled paged copy
    b = _Pool(mgr, "LWs", 8, nl, no, nt, nh, hd, 2, kv=KV.OperationalNHD, fill=0x12)
    ref = _host("LWs", 8, nl, no, nt, nh, hd, 2, fill=0x12)
    mgr.execute_transfer(a.h, sids, b.h, dids, TransferOptions(cast_mode=cast, cast_scales=t)).wait(20.0)
    b.download()
    _expected_pool_copy(a.twin, ref, sids, dids, cast, h, nl, no)
    _check_pairs([(b.twin, ref)])
    # execute_fanout: two destinations, distinct source lists
    c, d = (_Pool(mgr, "LWs", 8, nl, no, nt, nh, hd, 2, kv=KV.OperationalNHD, fill=0x34) for _ in range(2))
    rc, rd = _host("LWs", 8, nl, no, nt, nh, hd, 2, fill=0x34), _host("LWs", 8, nl, no, nt, nh, hd, 2, fill=0x34)
    mgr.execute_fanout(a.h, [c.h, d.h], [sids, [2, 3, 4]], [dids, dids], options=TransferOptions(cast_mode=cast, cast_scales=t)).wait(20.0)
    c.download()
    d.download()
    _expected_pool_copy(a.twin, rc, sids, dids, cast, h, nl, no)
    _expected_pool_copy(a.twin, rd, [2, 3, 4], dids, cast, h, nl, no)
    _check_pairs([(c.twin, rc), (d.twin, rd)])
    # execute_reshard and execute_gather: TP2 -> TP1 into a UniversalTP pool, both with the same scales
    halves = [_Pool(mgr, "LWs", 8, nl, no, nt, 2, hd, 1, kv=KV.OperationalNHD) for _ in range(2)]
    for i, p in enumerate(halves):
        randomize(p.twin, 60 + i)
        p.upload()
    plan = tp_reshard_plan(4, 2, 1, 0)
    sources = {r: (p.h, sids) for r, p in enumerate(halves)}
    g, e = (_Pool(mgr, "FC", 8, nl, no, nt, nh, hd, 2, kv=KV.UniversalTP, fill=0x56) for _ in range(2))
    ref = _host("FC", 8, nl, no, nt, nh, hd, 2, fill=0x56)
    mgr.execute_gather(sources, g.h, dids, plan, TransferOptions(cast_mode=cast, cast_scales=t)).wait(20.0)
    for n in mgr.execute_reshard(sources, e.h, dids, plan, TransferOptions(cast_mode=cast, cast_scales=t)):
        n.wait(20.0)
    g.download()
    e.download()
    for w in plan:
        for s, dd in zip(sids, dids):
            O.write_logical_block(ref, dd, reshard_block_scaled(O.read_logical_block(halves[w.src_rank].twin, s), O.read_logical_block(ref, dd),
                                                                int(KV.OperationalNHD), int(KV.UniversalTP), nl, no, nt, 2, nh, hd, int(cast), h,
                                                                w.src_head_begin, w.dst_head_begin, w.head_count))
    _check_pairs([(g.twin, ref), (e.twin, ref)])


def test_manager_rejections(mgr):
    nl, no, nt, nh, hd = 3, 2, 16, 2, 64
    t, _ = _scales(nl, no, 51)
    a = _Pool(mgr, "LWs", 4, nl, no, nt, nh, hd, 2, kv=KV.OperationalNHD)
    b = _Pool(mgr, "LWs", 4, nl, no, nt, nh, hd, 1, kv=KV.OperationalNHD)
    c = _Pool(mgr, "LWs", 4, nl, no, nt, nh, hd, 2, kv=KV.OperationalNHD)
    launches = K.launch_count()

    def err(opts, dst=b):
        with pytest.raises(KvbmError) as e:
            mgr.execute_transfer(a.h, [0], dst.h, [1], opts)
        return e.value

    e = err(TransferOptions(cast_scales=t), dst=c)
    assert e.code == ErrorCode.ERR and "need a cast_mode" in e.msg
    e = err(TransferOptions(cast_mode=CM.BF16_TO_FP8E4M3, cast_scales=t[:nl * no - 1]))
    assert e.code == ErrorCode.RANGE and "num_layers * outer_dim" in e.msg
    host = np.ones(nl * no, dtype=np.float32)   # pageable host memory: must never reach a kernel
    e = err(TransferOptions(cast_mode=CM.BF16_TO_FP8E4M3, cast_scales=host))
    assert e.code == ErrorCode.ERR and "pinned host memory" in e.msg
    with pytest.raises(KvbmError) as g:
        mgr.execute_gather({0: (a.h, [0])}, b.h, [1], [HeadWindow(0, 0, 0, 1)], TransferOptions(cast_mode=CM.BF16_TO_FP8E4M3, cast_scales=host))
    assert g.value.code == ErrorCode.ERR and "pinned host memory" in g.value.msg
    assert K.launch_count() == launches
    # pinned host memory mapped into the device is accepted
    pinned = torch.from_numpy(_scales(nl, no, 52)[1]).pin_memory()
    mgr.execute_transfer(a.h, [0], b.h, [1], TransferOptions(cast_mode=CM.BF16_TO_FP8E4M3, cast_scales=pinned)).wait(20.0)


# ---------------------------------------------------------------------------------------------------------------------
# full-size Llama-3-70B fp8 TP4 -> bf16 TP2 (80 layers, 8 KV heads x 128, 16-token pages, OperationalNHD layer-separate pools)
# ---------------------------------------------------------------------------------------------------------------------
def test_full_size_llama_fp8_tp4_to_bf16_tp2(mgr):
    NL, NO, NT, H, HD, NB = 80, 2, 16, 8, 128, 12
    t, h = _scales(NL, NO, 61)
    src = [_Pool(mgr, "LWs", NB, NL, NO, NT, 2, HD, 1, kv=KV.OperationalNHD) for _ in range(4)]
    for i, p in enumerate(src):
        randomize(p.twin, 70 + i)
        p.upload()
    sids, dids = [3, 11, 0, 7], [5, 1, 9, 2]
    sources = {r: (p.h, sids) for r, p in enumerate(src)}
    for r in range(2):
        plan = tp_reshard_plan(H, 4, 2, r)
        one = _Pool(mgr, "LWs", NB, NL, NO, NT, 4, HD, 2, kv=KV.OperationalNHD, fill=0x5A)
        per = _Pool(mgr, "LWs", NB, NL, NO, NT, 4, HD, 2, kv=KV.OperationalNHD, fill=0x5A)
        opts = TransferOptions(cast_mode=CM.FP8E4M3_TO_BF16, cast_scales=t)
        mgr.execute_gather(sources, one.h, dids, plan, opts).wait(60.0)
        for n in mgr.execute_reshard(sources, per.h, dids, plan, opts):
            n.wait(60.0)
        one.download()
        per.download()
        for x, y in zip(one.twin.buffers, per.twin.buffers):
            assert np.array_equal(x, y)
        ref = _host("LWs", NB, NL, NO, NT, 4, HD, 2, fill=0x5A)
        for s, d in list(zip(sids, dids))[:2]:   # two blocks against the oracle
            blk = O.read_logical_block(ref, d)
            for w in plan:
                blk = reshard_block_scaled(O.read_logical_block(src[w.src_rank].twin, s), blk, int(KV.OperationalNHD), int(KV.OperationalNHD),
                                           NL, NO, NT, 2, 4, HD, int(CM.FP8E4M3_TO_BF16), h, w.src_head_begin, w.dst_head_begin, w.head_count)
            assert np.array_equal(O.read_logical_block(one.twin, d), blk)


@pytest.mark.multigpu
def test_two_gpu_scaled_pull():
    """A bf16 decode pool on GPU 1 pulls a scaled fp8 prefill pool of GPU 0 over NVLink (scales on GPU 1, the launching device)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    nl, no, nt, nh, hd = 4, 2, 16, 2, 128
    m = TransferManager(device=1, worker_id=18)
    m.enable_peer_access(0)
    t = torch.from_numpy(_scales(nl, no, 71)[1]).to("cuda:1")
    h = t.cpu().numpy()
    a = _Pool(m, "LWs", 6, nl, no, nt, nh, hd, 1, kv=KV.OperationalNHD, device=0)
    b = _Pool(m, "LWs", 6, nl, no, nt, nh, hd, 2, kv=KV.OperationalNHD, device=1, fill=0x44)
    ref = _host("LWs", 6, nl, no, nt, nh, hd, 2, fill=0x44)
    randomize(a.twin, 71)
    a.upload()
    m.execute_transfer(a.h, [4, 1], b.h, [0, 5], TransferOptions(cast_mode=CM.FP8E4M3_TO_BF16, cast_scales=t)).wait(20.0)
    torch.cuda.synchronize(1)
    b.download()
    _expected_pool_copy(a.twin, ref, [4, 1], [0, 5], CM.FP8E4M3_TO_BF16, h, nl, no)
    _check_pairs([(b.twin, ref)])
    m.close()

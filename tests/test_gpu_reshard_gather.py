"""GPU parity of the re-shard gather: kvbm_kernels_paged_permute_gather and TransferManager.execute_gather, against a fold of
tests/reshard_oracle.reshard_block over the windows.  Destinations are pre-filled with a pattern and compared whole, so the
heads no window covers are checked untouched."""
import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import (ErrorCode, HeadWindow, KvbmError, LayoutConfig, StorageKind, TransferManager, TransferOptions,
                                  tp_reshard_plan)
from oracle import oracle as O
from tests.gpu_util import DevicePool, ids_dev, randomize, stream_ptr
from tests.reshard_oracle import reshard_block
from tests.test_gpu_permute import _host, _Pool

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
ALL = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]
UNIVERSAL = (KV.UniversalTP, KV.UniversalPP)
CASTS = [CM.FP8E4M3_TO_BF16, CM.BF16_TO_FP8E4M3]
ELEMS = {CM.NONE: (2, 2), CM.FP8E4M3_TO_BF16: (1, 2), CM.BF16_TO_FP8E4M3: (2, 1)}   # (source, destination) element bytes


class _Src:
    """One source pool of a kernel-level gather: its host twin, format, head count and block ids."""

    def __init__(self, kind, kv, nb, geom, nh, sids, elem, seed):
        nl, no, nt, hd = geom
        self.kv, self.nh, self.sids = kv, nh, sids
        self.host = _host("FC" if kv in UNIVERSAL else kind, nb, nl, no, nt, nh, hd, elem)
        randomize(self.host, seed)
        self.dev = DevicePool(self.host)
        self.ids = ids_dev(sids)


def _gather(entries, dst, dst_kv, dnh, dids, geom, cast=CM.NONE, lb=0, le=None, done=0, epoch=0, completion=0, value=0, row=None):
    """entries: (source, src_head_begin, dst_head_begin, head_count) per window.  Runs the kernel, downloads dst when it ran."""
    nl, no, nt, hd = geom
    D = DevicePool(dst)
    di = ids_dev(dids)
    srcs = [K.PermuteSource(K.PermuteSide(s.dev.desc, s.ids.data_ptr(), int(s.kv)), s.nh, sb, db, k) for s, sb, db, k in entries]
    rc = K.paged_permute_gather(srcs, K.PermuteSide(D.desc, di.data_ptr(), int(dst_kv)), dnh, len(dids), lb, nl if le is None else le, nt,
                                hd * ELEMS[cast][0] if row is None else row, int(cast), done_flag=done, epoch=epoch, completion_flag=completion, completion_value=value,
                                stream=stream_ptr())
    torch.cuda.synchronize()
    if rc == 0:
        D.download()
    return rc


def _expected(entries, ref, dst_kv, dnh, dids, geom, cast=CM.NONE, layers=None):
    nl, no, nt, hd = geom
    for i, d in enumerate(dids):
        blk = O.read_logical_block(ref, d)
        for s, sb, db, k in entries:
            blk = reshard_block(O.read_logical_block(s.host, s.sids[i]), blk, int(s.kv), int(dst_kv), nl, no, nt, s.nh, dnh,
                                hd * ELEMS[cast][0], int(cast), sb, db, k, layers=layers)
        O.write_logical_block(ref, d, blk)


def _check(dst, ref):
    for got, want in zip(dst.buffers, ref.buffers):
        assert np.array_equal(got, want)


def _three_sources(src_kvs, kinds, geom, cast=CM.NONE, seed=0):
    """Four windows into a 7-head destination from three pools of different formats and head counts; source 0 appears twice
    and destination head 2 is covered by none of them (a partial plan)."""
    se = ELEMS[cast][0]
    s0 = _Src(kinds[0], src_kvs[0], 7, geom, 4, [5, 0, 3, 6], se, seed + 1)
    s1 = _Src(kinds[1], src_kvs[1], 6, geom, 2, [1, 4, 0, 2], se, seed + 2)
    s2 = _Src(kinds[2], src_kvs[2], 5, geom, 3, [4, 4, 1, 0], se, seed + 3)
    return [(s0, 1, 0, 2), (s1, 0, 3, 2), (s2, 2, 5, 1), (s0, 3, 6, 1)]


@pytest.mark.parametrize("dst_kv", ALL, ids=lambda k: k.name)
@pytest.mark.parametrize("src_kv", ALL, ids=lambda k: k.name)
@pytest.mark.parametrize("kinds", [("FC", "FC", "FC", "FC"), ("LWs", "LWf", "FC", "LWs"), ("LWf", "LWs", "LWs", "LWf")], ids=lambda k: "-".join(k))
def test_every_format_pair_with_mixed_source_formats(src_kv, dst_kv, kinds):
    """Source 0 has src_kv, sources 1 and 2 the next two formats: every format meets every destination format, mixed."""
    geom = (3, 2, 16, 32)
    i = ALL.index(src_kv)
    kvs = [ALL[i], ALL[(i + 1) % 4], ALL[(i + 2) % 4]]
    entries = _three_sources(kvs, kinds, geom, seed=10 * int(src_kv) + int(dst_kv))
    dk = "FC" if dst_kv in UNIVERSAL else kinds[3]
    dst, ref = _host(dk, 9, 3, 2, 16, 7, 32, 2, fill=0xAB), _host(dk, 9, 3, 2, 16, 7, 32, 2, fill=0xAB)
    dids = [8, 2, 4, 0]
    assert _gather(entries, dst, dst_kv, 7, dids, geom) == 0
    _expected(entries, ref, dst_kv, 7, dids, geom)
    _check(dst, ref)


@pytest.mark.parametrize("cast", CASTS, ids=lambda c: c.name)
@pytest.mark.parametrize("dst_kv", ALL, ids=lambda k: k.name)
def test_both_casts(dst_kv, cast):
    geom = (3, 2, 16, 32)
    entries = _three_sources([KV.OperationalNHD, KV.UniversalTP, KV.OperationalHND], ("LWs", "FC", "LWf"), geom, cast, seed=int(cast))
    de = ELEMS[cast][1]
    dk = "FC" if dst_kv in UNIVERSAL else "LWs"
    dst, ref = _host(dk, 9, 3, 2, 16, 7, 32, de, fill=0x3C), _host(dk, 9, 3, 2, 16, 7, 32, de, fill=0x3C)
    dids = [3, 7, 1, 0]
    assert _gather(entries, dst, dst_kv, 7, dids, geom, cast) == 0
    _expected(entries, ref, dst_kv, 7, dids, geom, cast)
    _check(dst, ref)


@pytest.mark.parametrize("hd,nt", [(16, 5), (64, 16), (80, 16), (96, 3), (128, 16), (576, 7)], ids=lambda x: str(x))
@pytest.mark.parametrize("cast", [CM.NONE] + CASTS, ids=lambda c: c.name)
def test_head_dims_and_layer_ranges(hd, nt, cast):
    """head_dim 16 ... 576: 16 / 64 / 128 rows take the shift-and-mask walk, 80 / 96 / 576 the multiply-high."""
    nl, no = 4, 2
    geom = (nl, no, nt, hd)
    se, de = ELEMS[cast]
    for layers in (None, range(1, 3), range(3, 4)):
        a = _Src("LWs", KV.OperationalNHD, 4, geom, 2, [3, 0], se, hd + nt)
        b = _Src("FC", KV.UniversalPP, 3, geom, 1, [1, 2], se, hd + nt + 1)
        entries = [(a, 1, 0, 1), (b, 0, 2, 1), (a, 0, 1, 1)]
        dst, ref = _host("FC", 4, nl, no, nt, 4, hd, de, fill=0x66), _host("FC", 4, nl, no, nt, 4, hd, de, fill=0x66)
        lb, le = (0, nl) if layers is None else (layers.start, layers.stop)
        assert _gather(entries, dst, KV.UniversalTP, 4, [1, 2], geom, cast, lb, le) == 0
        _expected(entries, ref, KV.UniversalTP, 4, [1, 2], geom, cast, layers)
        _check(dst, ref)


def test_more_than_eight_covered_heads_and_sixteen_sources():
    """16 one-head windows (TP16 -> TP1 on 16 heads): the warps loop past 8 covered heads."""
    geom = nl, no, nt, hd = 2, 2, 16, 64
    srcs = [_Src("LWs", KV.OperationalNHD, 3, geom, 1, [2, 0], 2, 50 + r) for r in range(16)]
    entries = [(srcs[w.src_rank], w.src_head_begin, w.dst_head_begin, w.head_count) for w in tp_reshard_plan(16, 16, 1, 0)]
    assert len(entries) == 16
    dst, ref = _host("LWs", 3, nl, no, nt, 16, hd, 2, fill=0x11), _host("LWs", 3, nl, no, nt, 16, hd, 2, fill=0x11)
    assert _gather(entries, dst, KV.OperationalNHD, 16, [1, 2], geom) == 0
    _expected(entries, ref, KV.OperationalNHD, 16, [1, 2], geom)
    _check(dst, ref)


def test_one_window_equals_paged_permute_heads():
    geom = nl, no, nt, hd = 3, 2, 16, 80
    for cast in [CM.NONE] + CASTS:
        se, de = ELEMS[cast]
        s = _Src("LWs", KV.OperationalNHD, 6, geom, 4, [0, 5, 2], se, 4)
        a, b = _host("FC", 6, nl, no, nt, 2, hd, de, fill=0x77), _host("FC", 6, nl, no, nt, 2, hd, de, fill=0x77)
        assert _gather([(s, 1, 1, 1)], a, KV.UniversalTP, 2, [3, 1, 4], geom, cast) == 0
        B = DevicePool(b)
        di = ids_dev([3, 1, 4])
        K.check(K.paged_permute_heads(K.PermuteSide(s.dev.desc, s.ids.data_ptr(), int(KV.OperationalNHD)),
                                      K.PermuteSide(B.desc, di.data_ptr(), int(KV.UniversalTP)), 3, 0, nl, 4, 1, 2, 1, 1, nt, hd * se,
                                      int(cast), stream=stream_ptr()))
        torch.cuda.synchronize()
        B.download()
        assert np.array_equal(a.buffers[0], b.buffers[0]) and bool((a.buffers[0] != 0x77).any())


def test_signals_once_empty_gathers_and_argument_checks():
    geom = nl, no, nt, hd = 4, 2, 16, 64
    a = _Src("LWf", KV.OperationalNHD, 6, geom, 2, [0], 2, 9)
    b = _Src("FC", KV.UniversalTP, 6, geom, 2, [3], 2, 10)
    dst = _host("FC", 6, nl, no, nt, 4, hd, 2)
    ok = [(a, 0, 0, 2), (b, 0, 2, 2)]
    flags = torch.zeros(4, dtype=torch.int32, device="cuda:0")
    launches0 = K.launch_count()
    assert _gather(ok, dst, KV.UniversalPP, 4, [1], geom, done=flags.data_ptr(), epoch=7, completion=flags.data_ptr() + 4, value=8) == 0
    assert K.launch_count() - launches0 == 2                    # one gather launch + one signal launch for both windows
    a.sids, b.sids = [], []
    assert _gather(ok, dst, KV.UniversalPP, 4, [], geom, done=flags.data_ptr() + 8, epoch=9, completion=flags.data_ptr() + 12, value=10) == 0
    assert flags.cpu().tolist() == [7, 8, 9, 10]
    run = lambda e, **kw: _gather(e, dst, KV.UniversalPP, 4, [1], geom, **kw)  # noqa: E731
    inval = K.CUDA_ERROR_INVALID_VALUE
    assert run([(a, 0, 0, 2), (b, 0, 1, 2)]) == inval          # overlapping destination windows
    assert run([(a, 0, 0, 0)]) == inval                        # an empty window
    assert run([(a, 1, 0, 2)]) == inval                        # past the source's heads
    assert run([(a, 0, 3, 2)]) == inval                        # past the destination's heads
    assert run([(a, 0, 0, 1)] * 17) == inval                   # more than 16 sources
    assert run(ok, cast=3, row=hd * 2) == inval                # unknown cast mode
    assert run(ok, lb=0, le=nl + 1) == inval


# ---------------------------------------------------------------------------------------------------------------------
# through the TransferManager
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=7)
    yield m
    torch.cuda.synchronize()
    m.close()


def test_manager_gather_one_completion_after_every_window(mgr):
    nl, no, nt, hd = 4, 2, 16, 128
    # TP4 -> TP2 of an 8-head model: decode rank 1 takes heads from prefill ranks 2 (NHD) and 3 (HND), into UniversalTP
    s2 = _Pool(mgr, "LWs", 10, nl, no, nt, 2, hd, 2, kv=KV.OperationalNHD)
    s3 = _Pool(mgr, "LWf", 10, nl, no, nt, 2, hd, 2, kv=KV.OperationalHND)
    d = _Pool(mgr, "FC", 8, nl, no, nt, 4, hd, 2, kv=KV.UniversalTP, fill=0x21)
    ref = _host("FC", 8, nl, no, nt, 4, hd, 2, fill=0x21)
    for i, p in enumerate((s2, s3)):
        randomize(p.twin, 31 + i)
        p.upload()
    sids, dids = [9, 0, 4], [2, 7, 5]
    plan = tp_reshard_plan(8, 4, 2, 1)
    flag = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    launches0, moved0, h2d0 = K.launch_count(), mgr.bytes_moved(), mgr.h2d_bytes()
    note = mgr.execute_gather({2: (s2.h, sids), 3: (s3.h, sids)}, d.h, dids, plan, TransferOptions(done_flag=flag.data_ptr(), epoch=3))
    note.wait(20.0)
    assert K.launch_count() - launches0 == 2                    # the gather + the completion signal
    assert int(flag.item()) == 3
    assert mgr.bytes_moved() - moved0 == 3 * nl * no * nt * 4 * hd * 2
    assert mgr.h2d_bytes() - h2d0 == 3 * 3 * 4                  # one upload: two source tables + the destination's, int32
    d.download()
    for w in plan:
        src, kv = ((s2, KV.OperationalNHD), (s3, KV.OperationalHND))[w.src_rank - 2]
        for s, t in zip(sids, dids):
            O.write_logical_block(ref, t, reshard_block(O.read_logical_block(src.twin, s), O.read_logical_block(ref, t), int(kv), int(KV.UniversalTP),
                                                        nl, no, nt, 2, 4, hd * 2, 0, w.src_head_begin, w.dst_head_begin, w.head_count))
    assert np.array_equal(d.twin.buffers[0], ref.buffers[0])
    # a caller stream returns the completed notification; a layer range and the cast compose
    a8 = _Pool(mgr, "LWs", 10, nl, no, nt, 2, hd, 1, kv=KV.OperationalNHD)
    u = _Pool(mgr, "FC", 6, nl, no, nt, 4, hd, 2, kv=KV.UniversalPP, fill=0x44)
    ref_u = _host("FC", 6, nl, no, nt, 4, hd, 2, fill=0x44)
    randomize(a8.twin, 33)
    a8.upload()
    s = torch.cuda.Stream()
    n = mgr.execute_gather({0: (a8.h, [1, 2])}, u.h, [5, 0], [HeadWindow(0, 1, 3, 1), HeadWindow(0, 0, 0, 1)],
                           TransferOptions(cast_mode=CM.FP8E4M3_TO_BF16, layer_range=range(1, 3), cuda_stream=s.cuda_stream))
    assert n.token == 0
    s.synchronize()
    u.download()
    for sb, db in ((1, 3), (0, 0)):
        for x, y in zip([1, 2], [5, 0]):
            O.write_logical_block(ref_u, y, reshard_block(O.read_logical_block(a8.twin, x), O.read_logical_block(ref_u, y), int(KV.OperationalNHD),
                                                          int(KV.UniversalPP), nl, no, nt, 2, 4, hd, int(CM.FP8E4M3_TO_BF16), sb, db, 1,
                                                          layers=range(1, 3)))
    assert np.array_equal(u.twin.buffers[0], ref_u.buffers[0])


def test_manager_gather_rejections(mgr):
    nl, no, nt, hd = 3, 2, 16, 64
    a = _Pool(mgr, "LWs", 6, nl, no, nt, 2, hd, 2, kv=KV.OperationalNHD)
    b = _Pool(mgr, "LWs", 6, nl, no, nt, 4, hd, 2, kv=KV.OperationalNHD)
    plan = [HeadWindow(0, 0, 0, 2), HeadWindow(1, 0, 2, 2)]
    src = {0: (a.h, [0]), 1: (a.h, [1])}

    def err(fn):
        with pytest.raises(KvbmError) as e:
            fn()
        return e.value

    e = err(lambda: mgr.execute_gather(src, b.h, [2], [HeadWindow(0, 0, 0, 2), HeadWindow(1, 0, 1, 2)]))
    assert e.code == ErrorCode.OVERLAP
    e = err(lambda: mgr.execute_gather(src, b.h, [2], [HeadWindow(0, 0, 0, 1)] * 17))
    assert e.code == ErrorCode.UNSUPPORTED
    e = err(lambda: mgr.execute_gather(src, b.h, [2], plan, TransferOptions(head_window=(0, 0, 2))))
    assert e.code == ErrorCode.ERR
    e = err(lambda: mgr.execute_gather(src, b.h, [2], [HeadWindow(0, 1, 0, 2)]))
    assert e.code == ErrorCode.RANGE and "Head window" in e.msg
    ready = torch.zeros(nl, dtype=torch.int32, device="cuda:0")
    e = err(lambda: mgr.execute_gather(src, b.h, [2], plan, TransferOptions(layer_ready_flags=ready.data_ptr(), epoch=1)))
    assert e.code == ErrorCode.UNSUPPORTED and "layer streaming / multicast" in e.msg
    e = err(lambda: mgr.execute_gather(src, b.h, [2], plan, TransferOptions(multicast=1)))
    assert e.code == ErrorCode.UNSUPPORTED and "layer streaming / multicast" in e.msg
    e = err(lambda: mgr.execute_gather(src, b.h, [2], plan, TransferOptions(per_dst_done_flags=[ready.data_ptr()])))
    assert e.code == ErrorCode.UNSUPPORTED and "layer streaming / multicast" in e.msg
    unknown = _Pool(mgr, "LWs", 6, nl, no, nt, 2, hd, 2, kv=None)
    e = err(lambda: mgr.execute_gather({0: (a.h, [0]), 1: (unknown.h, [1])}, b.h, [2], plan))
    assert e.code == ErrorCode.UNSUPPORTED and "Layout transformation not supported" in e.msg
    e = err(lambda: mgr.execute_gather(src, b.h, [2], plan, TransferOptions(dst_kv_layout=int(KV.UniversalTP))))
    assert e.code == ErrorCode.INCOMPATIBLE and "fully contiguous" in e.msg
    d32 = _Pool(mgr, "LWs", 6, nl, no, nt, 2, 2 * hd, 2, kv=KV.OperationalNHD)       # head_dim 128 against 64
    e = err(lambda: mgr.execute_gather({0: (a.h, [0]), 1: (d32.h, [1])}, b.h, [2], plan))
    assert e.code == ErrorCode.INCOMPATIBLE and "Head row size mismatch" in e.msg
    other_layers = _Pool(mgr, "LWs", 6, nl + 1, no, nt, 2, hd, 2, kv=KV.OperationalNHD)
    e = err(lambda: mgr.execute_gather({0: (a.h, [0]), 1: (other_layers.h, [1])}, b.h, [2], plan))
    assert e.code == ErrorCode.INCOMPATIBLE and "incompatible layer counts" in e.msg
    e = err(lambda: mgr.execute_gather({0: (a.h, [0]), 1: (a.h, [9])}, b.h, [2], plan))      # block id past the pool
    assert e.code == ErrorCode.RANGE
    e = err(lambda: mgr.execute_gather(src, b.h, [2], plan, TransferOptions(layer_range=range(0, nl + 1))))
    assert e.code == ErrorCode.RANGE
    # one source in pinned host memory: the device source takes CudaAsyncD2D, the pinned one CudaAsyncH2D
    cfg = LayoutConfig(6, nl, no, nt, 2 * hd, num_heads=2)
    pinned = torch.zeros(cfg.required_bytes(), dtype=torch.uint8).pin_memory()
    hs = mgr.register_fully_contiguous(cfg, pinned.data_ptr(), pinned.numel(), StorageKind.Pinned, 0)
    mgr.set_kv_block_layout(hs, KV.OperationalNHD)
    e = err(lambda: mgr.execute_gather({0: (a.h, [0]), 1: (hs, [1])}, b.h, [2], plan))
    assert e.code == ErrorCode.UNSUPPORTED and "same CUDA strategy" in e.msg


# ---------------------------------------------------------------------------------------------------------------------
# full-size Llama-3-70B: 80 layers, 8 KV heads x 128, 16-token pages, engine pools OperationalNHD layer-separate; the gather
# against execute_reshard's per-window transfers on the same pools
# ---------------------------------------------------------------------------------------------------------------------
NL, NO, NT, H, HD = 80, 2, 16, 8, 128
NB = 20


def _tp_pools(mgr, tp, elem=2, fill=0, seed=None):
    nh = max(1, H // tp)
    pools = [_Pool(mgr, "LWs", NB, NL, NO, NT, nh, HD, elem, kv=KV.OperationalNHD, fill=fill) for _ in range(tp)]
    if seed is not None:
        gen = torch.Generator(device="cuda:0").manual_seed(seed)
        for p in pools:
            for t in p.mem:
                t.copy_(torch.randint(0, 256, t.shape, dtype=torch.uint8, device="cuda:0", generator=gen))
        torch.cuda.synchronize()
    return pools


@pytest.mark.parametrize("src_tp,dst_tp,cast", [(4, 2, CM.NONE), (2, 8, CM.NONE), (8, 1, CM.NONE), (4, 2, CM.FP8E4M3_TO_BF16)],
                         ids=lambda x: str(x))
def test_full_size_llama_gather_equals_execute_reshard(mgr, src_tp, dst_tp, cast):
    se, de = ELEMS[cast]
    src = _tp_pools(mgr, src_tp, se, seed=src_tp * 10 + dst_tp)
    one, per = _tp_pools(mgr, dst_tp, de, fill=0x5A), _tp_pools(mgr, dst_tp, de, fill=0x5A)
    rng = np.random.default_rng(src_tp * 10 + dst_tp)
    sids, dids = list(map(int, rng.permutation(NB)[:16])), list(map(int, rng.permutation(NB)[:16]))
    sources = {s: (p.h, sids) for s, p in enumerate(src)}
    flag = torch.zeros(dst_tp, dtype=torch.int32, device="cuda:0")
    notes = []
    for r in range(dst_tp):
        plan = tp_reshard_plan(H, src_tp, dst_tp, r)
        notes.append(mgr.execute_gather(sources, one[r].h, dids, plan, TransferOptions(cast_mode=cast, done_flag=flag[r:].data_ptr(), epoch=r + 1)))
        notes += mgr.execute_reshard(sources, per[r].h, dids, plan, TransferOptions(cast_mode=cast))
    for n in notes:
        n.wait(60.0)
    torch.cuda.synchronize()
    assert flag.cpu().tolist() == list(range(1, dst_tp + 1))
    for a, b in zip(one, per):
        for x, y in zip(a.mem, b.mem):
            assert torch.equal(x, y)
        assert bool((a.mem[0].view(NO, NB, -1)[:, [i for i in range(NB) if i not in dids]] == 0x5A).all())


@pytest.mark.multigpu
def test_decode_gpu_gathers_its_heads_from_two_prefill_gpus():
    """TP4 -> TP2 over NVLink as one gather: decode rank 0 on GPU 1 reads heads from prefill ranks 0 and 1 (GPUs 0 and 2 when
    there are three, else both on GPU 0) and assembles its 4-head UniversalTP blocks."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    nl, no, nt, hd = 4, 2, 16, 128
    devs = [0, 2] if torch.cuda.device_count() >= 3 else [0, 0]
    m = TransferManager(device=1, worker_id=8)
    for d in set(devs):
        m.enable_peer_access(d)
    src = [_Pool(m, "LWs", 8, nl, no, nt, 2, hd, 2, kv=KV.OperationalNHD, device=d) for d in devs]
    dst = _Pool(m, "FC", 8, nl, no, nt, 4, hd, 2, kv=KV.UniversalTP, device=1, fill=0x44)
    ref = _host("FC", 8, nl, no, nt, 4, hd, 2, fill=0x44)
    for i, p in enumerate(src):
        randomize(p.twin, 40 + i)
        p.upload()
    sids, dids = [7, 2, 5], [1, 6, 3]
    plan = tp_reshard_plan(8, 4, 2, 0)
    m.execute_gather({r: (p.h, sids) for r, p in enumerate(src)}, dst.h, dids, plan).wait(20.0)
    torch.cuda.synchronize(1)
    dst.download()
    for w in plan:
        for s, t in zip(sids, dids):
            O.write_logical_block(ref, t, reshard_block(O.read_logical_block(src[w.src_rank].twin, s), O.read_logical_block(ref, t),
                                                        int(KV.OperationalNHD), int(KV.UniversalTP), nl, no, nt, 2, 4, hd * 2, 0,
                                                        w.src_head_begin, w.dst_head_begin, w.head_count))
    assert np.array_equal(dst.twin.buffers[0], ref.buffers[0])
    m.close()

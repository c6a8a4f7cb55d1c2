"""GPU parity of the layout-transforming hand-off (kvbm_kernels_paged_permute and TransferManager transfers between layouts
whose KvBlockLayouts differ) against the oracle's dim_order definition (oracle.kv_layout_permute, itself checked against
the pinned K2 / K3 restatement in tests/test_oracle_kernels.py).

Reference: lib/kvbm-physical/src/layout/kv_block_layout.rs:40-119, transfer/executor/mod.rs:27-119 (select_transform_kernel
and the effective_*_layout overrides -- dead code there: validate_layout_compatibility, transfer/mod.rs:128-147, rejects every
pair these tests execute)."""
import itertools

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import (BlockDimension, ErrorCode, KvbmError, LayoutConfig, StorageKind, TransferManager,
                                  TransferOptions)
from oracle import oracle as O
from tests.gpu_util import DevicePool, ids_dev, randomize, stream_ptr

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
ALL = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]
UNIVERSAL = (KV.UniversalTP, KV.UniversalPP)


def _host(kind, nb, nl, no, nt, nh, hd, elem, fill=0):
    k, bd = {"FC": (O.FC, O.BLOCK_IS_FIRST_DIM), "LWf": (O.LW, O.BLOCK_IS_FIRST_DIM), "LWs": (O.LW, O.BLOCK_IS_SECOND_DIM)}[kind]
    return O.Layout(k, nb, nl, no, nt, nh * hd, elem, block_dim=bd, fill=fill, allow_fp8=(elem == 1))


def _expected(src, ref, sids, dids, src_kv, dst_kv, nl, no, nt, nh, row, layers=None):
    """ref (a host twin of the destination before the transfer) after the transfer, per the oracle."""
    for s, d in zip(sids, dids):
        blk = O.read_logical_block(src, s)
        old = O.read_logical_block(ref, d)
        O.write_logical_block(ref, d, O.kv_layout_permute(blk, int(src_kv), int(dst_kv), nl, no, nt, nh, row, layers=layers, dst_old=old))


def _run_kernel(src, dst, sids, dids, src_kv, dst_kv, nl, nh, nt, row, lb=0, le=None, done=0, epoch=0):
    S, D = DevicePool(src), DevicePool(dst)
    si, di = ids_dev(sids), ids_dev(dids)
    rc = K.paged_permute(K.PermuteSide(S.desc, si.data_ptr(), int(src_kv)), K.PermuteSide(D.desc, di.data_ptr(), int(dst_kv)),
                         len(sids), lb, nl if le is None else le, nh, nt, row, done_flag=done, epoch=epoch, stream=stream_ptr())
    torch.cuda.synchronize()
    if rc == 0:
        D.download()
    return rc


@pytest.mark.parametrize("src_kv,dst_kv", list(itertools.product(ALL, ALL)), ids=lambda k: k.name)
@pytest.mark.parametrize("kinds", [("FC", "FC"), ("LWf", "LWs"), ("LWs", "FC")], ids=lambda k: "-".join(k))
def test_every_pair_of_layouts_matches_the_oracle(src_kv, dst_kv, kinds):
    nl, no, nt, nh, hd, elem = 3, 2, 16, 4, 32, 2
    row = hd * elem
    sk = "FC" if src_kv in UNIVERSAL else kinds[0]
    dk = "FC" if dst_kv in UNIVERSAL else kinds[1]
    src, dst, ref = _host(sk, 7, nl, no, nt, nh, hd, elem), _host(dk, 9, nl, no, nt, nh, hd, elem, 0xAB), _host(dk, 9, nl, no, nt, nh, hd, elem, 0xAB)
    randomize(src, 11 * int(src_kv) + int(dst_kv))
    sids, dids = [5, 0, 3, 6], [8, 2, 4, 0]
    assert _run_kernel(src, dst, sids, dids, src_kv, dst_kv, nl, nh, nt, row) == 0
    _expected(src, ref, sids, dids, src_kv, dst_kv, nl, no, nt, nh, row)
    for got, want in zip(dst.buffers, ref.buffers):        # moved blocks AND every untouched byte
        assert np.array_equal(got, want)


@pytest.mark.parametrize("geom", [(1, 1, 1, 1, 8, 2), (2, 2, 5, 3, 128, 1), (2, 1, 64, 8, 128, 2), (1, 2, 3, 2, 1024, 4), (4, 2, 16, 40, 64, 2),
                                  (2, 2, 16, 8, 80, 2), (2, 2, 16, 4, 96, 2), (2, 1, 16, 1, 576, 2), (1, 2, 7, 3, 24, 2), (2, 2, 33, 2, 40, 2)],
                         ids=lambda g: "nl%d-no%d-nt%d-nh%d-hd%d-e%d" % g)
@pytest.mark.parametrize("src_kv,dst_kv", [(KV.OperationalNHD, KV.UniversalTP), (KV.UniversalTP, KV.OperationalHND),
                                           (KV.OperationalHND, KV.OperationalNHD), (KV.UniversalPP, KV.UniversalTP)], ids=lambda k: k.name)
def test_row_sizes_head_counts_and_odd_pages(geom, src_kv, dst_kv):
    """16 B ... 4 KiB rows, one head (a single warp) ... 40 heads (warps loop), page sizes that are not powers of two,
    fp8 (1-byte) elements; rows that are not a power of two (head_dim 80 / 96 / 40 / 24, MLA's 576-wide single head) take the
    incremental (token, column) walk."""
    nl, no, nt, nh, hd, elem = geom
    row = hd * elem
    sk = "FC" if src_kv in UNIVERSAL else "LWs"
    dk = "FC" if dst_kv in UNIVERSAL else "LWf"
    src, dst, ref = _host(sk, 5, nl, no, nt, nh, hd, elem), _host(dk, 5, nl, no, nt, nh, hd, elem, 0x5A), _host(dk, 5, nl, no, nt, nh, hd, elem, 0x5A)
    randomize(src, 3)
    sids, dids = [4, 1, 2], [0, 3, 1]
    assert _run_kernel(src, dst, sids, dids, src_kv, dst_kv, nl, nh, nt, row) == 0
    _expected(src, ref, sids, dids, src_kv, dst_kv, nl, no, nt, nh, row)
    for got, want in zip(dst.buffers, ref.buffers):
        assert np.array_equal(got, want)


def test_layer_ranges_signals_and_argument_checks():
    nl, no, nt, nh, hd, elem = 4, 2, 16, 4, 64, 2
    row = hd * elem
    src = _host("LWf", 6, nl, no, nt, nh, hd, elem)
    randomize(src, 9)
    for lb, le in ((0, 1), (1, 3), (3, 4), (2, 2)):
        dst, ref = _host("FC", 6, nl, no, nt, nh, hd, elem, 0x33), _host("FC", 6, nl, no, nt, nh, hd, elem, 0x33)
        assert _run_kernel(src, dst, [1, 2], [5, 0], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, row, lb, le) == 0
        if le > lb:
            _expected(src, ref, [1, 2], [5, 0], KV.OperationalNHD, KV.UniversalTP, nl, no, nt, nh, row, layers=range(lb, le))
        assert np.array_equal(dst.buffers[0], ref.buffers[0])
    # done flag: epoch arrives after the data (also for an empty transfer)
    flag = torch.zeros(2, dtype=torch.int32, device="cuda:0")
    dst = _host("FC", 6, nl, no, nt, nh, hd, elem)
    assert _run_kernel(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalPP, nl, nh, nt, row, done=flag.data_ptr(), epoch=7) == 0
    assert _run_kernel(src, dst, [], [], KV.OperationalNHD, KV.UniversalPP, nl, nh, nt, row, done=flag.data_ptr() + 4, epoch=9) == 0
    assert flag.cpu().tolist() == [7, 9]
    # contract violations are cudaErrorInvalidValue, nothing is launched
    inval = K.CUDA_ERROR_INVALID_VALUE
    assert _run_kernel(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, 48) == inval          # region != nt*nh*row
    assert _run_kernel(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, 8) == inval           # row < 16 B
    assert _run_kernel(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt * 16, 8) == inval      # ... even when the region size fits
    assert _run_kernel(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh * 16, nt, 8) == inval
    assert _run_kernel(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh * 2, nt, row) == inval     # region != nt*nh*row
    assert _run_kernel(src, dst, [0], [1], KV.Unknown, KV.UniversalTP, nl, nh, nt, row) == inval
    assert _run_kernel(src, dst, [0], [1], KV.Custom, KV.UniversalTP, nl, nh, nt, row) == inval
    assert _run_kernel(src, dst, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, row, 0, nl + 1) == inval
    other = _host("FC", 6, nl + 1, no, nt, nh, hd, elem)
    assert _run_kernel(src, other, [0], [1], KV.OperationalNHD, KV.UniversalTP, nl, nh, nt, row) == inval       # layer counts differ


def test_agrees_with_the_legacy_k2_k3_symbols():
    """The pointer-table kernels the reference exports (tensor_kernels.cu:306-360) and the paged form write the same bytes,
    for rows that are a power-of-two number of 16 B vectors (hd 128) and rows that are not (hd 80)."""
    nl, no, nt, nh, elem = 5, 2, 16, 8, 2
    nb = 6
    for hd in (128, 80):
        row = hd * elem
        src = _host("LWs", nb, nl, no, nt, nh, hd, elem)
        randomize(src, 21)
        S = DevicePool(src)
        uni_a = torch.zeros(nb * nl * no * nt * nh * row, dtype=torch.uint8, device="cuda:0")
        uni_b = torch.zeros_like(uni_a)
        bs = nl * no * nt * nh * row
        # legacy: host-built pointer tables
        chunk_ptrs = torch.tensor([S.region_addr(b, l, o) for b in range(nb) for l in range(nl) for o in range(no)], dtype=torch.int64, device="cuda:0")
        uni_ptrs = torch.tensor([uni_a.data_ptr() + b * bs for b in range(nb)], dtype=torch.int64, device="cuda:0")
        K.check(K.universal_from_block(uni_ptrs.data_ptr(), chunk_ptrs.data_ptr(), nb, nh, nl, no, nt, hd, K.TensorDataType.BF16,
                                       K.BlockLayout.NHD, stream_ptr()))
        # paged: layouts + block tables only
        lb = torch.tensor([uni_b.data_ptr() + l * no * nt * nh * row for l in range(nl)], dtype=torch.int64, device="cuda:0")
        udesc = K.PagedLayout(lb.data_ptr(), bs, nt * nh * row, nt * nh * row, nl, no, nb)
        ids = ids_dev(range(nb))
        K.check(K.paged_permute(K.PermuteSide(S.desc, ids.data_ptr(), int(KV.OperationalNHD)), K.PermuteSide(udesc, ids.data_ptr(), int(KV.UniversalTP)),
                                nb, 0, nl, nh, nt, row, stream=stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(uni_a, uni_b) and bool(uni_a.any()), hd


# ---------------------------------------------------------------------------------------------------------------------
# through the TransferManager
# ---------------------------------------------------------------------------------------------------------------------
class _Pool:
    def __init__(self, mgr, kind, nb, nl, no, nt, nh, hd, elem, kv, device=0, fill=0):
        self.twin = _host(kind, nb, nl, no, nt, nh, hd, elem, fill)
        self.cfg = LayoutConfig(nb, nl, no, nt, nh * hd, dtype_width_bytes=elem, num_heads=nh, allow_fp8=(elem == 1))
        self.mem = [torch.from_numpy(b.copy()).to(f"cuda:{device}") for b in self.twin.buffers]
        ptrs, sizes = [t.data_ptr() for t in self.mem], [t.numel() for t in self.mem]
        if kind == "FC":
            self.h = mgr.register_fully_contiguous(self.cfg, ptrs[0], sizes[0], StorageKind.Device, device)
        else:
            bd = BlockDimension.BlockIsSecondDim if kind == "LWs" else BlockDimension.BlockIsFirstDim
            self.h = mgr.register_layer_separate(self.cfg, ptrs, sizes, bd, StorageKind.Device, device)
        if kv is not None:
            mgr.set_kv_block_layout(self.h, kv)

    def upload(self):
        for t, b in zip(self.mem, self.twin.buffers):
            t.copy_(torch.from_numpy(b))
        torch.cuda.synchronize()

    def download(self):
        torch.cuda.synchronize()
        for t, b in zip(self.mem, self.twin.buffers):
            b[:] = t.cpu().numpy()


@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=5)
    yield m
    torch.cuda.synchronize()
    m.close()


def test_manager_turns_a_format_mismatch_into_one_permuting_launch(mgr):
    nl, no, nt, nh, hd, elem = 4, 2, 16, 8, 128, 2
    row = hd * elem
    g = (nl, no, nt, nh, hd, elem)
    op = _Pool(mgr, "LWs", 12, *g, kv=KV.OperationalNHD)          # the engine's pool (vLLM layout)
    uni = _Pool(mgr, "FC", 10, *g, kv=KV.UniversalTP, fill=0x11)  # storage / re-shard format
    ref = _host("FC", 10, *g, fill=0x11)
    randomize(op.twin, 77)
    op.upload()
    sids, dids = [3, 11, 0, 7], [9, 1, 4, 2]
    launches0 = K.launch_count()
    note = mgr.execute_transfer(op.h, sids, uni.h, dids)
    note.wait(20.0)
    assert K.launch_count() - launches0 == 2                      # the permuting kernel + the completion signal
    uni.download()
    _expected(op.twin, ref, sids, dids, KV.OperationalNHD, KV.UniversalTP, nl, no, nt, nh, row)
    assert np.array_equal(uni.twin.buffers[0], ref.buffers[0])
    # back into a different operational format on a third pool: UniversalTP -> OperationalHND
    hnd = _Pool(mgr, "LWf", 8, *g, kv=KV.OperationalHND)
    ref2 = _host("LWf", 8, *g)
    mgr.execute_transfer(uni.h, dids, hnd.h, [0, 1, 2, 3]).wait(20.0)
    hnd.download()
    _expected(uni.twin, ref2, dids, [0, 1, 2, 3], KV.UniversalTP, KV.OperationalHND, nl, no, nt, nh, row)
    for a, b in zip(hnd.twin.buffers, ref2.buffers):
        assert np.array_equal(a, b)
    # which must equal a direct NHD -> HND transpose of the original blocks
    direct = _Pool(mgr, "LWf", 8, *g, kv=KV.OperationalHND)
    mgr.execute_transfer(op.h, sids, direct.h, [0, 1, 2, 3]).wait(20.0)
    direct.download()
    for a, b in zip(direct.twin.buffers, hnd.twin.buffers):
        assert np.array_equal(a, b)
    # equal formats stay the plain paged copy (one launch, bit-identical blocks)
    twin_pool = _Pool(mgr, "FC", 12, *g, kv=KV.OperationalNHD)
    launches0 = K.launch_count()
    mgr.execute_transfer(op.h, [3], twin_pool.h, [5]).wait(20.0)
    assert K.launch_count() - launches0 == 1
    twin_pool.download()
    assert np.array_equal(O.read_logical_block(twin_pool.twin, 5), O.read_logical_block(op.twin, 3))


def test_manager_overrides_layer_ranges_done_flag_and_rejections(mgr):
    nl, no, nt, nh, hd, elem = 3, 2, 16, 4, 64, 2
    row = hd * elem
    g = (nl, no, nt, nh, hd, elem)
    a = _Pool(mgr, "FC", 6, *g, kv=None)             # Unknown: formats come from the options (options.rs:63-80)
    b = _Pool(mgr, "FC", 6, *g, kv=None, fill=0x22)
    ref = _host("FC", 6, *g, fill=0x22)
    randomize(a.twin, 5)
    a.upload()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    o = TransferOptions(src_kv_layout=int(KV.OperationalHND), dst_kv_layout=int(KV.UniversalPP), layer_range=range(1, 3),
                        done_flag=flag.data_ptr(), epoch=41)
    mgr.execute_transfer(a.h, [2, 4], b.h, [0, 5], o).wait(20.0)
    b.download()
    assert int(flag.item()) == 41
    _expected(a.twin, ref, [2, 4], [0, 5], KV.OperationalHND, KV.UniversalPP, nl, no, nt, nh, row, layers=range(1, 3))
    assert np.array_equal(b.twin.buffers[0], ref.buffers[0])
    # rejections
    with pytest.raises(KvbmError) as e:                          # Unknown -> known: the reference's error
        mgr.execute_transfer(a.h, [0], b.h, [1], TransferOptions(dst_kv_layout=int(KV.UniversalTP)))
    assert e.value.code == ErrorCode.UNSUPPORTED and "Layout transformation not supported" in e.value.msg
    lw = _Pool(mgr, "LWf", 6, *g, kv=KV.OperationalNHD)
    with pytest.raises(KvbmError) as e:                          # a universal format cannot live in a layer-separate pool
        mgr.execute_transfer(a.h, [0], lw.h, [1], TransferOptions(src_kv_layout=int(KV.OperationalNHD), dst_kv_layout=int(KV.UniversalTP)))
    assert e.value.code == ErrorCode.INCOMPATIBLE and "fully contiguous" in e.value.msg
    with pytest.raises(KvbmError) as e:                          # validation still runs first
        mgr.execute_transfer(a.h, [0, 0], b.h, [1, 1], o)
    assert e.value.code == ErrorCode.DUPLICATE_DST
    ready = torch.zeros(nl, dtype=torch.int32, device="cuda:0")
    with pytest.raises(KvbmError) as e:
        mgr.execute_transfer(a.h, [0], b.h, [1], TransferOptions(src_kv_layout=4, dst_kv_layout=1, layer_ready_flags=ready.data_ptr(), epoch=1))
    assert e.value.code == ErrorCode.UNSUPPORTED and "layer streaming" in e.value.msg


def test_full_size_tp_reshard_round_trip_is_the_identity(mgr):
    """Llama-3-70B KV geometry (80 layers, 8 KV heads x 128, bf16, 16-token pages): engine pool -> universal -> engine pool.
    Property check at full size (oracle on two blocks only: it is a numpy transpose of 5 MiB per block)."""
    nl, no, nt, nh, hd, elem = 80, 2, 16, 8, 128, 2
    row = hd * elem
    nb, n = 72, 64
    g = (nl, no, nt, nh, hd, elem)
    op = _Pool(mgr, "LWs", nb, *g, kv=KV.OperationalNHD)
    uni = _Pool(mgr, "FC", nb, *g, kv=KV.UniversalTP)
    back = _Pool(mgr, "LWs", nb, *g, kv=KV.OperationalNHD)
    gen = torch.Generator(device="cuda:0").manual_seed(1)
    for t in op.mem:
        t.copy_(torch.randint(0, 256, t.shape, dtype=torch.uint8, device="cuda:0", generator=gen))
    torch.cuda.synchronize()        # the manager's streams are non-blocking: they do not wait for torch's fill
    rng = np.random.default_rng(2)
    s, u, d = (list(map(int, rng.permutation(nb)[:n])) for _ in range(3))
    mgr.execute_transfer(op.h, s, uni.h, u).wait(30.0)
    mgr.execute_transfer(uni.h, u, back.h, d).wait(30.0)
    torch.cuda.synchronize()
    region = nt * nh * row
    for l in (0, 41, 79):           # block-is-second-dim: [outer][block][region] per layer
        src_l, dst_l = op.mem[l].view(no, nb, region), back.mem[l].view(no, nb, region)
        assert torch.equal(src_l[:, s, :], dst_l[:, d, :])
    op.download()
    uni.download()
    for i in (0, n - 1):
        want = O.kv_layout_permute(O.read_logical_block(op.twin, s[i]), int(KV.OperationalNHD), int(KV.UniversalTP), nl, no, nt, nh, row)
        assert np.array_equal(O.read_logical_block(uni.twin, u[i]), want)


@pytest.mark.multigpu
def test_permuting_pull_over_nvlink():
    """Decode-side launch: the prefill GPU's operational pool is read over NVLink and lands in universal format locally."""
    nl, no, nt, nh, hd, elem = 4, 2, 16, 8, 128, 2
    row = hd * elem
    g = (nl, no, nt, nh, hd, elem)
    mgr = TransferManager(device=1, worker_id=6)
    mgr.enable_peer_access(0)
    src = _Pool(mgr, "LWs", 16, *g, kv=KV.OperationalNHD, device=0)
    dst = _Pool(mgr, "FC", 16, *g, kv=KV.UniversalTP, device=1, fill=0x44)
    ref = _host("FC", 16, *g, fill=0x44)
    randomize(src.twin, 8)
    src.upload()
    torch.cuda.synchronize(0)
    sids, dids = [15, 2, 9, 4, 0], [1, 14, 3, 8, 6]
    mgr.execute_transfer(src.h, sids, dst.h, dids).wait(20.0)
    torch.cuda.synchronize(1)
    dst.download()
    _expected(src.twin, ref, sids, dids, KV.OperationalNHD, KV.UniversalTP, nl, no, nt, nh, row)
    assert np.array_equal(dst.twin.buffers[0], ref.buffers[0])
    mgr.close()

"""The permuting kernels (the paged permute, the gather, re-paging and the re-paging gather) and the paged copy at the limits their
launchers accept, each paired with its first rejected neighbour, and past 4 GiB, against the oracles:

- warps that loop over heads past 8, and the gather's 16 sources / 256 covered heads (also through the manager);
- the walk's smallest and largest rows, the multiply-high row split and the small page's split at their bounds;
- token positions at the 32-bit bound (kernels) and at 2^31 (manager);
- block offsets past 2^32 in one > 4 GiB fully contiguous pool, as destination and as source;
- manager hand-offs whose id lists outgrow a staging slot's arena share, then many short hand-offs reusing the slots.

Pools start from random bytes (the > 4 GiB pool from a fill function of the byte offset), every destination keeps blocks no id
names, and whole destination pools are compared.  A rejected neighbour returns cudaErrorInvalidValue (the manager: its error code)
before any launch, so K.launch_count() stays put."""
import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import ErrorCode, KvbmError, LayoutConfig, StorageKind, TransferManager, tp_reshard_plan
from oracle import oracle as O
from tests.cast_oracle import cast_bytes
from tests.gpu_util import DevicePool, ids_dev, randomize, stream_ptr
from tests.repage_gather_oracle import repage_gather
from tests.repage_oracle import repage, table_slice
from tests.reshard_oracle import reshard_block
from tests.test_gpu_permute import _host, _Pool

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
INVAL = K.CUDA_ERROR_INVALID_VALUE
UNIVERSAL = (KV.UniversalTP, KV.UniversalPP)
ELEMS = {CM.NONE: (2, 2), CM.FP8E4M3_TO_BF16: (1, 2), CM.BF16_TO_FP8E4M3: (2, 1)}   # (source, destination) element bytes


def _kind(kv, pref):
    return "FC" if kv in UNIVERSAL else pref


def _scales(nl, no):
    """One distinct dequantisation scale per (layer, outer) pair."""
    return np.array([0.3 + 0.55 * i for i in range(nl * no)], dtype=np.float32)


def _rejected(run):
    """run() returns cudaErrorInvalidValue and launches nothing."""
    before = K.launch_count()
    assert run() == INVAL
    assert K.launch_count() == before


def _windows(plan):
    """A tp_reshard_plan as (source index, src_head_begin, dst_head_begin, head_count), sources numbered in rank order."""
    index = {r: i for i, r in enumerate(sorted({w.src_rank for w in plan}))}
    return [(index[w.src_rank], w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan]


class _Range:
    """Host twins for tokens [tb, te) of one sequence: per source a pool of page ps holding the blocks the range touches (plus
    one no id names) in a shuffled table, and a destination pool of page pd likewise (plus a guard block).  The block-table
    kernels (permute, gather) take ps == pd, tb = 0 and te = n * ps: block sids[i] -> dids[i].  One oracle for all four: the
    re-paging gather's, which is the gather for equal pages and re-paging for one full window."""

    def __init__(self, ps, pd, tb, te, geom, cast, src_nhs, dst_nh, src_kvs, dst_kv, seed, src_kind="LWs", dst_kind="LWf"):
        self.nl, self.no, self.hd = geom
        self.ps, self.pd, self.tb, self.te, self.cast = ps, pd, tb, te, cast
        se, de = ELEMS[cast]
        self.src_row = self.hd * se
        self.src_nhs, self.dst_nh = list(src_nhs), dst_nh
        self.src_kvs = [src_kvs[i % len(src_kvs)] for i in range(len(self.src_nhs))]
        self.dst_kv = dst_kv
        rng = np.random.default_rng(seed)
        ns, nd = -(-te // ps) - tb // ps, -(-te // pd) - tb // pd
        self.src, self.sids = [], []
        for i, (nh, kv) in enumerate(zip(self.src_nhs, self.src_kvs)):
            h = _host(_kind(kv, src_kind), ns + 1, self.nl, self.no, ps, nh, self.hd, se)
            randomize(h, seed + 10 + i)
            self.src.append(h)
            self.sids.append([int(x) for x in rng.permutation(ns + 1)[:ns]])
        self.dst = _host(_kind(dst_kv, dst_kind), nd + 1, self.nl, self.no, pd, dst_nh, self.hd, de)
        self.ref = _host(_kind(dst_kv, dst_kind), nd + 1, self.nl, self.no, pd, dst_nh, self.hd, de)
        randomize(self.dst, seed + 1)
        for a, b in zip(self.ref.buffers, self.dst.buffers):
            a[:] = b
        guard = int(rng.integers(0, nd + 1))
        self.dids = [b for b in rng.permutation(nd + 1).tolist() if b != guard]

    def launch(self, kernel, windows=None, scales=None, te=None):
        """One launch of `kernel` ("permute", "gather", "repage", "repage_gather") over the range (te overrides its end); the
        destination twin holds the result when it returns 0.  Id tables carry two spare entries, so a longer range still names
        blocks of the pools."""
        te = self.te if te is None else te
        windows = windows or [(0, 0, 0, self.dst_nh)]
        S = [DevicePool(h) for h in self.src]
        D = DevicePool(self.dst)
        si = [ids_dev(x + x[:1] * 2) for x in self.sids]
        di = ids_dev(self.dids + self.dids[:1] * 2)
        sides = [K.PermuteSide(p.desc, i.data_ptr(), int(kv)) for p, i, kv in zip(S, si, self.src_kvs)]
        dside = K.PermuteSide(D.desc, di.data_ptr(), int(self.dst_kv))
        srcs = [K.PermuteSource(sides[s], self.src_nhs[s], sb, db, k) for s, sb, db, k in windows]
        sc = None if scales is None else torch.from_numpy(scales).cuda()
        n, st = len(self.dids), stream_ptr()
        if kernel == "permute":
            rc = K.paged_permute_heads(sides[0], dside, n, 0, self.nl, self.src_nhs[0], 0, self.dst_nh, 0, self.dst_nh, self.ps, self.src_row,
                                       int(self.cast), stream=st, cast_scales=sc)
        elif kernel == "gather":
            rc = K.paged_permute_gather(srcs, dside, self.dst_nh, n, 0, self.nl, self.ps, self.src_row, int(self.cast), stream=st, cast_scales=sc)
        elif kernel == "repage":
            rc = K.paged_repage(sides[0], self.ps, dside, self.pd, self.tb, te, 0, self.nl, self.dst_nh, self.src_row, int(self.cast), sc,
                                stream=st)
        else:
            rc = K.paged_repage_gather(srcs, self.ps, dside, self.dst_nh, self.pd, self.tb, te, 0, self.nl, self.src_row, int(self.cast), sc,
                                       stream=st)
        torch.cuda.synchronize()
        if rc == 0:
            D.download()
        return rc

    def check(self, windows=None, scales=None):
        windows = windows or [(0, 0, 0, self.dst_nh)]
        sources = [([O.read_logical_block(h, b) for b in ids], int(kv), nh)
                   for h, ids, kv, nh in zip(self.src, self.sids, self.src_kvs, self.src_nhs)]
        new = repage_gather(sources, windows, [O.read_logical_block(self.ref, b) for b in self.dids], int(self.dst_kv), self.dst_nh, self.nl,
                            self.no, self.ps, self.pd, self.src_row, self.tb, self.te, int(self.cast), scales)
        for b, blk in zip(self.dids, new):
            O.write_logical_block(self.ref, b, blk)
        for got, want in zip(self.dst.buffers, self.ref.buffers):
            assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------------------------------
# 1. heads past 8, and the gathers' maxima
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nh,ps,pd,cast,scaled", [(9, 16, 64, CM.NONE, False), (12, 64, 16, CM.NONE, False), (40, 16, 64, CM.NONE, False),
                                                  (40, 64, 16, CM.NONE, False), (12, 6, 48, CM.NONE, False),
                                                  (12, 16, 64, CM.FP8E4M3_TO_BF16, True), (40, 64, 16, CM.BF16_TO_FP8E4M3, True)],
                         ids=lambda x: str(getattr(x, "name", x)))
def test_repage_warps_loop_over_heads_past_eight(nh, ps, pd, cast, scaled):
    """A CTA has at most 8 warps, so heads 8.. are a warp's second (.. fifth) head; 12 is no multiple of 8."""
    big = max(ps, pd)
    c = _Range(ps, pd, 5, 2 * big - 3, (2, 2, 32), cast, [nh], nh, [KV.OperationalNHD], KV.OperationalNHD, nh + ps, dst_kind="FC")
    scales = _scales(2, 2) if scaled else None
    assert c.launch("repage", scales=scales) == 0
    c.check(scales=scales)


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16)], ids=str)
def test_repage_takes_more_than_256_heads(ps, pd):
    """kvbm_kernels_paged_repage has no head limit: 300 heads of a 16 B row, 37 or 38 per warp.  The same full window through
    kvbm_kernels_paged_repage_gather is past the gather's 256 heads."""
    nh = 300
    c = _Range(ps, pd, 5, 2 * max(ps, pd) - 3, (2, 2, 8), CM.NONE, [nh], nh, [KV.OperationalNHD], KV.OperationalHND, nh + ps)
    _rejected(lambda: c.launch("repage_gather"))
    assert c.launch("repage") == 0
    c.check()


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16)], ids=str)
def test_repage_gather_covers_more_than_eight_heads(ps, pd):
    """TP4 -> TP1 on 32 KV heads: four 8-head windows, 32 covered heads over 8 warps."""
    windows = _windows(tp_reshard_plan(32, 4, 1, 0))
    c = _Range(ps, pd, 3, 2 * max(ps, pd) - 5, (2, 2, 32), CM.NONE, [8] * 4, 32, [KV.OperationalHND, KV.OperationalNHD], KV.OperationalNHD, 17)
    assert c.launch("repage_gather", windows) == 0
    c.check(windows)


@pytest.mark.parametrize("kernel,ps,pd", [("gather", 16, 16), ("repage_gather", 16, 64), ("repage_gather", 64, 16)], ids=str)
def test_gathers_at_sixteen_sources_and_256_heads(kernel, ps, pd):
    """tp_reshard_plan(256, 16, 1, 0): 16 sources of 16 heads cover 256 destination heads.  Neighbours: 17 sources (255 heads),
    and 257 covered heads (a 17-head window) over 16 sources."""
    tb, te = (0, 2 * ps) if kernel == "gather" else (5, 2 * max(ps, pd) - 3)
    windows = _windows(tp_reshard_plan(256, 16, 1, 0))
    assert len(windows) == K.GATHER_MAX_SOURCES and sum(w[3] for w in windows) == K.GATHER_MAX_HEADS
    c = _Range(ps, pd, tb, te, (2, 2, 16), CM.NONE, [16] * 16, 256, [KV.OperationalNHD, KV.UniversalPP, KV.OperationalHND],
               KV.OperationalNHD, 3, src_kind="FC")
    assert c.launch(kernel, windows) == 0
    c.check(windows)
    _rejected(lambda: c.launch(kernel, [(j % 16, 0, 15 * j, 15) for j in range(17)]))
    n = _Range(ps, pd, tb, te, (1, 1, 16), CM.NONE, [16] * 15 + [17], 257, [KV.OperationalNHD], KV.OperationalNHD, 4)
    _rejected(lambda: n.launch(kernel, [(i, 0, 16 * i, 16) for i in range(15)] + [(15, 0, 240, 17)]))


def test_manager_repage_gather_takes_sixteen_windows():
    """execute_repage_gather with the 16 windows of TP16 -> TP1 on 256 heads; a 17th window is UNSUPPORTED, nothing launched."""
    mgr = TransferManager(device=0, worker_id=51)
    try:
        nl, no, hd, ps, pd = 2, 2, 16, 16, 64
        tb, te = 5, 125
        plan = tp_reshard_plan(256, 16, 1, 0)
        ns, nd = -(-te // ps), -(-te // pd)
        src = {r: _Pool(mgr, "LWs", ns + 1, nl, no, ps, 16, hd, 2, kv=KV.OperationalNHD) for r in range(16)}
        dst = _Pool(mgr, "LWs", nd + 1, nl, no, pd, 256, hd, 2, kv=KV.OperationalHND)
        for r, p in src.items():
            randomize(p.twin, 60 + r)
            p.upload()
        randomize(dst.twin, 59)
        dst.upload()
        ref = _host("LWs", nd + 1, nl, no, pd, 256, hd, 2)
        for a, b in zip(ref.buffers, dst.twin.buffers):
            a[:] = b
        stab = {r: [(i * 5 + r) % (ns + 1) for i in range(ns)] for r in range(16)}
        dtab = list(range(nd, 0, -1))                 # block 0 is the guard
        sources = {r: (src[r].h, stab[r]) for r in range(16)}
        mgr.execute_repage_gather(sources, dst.h, dtab, plan, range(tb, te)).wait(20.0)
        torch.cuda.synchronize()
        dst.download()
        new = repage_gather([([O.read_logical_block(src[r].twin, b) for b in stab[r]], int(KV.OperationalNHD), 16) for r in range(16)],
                            _windows(plan), [O.read_logical_block(ref, b) for b in dtab], int(KV.OperationalHND), 256, nl, no, ps, pd, hd * 2,
                            tb, te)
        for b, blk in zip(dtab, new):
            O.write_logical_block(ref, b, blk)
        for a, b in zip(dst.twin.buffers, ref.buffers):
            assert np.array_equal(a, b)
        w0 = plan[0]
        split = [type(w0)(w0.src_rank, w0.src_head_begin, w0.dst_head_begin, 8),
                 type(w0)(w0.src_rank, w0.src_head_begin + 8, w0.dst_head_begin + 8, w0.head_count - 8)] + plan[1:]
        before = K.launch_count()
        with pytest.raises(KvbmError) as e:
            mgr.execute_repage_gather(sources, dst.h, dtab, split, range(tb, te))
        assert e.value.code == ErrorCode.UNSUPPORTED and K.launch_count() == before
    finally:
        torch.cuda.synchronize()
        mgr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. row and page extremes
# ---------------------------------------------------------------------------------------------------------------------
# (cast, head_dim accepted, head_dim of the first rejected neighbour): the walk counts 16 B vectors of the fp8 side's row under a
# cast, else of the row; it takes 16 B ... 64 KiB, so the bf16 side of a cast reaches 128 KiB
ROWS = {"16B": (CM.NONE, 8, 4), "bf16_32B_to_fp8_16B": (CM.BF16_TO_FP8E4M3, 16, 8), "fp8_16B_to_bf16_32B": (CM.FP8E4M3_TO_BF16, 16, 8),
        "64KiB": (CM.NONE, 32768, 32776), "fp8_64KiB_to_bf16_128KiB": (CM.FP8E4M3_TO_BF16, 65536, 65552),
        "bf16_128KiB_to_fp8_64KiB": (CM.BF16_TO_FP8E4M3, 65536, 65552)}


def _row_case(kernel, cast, hd, seed):
    large = hd > 1024
    nl, no, nt = (1, 1, 2) if large else (2, 2, 16)
    ps, pd = {"permute": (nt, nt), "gather": (nt, nt), "repage": (nt // 2, nt), "repage_gather": (nt, nt // 2)}[kernel]
    tb, te = (0, 2 * nt) if ps == pd else (1, 2 * nt - 1)
    gather = kernel in ("gather", "repage_gather")
    src_nhs, dst_nh = ([1, 1], 2) if gather else ([2], 2)
    c = _Range(ps, pd, tb, te, (nl, no, hd), cast, src_nhs, dst_nh, [KV.OperationalHND], KV.OperationalNHD, seed)
    return c, ([(0, 0, 1, 1), (1, 0, 0, 1)] if gather else None)


@pytest.mark.parametrize("row", list(ROWS))
@pytest.mark.parametrize("kernel", ["permute", "gather", "repage", "repage_gather"])
def test_smallest_and_largest_rows(kernel, row):
    cast, hd, bad = ROWS[row]
    c, windows = _row_case(kernel, cast, hd, 7)
    assert c.launch(kernel, windows) == 0
    c.check(windows)
    n, windows = _row_case(kernel, cast, bad, 8)
    _rejected(lambda: n.launch(kernel, windows))


V_BOUND = 4095                    # 16 B vectors per row: 65 520 B, not a power of two, so the row split is a multiply-high


def test_row_split_bound_holds_for_the_chosen_row():
    """row_split takes nt while nt * V < 2^32 // V: 256 for V = 4095, not 257."""
    assert 256 * V_BOUND < 2**32 // V_BOUND <= 257 * V_BOUND


@pytest.mark.parametrize("kernel,cast", [("permute", CM.NONE), ("permute", CM.FP8E4M3_TO_BF16), ("repage", CM.NONE)],
                         ids=["permute", "permute_fp8_to_bf16", "repage"])
def test_multiply_high_row_split_at_its_bound(kernel, cast):
    """V = 4095 vectors per walk row at the largest page the launcher takes for it (256), every vector of a head's 256 rows; a page
    of 257 is rejected.  Under the cast the walk row is the fp8 side's: head_dim 65 520 (a bf16 row of 131 040 B)."""
    hd = V_BOUND * 16 // ELEMS[cast][0]
    if kernel == "permute":
        c = _Range(256, 256, 0, 512, (1, 1, hd), cast, [1], 1, [KV.OperationalNHD], KV.UniversalTP, 11)
        n = _Range(257, 257, 0, 257, (1, 1, hd), cast, [1], 1, [KV.OperationalNHD], KV.UniversalTP, 12)
    else:
        c = _Range(256, 16, 5, 2 * 256 - 3, (1, 1, hd), cast, [1], 1, [KV.OperationalNHD], KV.OperationalHND, 13)
        n = _Range(257, 1, 0, 3, (1, 1, hd), cast, [1], 1, [KV.OperationalNHD], KV.OperationalHND, 14)
    assert c.launch(kernel) == 0
    c.check()
    _rejected(lambda: n.launch(kernel))


SMALL_PAGE = 3 * 1024                                 # not a power of two: the page split is a multiply-high by ceil(2^32 / 3072)
BIG_PAGE = SMALL_PAGE * (2**32 // SMALL_PAGE**2)      # 3072 * 455: the largest multiple with big_page * small_page < 2^32


@pytest.mark.parametrize("ps,pd", [(SMALL_PAGE, BIG_PAGE), (BIG_PAGE, SMALL_PAGE)], ids=["small_to_big", "big_to_small"])
def test_small_page_split_at_its_bound(ps, pd):
    """A non-power-of-two small page at a ratio of 455, so the page split runs q up to BIG_PAGE - 1 = 1 397 759, just below
    2^32 / 3072.  The next multiple (ratio 456) is rejected."""
    assert BIG_PAGE * SMALL_PAGE < 2**32 <= (BIG_PAGE + SMALL_PAGE) * SMALL_PAGE
    c = _Range(ps, pd, 1000, BIG_PAGE + 5000, (1, 1, 8), CM.NONE, [1], 1, [KV.OperationalNHD], KV.OperationalNHD, 21)
    assert c.launch("repage") == 0
    c.check()
    nb = BIG_PAGE + SMALL_PAGE
    n = _Range(SMALL_PAGE if ps < pd else nb, nb if ps < pd else SMALL_PAGE, 0, 1, (1, 1, 8), CM.NONE, [1], 1, [KV.OperationalNHD],
               KV.OperationalNHD, 22)
    _rejected(lambda: n.launch("repage"))


# ---------------------------------------------------------------------------------------------------------------------
# 3. token positions at the 32-bit bound
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["repage", "repage_gather"])
@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (48, 16), (16, 48), (1, 16), (16, 1)], ids=str)
def test_token_positions_at_the_32_bit_bound(ps, pd, kernel):
    """token_end is the largest the kernel takes for the page pair (the range's last block of the larger page ends at
    te_max < 2^32), the range starts mid-block; te_max + 1 is rejected."""
    big = max(ps, pd)
    te = (2**32 - 1) // big * big
    tb = te - 2 * big - 3
    if kernel == "repage":
        c = _Range(ps, pd, tb, te, (2, 2, 32), CM.NONE, [4], 4, [KV.OperationalNHD], KV.OperationalHND, ps + pd)
        windows = None
    else:
        c = _Range(ps, pd, tb, te, (2, 2, 32), CM.NONE, [2, 2], 4, [KV.OperationalHND, KV.OperationalNHD], KV.OperationalNHD, ps + pd)
        windows = _windows(tp_reshard_plan(4, 2, 1, 0))
    assert c.launch(kernel, windows) == 0
    c.check(windows)
    _rejected(lambda: c.launch(kernel, windows, te=te + 1))


def test_manager_token_range_ends_at_2_pow_31():
    """execute_repage takes a range ending at 2^31; one token more is a RANGE error and launches nothing."""
    mgr = TransferManager(device=0, worker_id=52)
    try:
        nl, no, nh, hd, ps, pd = 2, 2, 4, 32, 16, 64
        tb, te = 2**31 - 77, 2**31
        ns, nd = -(-te // ps) - tb // ps, -(-te // pd) - tb // pd
        src = _Pool(mgr, "LWs", ns + 1, nl, no, ps, nh, hd, 2, kv=KV.OperationalNHD)
        dst = _Pool(mgr, "LWf", nd + 1, nl, no, pd, nh, hd, 2, kv=KV.OperationalHND)
        randomize(src.twin, 71)
        randomize(dst.twin, 72)
        src.upload()
        dst.upload()
        ref = _host("LWf", nd + 1, nl, no, pd, nh, hd, 2)
        for a, b in zip(ref.buffers, dst.twin.buffers):
            a[:] = b
        sids, dids = list(range(ns, 0, -1)), list(range(1, nd + 1))
        mgr.execute_repage(src.h, sids, dst.h, dids, range(tb, te)).wait(20.0)
        torch.cuda.synchronize()
        dst.download()
        new = repage([O.read_logical_block(src.twin, b) for b in sids], [O.read_logical_block(ref, b) for b in dids], int(KV.OperationalNHD),
                     int(KV.OperationalHND), nl, no, nh, ps, pd, hd * 2, tb, te)
        for b, blk in zip(dids, new):
            O.write_logical_block(ref, b, blk)
        for a, b in zip(dst.twin.buffers, ref.buffers):
            assert np.array_equal(a, b)
        before = K.launch_count()
        with pytest.raises(KvbmError) as e:
            mgr.execute_repage(src.h, sids, dst.h, dids, range(tb, te + 1))
        assert e.value.code == ErrorCode.RANGE and K.launch_count() == before
    finally:
        torch.cuda.synchronize()
        mgr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. long sequences through the manager: id lists past a staging slot's arena share, then many short hand-offs
# ---------------------------------------------------------------------------------------------------------------------
DIM_ORDER = {KV.UniversalTP: "hlot", KV.UniversalPP: "lhot", KV.OperationalHND: "loht", KV.OperationalNHD: "loth"}


class _DevPool:
    """A fully contiguous device pool of random bytes registered with a manager, in format kv.  view(): its
    [block, token, layer, outer, head, row] view, written from the format's dim order (a block is its dims in that order)."""

    def __init__(self, mgr, nb, nl, no, nt, nh, hd, kv, gen):
        self.nb, self.nl, self.no, self.nt, self.nh, self.row, self.kv = nb, nl, no, nt, nh, hd * 2, kv
        self.bs = nl * no * nt * nh * self.row
        self.gen = gen
        self.mem = torch.empty(nb * self.bs, dtype=torch.uint8, device="cuda")
        self.randomize()
        cfg = LayoutConfig(nb, nl, no, nt, nh * hd, dtype_width_bytes=2, num_heads=nh)
        self.h = mgr.register_fully_contiguous(cfg, self.mem.data_ptr(), self.mem.numel(), StorageKind.Device, 0)
        mgr.set_kv_block_layout(self.h, kv)

    def randomize(self):
        self.mem.copy_(torch.randint(0, 256, self.mem.shape, dtype=torch.uint8, device="cuda", generator=self.gen))
        torch.cuda.synchronize()      # the manager's streams do not wait for torch's

    def view(self, mem=None):
        order = DIM_ORDER[self.kv]
        size = {"h": self.nh, "l": self.nl, "o": self.no, "t": self.nt}
        v = (self.mem if mem is None else mem).view(self.nb, *[size[c] for c in order], self.row)
        return v.permute(0, *[1 + order.index(c) for c in "tloh"], 5)

    def block(self, b, mem=None):
        return (self.mem if mem is None else mem)[b * self.bs:(b + 1) * self.bs].cpu().numpy()


def _torch_expect(exp, dst, dtab, tb, te, sources, windows):
    """exp (a copy of dst's bytes) after tokens [tb, te) of each window's source heads land on its destination heads.  Tables
    are whole sequences' (entry i holds tokens i * page ..); each side's sequence view is the blocks the range touches along the
    token axis."""
    dv = dst.view(exp)
    t = torch.tensor(table_slice(dtab, tb, te, dst.nt), device="cuda")
    d0 = tb // dst.nt * dst.nt
    seq = dv[t].flatten(0, 1)
    for s, sb, db, k in windows:
        pool, tab = sources[s]
        s0 = tb // pool.nt * pool.nt
        sseq = pool.view()[torch.tensor(table_slice(tab, tb, te, pool.nt), device="cuda")].flatten(0, 1)
        seq[tb - d0:te - d0, :, :, db:db + k] = sseq[tb - s0:te - s0, :, :, sb:sb + k]
    dv[t] = seq.view(len(t), dst.nt, *seq.shape[1:])


def test_manager_long_sequences_grow_and_reuse_staging_slots():
    """Llama-3-8B's KV geometry on 4 layers: one-token pages -> 16-token pages over 32 768 tokens (32 768 + 2 048 ids, past a
    slot's 4 096), and TP8 one-token -> TP2 16-token (4 * 32 768 + 2 048 ids), then 72 short hand-offs issued back to back.
    Expected pools from torch indexing over the token view, cross-checked with the numpy oracles on sampled blocks."""
    mgr = TransferManager(device=0, worker_id=53)
    try:
        nl, no, hd, T = 4, 2, 128, 32768
        gen = torch.Generator(device="cuda").manual_seed(5)
        rng = np.random.default_rng(6)
        src = _DevPool(mgr, T + 1, nl, no, 1, 8, hd, KV.OperationalNHD, gen)
        dst = _DevPool(mgr, T // 16 + 1, nl, no, 16, 8, hd, KV.OperationalHND, gen)
        plan = tp_reshard_plan(8, 8, 2, 0)
        windows = _windows(plan)
        ranks = sorted({w.src_rank for w in plan})
        gsrc = [_DevPool(mgr, T + 1, nl, no, 1, 1, hd, KV.OperationalNHD, gen) for _ in ranks]
        gdst = _DevPool(mgr, T // 16 + 1, nl, no, 16, 4, hd, KV.UniversalTP, gen)
        stab = [int(x) for x in rng.permutation(T + 1)[:T]]
        gtab = [[int(x) for x in rng.permutation(T + 1)[:T]] for _ in ranks]
        dtab = [int(x) + 1 for x in rng.permutation(T // 16)]            # block 0 of either destination is the guard
        tb, te = 5, T

        def check_long(pool, sources, wins, handoff, oracle):
            exp = pool.mem.clone()
            sample = [0, len(dtab) // 2, len(dtab) - 1]
            old = {k: pool.block(dtab[k]) for k in sample}
            handoff().wait(60.0)
            torch.cuda.synchronize()
            _torch_expect(exp, pool, dtab, tb, te, sources, wins)
            for k in sample:                                               # the torch reference against the numpy oracle
                a, b = max(tb, k * 16), min(te, (k + 1) * 16)
                blocks = [[p.block(x) for x in table_slice(tab, a, b, 1)] for p, tab in sources]
                assert np.array_equal(oracle(blocks, old[k], a, b), pool.block(dtab[k], exp))
            assert torch.equal(pool.mem, exp)

        check_long(dst, [(src, stab)], [(0, 0, 0, 8)],
                   lambda: mgr.execute_repage(src.h, table_slice(stab, tb, te, 1), dst.h, table_slice(dtab, tb, te, 16), range(tb, te)),
                   lambda blocks, old, a, b: repage(blocks[0], [old], int(KV.OperationalNHD), int(KV.OperationalHND), nl, no, 8, 1, 16,
                                                    hd * 2, a, b)[0])
        gsources = [(p, tab) for p, tab in zip(gsrc, gtab)]
        check_long(gdst, gsources, windows,
                   lambda: mgr.execute_repage_gather({r: (gsrc[i].h, table_slice(gtab[i], tb, te, 1)) for i, r in enumerate(ranks)}, gdst.h,
                                                     table_slice(dtab, tb, te, 16), plan, range(tb, te)),
                   lambda blocks, old, a, b: repage_gather([(x, int(KV.OperationalNHD), 1) for x in blocks], windows, [old],
                                                           int(KV.UniversalTP), 4, nl, no, 1, 16, hd * 2, a, b)[0])

        # short hand-offs on disjoint destination blocks, back to back: the slots the long ones grew are reused
        dst.randomize()
        gdst.randomize()
        exp, gexp = dst.mem.clone(), gdst.mem.clone()
        notes, done = [], []
        for i in range(72):
            a = i * 448 + 7 + i % 5
            b = a + 40 + 37 * (i % 7)
            if i % 9 == 8:
                notes.append(mgr.execute_repage_gather({r: (gsrc[j].h, table_slice(gtab[j], a, b, 1)) for j, r in enumerate(ranks)}, gdst.h,
                                                       table_slice(dtab, a, b, 16), plan, range(a, b)))
                done.append((gexp, gdst, a, b, gsources, windows))
            else:
                notes.append(mgr.execute_repage(src.h, table_slice(stab, a, b, 1), dst.h, table_slice(dtab, a, b, 16), range(a, b)))
                done.append((exp, dst, a, b, [(src, stab)], [(0, 0, 0, 8)]))
        for note in notes:
            note.wait(60.0)
        torch.cuda.synchronize()
        for e, pool, a, b, sources, wins in done:
            _torch_expect(e, pool, dtab, a, b, sources, wins)
        assert torch.equal(dst.mem, exp)
        assert torch.equal(gdst.mem, gexp)
    finally:
        torch.cuda.synchronize()
        mgr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. one fully contiguous pool past 4 GiB: block offsets id * block_stride >= 2^32
# ---------------------------------------------------------------------------------------------------------------------
BNL, BNO, BNT, BNH, BHD = 4, 2, 16, 8, 128          # bf16: 32 KiB regions, 256 KiB blocks
BREGION = BNT * BNH * BHD * 2
BBLOCK = BNL * BNO * BREGION
BNB = (1 << 32) // BBLOCK + 64                      # 16 448 blocks (4.02 GiB): block 16 384 starts at byte 2^32
WRAP = (1 << 32) // BBLOCK                          # a block offset truncated to 32 bits lands WRAP blocks lower
BIG_IDS = [WRAP + 63, WRAP + 5, WRAP + 32, WRAP]    # the moved blocks, all past 2^32
CHUNK_WORDS = 1 << 24                               # 64 MiB per device-side comparison


def _fill_words(first, n):
    """The pool's fill: int32 word w holds a hash of w (every product below 2^63)."""
    x = torch.arange(first, first + n, dtype=torch.int64, device="cuda")
    x = (x * 0x2C1B3C6D + 0x3A8F05C5) & 0xFFFFFFFF
    x ^= x >> 15
    x = (x * 0x045D9F3B) & 0xFFFFFFFF
    x ^= x >> 13
    return (x - ((x >> 31) << 32)).to(torch.int32)


class _BigPool:
    """BNB blocks of BNL x BNO regions in one allocation, filled by _fill_words and never mirrored on the host."""

    def __init__(self):
        self.mem = torch.empty(BNB * BBLOCK, dtype=torch.uint8, device="cuda")
        self.words = self.mem.view(torch.int32)
        self.refill()
        base = self.mem.data_ptr()
        self.layer_base = torch.tensor([base + l * BNO * BREGION for l in range(BNL)], dtype=torch.int64, device="cuda")
        self.desc = K.PagedLayout(self.layer_base.data_ptr(), BBLOCK, BREGION, BREGION, BNL, BNO, BNB)

    def refill(self):
        for s in range(0, self.words.numel(), CHUNK_WORDS):
            n = min(CHUNK_WORDS, self.words.numel() - s)
            self.words[s:s + n] = _fill_words(s, n)

    def block(self, b):
        return self.mem[b * BBLOCK:(b + 1) * BBLOCK].cpu().numpy()

    def assert_filled(self, ids):
        w = BBLOCK // 4
        for b in ids:
            assert torch.equal(self.words[b * w:(b + 1) * w], _fill_words(b * w, w)), f"block {b} changed"

    def restore(self, ids):
        w = BBLOCK // 4
        for b in ids:
            self.words[b * w:(b + 1) * w] = _fill_words(b * w, w)

    def assert_all_filled(self):
        for s in range(0, self.words.numel(), CHUNK_WORDS):
            n = min(CHUNK_WORDS, self.words.numel() - s)
            if not torch.equal(self.words[s:s + n], _fill_words(s, n)):
                bad = int((self.words[s:s + n] != _fill_words(s, n)).nonzero()[0]) + s
                raise AssertionError(f"byte {4 * bad} (block {4 * bad // BBLOCK}) of the pool changed")


@pytest.fixture(scope="module")
def big_pool():
    free, _ = torch.cuda.mem_get_info()
    if free < 10 * 2**30:
        pytest.skip(f"a {BNB * BBLOCK / 2**30:.2f} GiB pool and its checks want about 10 GiB free; {free / 2**30:.1f} GiB are")
    pool = _BigPool()
    yield pool
    pool.mem = pool.words = pool.layer_base = None
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _into_big(big, launch, want):
    """launch() writes BIG_IDS of the big pool; want(old) maps their blocks before it to the blocks after it.  Checks the moved
    blocks, the blocks a 32-bit offset would hit (inside the same allocation), and after restoring the moved blocks every byte."""
    old = [big.block(b) for b in BIG_IDS]
    try:
        assert launch() == 0
        torch.cuda.synchronize()
        for b, w in zip(BIG_IDS, want(old)):
            assert np.array_equal(big.block(b), w), f"block {b}"
        big.assert_filled([b - WRAP for b in BIG_IDS])
        big.restore(BIG_IDS)
        big.assert_all_filled()
    except BaseException:
        big.refill()             # the next case starts from the fill, whatever this one wrote
        raise


def _src_twin(kind, nb, nh, elem, seed, nt=BNT):
    h = _host(kind, nb, BNL, BNO, nt, nh, BHD, elem)
    randomize(h, seed)
    return h


SIDS = [4, 1, 5, 0]


def _big_side(big, ids_t, kv):
    return K.PermuteSide(big.desc, ids_t.data_ptr(), int(kv))


@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16], ids=lambda c: c.name)
def test_big_pool_paged_copy(big_pool, cast):
    src = _src_twin("LWs", 6, BNH, ELEMS[cast][0], 31)
    S, si, di = DevicePool(src), ids_dev(SIDS), ids_dev(BIG_IDS)
    dsts = [K.PagedDst(big_pool.desc, si.data_ptr(), di.data_ptr(), 0, 0)]
    _into_big(big_pool, lambda: K.paged_copy(S.desc, dsts, len(SIDS), 0, BNL, int(cast), None, stream_ptr()),
              lambda old: [cast_bytes(O.read_logical_block(src, s), int(cast)) for s in SIDS])


def test_big_pool_permute(big_pool):
    src = _src_twin("LWs", 6, BNH, 2, 32)
    S, si, di = DevicePool(src), ids_dev(SIDS), ids_dev(BIG_IDS)
    _into_big(big_pool, lambda: K.paged_permute(K.PermuteSide(S.desc, si.data_ptr(), int(KV.OperationalNHD)), _big_side(big_pool, di, KV.UniversalTP),
                                                len(SIDS), 0, BNL, BNH, BNT, BHD * 2, stream=stream_ptr()),
              lambda old: [O.kv_layout_permute(O.read_logical_block(src, s), int(KV.OperationalNHD), int(KV.UniversalTP), BNL, BNO, BNT, BNH,
                                               BHD * 2) for s in SIDS])


def test_big_pool_gather(big_pool):
    """TP4 -> TP1: four 2-head sources into the big pool's 8 heads."""
    windows = _windows(tp_reshard_plan(BNH, 4, 1, 0))
    srcs = [_src_twin("LWf", 6, 2, 2, 40 + i) for i in range(4)]
    S, si, di = [DevicePool(s) for s in srcs], ids_dev(SIDS), ids_dev(BIG_IDS)
    ps = [K.PermuteSource(K.PermuteSide(S[s].desc, si.data_ptr(), int(KV.OperationalNHD)), 2, sb, db, k) for s, sb, db, k in windows]

    def want(old):
        out = []
        for i, s in enumerate(SIDS):
            blk = old[i]
            for j, sb, db, k in windows:
                blk = reshard_block(O.read_logical_block(srcs[j], s), blk, int(KV.OperationalNHD), int(KV.UniversalPP), BNL, BNO, BNT, 2, BNH,
                                    BHD * 2, 0, sb, db, k)
            out.append(blk)
        return out
    _into_big(big_pool, lambda: K.paged_permute_gather(ps, _big_side(big_pool, di, KV.UniversalPP), BNH, len(SIDS), 0, BNL, BNT, BHD * 2,
                                                       stream=stream_ptr()), want)


def test_big_pool_repage(big_pool):
    """Page 4 -> the big pool's page 16 (the big pool is the larger page's side), tokens 5 .. 61 of the sequence whose
    destination table is BIG_IDS."""
    tb, te, ps = 5, 61, 4
    ns = -(-te // ps) - tb // ps
    src = _src_twin("LWs", ns + 1, BNH, 2, 50, nt=ps)
    sids = list(range(ns, 0, -1))
    S, si, di = DevicePool(src), ids_dev(sids), ids_dev(BIG_IDS)
    _into_big(big_pool, lambda: K.paged_repage(K.PermuteSide(S.desc, si.data_ptr(), int(KV.OperationalNHD)), ps,
                                               _big_side(big_pool, di, KV.OperationalHND), BNT, tb, te, 0, BNL, BNH, BHD * 2, stream=stream_ptr()),
              lambda old: repage([O.read_logical_block(src, b) for b in sids], old, int(KV.OperationalNHD), int(KV.OperationalHND), BNL, BNO,
                                 BNH, ps, BNT, BHD * 2, tb, te))


def test_big_pool_repage_gather(big_pool):
    """TP4 one-token pages -> the big pool's 16-token pages, tokens 5 .. 61."""
    tb, te = 5, 61
    windows = _windows(tp_reshard_plan(BNH, 4, 1, 0))
    srcs = [_src_twin("LWs", te - tb + 1, 2, 2, 60 + i, nt=1) for i in range(4)]
    sids = [[(7 * k + i) % (te - tb + 1) for k in range(te - tb)] for i in range(4)]
    S, si, di = [DevicePool(s) for s in srcs], [ids_dev(x) for x in sids], ids_dev(BIG_IDS)
    ps = [K.PermuteSource(K.PermuteSide(S[s].desc, si[s].data_ptr(), int(KV.OperationalNHD)), 2, sb, db, k) for s, sb, db, k in windows]
    _into_big(big_pool, lambda: K.paged_repage_gather(ps, 1, _big_side(big_pool, di, KV.UniversalTP), BNH, BNT, tb, te, 0, BNL, BHD * 2,
                                                      stream=stream_ptr()),
              lambda old: repage_gather([([O.read_logical_block(srcs[i], b) for b in sids[i]], int(KV.OperationalNHD), 2) for i in range(4)],
                                        windows, old, int(KV.UniversalTP), BNH, BNL, BNO, 1, BNT, BHD * 2, tb, te))


@pytest.mark.parametrize("kernel", ["permute", "repage"])
def test_big_pool_as_source(big_pool, kernel):
    """Blocks past 2^32 of the big pool are read: by the permute, and by re-paging into 32-token pages (the big pool is the
    smaller page's side).  The pool keeps every byte."""
    olds = [big_pool.block(b) for b in BIG_IDS]
    nt = BNT if kernel == "permute" else 32
    tb, te = (0, len(BIG_IDS) * BNT) if kernel == "permute" else (5, 61)
    nd = -(-te // nt) - tb // nt
    dst, ref = _host("LWf", nd + 2, BNL, BNO, nt, BNH, BHD, 2), _host("LWf", nd + 2, BNL, BNO, nt, BNH, BHD, 2)
    randomize(dst, 70)
    for a, b in zip(ref.buffers, dst.buffers):
        a[:] = b
    dids = list(range(nd + 1, 1, -1))                          # blocks 0 and 1 are guards
    D, si, di = DevicePool(dst), ids_dev(BIG_IDS), ids_dev(dids)
    dside = K.PermuteSide(D.desc, di.data_ptr(), int(KV.OperationalNHD))
    if kernel == "permute":
        rc = K.paged_permute(_big_side(big_pool, si, KV.UniversalTP), dside, len(BIG_IDS), 0, BNL, BNH, BNT, BHD * 2, stream=stream_ptr())
        new = [O.kv_layout_permute(o, int(KV.UniversalTP), int(KV.OperationalNHD), BNL, BNO, BNT, BNH, BHD * 2) for o in olds]
    else:
        rc = K.paged_repage(_big_side(big_pool, si, KV.UniversalTP), BNT, dside, nt, tb, te, 0, BNL, BNH, BHD * 2, stream=stream_ptr())
        new = repage(olds, [O.read_logical_block(ref, b) for b in dids], int(KV.UniversalTP), int(KV.OperationalNHD), BNL, BNO, BNH, BNT, nt,
                     BHD * 2, tb, te)
    assert rc == 0
    torch.cuda.synchronize()
    D.download()
    for b, blk in zip(dids, new):
        O.write_logical_block(ref, b, blk)
    for got, want in zip(dst.buffers, ref.buffers):
        assert np.array_equal(got, want)
    try:
        big_pool.assert_all_filled()
    except BaseException:
        big_pool.refill()
        raise


def test_big_pool_through_the_manager(big_pool):
    """The big pool registered with register_fully_contiguous as UniversalTP; an OperationalNHD pool's blocks land past 2^32."""
    mgr = TransferManager(device=0, worker_id=54)
    try:
        cfg = LayoutConfig(BNB, BNL, BNO, BNT, BNH * BHD, dtype_width_bytes=2, num_heads=BNH)
        h = mgr.register_fully_contiguous(cfg, big_pool.mem.data_ptr(), big_pool.mem.numel(), StorageKind.Device, 0)
        mgr.set_kv_block_layout(h, KV.UniversalTP)
        src = _Pool(mgr, "LWs", 6, BNL, BNO, BNT, BNH, BHD, 2, kv=KV.OperationalNHD)
        randomize(src.twin, 80)
        src.upload()
        _into_big(big_pool, lambda: mgr.execute_transfer(src.h, SIDS, h, BIG_IDS).wait(30.0) or 0,
                  lambda old: [O.kv_layout_permute(O.read_logical_block(src.twin, s), int(KV.OperationalNHD), int(KV.UniversalTP), BNL, BNO, BNT,
                                                   BNH, BHD * 2) for s in SIDS])
    finally:
        torch.cuda.synchronize()
        mgr.close()

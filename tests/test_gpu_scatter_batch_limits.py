"""The re-paging scatter (kvbm_kernels_paged_repage_scatter, TransferManager.execute_repage_scatter) and the batch re-paging gather
(kvbm_kernels_paged_stage_repage_gather_batch, TransferManager.execute_repage_batch) at the limits their launchers accept, each
paired with its first rejected neighbour, and past 4 GiB, against the oracles:

- the scatter's entry, pair and stage tables at their maxima: warps that loop past 8 entries with uneven pair counts, 256 pairs
  over 4 stages, 16 stages, one pool behind two stages of one table with layer shifts of both signs;
- every (source, destination) format pair under a PP layer shift, so universal targets stride over their own layer count;
- the walk's smallest and largest rows, the multiply-high row split and the small page's split at their bounds;
- token positions at the 32-bit bound (kernels) and at 2^31 (manager), a batch's wrapped small_k among them;
- block offsets past 2^32 in the > 4 GiB pool of tests/test_gpu_transform_limits.py, on every address path of both kernels;
- manager id lists past a staging slot's arena share, then many short scatters reusing the slots.

Pools start from random bytes, every destination keeps blocks no table names, and whole destination pools are compared with
tests/scatter_oracle.py or tests/repage_batch_oracle.py; every scatter is also compared with one
kvbm_kernels_paged_stage_repage_gather launch per target.  A rejected neighbour returns cudaErrorInvalidValue (the manager: its
error code) before any launch, so K.launch_count() stays put."""
import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import (ErrorCode, KvbmError, LayoutConfig, ScatterWindow, StorageKind, TransferManager, tp_pp_reshard_plan,
                                  tp_pp_scatter_plan)
from tests.gpu_util import ids_dev, stream_ptr
from tests.repage_batch_oracle import repage_batch
from tests.repage_oracle import table_slice
from tests.scatter_oracle import repage_scatter
from tests.test_gpu_repage_batch import BatchRig, _requests, plan_rig
from tests.test_gpu_repage_scatter import ALL, ScatterRig, _plan_rig
from tests.test_gpu_stage_gather import ELEMS, _register
from tests.test_gpu_transform_limits import (BHD, BIG_IDS, BIG_PAGE, BNB, BNH, BNL, BNO, BNT, ROWS, SMALL_PAGE, V_BOUND, _DevPool,
                                             _into_big, _rejected, _torch_expect, big_pool)  # noqa: F401  (big_pool: the fixture)
from tests.test_gpu_transform_stream import Pool

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
NHD, HND, UTP, UPP = KV.OperationalNHD, KV.OperationalHND, KV.UniversalTP, KV.UniversalPP
PAGE_PAIRS = [(16, 64), (64, 16), (48, 16), (16, 48), (1, 16), (16, 1)]


class SpanRig(ScatterRig):
    """ScatterRig over a range anywhere below 2^32: its pools and tables hold only the blocks the range touches (and two no table
    names).  They are built for the same range moved down by whole blocks of the larger page, which keeps every slot, block
    count and unit of the range."""

    def __init__(self, src, dsts, targets, ps, pd, tokens, **kw):
        shift = tokens.start // max(ps, pd) * max(ps, pd)
        super().__init__(src, dsts, targets, ps=ps, pd=pd, tokens=range(tokens.start - shift, tokens.stop - shift), **kw)
        self.tb, self.te = tokens.start, tokens.stop


def _replicated(nl, hd, cast, ps, pd, tokens, seed, no=1):
    """A one-head source into two targets on one pool of two heads, through one table: the head replicated."""
    return ScatterRig((nl, 1, HND), [(nl, 2, NHD)], [(0, 0, 0, nl, 0, 0, 1), (0, 0, 0, nl, 0, 1, 1)], ps=ps, pd=pd, tokens=tokens, no=no,
                      hd=hd, cast=cast, seed=seed)


def _batch3(nl, hd, cast, ps, pd, seqs, seed, no=1):
    """A one-head source read by two windows into the two heads of the destination (the head replicated), over 3 sequences."""
    return BatchRig([(nl, 1, HND)], [(0, 0, 0, nl, 0, 0, 1), (0, 0, 0, nl, 0, 1, 1)], nl, 2, NHD, seqs, ps=ps, pd=pd, no=no, hd=hd, cast=cast,
                    seed=seed)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the scatter's entry, pair and stage tables at their maxima
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ps,pd,cast,scaled", [(16, 64, CM.NONE, False), (64, 16, CM.NONE, False), (16, 64, CM.FP8E4M3_TO_BF16, True)],
                         ids=["16_64", "64_16", "16_64_fp8_to_bf16_scaled"])
def test_scatter_warps_loop_past_eight_entries_with_uneven_pairs(ps, pd, cast, scaled):
    """40 source heads in one stage: all to one pool, heads 0-9 and 30-39 also to a second pool (one table), so entries 0-9 and
    30-39 have two pairs and 10-29 one; a warp takes entries w, w + 8, .. w + 32."""
    r = ScatterRig((2, 40, NHD), [(2, 40, HND), (2, 20, UTP)], [(0, 0, 0, 2, 0, 0, 40), (1, 0, 0, 2, 0, 0, 10), (1, 0, 0, 2, 30, 10, 10)],
                   ps=ps, pd=pd, hd=32, cast=cast, scaled=scaled, seed=40 + ps)
    r.run_and_check()


# (source layer, [(src_head_begin, head_count) per target]): 112 + 64 + 48 + 32 = 256 pairs over 64, 16, 8 and 26 entries
PAIR_STAGES = [(0, [(0, 64), (8, 48)]), (1, [(16, 16)] * 4), (2, [(56, 8)] * 6), (3, [(0, 8), (2, 8), (40, 8), (50, 8)])]


def _pairs_rig(last_count, ps, pd):
    wins = [(sl, sb, k) for sl, ws in PAIR_STAGES for sb, k in ws]
    wins[-1] = wins[-1][:2] + (last_count,)
    dsts = [(2, k + 3, ALL[t % 4]) for t, (_sl, _sb, k) in enumerate(wins)]
    targets = [(t, sl, t % 2, 1, sb, t % 3, k) for t, (sl, sb, k) in enumerate(wins)]
    return ScatterRig((4, 64, HND), dsts, targets, ps=ps, pd=pd, hd=8, no=1, seed=last_count)


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16)], ids=str)
def test_scatter_takes_256_pairs_over_four_stages(ps, pd):
    """16 targets, 256 (target, head) pairs over 4 one-layer stages of 64, 16, 8 and 26 entries; one pair more is rejected."""
    r = _pairs_rig(8, ps, pd)
    assert len(r.targets) == K.GATHER_MAX_SOURCES and sum(t[6] for t in r.targets) == K.GATHER_MAX_HEADS
    r.run_and_check()
    n = _pairs_rig(9, ps, pd)
    _rejected(lambda: n.launch())


@pytest.mark.parametrize("layers,ps,pd", [(None, 16, 64), (range(3, 13), 64, 16)], ids=["all_layers", "layers_3_13"])
def test_scatter_takes_sixteen_stages(layers, ps, pd):
    """A PP1 -> PP16-like push: target t takes source layer t into its own one-layer pool, one stage each; 17 targets are
    rejected."""
    dsts = [(1, 4, ALL[t % 4]) for t in range(17)]
    targets = [(t, t, 0, 1, 0, 0, 4) for t in range(16)]
    r = ScatterRig((16, 4, NHD), dsts[:16], targets, ps=ps, pd=pd, hd=32, no=1, layers=layers, seed=16)
    r.run_and_check()
    n = ScatterRig((16, 4, NHD), dsts, targets + [(16, 15, 0, 1, 0, 0, 4)], ps=ps, pd=pd, hd=32, no=1, layers=layers, seed=17)
    _rejected(lambda: n.launch())


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16)], ids=str)
def test_one_pool_behind_two_stages_with_layer_shifts_of_both_signs(ps, pd):
    """Source layers 0-1 -> layers 2-3 and 2-3 -> 0-1 of one pool, through its one table, in both formats' strides."""
    for kv in (UTP, NHD):
        r = ScatterRig((4, 4, HND), [(4, 4, kv)], [(0, 0, 2, 2, 0, 0, 4), (0, 2, 0, 2, 0, 0, 4)], ps=ps, pd=pd, hd=32, seed=int(kv) + ps)
        r.run_and_check()


# ---------------------------------------------------------------------------------------------------------------------
# 2. every format pair under a PP layer shift
# ---------------------------------------------------------------------------------------------------------------------
SHIFT_PLANS = {"pp2tp2_rank3_to_pp3tp2": (4, 12, 2, 2, 2, 3, 3),     # a 6-layer source into 4-layer targets
               "pp3tp2_rank2_to_pp2tp2": (4, 12, 2, 3, 2, 2, 2)}     # a 4-layer source into 6-layer targets


def test_the_shift_plans_shapes():
    for name, want in (("pp2tp2_rank3_to_pp3tp2", [(0, 2, 2), (2, 0, 4)]), ("pp3tp2_rank2_to_pp2tp2", [(0, 4, 2), (2, 0, 2)])):
        assert [(w.src_layer_begin, w.dst_layer_begin, w.layer_count) for w in tp_pp_scatter_plan(*SHIFT_PLANS[name])] == want


@pytest.mark.parametrize("dst_kv", ALL, ids=lambda k: k.name)
@pytest.mark.parametrize("src_kv", ALL, ids=lambda k: k.name)
@pytest.mark.parametrize("plan", list(SHIFT_PLANS))
def test_every_format_pair_under_a_layer_shift(plan, src_kv, dst_kv):
    ps, pd = (16, 64) if (int(src_kv) + int(dst_kv)) % 2 else (64, 16)
    r = _plan_rig(*SHIFT_PLANS[plan], src_kv=src_kv, dst_kvs=(dst_kv,), ps=ps, pd=pd, hd=32, seed=4 * int(src_kv) + int(dst_kv))
    r.run_and_check()


# ---------------------------------------------------------------------------------------------------------------------
# 3. row and page extremes
# ---------------------------------------------------------------------------------------------------------------------
def _row_geometry(hd):
    return (1, 1, 2) if hd > 1024 else (2, 2, 16)     # nl, no, nt


@pytest.mark.parametrize("row", list(ROWS))
def test_scatter_smallest_and_largest_rows(row):
    cast, hd, bad = ROWS[row]
    nl, no, nt = _row_geometry(hd)
    r = _replicated(nl, hd, cast, nt // 2, nt, range(1, 2 * nt - 1), 7, no=no)
    r.run_and_check()
    nl, no, nt = _row_geometry(bad)
    n = _replicated(nl, bad, cast, nt // 2, nt, range(1, 2 * nt - 1), 8, no=no)
    _rejected(lambda: n.launch())


@pytest.mark.parametrize("row", list(ROWS))
def test_batch_smallest_and_largest_rows(row):
    cast, hd, bad = ROWS[row]
    for h, seed in ((hd, 7), (bad, 8)):
        nl, no, nt = _row_geometry(h)
        r = _batch3(nl, h, cast, nt, nt // 2, [(1, 2 * nt - 1), (2 * nt + 1, 2 * nt + 2), (3 * nt, 5 * nt)], seed, no=no)
        if h == hd:
            assert r.run() == 0
            r.check()
        else:
            _rejected(r.run)


@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16], ids=lambda c: c.name)
def test_multiply_high_row_split_at_its_bound(cast):
    """V = 4095 vectors per walk row at page 256, the largest page the launchers take for it; page 257 is rejected."""
    hd = V_BOUND * 16 // ELEMS[cast][0]
    r = _replicated(1, hd, cast, 256, 16, range(5, 2 * 256 - 3), 11)
    r.run_and_check()
    _rejected(lambda: _replicated(1, hd, cast, 257, 1, range(0, 3), 12).launch())
    b = _batch3(1, hd, cast, 256, 16, [(5, 300), (767, 769), (1027, 1224)], 13)
    assert b.run() == 0
    b.check()
    _rejected(_batch3(1, hd, cast, 257, 1, [(0, 3), (300, 301), (600, 700)], 14).run)


@pytest.mark.parametrize("ps,pd", [(SMALL_PAGE, BIG_PAGE), (BIG_PAGE, SMALL_PAGE)], ids=["small_to_big", "big_to_small"])
def test_small_page_split_at_its_bound(ps, pd):
    """A 3072-token small page under a 455x larger one, the source on either side; the next multiple (ratio 456) is rejected."""
    r = _replicated(1, 8, CM.NONE, ps, pd, range(1000, BIG_PAGE + 5000), 21)
    r.run_and_check()
    nb = BIG_PAGE + SMALL_PAGE
    nps, npd = (SMALL_PAGE, nb) if ps < pd else (nb, SMALL_PAGE)
    _rejected(lambda: _replicated(1, 8, CM.NONE, nps, npd, range(0, 1), 22).launch())
    b = _batch3(1, 8, CM.NONE, ps, pd, [(1000, BIG_PAGE + 5000), (2 * BIG_PAGE + 1, 2 * BIG_PAGE + 2), (3 * BIG_PAGE + 10, 3 * BIG_PAGE + 3100)], 23)
    assert b.run() == 0
    b.check()
    assert K.repage_batch_units(b.seqs, nps, npd) is None
    args = list(b.args())
    args[1], args[4] = nps, npd
    _rejected(lambda: K.paged_stage_repage_gather_batch(*args, stream=stream_ptr()))


# ---------------------------------------------------------------------------------------------------------------------
# 4. token positions at the 32-bit bound (kernels) and at 2^31 (manager)
# ---------------------------------------------------------------------------------------------------------------------
def _te_max(ps, pd):
    """The largest token_end the kernels take for the page pair: the last block of the larger page ends below 2^32."""
    big = max(ps, pd)
    return (2**32 - 1) // big * big


@pytest.mark.parametrize("ps,pd", PAGE_PAIRS, ids=str)
def test_scatter_token_positions_at_the_32_bit_bound(ps, pd):
    big, te = max(ps, pd), _te_max(ps, pd)
    tb = te - 2 * big - 3
    r = SpanRig((2, 4, NHD), [(2, 4, HND), (2, 2, UTP)], [(0, 0, 0, 2, 0, 0, 4), (1, 0, 0, 2, 2, 0, 2)], ps, pd, range(tb, te), hd=32,
                seed=ps + pd)
    r.run_and_check()
    _rejected(lambda: r.launch(tokens=range(tb, te + 1)))


@pytest.mark.parametrize("ps,pd", PAGE_PAIRS, ids=str)
def test_batch_token_positions_at_the_32_bit_bound(ps, pd):
    """The first sequence ends at te_max and starts mid-block, so its first unit's small_k wraps below 0 (also when the small
    table is the source's); then a sequence from 0, and one across 2^31.  A sequence ending at te_max + 1 is rejected by the
    unit table and by the launch."""
    big, te = max(ps, pd), _te_max(ps, pd)
    mid = 2**31 // big * big - big // 2 - 1
    seqs = [(te - 2 * big - 3, te), (0, 2 * big + 3), (mid, mid + 2 * big + 5)]
    r = BatchRig([(2, 2, HND), (2, 2, NHD)], [(0, 0, 0, 2, 0, 0, 2), (1, 0, 0, 2, 0, 2, 2)], 2, 4, UTP, seqs, ps=ps, pd=pd, hd=32, seed=ps + pd)
    assert (r.units_np[:, 2] >= 2**31).any()                      # a wrapped small_k
    assert r.run() == 0
    r.check()
    bad = seqs + [(te - 5, te + 1)]
    assert K.repage_batch_units(bad, ps, pd) is None
    args = list(r.args())
    args[5] = bad
    _rejected(lambda: K.paged_stage_repage_gather_batch(*args, stream=stream_ptr()))


@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=61)
    yield m
    torch.cuda.synchronize()
    m.close()


def _plan_of(r):
    return [ScatterWindow(p, sl, dl, c, sb, db, k) for p, sl, dl, c, sb, db, k in r.targets]


def _ids(a):
    return [int(x) for x in a]


def test_manager_scatter_range_ends_at_2_pow_31(mgr):
    """execute_repage_scatter takes tokens ending at 2^31; one token more is a RANGE error and launches nothing."""
    tb, te = 2**31 - 77, 2**31
    r = SpanRig((2, 4, NHD), [(2, 4, HND), (2, 2, UPP)], [(0, 0, 0, 2, 0, 0, 4), (1, 0, 0, 2, 2, 0, 2)], 16, 64, range(tb, te), hd=32, seed=31)
    sh = _register(mgr, r.src, r.src.kv)
    dhs = [_register(mgr, p, p.kv) for p in r.dsts]
    call = lambda tokens: mgr.execute_repage_scatter(sh, _ids(r.sids), dhs, [_ids(d) for d in r.dids], _plan_of(r), tokens)  # noqa: E731
    call(range(tb, te)).wait(20.0)
    torch.cuda.synchronize()
    for p, want in zip(r.dsts, r.expected()):
        assert np.array_equal(p.buf.cpu().numpy(), want)
    before = K.launch_count()
    with pytest.raises(KvbmError) as e:
        call(range(tb, te + 1))
    assert e.value.code == ErrorCode.RANGE and K.launch_count() == before


def test_manager_batch_range_ends_at_2_pow_31(mgr):
    """execute_repage_batch takes a sequence ending at 2^31 beside others; one token more is a RANGE error, nothing launched."""
    plan = tp_pp_reshard_plan(8, 4, 2, 2, 1, 1, 0)
    seqs = [(2**31 - 77, 2**31), (5, 130), (2**31 - 300, 2**31 - 200)]
    r = plan_rig(8, 4, 2, 2, 1, 1, 0, seqs, src_kv=UTP, dst_kv=NHD, seed=32)
    ranks = sorted({w.src_rank for w in plan})
    hs = {rk: _register(mgr, r.srcs[i], r.srcs[i].kv) for i, rk in enumerate(ranks)}
    dh = _register(mgr, r.dst, r.dst.kv)
    reqs = _requests(r, ranks)
    mgr.execute_repage_batch(hs, dh, reqs, plan).wait(20.0)
    torch.cuda.synchronize()
    r.check()
    before = K.launch_count()
    with pytest.raises(KvbmError) as e:
        mgr.execute_repage_batch(hs, dh, [(range(2**31 - 77, 2**31 + 1),) + reqs[0][1:]] + reqs[1:], plan)
    assert e.value.code == ErrorCode.RANGE and K.launch_count() == before


# ---------------------------------------------------------------------------------------------------------------------
# 5. block offsets past 2^32: the big pool of tests/test_gpu_transform_limits.py
# ---------------------------------------------------------------------------------------------------------------------
TOKENS = range(5, 61)            # big-pool page 16: blocks 0 .. 3 of the sequence, whose table is BIG_IDS


def _big_side(big, ids_t, kv):
    return K.PermuteSide(big.desc, ids_t.data_ptr(), int(kv))


def _src_pool(nh, page, kv, seed, nl=BNL):
    n = -(-TOKENS.stop // page) - TOKENS.start // page
    p = Pool(n + 2, nl, BNO, page, nh, BHD * 2, kv, seed)
    ids = np.random.default_rng(seed).permutation(n + 2)[:n].astype(np.int32)
    return p, ids, torch.from_numpy(ids).cuda()


def _gathers(src_side, src_nh, ps, targets, pd):
    """One kvbm_kernels_paged_stage_repage_gather launch per target (side, num_heads, sl, dl, c, sb, db, k); the first error."""
    for side, nh, sl, dl, c, sb, db, k in targets:
        rc = K.paged_stage_repage_gather([K.StageSource(K.PermuteSource(src_side, src_nh, sb, db, k), sl, dl, c)], ps, side, nh, pd, TOKENS.start,
                                         TOKENS.stop, dl, dl + c, BHD * 2, stream=stream_ptr())
        if rc:
            return rc
    return 0


def _scatter(src_side, src_nh, ps, targets, pd):
    kt = [K.ScatterTarget(side, nh, sb, db, k, sl, dl, c, 0) for side, nh, sl, dl, c, sb, db, k in targets]
    return K.paged_repage_scatter(src_side, src_nh, ps, kt, pd, TOKENS.start, TOKENS.stop, 0, BNL, BHD * 2, stream=stream_ptr())


@pytest.mark.parametrize("ps,big_kv", [(4, UTP), (64, HND)], ids=["source_page_4", "source_page_64"])
def test_big_pool_as_scatter_destination(big_pool, ps, big_kv):
    """The big pool is two targets (heads 0-3 and 4-7 of it from the same 4 source heads, so replicated heads land past 2^32) next
    to a small pool.  Source page 4: the big pool is the larger page's side, its block from the target's table (side_block);
    source page 64: it is the small side, its block per vector (repage_small)."""
    src, sids, sids_t = _src_pool(4, ps, NHD, 90 + ps)
    small = Pool(6, BNL, BNO, BNT, 4, BHD * 2, UPP, 91)
    small0 = small.buf.clone()
    dids = np.array([4, 1, 5, 2], dtype=np.int32)                  # blocks 0 and 3 are guards
    bi, di = ids_dev(BIG_IDS), torch.from_numpy(dids).cuda()
    bside, sside = _big_side(big_pool, bi, big_kv), small.side(di)
    targets = [(bside, BNH, 0, 0, BNL, 0, 0, 4), (bside, BNH, 0, 0, BNL, 0, 4, 4), (sside, 4, 0, 0, BNL, 0, 0, 4)]
    want_small = {}

    def want(old):
        pools = [np.stack(old), small0.cpu().numpy()]
        ts = [(0, list(range(4)), int(big_kv), BNH, BNL, (0, 0, BNL, 0, 0, 4)), (0, list(range(4)), int(big_kv), BNH, BNL, (0, 0, BNL, 0, 4, 4)),
              (1, dids, int(UPP), 4, BNL, (0, 0, BNL, 0, 0, 4))]
        repage_scatter(([src.final_np[b] for b in sids], src.kv, 4, BNL), ts, pools, BNO, ps, BNT, BHD * 2, TOKENS.start, TOKENS.stop)
        want_small["pool"] = pools[1]
        return list(pools[0])

    for launch in (lambda: _scatter(src.side(sids_t), 4, ps, targets, BNT), lambda: _gathers(src.side(sids_t), 4, ps, targets, BNT)):
        small.buf.copy_(small0)
        _into_big(big_pool, launch, want)
        assert np.array_equal(small.buf.cpu().numpy(), want_small["pool"])


@pytest.mark.parametrize("pd", [4, 32])
def test_big_pool_as_scatter_source(big_pool, pd):
    """Blocks past 2^32 read once and stored to two small pools: page 4 reads them as the larger page's side, page 32 as the
    small side.  The big pool keeps every byte."""
    olds = [big_pool.block(b) for b in BIG_IDS]
    nd = -(-TOKENS.stop // pd) - TOKENS.start // pd
    dsts = [Pool(nd + 2, BNL, BNO, pd, BNH, BHD * 2, NHD, 93), Pool(nd + 2, BNL, BNO, pd, 4, BHD * 2, UTP, 94)]
    init = [p.buf.clone() for p in dsts]
    dids = [np.random.default_rng(95 + i).permutation(nd + 2)[:nd].astype(np.int32) for i in range(2)]
    dids_t = [torch.from_numpy(x).cuda() for x in dids]
    bi = ids_dev(BIG_IDS)
    sside = _big_side(big_pool, bi, UPP)
    targets = [(dsts[0].side(dids_t[0]), BNH, 0, 0, BNL, 0, 0, BNH), (dsts[1].side(dids_t[1]), 4, 0, 0, BNL, 4, 0, 4)]
    pools = [x.cpu().numpy() for x in init]
    repage_scatter((olds, int(UPP), BNH, BNL), [(0, dids[0], int(NHD), BNH, BNL, (0, 0, BNL, 0, 0, BNH)), (1, dids[1], int(UTP), 4, BNL, (0, 0, BNL, 4, 0, 4))],
                   pools, BNO, BNT, pd, BHD * 2, TOKENS.start, TOKENS.stop)
    try:
        for launch in (_scatter, _gathers):
            for p, x in zip(dsts, init):
                p.buf.copy_(x)
            assert launch(sside, BNH, BNT, targets, pd) == 0
            torch.cuda.synchronize()
            for p, want in zip(dsts, pools):
                assert np.array_equal(p.buf.cpu().numpy(), want)
        big_pool.assert_all_filled()
    except BaseException:
        big_pool.refill()
        raise


BATCH_SEQS = [(5, 29), (115, 141)]     # two big-pool blocks each, at page 16: the concatenated table is BIG_IDS


def test_big_pool_as_batch_destination(big_pool):
    """TP2 at page 4 -> the big pool's 8 heads at page 16 (the larger page's side), two sequences splitting BIG_IDS."""
    units, ns, nd = K.repage_batch_units(BATCH_SEQS, 4, BNT)
    assert nd == len(BIG_IDS)
    srcs = [Pool(ns + 2, BNL, BNO, 4, 4, BHD * 2, HND, 96 + s) for s in range(2)]
    sids = [np.random.default_rng(98 + s).permutation(ns + 2)[:ns].astype(np.int32) for s in range(2)]
    sids_t = [torch.from_numpy(x).cuda() for x in sids]
    units_t = torch.from_numpy(units.view(np.int32)).cuda()
    windows = [(0, 0, 0, BNL, 0, 0, 4), (1, 0, 0, BNL, 0, 4, 4)]
    bi = ids_dev(BIG_IDS)
    sources = [K.StageSource(K.PermuteSource(srcs[s].side(sids_t[s]), 4, sb, db, k), sl, dl, c) for s, sl, dl, c, sb, db, k in windows]
    counts = [-(-te // 4) - tb // 4 for tb, te in BATCH_SEQS]
    per_seq = lambda ids: np.split(ids, np.cumsum(counts)[:-1])  # noqa: E731

    def want(old):
        seqs = [(tb, te, [per_seq(sids[0])[i], per_seq(sids[1])[i]], [2 * i, 2 * i + 1]) for i, (tb, te) in enumerate(BATCH_SEQS)]
        return list(repage_batch([(p.final_np, p.kv, 4, BNL) for p in srcs], windows, np.stack(old), int(UTP), BNH, BNL, BNO, 4, BNT, BHD * 2,
                                 seqs))
    _into_big(big_pool, lambda: K.paged_stage_repage_gather_batch(sources, 4, _big_side(big_pool, bi, UTP), BNH, BNT, BATCH_SEQS,
                                                                  units_t.data_ptr(), len(units), 0, BNL, BHD * 2, stream=stream_ptr()), want)


def test_big_pool_as_batch_source(big_pool):
    """The big pool's blocks past 2^32 as the small side (page 16 -> 32) of two sequences; it keeps every byte."""
    olds = [big_pool.block(b) for b in BIG_IDS]
    units, ns, nd = K.repage_batch_units(BATCH_SEQS, BNT, 32)
    assert ns == len(BIG_IDS)
    dst = Pool(nd + 2, BNL, BNO, 32, BNH, BHD * 2, NHD, 99)
    init = dst.buf.cpu().numpy()
    dids = np.random.default_rng(100).permutation(nd + 2)[:nd].astype(np.int32)
    units_t, dids_t, bi = torch.from_numpy(units.view(np.int32)).cuda(), torch.from_numpy(dids).cuda(), ids_dev(BIG_IDS)
    src = K.StageSource(K.PermuteSource(_big_side(big_pool, bi, UTP), BNH, 0, 0, BNH), 0, 0, BNL)
    rc = K.paged_stage_repage_gather_batch([src], BNT, dst.side(dids_t), BNH, 32, BATCH_SEQS, units_t.data_ptr(), len(units), 0, BNL, BHD * 2,
                                           stream=stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    n0 = -(-BATCH_SEQS[0][1] // 32) - BATCH_SEQS[0][0] // 32
    want = repage_batch([(np.stack(olds), int(UTP), BNH, BNL)], [(0, 0, 0, BNL, 0, 0, BNH)], init, int(NHD), BNH, BNL, BNO, BNT, 32, BHD * 2,
                        [(tb, te, [[2 * i, 2 * i + 1]], d) for i, ((tb, te), d) in enumerate(zip(BATCH_SEQS, (dids[:n0], dids[n0:])))])
    assert np.array_equal(dst.buf.cpu().numpy(), want)
    try:
        big_pool.assert_all_filled()
    except BaseException:
        big_pool.refill()
        raise


def test_big_pool_as_manager_scatter_destination(big_pool):
    """The big pool registered as one destination of execute_repage_scatter, taking the source's 4 heads twice, next to a small
    pool: page 4 -> 16."""
    m = TransferManager(device=0, worker_id=62)
    try:
        cfg = LayoutConfig(BNB, BNL, BNO, BNT, BNH * BHD, dtype_width_bytes=2, num_heads=BNH)
        bh = m.register_fully_contiguous(cfg, big_pool.mem.data_ptr(), big_pool.mem.numel(), StorageKind.Device, 0)
        m.set_kv_block_layout(bh, UTP)
        src, sids, _ = _src_pool(4, 4, NHD, 101)
        small = Pool(6, BNL, BNO, BNT, 4, BHD * 2, HND, 102)
        small0 = small.buf.cpu().numpy()
        dids = [3, 0, 5, 1]
        sh, smh = _register(m, src, src.kv), _register(m, small, small.kv)
        plan = [ScatterWindow(0, 0, 0, BNL, 0, 0, 4), ScatterWindow(0, 0, 0, BNL, 0, 4, 4), ScatterWindow(1, 0, 0, BNL, 0, 0, 4)]
        want_small = {}

        def want(old):
            pools = [np.stack(old), small0.copy()]
            repage_scatter(([src.final_np[b] for b in sids], src.kv, 4, BNL),
                           [(w.dst_rank, list(range(4)) if w.dst_rank == 0 else dids, int(UTP if w.dst_rank == 0 else HND), BNH if w.dst_rank == 0 else 4,
                             BNL, (w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count))
                            for w in plan], pools, BNO, 4, BNT, BHD * 2, TOKENS.start, TOKENS.stop)
            want_small["pool"] = pools[1]
            return list(pools[0])
        _into_big(big_pool, lambda: m.execute_repage_scatter(sh, _ids(sids), [bh, smh], [BIG_IDS, dids], plan, TOKENS).wait(30.0) or 0, want)
        assert np.array_equal(small.buf.cpu().numpy(), want_small["pool"])
    finally:
        torch.cuda.synchronize()
        m.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. manager id lists past a staging slot's arena share (4096 ids), then many short scatters reusing the slots
# ---------------------------------------------------------------------------------------------------------------------
def test_manager_scatter_id_lists_grow_and_reuse_staging_slots():
    """Llama-3-8B's KV geometry on 4 layers: one-token pages of 8 heads -> 8 TP destinations of 16-token pages over 32 768 tokens
    (32 768 + 8 x 2 048 ids), then 72 short scatters back to back on disjoint blocks.  Expected pools from torch indexing over the
    token view, cross-checked with the numpy oracle on sampled blocks."""
    m = TransferManager(device=0, worker_id=63)
    try:
        nl, no, hd, T = 4, 2, 128, 32768
        gen = torch.Generator(device="cuda").manual_seed(8)
        rng = np.random.default_rng(9)
        src = _DevPool(m, T + 1, nl, no, 1, 8, hd, NHD, gen)
        dsts = [_DevPool(m, T // 16 + 1, nl, no, 16, 1, hd, ALL[d % 4], gen) for d in range(8)]
        plan = tp_pp_scatter_plan(8, nl, 1, 1, 8, 1, 0)
        assert [w.dst_rank for w in plan] == list(range(8))
        stab = [int(x) for x in rng.permutation(T + 1)[:T]]
        dtabs = [[int(x) + 1 for x in rng.permutation(T // 16)] for _ in dsts]       # block 0 of every destination is the guard
        tb, te = 5, T

        def scatter(a, b, n=8):
            return m.execute_repage_scatter(src.h, table_slice(stab, a, b, 1), [d.h for d in dsts[:n]], [table_slice(t, a, b, 16) for t in dtabs[:n]],
                                            plan[:n], range(a, b))

        def expect(exps, a, b, n=8):
            for w in plan[:n]:
                _torch_expect(exps[w.dst_rank], dsts[w.dst_rank], dtabs[w.dst_rank], a, b, [(src, stab)],
                              [(0, w.src_head_begin, w.dst_head_begin, w.head_count)])

        exps = [d.mem.clone() for d in dsts]
        sample = [0, T // 32, T // 16 - 1]
        olds = {(d, k): dsts[d].block(dtabs[d][k]) for d in (0, 7) for k in sample}
        scatter(tb, te).wait(60.0)
        torch.cuda.synchronize()
        expect(exps, tb, te)
        for (d, k), old in olds.items():                                    # the torch reference against the numpy oracle
            a, b = max(tb, k * 16), min(te, (k + 1) * 16)
            w = plan[d]
            pools = [old[None].copy()]
            repage_scatter(([src.block(x) for x in table_slice(stab, a, b, 1)], int(NHD), 8, nl),
                           [(0, [0], int(dsts[d].kv), 1, nl, (0, 0, nl, w.src_head_begin, w.dst_head_begin, w.head_count))], pools, no, 1, 16,
                           hd * 2, a, b)
            assert np.array_equal(pools[0][0], dsts[d].block(dtabs[d][k], exps[d]))
        for d, e in zip(dsts, exps):
            assert torch.equal(d.mem, e)

        for d in dsts:
            d.randomize()
        exps = [d.mem.clone() for d in dsts]
        notes, done = [], []
        for i in range(72):
            a = i * 448 + 7 + i % 5
            b = a + 40 + 37 * (i % 7)
            n = 4 if i % 9 == 8 else 8                                       # some to the first 4 destinations only
            notes.append(scatter(a, b, n))
            done.append((a, b, n))
        for note in notes:
            note.wait(60.0)
        torch.cuda.synchronize()
        for a, b, n in done:
            expect(exps, a, b, n)
        for d, e in zip(dsts, exps):
            assert torch.equal(d.mem, e)
    finally:
        torch.cuda.synchronize()
        m.close()


def test_manager_batch_id_lists_outgrow_a_staging_slot(mgr):
    """300 sequences of 230-269 tokens, one-token pages -> 16-token pages: about 75 000 source and 4 800 destination ids in one
    execute_repage_batch, each side past a slot's 4 096."""
    plan = tp_pp_reshard_plan(2, 2, 1, 1, 1, 1, 0)
    seqs = [(i * 7 % 16 + i, i * 7 % 16 + i + 230 + i % 40) for i in range(300)]
    r = plan_rig(2, 2, 1, 1, 1, 1, 0, seqs, src_kv=HND, dst_kv=UTP, ps=1, pd=16, seed=33)
    assert min(len(np.concatenate(r.sids[0])), len(np.concatenate(r.dids))) > 4096
    ranks = sorted({w.src_rank for w in plan})
    hs = {rk: _register(mgr, r.srcs[i], r.srcs[i].kv) for i, rk in enumerate(ranks)}
    dh = _register(mgr, r.dst, r.dst.kv)
    mgr.execute_repage_batch(hs, dh, _requests(r, ranks), plan).wait(30.0)
    torch.cuda.synchronize()
    r.check()

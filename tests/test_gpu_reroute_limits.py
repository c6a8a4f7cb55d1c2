"""The batch re-paging scatter (kvbm_kernels_paged_repage_scatter_batch), the routed scatter
(kvbm_kernels_paged_repage_scatter_routed, TransferManager.execute_repage_scatter_routed), the routed gather
(kvbm_kernels_paged_stage_repage_gather_routed, TransferManager.execute_repage_batch_routed) and the any-page gather
(kvbm_kernels_paged_stage_repage_gather_anypage) at the limits their launchers accept, each paired with its first rejected
neighbour where it has one, and past 4 GiB, against the oracles:

- block offsets past 2^32 in the > 4 GiB pool of tests/test_gpu_transform_limits.py, as the destination and as the source of
  each family, on the larger page's side (block ids[j]) and on the smaller page's side (block ids[small_k + b]); the any-page
  pairs (24 and 6 against the pool's 16) run with a nonzero phase.  In the routed cases every unrouted position of a big-pool
  table names a big-pool block past 2^32 that must keep its bytes;
- the streamed form of each family, flags released before the launch, in both gate modes, into the big pool;
- the routing tables at their maxima: a routed scatter of 16 targets and 256 (target, head) pairs whose masks route 31, 16 or 1
  entries of one stage, and a routed gather of 16 sources over 256 heads under masks of the last, the first and every source;
- the manager's 32-bit masks: 32 destinations (32 sources) whose windows read or write ranks 16-31, sequences routed to rank 31
  alone, next to the 33-rank rejection;
- the any-page arithmetic at its bounds together: the largest pair the exactness bound accepts at a prime small page with the
  phase at its maximum next to the first rejected pair, the multiply-high row split at V = 4095 with a nonzero phase, and units
  across 2^31 with the last big block ending below 2^32.

Pools start from random bytes (the big pool from its hash fill), every destination keeps blocks no table names, and whole
destination pools are compared with tests/scatter_batch_oracle.py, tests/scatter_oracle.py (per sequence, through the routed
rig), tests/stage_repage_oracle.py and tests/repage_batch_oracle.py.  A wrongly computed index stays inside the allocations: the
id tables are full length, unrouted positions name real blocks, and a block offset cut to 32 bits lands WRAP blocks lower in the
same pool, on a block that must keep its fill.  A rejected neighbour returns its error before any launch, so K.launch_count()
stays put.  There is no profiler here: every launch is followed by a device synchronize before its check.

Not covered: the accepted neighbour of the num_units x layers x outer_dim < 2^31 bound, which needs a 16 GiB unit table or 2^31
CTAs; its rejection is a CPU case (tests/test_scatter_route_host.py, tests/test_gather_route_host.py)."""
import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import ErrorCode, KvbmError, LayoutConfig, ScatterWindow, ShardWindow, StorageKind, TransferManager
from tests.gpu_util import stream_ptr
from tests.scatter_batch_oracle import table_len
from tests.test_gpu_gather_route import GatherRig
from tests.test_gpu_gather_route import _register as _register_gather_pool
from tests.test_gpu_repage_anypage import AnyRig, any_rig
from tests.test_gpu_scatter_route import RouteRig
from tests.test_gpu_scatter_route import _register as _register_pool
from tests.test_gpu_scatter_seqs import BatchRig as SeqsRig
from tests.test_gpu_gather_route import _managed as _managed_gather
from tests.test_gpu_repage_batch import _requests
from tests.test_gpu_scatter_route import _managed as _managed_route
from tests.test_gpu_scatter_seqs import _managed as _managed_seqs
from tests.test_gpu_transform_limits import (BHD, BIG_IDS, BNB, BNH, BNL, BNO, BNT, V_BOUND, WRAP, _into_big, _rejected,
                                             big_pool)  # noqa: F401  (big_pool: the fixture)

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
NHD, HND, UTP, UPP = KV.OperationalNHD, KV.OperationalHND, KV.UniversalTP, KV.UniversalPP
BATCH_SEQS = [(5, 29), (115, 141)]     # two big-pool blocks each at page 16: four destination blocks in all
UNROUTED = [WRAP + 40, WRAP + 41]      # big-pool blocks that only unrouted table positions name
GEOM = dict(no=BNO, hd=BHD)           # bf16 rows of the big pool's head_dim, its outer dimension


def _sync():
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# a rig pool standing in for the big pool: same geometry, its side pointed at the big pool through a remapped table
# ---------------------------------------------------------------------------------------------------------------------
def _point_at_big(big, pool, table, remap):
    """pool.side(...) now names the big pool, with `table` (the pool's concatenated ids) mapped through `remap`."""
    assert (pool.nl, pool.no, pool.page, pool.nh, pool.row) == (BNL, BNO, BNT, BNH, BHD * 2)
    t = torch.tensor([remap[int(x)] for x in table] or [0], dtype=torch.int32, device="cuda")
    kv = pool.kv
    pool.side = lambda _ids: K.PermuteSide(big.desc, t.data_ptr(), kv)
    pool.big_table = t


def _as_destination(big, pool, table, unrouted=()):
    """Map the table's routed ids (at most 4) to BIG_IDS and the ids of `unrouted` to UNROUTED; returns {rig id: big id}."""
    routed = [int(x) for x in dict.fromkeys(int(y) for y in table) if int(x) not in unrouted]
    assert len(routed) <= len(BIG_IDS) and len(unrouted) <= len(UNROUTED)
    remap = dict(zip(routed, BIG_IDS))
    remap.update(zip(unrouted, UNROUTED))
    _point_at_big(big, pool, table, remap)
    return remap


def _as_source(big, pool, table):
    """Map every id the table names to its own big-pool block past 2^32, whose bytes become the rig pool's final bytes."""
    ids = list(dict.fromkeys(int(y) for y in table))
    remap = {x: WRAP + 2 + 3 * k for k, x in enumerate(ids)}
    assert max(remap.values()) < WRAP + 64
    for x, b in remap.items():
        pool.final_np[x] = big.block(b)
    _point_at_big(big, pool, table, remap)


def _into_big_rows(big, launch, initial, remap, expected):
    """_into_big with a rig: the big blocks' old bytes become rows of the rig pool's initial tensor, `expected()` is the rig's
    oracle pool (numpy) for that stand-in; returns what expected() returned, for the rig's other pools."""
    inv = {b: x for x, b in remap.items()}
    out = {}

    def want(old):
        for b, blk in zip(BIG_IDS, old):
            if b in inv:
                initial[inv[b]] = torch.from_numpy(blk).cuda()
        out["pools"], pool = expected()
        return [pool[inv[b]] if b in inv else o for b, o in zip(BIG_IDS, old)]
    _into_big(big, lambda: launch() or 0, want)
    return out["pools"]


def _check_filled(big):
    try:
        big.assert_all_filled()
    except BaseException:
        big.refill()
        raise


# ---------------------------------------------------------------------------------------------------------------------
# 1. each family into and out of the big pool, on both address paths
# ---------------------------------------------------------------------------------------------------------------------
def _seqs_dst(ps):
    """A 4-head source into the big pool's heads 0-3 and 4-7 (two targets, one table) and a small pool."""
    return SeqsRig((BNL, 4, NHD), [(BNL, BNH, UTP), (BNL, 4, HND)], [(0, 0, 0, BNL, 0, 0, 4), (0, 0, 0, BNL, 0, 4, 4), (1, 0, 0, BNL, 0, 0, 4)],
                   BATCH_SEQS, ps=ps, pd=BNT, seed=ps, **GEOM)


def _route_dst(ps, masks=(0b111, 0b100, 0b010)):
    """As _seqs_dst, routed: sequence 0 to every target, 1 to the small pool only (its big-pool positions unrouted), 2 to the big
    pool's heads 4-7 only (the manager, which routes whole destinations: to the big pool)."""
    return RouteRig((BNL, 4, NHD), [(BNL, BNH, UTP), (BNL, 4, HND)], [(0, 0, 0, BNL, 0, 0, 4), (0, 0, 0, BNL, 0, 4, 4), (1, 0, 0, BNL, 0, 0, 4)],
                    [(tb, te, m) for (tb, te), m in zip([(5, 29), (40, 60), (115, 141)], masks)], ps=ps, pd=BNT, seed=ps + 1, **GEOM)


def _fanin_dst(ps):
    """TP2 -> the big pool's 8 heads: sequence 0 from both sources, 1 from source 0 only, 2 from source 1 only."""
    return GatherRig([(BNL, 4, HND), (BNL, 4, NHD)], [(0, 0, 0, BNL, 0, 0, 4), (1, 0, 0, BNL, 0, 4, 4)], (BNL, BNH, UTP),
                     [(5, 29, 0b11), (40, 47, 0b01), (115, 120, 0b10)], ps=ps, pd=BNT, seed=ps + 2, **GEOM)


def _any_dst(ps):
    return AnyRig([(BNL, 4, HND), (BNL, 4, NHD)], [(0, 0, 0, BNL, 0, 0, 4), (1, 0, 0, BNL, 0, 4, 4)], BNL, BNH, UTP, BATCH_SEQS, ps=ps, pd=BNT,
                  seed=ps + 3, **GEOM)


def _dst_case(family, ps, manager=False):
    """(rig, stand-in pool, its table, unrouted ids, initial tensor (rows by rig id), launch, expected() -> (all pools, stand-in's))."""
    if family == "batch_scatter":
        r = _seqs_dst(ps)
        return r, r.dsts[0], r.dids[0], (), r.initial[0], r.launch, lambda: (lambda p: (p, p[0]))(r.expected())
    if family == "routed_scatter":
        r = _route_dst(ps, (0b111, 0b100, 0b011)) if manager else _route_dst(ps)
        return r, r.dsts[0], r.dids[0], tuple(r.sentinel[0]), r.initial[0], r.launch, lambda: (lambda p: (p, p[0]))(r.expected())
    if family == "routed_gather":
        r = _fanin_dst(ps)
        return r, r.dst, r.dids, (), r.initial, r.launch, lambda: (lambda p: (p, p))(r.expected())
    r = _any_dst(ps)
    assert (r.any_np[:, 3] != 0).any(), "a nonzero phase"
    return r, r.dst, np.concatenate(r.dids), (), r.initial, r.run, lambda: (lambda p: (p, p))(r.expected())


# (source page) per family: the big pool on the larger page's side, then on the smaller page's side
DST_PAGES = {"batch_scatter": (4, 64), "routed_scatter": (4, 64), "routed_gather": (4, 64), "anypage": (6, 24)}


@pytest.mark.parametrize("side", ["larger_page_side", "smaller_page_side"])
@pytest.mark.parametrize("family", list(DST_PAGES))
def test_big_pool_as_destination(big_pool, family, side):
    ps = DST_PAGES[family][side == "smaller_page_side"]
    r, pool, table, unrouted, initial, launch, expected = _dst_case(family, ps)
    remap = _as_destination(big_pool, pool, table, unrouted)
    pools = _into_big_rows(big_pool, launch, initial, remap, expected)
    if family in ("batch_scatter", "routed_scatter"):           # the small pool beside the big one
        assert np.array_equal(r.dsts[1].buf.cpu().numpy(), pools[1])
    _sync()


def _seqs_src(pd):
    return SeqsRig((BNL, BNH, UTP), [(BNL, BNH, NHD), (BNL, 4, UTP)], [(0, 0, 0, BNL, 0, 0, BNH), (1, 0, 0, BNL, 4, 0, 4)], BATCH_SEQS, ps=BNT,
                   pd=pd, seed=pd + 4, **GEOM)


def _route_src(pd):
    return RouteRig((BNL, BNH, UTP), [(BNL, BNH, NHD), (BNL, 4, UTP)], [(0, 0, 0, BNL, 0, 0, BNH), (1, 0, 0, BNL, 4, 0, 4)],
                    [(5, 29, 0b11), (40, 60, 0b10), (115, 141, 0b01)], ps=BNT, pd=pd, seed=pd + 5, **GEOM)


def _fanin_src(pd):
    """Two 8-head workers writing the same destination heads, each sequence from one: the big pool is worker 0, its positions
    for worker 1's sequence unrouted."""
    return GatherRig([(BNL, BNH, UTP), (BNL, BNH, HND)], [(0, 0, 0, BNL, 0, 0, BNH), (1, 0, 0, BNL, 0, 0, BNH)], (BNL, BNH, NHD),
                     [(5, 29, 0b01), (40, 60, 0b10), (115, 141, 0b01)], ps=BNT, pd=pd, seed=pd + 6, **GEOM)


def _any_src(pd):
    return AnyRig([(BNL, BNH, UTP)], [(0, 0, 0, BNL, 0, 0, BNH)], BNL, BNH, NHD, BATCH_SEQS, ps=BNT, pd=pd, seed=pd + 7, **GEOM)


# (destination page) per family: the big pool on the larger page's side, then on the smaller page's side
SRC_PAGES = {"batch_scatter": (4, 32), "routed_scatter": (4, 32), "routed_gather": (4, 32), "anypage": (6, 24)}


@pytest.mark.parametrize("side", ["larger_page_side", "smaller_page_side"])
@pytest.mark.parametrize("family", list(SRC_PAGES))
def test_big_pool_as_source(big_pool, family, side):
    pd = SRC_PAGES[family][side == "smaller_page_side"]
    if family == "batch_scatter":
        r = _seqs_src(pd)
        _as_source(big_pool, r.src, r.sids)
        assert r.launch() == 0
        _sync()
        for p, want in zip(r.dsts, r.expected()):
            assert np.array_equal(p.buf.cpu().numpy(), want)
    elif family == "routed_scatter":
        r = _route_src(pd)
        _as_source(big_pool, r.src, r.sids)
        assert r.launch() == 0
        _sync()
        r.check_pools()
    elif family == "routed_gather":
        r = _fanin_src(pd)
        _as_source(big_pool, r.srcs[0], r.sids[0])
        assert r.launch() == 0
        _sync()
        assert np.array_equal(r.dst.buf.cpu().numpy(), r.expected())
    else:
        r = _any_src(pd)
        assert (r.any_np[:, 3] != 0).any(), "a nonzero phase"
        _as_source(big_pool, r.srcs[0], np.concatenate(r.sids[0]))
        assert r.run() == 0
        r.check()
    _check_filled(big_pool)
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# 2. the streamed form of each family into the big pool, flags released before the launch
# ---------------------------------------------------------------------------------------------------------------------
GUARDED = 64     # ready words: every layer and the words after them, all released


def _stream_desc(epoch, gate_mode, ready, nl, n_ready):
    st = K.PermuteStream()
    for j in range(n_ready):
        st.layer_ready_flags[j] = ready.data_ptr()
    flags = torch.zeros(nl + 2, dtype=torch.int32, device="cuda")
    ws = torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device="cuda")
    st.layer_done_flags, st.done_flag, st.completion_flag = flags.data_ptr(), flags[nl:].data_ptr(), flags[nl + 1:].data_ptr()
    st.epoch, st.sync_workspace, st.completion_value = epoch, ws.data_ptr(), epoch + 1
    st.gate_mode, st.gate_timeout_ms, st.max_ctas = gate_mode, 10000, 4
    return st, flags, ws


@pytest.mark.parametrize("gate_mode", [K.GATE_SPIN, K.GATE_STREAM_WAIT], ids=["spin", "stream_wait"])
@pytest.mark.parametrize("family", list(DST_PAGES))
def test_streamed_into_the_big_pool(big_pool, family, gate_mode):
    epoch = 9
    r, pool, table, unrouted, initial, _launch, expected = _dst_case(family, DST_PAGES[family][0])
    remap = _as_destination(big_pool, pool, table, unrouted)
    ready = torch.full((GUARDED,), epoch, dtype=torch.int32, device="cuda")
    nw = len(r.windows) if family in ("routed_gather", "anypage") else 1
    st, flags, ws = _stream_desc(epoch, gate_mode, ready, BNL, nw)
    _sync()
    if family == "batch_scatter":
        launch = lambda: K.paged_repage_scatter_batch_streamed(r.src.side(r.sids_t), r.src.nh, r.ps, r.kernel_targets(), r.pd, r.seqs,  # noqa: E731
                                                               r.units_t.data_ptr(), r.nu, r.lb, r.le, r.row, r.cast, r.scales, st, stream_ptr())
    elif family == "routed_scatter":
        launch = lambda: K.paged_repage_scatter_routed_streamed(r.src.side(r.sids_t), r.src.nh, r.ps, r.kernel_targets(), r.pd, r.seqs,  # noqa: E731
                                                                r.units_t.data_ptr(), r.nu, r.lb, r.le, r.row, r.cast, r.scales, st, stream_ptr())
    elif family == "routed_gather":
        launch = lambda: K.paged_stage_repage_gather_routed_streamed(*r.args(), st, stream_ptr())  # noqa: E731
    else:
        launch = lambda: K.paged_stage_repage_gather_anypage_streamed(*r.args(), st, stream_ptr())  # noqa: E731
    pools = _into_big_rows(big_pool, launch, initial, remap, expected)
    if family in ("batch_scatter", "routed_scatter"):
        assert np.array_equal(r.dsts[1].buf.cpu().numpy(), pools[1])
    assert flags.tolist() == [epoch] * (BNL + 1) + [epoch + 1]
    assert not ws.any().item(), "the workspace must be left zeroed"
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# 3. the routing tables at their maxima
# ---------------------------------------------------------------------------------------------------------------------
# routed scatter: targets 0-13 take source heads 0-15, target 14 head 47 alone, target 15 heads 16-46: 224 + 1 + 31 = 256 pairs
ROUTE_WINDOWS = [(0, 16)] * 14 + [(47, 1), (16, 31)]
ROUTE_MASKS = [1 << 15, 1 << 14, 0x5555, 0xAAAA, 1 << 0, 0xFFFF, (1 << 14) | (1 << 15), 0x3FFF]


def test_routed_scatter_at_16_targets_and_256_pairs():
    """One stage of 48 source heads; the masks route 31 entries (bit 15 alone), 1 entry (bit 14 alone), 16 and 48 in one launch,
    so one sequence's warps loop past 8 entries while another's is one warp.  A 17th target is rejected, with the pairs still at
    256 (target 15 gives up a head to it)."""
    dsts = [(2, k + (t % 3), (UTP, HND, NHD, UPP)[t % 4]) for t, (_sb, k) in enumerate(ROUTE_WINDOWS)]
    targets = [(t, 0, 0, 2, sb, t % 3, k) for t, (sb, k) in enumerate(ROUTE_WINDOWS)]
    seqs = [(3 + 70 * i, 3 + 70 * i + 40 + 7 * i, m) for i, m in enumerate(ROUTE_MASKS)]
    r = RouteRig((2, 48, HND), dsts, targets, seqs, ps=16, pd=64, no=1, hd=32, seed=256)
    assert len(r.targets) == K.GATHER_MAX_SOURCES and sum(t[6] for t in r.targets) == K.GATHER_MAX_HEADS
    r.run_and_check()
    ntargets = targets[:15] + [targets[15][:6] + (30,), (16, 0, 0, 2, 46, 0, 1)]
    assert len(ntargets) == K.GATHER_MAX_SOURCES + 1 and sum(t[6] for t in ntargets) == K.GATHER_MAX_HEADS
    n = RouteRig((2, 48, HND), dsts + [(2, 1, NHD)], ntargets, seqs, ps=16, pd=64, no=1, hd=32, seed=257)
    _rejected(lambda: n.launch())
    _sync()


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16)], ids=str)
def test_routed_gather_at_16_sources_and_256_heads(ps, pd):
    """16 sources of 16 heads into 256 destination heads, one stage: sequences from the last source only, the first only, every
    source, and alternating halves; 16 routed entries under one mask make the CTA's 8 warps loop.  A 17th source is rejected,
    with the covered heads still at 256 (source 15 gives up 8 of its heads to it)."""
    pools = [(2, 16, (HND, NHD, UTP, UPP)[p % 4]) for p in range(16)]
    windows = [(p, 0, 0, 2, 0, 16 * p, 16) for p in range(16)]
    masks = [1 << 15, 1, 0xFFFF, 0x5555, 0xAAAA, 1 << 15]
    seqs = [(5 + 90 * i, 5 + 90 * i + 50 + 9 * i, m) for i, m in enumerate(masks)]
    r = GatherRig(pools, windows, (2, 256, NHD), seqs, ps=ps, pd=pd, no=1, hd=8, seed=ps)
    r.run_and_check()
    nwindows = windows[:15] + [(15, 0, 0, 2, 0, 240, 8), (16, 0, 0, 2, 0, 248, 8)]
    assert len(nwindows) == K.GATHER_MAX_SOURCES + 1 and sum(w[6] for w in nwindows) == K.GATHER_MAX_HEADS
    n = GatherRig(pools + [(2, 8, HND)], nwindows, (2, 256, NHD), seqs, ps=ps, pd=pd, no=1, hd=8, seed=ps + 1)
    _rejected(lambda: n.launch())
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# 4. the manager's 32-bit masks: windows on ranks 16-31, sequences routed to rank 31 alone, next to 33 ranks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=67)
    yield m
    _sync()
    m.close()


# masks over the 16 rig pools, pool p being manager rank 16 + p
HIGH_MASKS = [1 << 15, 1 << 15, 1, 0xFFFF, 0x8001, 0x00F0, 1 << 15, 0x7FFF]


def test_manager_routed_scatter_to_32_destinations(mgr):
    """execute_repage_scatter_routed with 32 destinations, windows writing 16-31 only; several sequences go to destination 31
    alone.  Destinations 0-15 are registered pools no window writes and keep their bytes.  33 destinations: UNSUPPORTED, nothing
    launched."""
    dsts = [(2, 1, (NHD, UTP)[p % 2]) for p in range(16)]
    targets = [(p, 0, 0, 2, p, 0, 1) for p in range(16)]
    seqs = [(7 + 100 * i, 7 + 100 * i + 60 + 5 * i, m) for i, m in enumerate(HIGH_MASKS)]
    r = RouteRig((2, 16, HND), dsts, targets, seqs, ps=16, pd=64, no=1, hd=32, seed=32)
    idle = [RouteRig((2, 1, HND), [(2, 1, NHD)], [(0, 0, 0, 2, 0, 0, 1)], [(0, 1, 1)], ps=16, pd=64, no=1, hd=32, seed=40 + k).dsts[0]
            for k in range(17)]
    idle0 = [p.buf.clone() for p in idle]
    sh = _register_pool(mgr, r.src, KV(r.src.kv))
    dhs = [_register_pool(mgr, p, KV(p.kv)) for p in idle[:16]] + [_register_pool(mgr, p, KV(p.kv)) for p in r.dsts]
    extra = _register_pool(mgr, idle[16], KV(idle[16].kv))
    plan = [ScatterWindow(16 + p, sl, dl, c, sb, db, k) for p, sl, dl, c, sb, db, k in r.targets]
    reqs, so, do = [], 0, 0
    for tb, te, m in r.seqs:
        a, b = table_len(tb, te, r.ps), table_len(tb, te, r.pd)
        reqs.append((range(tb, te), [int(x) for x in r.sids[so:so + a]],
                     {16 + p: [int(x) for x in r.dids[p][do:do + b]] for p in range(16) if (m >> p) & 1}))
        so, do = so + a, do + b
    assert sum(set(q[2]) == {31} for q in reqs) >= 3
    mgr.execute_repage_scatter_routed(sh, dhs, reqs, plan).wait(20.0)
    _sync()
    r.check_pools()
    assert all(torch.equal(p.buf, x) for p, x in zip(idle, idle0))
    before = K.launch_count()
    with pytest.raises(KvbmError) as e:
        mgr.execute_repage_scatter_routed(sh, dhs + [extra], reqs, plan)
    assert e.value.code == ErrorCode.UNSUPPORTED and K.launch_count() == before
    _sync()


def _c_batch_routed(mgr, handles, dh, reqs, plan):
    """kvbm_manager_execute_repage_batch_routed with the source list as given (TransferManager.execute_repage_batch_routed passes
    only the ranks its plan reads, so its masks never reach bit 16): reqs are (tokens, {source rank: ids}, dst ids); the mask is
    the dict's keys.  Returns the notification or raises the error."""
    import ctypes as C
    from dynamo_b200 import physical as P
    keep, n = [], len(handles)
    cs = (P._CRepageRouteSeq * max(1, len(reqs)))()
    for c, (tokens, ids, dids) in zip(cs, reqs):
        arrs = {r: (C.c_size_t * max(1, len(x)))(*x) for r, x in ids.items()}
        sp = (C.c_void_p * n)(*[C.addressof(arrs[r]) if r in arrs else None for r in range(n)])
        d = (C.c_size_t * max(1, len(dids)))(*dids)
        keep += [arrs, sp, d]
        c.token_begin, c.token_end, c.src_ids, c.n_src = tokens.start, tokens.stop, C.addressof(sp), len(next(iter(ids.values())))
        c.dst_ids, c.n_dst, c.src_mask = C.addressof(d), len(dids), sum(1 << r for r in ids)
    ws = (P._CShardWindow * len(plan))(*[P._CShardWindow(w.src_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin,
                                                          w.dst_head_begin, w.head_count) for w in plan])
    srcs = (C.c_uint64 * n)(*handles)
    o, tok = P.TransferOptions()._c(), C.c_uint64()
    P._check(P.lib().kvbm_manager_execute_repage_batch_routed(mgr._h, n, srcs, dh, cs, len(reqs), ws, len(plan), None, C.byref(o),
                                                             C.byref(tok)))
    return P.TransferCompleteNotification(mgr, tok.value)


def test_manager_routed_gather_from_32_sources(mgr):
    """The routed gather's C entry with 32 sources, windows reading 16-31 only; several sequences come from source 31 alone, so
    its window mask is bit 15 and its source mask bit 31.  33 sources: UNSUPPORTED, nothing launched."""
    pools = [(2, 1, (HND, UTP)[p % 2]) for p in range(16)]
    windows = [(p, 0, 0, 2, 0, p, 1) for p in range(16)]
    seqs = [(7 + 100 * i, 7 + 100 * i + 60 + 5 * i, m) for i, m in enumerate(HIGH_MASKS)]
    r = GatherRig(pools, windows, (2, 16, NHD), seqs, ps=64, pd=16, no=1, hd=32, seed=33)
    idle = GatherRig([(2, 1, HND)], [(0, 0, 0, 2, 0, 0, 1)], (2, 1, NHD), [(0, 1, 1)], ps=64, pd=16, no=1, hd=32, seed=34).srcs[0]
    handles = [_register_gather_pool(mgr, idle)] * 16 + [_register_gather_pool(mgr, x) for x in r.srcs]
    dh = _register_gather_pool(mgr, r.dst)
    plan = [ShardWindow(16 + p, sl, dl, c, sb, db, k) for p, sl, dl, c, sb, db, k in r.windows]
    reqs, so, do = [], 0, 0
    for tb, te, m in r.seqs:
        a, b = table_len(tb, te, r.ps), table_len(tb, te, r.pd)
        reqs.append((range(tb, te), {16 + p: [int(x) for x in r.sids[p][so:so + a]] for p in range(16) if (m >> p) & 1},
                     [int(x) for x in r.dids[do:do + b]]))
        so, do = so + a, do + b
    assert sum(set(q[1]) == {31} for q in reqs) >= 3
    _c_batch_routed(mgr, handles, dh, reqs, plan).wait(20.0)
    _sync()
    r.check_pool()
    before = K.launch_count()
    with pytest.raises(KvbmError) as e:
        _c_batch_routed(mgr, handles + handles[:1], dh, reqs, plan)
    assert e.value.code == ErrorCode.UNSUPPORTED and K.launch_count() == before
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# 5. the any-page arithmetic at its bounds together
# ---------------------------------------------------------------------------------------------------------------------
def _largest_big(small):
    """The largest big page that small does not divide and the exactness bound accepts (a multiple of small, whose factor is
    only big, goes further)."""
    big = 2 * small - 1
    while (big + small - int(np.gcd(big, small))) * small >= (1 << 32):
        big -= 1
    return big


@pytest.mark.parametrize("direction", ["small_to_big", "big_to_small"])
def test_anypage_largest_pair_at_the_largest_phase(direction):
    """Small page 46 337 (prime) under the largest big page it does not divide that the exactness bound takes (46 353), in a big
    block whose phase is small - 1, the largest, beside a sequence across 2^31 and one whose last big block ends below 2^32.  The next big page is rejected by
    the unit helper and by the launch, which launches nothing."""
    small = 46337
    big = _largest_big(small)
    assert int(np.gcd(big, small)) == 1
    j = next(j for j in range(1, small) if (j * big) % small == small - 1)
    mid = (1 << 31) // big * big
    last = ((1 << 32) - 1) // big * big
    seqs = [(j * big + 3, (j + 1) * big), (mid - 7, mid + 9), (last - small - 5, last)]
    ps, pd = (small, big) if direction == "small_to_big" else (big, small)
    r = any_rig(2, 1, 1, 1, 1, 1, 0, seqs, ps=ps, pd=pd, hd=8, no=1, seed=5)
    assert int(r.any_np[:, 3].max()) == small - 1
    assert r.run() == 0
    r.check()
    bps, bpd = (small, big + 1) if direction == "small_to_big" else (big + 1, small)
    assert K.repage_anypage_units(seqs, bps, bpd) is None
    args = list(r.args())
    args[1], args[4] = bps, bpd
    _rejected(lambda: K.paged_stage_repage_gather_anypage(*args, stream=stream_ptr()))
    _sync()


@pytest.mark.parametrize("ps,pd", [(24, 16), (16, 24)], ids=str)
def test_anypage_row_split_at_its_bound_with_a_phase(ps, pd):
    """V = 4095 vectors per walk row (the multiply-high split) with 24 <-> 16 pages, in big blocks of phase 8."""
    hd = V_BOUND * 16 // 2
    seqs = [(24 + 5, 3 * 24 - 1), (5 * 24 + 1, 5 * 24 + 2), (7 * 24 + 17, 9 * 24 + 3)]
    r = any_rig(1, 1, 1, 1, 1, 1, 0, seqs, ps=ps, pd=pd, hd=hd, no=1, seed=ps)
    assert 8 in set(int(x) for x in r.any_np[:, 3])
    assert r.run() == 0
    r.check()
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# 6. each family's manager entry into the big pool, registered as one fully contiguous layout
# ---------------------------------------------------------------------------------------------------------------------
def _register_big(mgr, big, kv):
    cfg = LayoutConfig(BNB, BNL, BNO, BNT, BNH * BHD, dtype_width_bytes=2, num_heads=BNH)
    h = mgr.register_fully_contiguous(cfg, big.mem.data_ptr(), big.mem.numel(), StorageKind.Device, 0)
    mgr.set_kv_block_layout(h, KV(kv))
    return h


@pytest.mark.parametrize("family", list(DST_PAGES))
def test_manager_into_the_big_pool(big_pool, mgr, family):
    """execute_repage_scatter_batch, execute_repage_scatter_routed, execute_repage_batch_routed and execute_repage_anypage with
    the big pool as the destination (the larger page's side): the staged tables name blocks past 2^32, and a routed scatter's
    unrouted positions are the manager's padding."""
    r, pool, table, unrouted, initial, _launch, expected = _dst_case(family, DST_PAGES[family][0], manager=True)
    remap = _as_destination(big_pool, pool, table, unrouted)
    bh = _register_big(mgr, big_pool, pool.kv)
    big = lambda xs: [remap[int(x)] for x in xs]  # noqa: E731
    if family == "batch_scatter":
        sh, dhs, plan, reqs = _managed_seqs(mgr, r)
        reqs = [(t, s, [big(d[0])] + d[1:]) for t, s, d in reqs]
        launch = lambda: mgr.execute_repage_scatter_batch(sh, [bh] + dhs[1:], reqs, plan).wait(30.0)  # noqa: E731
    elif family == "routed_scatter":
        sh, dhs, plan, reqs = _managed_route(mgr, r)
        reqs = [(t, s, {p: big(x) if p == 0 else x for p, x in d.items()}) for t, s, d in reqs]
        launch = lambda: mgr.execute_repage_scatter_routed(sh, [bh] + dhs[1:], reqs, plan).wait(30.0)  # noqa: E731
    elif family == "routed_gather":
        sources, _dh, plan, reqs = _managed_gather(mgr, r)
        reqs = [(t, s, big(d)) for t, s, d in reqs]
        launch = lambda: mgr.execute_repage_batch_routed(sources, bh, reqs, plan).wait(30.0)  # noqa: E731
    else:
        hs = {s: _register_pool(mgr, p, KV(p.kv)) for s, p in enumerate(r.srcs)}
        plan = [ShardWindow(*w) for w in r.windows]
        reqs = [(t, s, big(d)) for t, s, d in _requests(r, list(hs))]
        launch = lambda: mgr.execute_repage_anypage(hs, bh, reqs, plan).wait(30.0)  # noqa: E731
    pools = _into_big_rows(big_pool, launch, initial, remap, expected)
    if family in ("batch_scatter", "routed_scatter"):
        assert np.array_equal(r.dsts[1].buf.cpu().numpy(), pools[1])
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# 7. manager id lists past a staging slot's arena (4096 ids), then many short calls that reuse the slots
# ---------------------------------------------------------------------------------------------------------------------
ARENA_IDS = 4096
SHORT = 5         # sequences per short call


def _arena_seqs(n, length=61, step=80):
    return [(3 + step * i, 3 + step * i + length) for i in range(n)]


def _short_calls(call, reqs):
    """len(reqs) / SHORT calls back to back, waited on together."""
    notes = [call(reqs[i:i + SHORT]) for i in range(0, len(reqs), SHORT)]
    assert len(notes) > 64
    for note in notes:
        note.wait(30.0)
    _sync()


def test_manager_routed_scatter_ids_past_the_arena(mgr):
    """350 sequences of 4 blocks, each to one of two destinations: the routed ids (1400 source + 2 x 700) fit a slot's arena,
    the staged tables with the manager's padding of unrouted positions (1400 + 2 x 1400) do not.  Then 70 calls of 5 sequences."""
    r = RouteRig((2, 2, HND), [(2, 2, NHD), (2, 2, UTP)], [(0, 0, 0, 2, 0, 0, 2), (1, 0, 0, 2, 0, 0, 2)],
                 [(tb, te, 1 + i % 2) for i, (tb, te) in enumerate(_arena_seqs(350))], ps=16, pd=16, no=1, hd=32, seed=4096)
    n = len(r.sids)
    assert 2 * n < ARENA_IDS < 3 * n
    sh, dhs, plan, reqs = _managed_route(mgr, r)
    mgr.execute_repage_scatter_routed(sh, dhs, reqs, plan).wait(30.0)
    _sync()
    want = r.expected()
    r.check_pools(want)
    r.reset_pools()
    _short_calls(lambda q: mgr.execute_repage_scatter_routed(sh, dhs, q, plan), reqs)
    r.check_pools(want)


def test_manager_routed_gather_ids_past_the_arena(mgr):
    """350 sequences of 4 blocks, each from one of two workers writing the same heads: the routed ids (2 x 700 source + 1400)
    fit a slot's arena, the staged tables with the padding (2 x 1400 + 1400) do not.  Then 70 calls of 5 sequences."""
    r = GatherRig([(2, 2, HND), (2, 2, NHD)], [(0, 0, 0, 2, 0, 0, 2), (1, 0, 0, 2, 0, 0, 2)], (2, 2, UTP),
                  [(tb, te, 1 + i % 2) for i, (tb, te) in enumerate(_arena_seqs(350))], ps=16, pd=16, no=1, hd=32, seed=4097)
    n = len(r.dids)
    assert 2 * n < ARENA_IDS < 3 * n
    sources, dh, plan, reqs = _managed_gather(mgr, r)
    mgr.execute_repage_batch_routed(sources, dh, reqs, plan).wait(30.0)
    _sync()
    want = r.expected()
    r.check_pool(want)
    r.reset()
    _short_calls(lambda q: mgr.execute_repage_batch_routed(sources, dh, q, plan), reqs)
    r.check_pool(want)


def test_manager_anypage_ids_past_the_arena(mgr):
    """400 sequences of 100 tokens at 24 -> 16: about 2 000 source and 2 900 destination ids in one execute_repage_anypage.
    Then 80 calls of 5 sequences."""
    seqs = _arena_seqs(400, length=100, step=130)
    r = any_rig(2, 2, 1, 1, 1, 1, 0, seqs, ps=24, pd=16, no=1, hd=32, seed=4098)
    assert sum(len(x) for x in r.sids[0]) + sum(len(x) for x in r.dids) > ARENA_IDS
    hs = {s: _register_pool(mgr, p, KV(p.kv)) for s, p in enumerate(r.srcs)}
    dh = _register_pool(mgr, r.dst, KV(r.dst.kv))
    plan = [ShardWindow(*w) for w in r.windows]
    reqs = _requests(r, list(hs))
    mgr.execute_repage_anypage(hs, dh, reqs, plan).wait(30.0)
    _sync()
    r.check()
    r.dst.buf.copy_(r.initial)
    _short_calls(lambda q: mgr.execute_repage_anypage(hs, dh, q, plan), reqs)
    r.check()

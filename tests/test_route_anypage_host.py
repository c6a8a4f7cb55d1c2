"""CPU checks of routed re-paging between pages that need not divide (each sequence of a batch pushed to, or pulled from, its own
workers in one launch, for any two page sizes): the exported symbols and the C layout of kvbm_route_anypage_unit, the unit table of
kvbm_kernels_repage_route_anypage_units against its definition and against the routed and anypage helpers, its 16-bit mask rule,
the exactness bound at its edge, the kernel entries' argument checks that return before any CUDA call, the manager's rejections on a
host-only manager against the routed entries', a 24 -> 64 push and pull only the new entries accept, and the 80 instantiations in
the built library.  The GPU cases are in tests/test_gpu_route_anypage.py."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, KvbmError, LayoutConfig, ScatterWindow, ShardWindow, StorageKind, TransferManager, TransferOptions
from tests.test_repage_anypage_host import _random_batch, anypage_units
from tests.test_scatter_route_host import _c_layout

KV = K.KvBlockLayout
INVAL = K.CUDA_ERROR_INVALID_VALUE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO, ROW = 2, 128
CUDA_ONLY = "direct CUDA strategy only"

KERNEL_ENTRIES = ("kvbm_kernels_repage_route_anypage_units", "kvbm_kernels_paged_repage_scatter_routed_anypage",
                  "kvbm_kernels_paged_repage_scatter_routed_anypage_streamed", "kvbm_kernels_paged_stage_repage_gather_routed_anypage",
                  "kvbm_kernels_paged_stage_repage_gather_routed_anypage_streamed")
MANAGER_ENTRIES = ("kvbm_manager_execute_repage_scatter_routed_anypage", "kvbm_manager_execute_repage_batch_routed_anypage")


def test_route_anypage_symbols_are_exported_and_listed():
    for name in KERNEL_ENTRIES:
        assert name in K.EXPORTED_SYMBOLS and callable(getattr(K.lib(), name))
    for name in MANAGER_ENTRIES:
        assert name in P.EXPORTED_SYMBOLS and callable(getattr(P.lib(), name))


def test_the_route_anypage_unit_mirror_matches_the_c_struct():
    names = ["q0", "tokens", "small_k", "route"]
    assert [f[0] for f in K.RouteAnypageUnit._fields_] == names
    got = _c_layout("kvbm_kernels.h", "kvbm_route_anypage_unit", names)
    assert got[:-1] == [getattr(K.RouteAnypageUnit, f).offset for f in names] == [0, 4, 8, 12]
    assert got[-1] == C.sizeof(K.RouteAnypageUnit) == 16


# ---------------------------------------------------------------------------------------------------------------------
# the unit table
# ---------------------------------------------------------------------------------------------------------------------
def route_anypage_units(seqs, ps, pd):
    """The table from its definition: anypage_units over the ranges, each record's fourth word its sequence's mask | phase << 16."""
    units, a, b = anypage_units([(tb, te) for tb, te, _ in seqs], ps, pd)
    masks = [m for tb, te, m in seqs for _ in range(tb // max(ps, pd), -(-te // max(ps, pd))) if tb != te]
    out = units.copy()
    out[:, 3] = np.array(masks, dtype=np.uint32).reshape(-1) | (units[:, 3] << 16)
    return out, a, b


def _masks(rng, seqs):
    return [(tb, te, int(rng.integers(1, 1 << 16))) for tb, te in seqs]


NAMED = [(544, 64), (64, 544), (24, 16), (16, 24), (48, 64), (64, 48), (3, 5), (5, 3), (600, 599), (1, 7)]


def _pairs():
    rng = np.random.default_rng(11)
    return NAMED + [(int(a), int(b)) for a, b in rng.integers(1, 601, size=(12, 2))]


@pytest.mark.parametrize("ps,pd", _pairs(), ids=str)
def test_unit_table_against_its_definition(ps, pd):
    rng = np.random.default_rng(1000 * ps + pd)
    for _ in range(10):
        seqs = _masks(rng, _random_batch(rng, max(ps, pd), min(ps, pd)))
        got = K.repage_route_anypage_units(seqs, ps, pd)
        want = route_anypage_units(seqs, ps, pd)
        assert got is not None
        assert np.array_equal(got[0], want[0]) and got[1:] == want[1:]
        # the two halves of the fourth word: the anypage helper's phase and the routed helper's mask
        phases = K.repage_anypage_units([(tb, te) for tb, te, _ in seqs], ps, pd)
        assert np.array_equal(got[0][:, :3], phases[0][:, :3]) and np.array_equal(got[0][:, 3] >> 16, phases[0][:, 3])
        assert got[1:] == phases[1:]
        flat = [m for tb, te, m in seqs for _ in range(tb // max(ps, pd), -(-te // max(ps, pd))) if tb != te]
        assert (got[0][:, 3] & 0xFFFF).tolist() == flat


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (16, 16), (1, 16), (48, 96), (96, 48), (64, 544 * 64)], ids=str)
def test_dividing_pairs_give_the_routed_table_byte_for_byte(ps, pd):
    rng = np.random.default_rng(ps * 7 + pd)
    for _ in range(10):
        seqs = _masks(rng, _random_batch(rng, max(ps, pd), min(ps, pd)))
        got = K.repage_route_anypage_units(seqs, ps, pd)
        want = K.repage_route_units(seqs, ps, pd)
        assert got is not None and want is not None
        assert got[0].tobytes() == want[0].tobytes() and got[1:] == want[1:]


def test_a_mask_bit_16_is_rejected_next_to_bit_15_at_a_phase_past_2_pow_15():
    """46337 / 46353 is the largest non-dividing pair the bound takes; the range puts a big block's slot 0 at slot small - 1 of its
    small block, so the phase fills the high half's top bit and bit 15 of the mask sits next to it."""
    small, big = 46337, 46353
    j = next(j for j in range(1, small) if j * big % small == small - 1)
    seqs = [(j * big, j * big + 7, 1 << 15)]
    got = K.repage_route_anypage_units(seqs, big, small)
    assert got is not None and len(got[0]) == 1
    assert got[0][0, 3] == (1 << 15) | ((small - 1) << 16) and (small - 1) >= 1 << 15
    assert K.repage_route_anypage_units([(j * big, j * big + 7, 1 << 16)], big, small) is None
    assert K.repage_route_anypage_units([(0, 0, 1 << 16)], big, small) is None          # also on an empty sequence
    # nothing is written on a rejection
    n, a, b = C.c_size_t(), C.c_size_t(), C.c_size_t()
    out = np.full((2, 4), 0xDEAD, dtype=np.uint32)
    arr = K._route_seqs([(0, 100, 1), (0, 100, 1 << 20)])
    assert K.lib().kvbm_kernels_repage_route_anypage_units(C.cast(arr, C.c_void_p), 2, 24, 64, out.ctypes.data, 2, C.byref(n), C.byref(a),
                                                           C.byref(b)) != 0
    assert (out == 0xDEAD).all()


def _bound_pair(small):
    big = (1 << 32) // small
    while (big + small - math.gcd(big, small)) * small >= (1 << 32):
        big -= 1
    return big


def test_the_helper_shares_the_anypage_rules_and_bound():
    top = (1 << 32) - 64
    for seqs, ps, pd in (([(9, 8)], 24, 64), ([(0, 64)], 0, 64), ([(top, top + 1)], 24, 64)):
        assert K.repage_anypage_units(seqs, ps, pd) is None
        assert K.repage_route_anypage_units([s + (1,) for s in seqs], ps, pd) is None
    for small in (600, 40000, 46337):
        big = _bound_pair(small)
        for a, b in ((small, big), (big, small)):
            assert K.repage_route_anypage_units([(0, 5, 1)], a, b) is not None
            a1, b1 = a + (a == big), b + (b == big)
            assert K.repage_route_anypage_units([(0, 5, 1)], a1, b1) is None
            assert K.repage_anypage_units([(0, 5)], a1, b1) is None
    n, a, b = C.c_size_t(), C.c_size_t(), C.c_size_t()
    assert K.lib().kvbm_kernels_repage_route_anypage_units(None, 2, 24, 64, None, 0, C.byref(n), C.byref(a), C.byref(b)) != 0
    # capacity below the count: counted, min(count, cap) written
    seqs = [(3, 200, 5), (7, 90, 2)]
    full = K.repage_route_anypage_units(seqs, 24, 64)[0]
    out = np.full((2, 4), 0xDEAD, dtype=np.uint32)
    arr = K._route_seqs(seqs)
    assert K.lib().kvbm_kernels_repage_route_anypage_units(C.cast(arr, C.c_void_p), 2, 24, 64, out.ctypes.data, 2, C.byref(n), C.byref(a),
                                                           C.byref(b)) == 0
    assert n.value == len(full) > 2 and np.array_equal(out, full[:2])


# ---------------------------------------------------------------------------------------------------------------------
# the kernel entries' argument checks (descriptors no check dereferences)
# ---------------------------------------------------------------------------------------------------------------------
def _side(nh, nl, page, no=NO, ids=0x2000, base=0x1000):
    reg = page * nh * ROW
    return K.PermuteSide(K.PagedLayout(base, reg, 8 * reg, reg, nl, no, 8), ids, int(KV.OperationalNHD))


def _t(nh, nl, sb, db, k, sl, dl, c, page=64, **kw):
    return K.ScatterTarget(_side(nh, nl, page, **kw), nh, sb, db, k, sl, dl, c, None)


def _s(nh, nl, sb, db, k, sl, dl, c, page=24, **kw):
    return K.StageSource(K.PermuteSource(_side(nh, nl, page, **kw), nh, sb, db, k), sl, dl, c)


TARGETS = [_t(2, 4, 0, 0, 2, 0, 0, 4, ids=0x2100), _t(2, 4, 2, 0, 2, 0, 0, 4, ids=0x2200, base=0x1100), _t(2, 2, 0, 0, 2, 4, 0, 2, base=0x1200)]
SOURCES = [_s(2, 4, 0, 0, 2, 0, 0, 4, ids=0x2100), _s(2, 4, 0, 0, 2, 0, 0, 4, ids=0x2200, base=0x1100)]
SCATTER_SEQS = [(0, 64, 0b011), (70, 130, 0b100)]
GATHER_SEQS = [(0, 64, 0b01), (70, 130, 0b10)]


def _n(seqs, ps, pd, helper):
    u = helper(seqs, ps, pd)
    return len(u[0]) if u is not None else 0


def _rs(targets=TARGETS, seqs=SCATTER_SEQS, ps=24, pd=64, lb=0, le=6, cast=0, scales=None, units=None, streamed=False, routed=False):
    """The routed anypage scatter (or, routed=True, the routed scatter) on descriptors no check dereferences."""
    helper = K.repage_route_units if routed else K.repage_route_anypage_units
    units = units if units is not None else (0x7000, _n(seqs, ps, pd, helper))
    s = _side(4, 6, ps)
    if routed:
        f = K.paged_repage_scatter_routed_streamed if streamed is not False else K.paged_repage_scatter_routed
    else:
        f = K.paged_repage_scatter_routed_anypage_streamed if streamed is not False else K.paged_repage_scatter_routed_anypage
    if streamed is not False:
        return f(s, 4, ps, targets, pd, seqs, *units, lb, le, ROW, cast, scales, streamed)
    return f(s, 4, ps, targets, pd, seqs, *units, lb, le, ROW, cast, scales)


def _rg(srcs=SOURCES, seqs=GATHER_SEQS, ps=24, pd=64, lb=0, le=4, cast=0, scales=None, units=None, streamed=False, routed=False):
    helper = K.repage_route_units if routed else K.repage_route_anypage_units
    units = units if units is not None else (0x7000, _n(seqs, ps, pd, helper))
    d = _side(2, 4, pd)
    if routed:
        f = K.paged_stage_repage_gather_routed_streamed if streamed is not False else K.paged_stage_repage_gather_routed
    else:
        f = K.paged_stage_repage_gather_routed_anypage_streamed if streamed is not False else K.paged_stage_repage_gather_routed_anypage
    if streamed is not False:
        return f(srcs, ps, d, 2, pd, seqs, *units, lb, le, ROW, cast, scales, streamed)
    return f(srcs, ps, d, 2, pd, seqs, *units, lb, le, ROW, cast, scales)


def test_scatter_argument_checks_before_any_cuda_call():
    # nothing to move signals (nothing to signal here)
    assert _rs(seqs=[]) == 0 and _rs(seqs=[(9, 9, 1), (70, 70, 4)]) == 0 and _rs(lb=3, le=3) == 0
    # the routing first: a mask of 0, a bit at num_targets or above, also on an empty sequence, even with a wrong unit count
    for seqs in ([(0, 64, 0b011), (70, 130, 0)], [(0, 64, 0b1011)], [(0, 64, 1 << 31)], [(0, 64, 1), (9, 9, 0)], [(0, 64, 1), (9, 9, 8)]):
        assert _rs(seqs=seqs) == INVAL and _rs(seqs=seqs, units=(0x7000, 999)) == INVAL
    sixteen = [_t(2, 6, 0, 0, 2, 0, 0, 6, ids=0x3000 + 0x100 * i, base=0x4000 + 0x100 * i) for i in range(16)]
    assert _rs(targets=sixteen, seqs=[(0, 64, 1 << 16)], units=(0x7000, 1)) == INVAL
    # the batch's rules with the new helper's count: a reversed range, a count other than the helper's, a null table, a null seqs
    assert _rs(seqs=[(0, 64, 1), (9, 8, 1)], units=(0x7000, 2)) == INVAL
    n = _n(SCATTER_SEQS, 24, 64, K.repage_route_anypage_units)
    assert _rs(units=(0x7000, n + 1)) == INVAL and _rs(units=(0x7000, n - 1)) == INVAL and _rs(units=(0, n)) == INVAL
    arr = (K.ScatterTarget * 3)(*TARGETS)
    assert K.lib().kvbm_kernels_paged_repage_scatter_routed_anypage(C.byref(_side(4, 6, 24)), 4, 24, arr, 3, 64, None, 2, 0x7000, n, 0, 6,
                                                                   ROW, 0, None, 0, None, 0, None) == INVAL
    # pages just past the exactness bound, in both directions, next to the pair just inside it (an empty layer range then moves
    # nothing and returns before any CUDA call)
    small = 600
    big = _bound_pair(small)
    for a, b in ((small, big), (big, small)):
        for x, y, want in ((a, b, 0), (a + (a == big), b + (b == big), INVAL)):
            tg = [_t(2, 4, 0, 0, 2, 0, 0, 4, page=y)]
            assert _rs(targets=tg, seqs=[(0, 5, 1)], ps=x, pd=y, units=(0x7000, 1), lb=2, le=2) == want
    # the single scatter's rules
    assert _rs(lb=4, le=3) == INVAL and _rs(le=7) == INVAL
    assert _rs(targets=[]) == INVAL and _rs(targets=[TARGETS[0]] * 17, seqs=[(0, 64, 1)]) == INVAL
    assert _rs(cast=3) == INVAL and _rs(scales=0x5000) == INVAL
    assert _rs(targets=TARGETS[:2], seqs=[(0, 64, 1)]) == INVAL                    # source layers 4..6 uncovered
    assert _rs(targets=TARGETS[:2] + [_t(2, 2, 0, 0, 2, 3, 0, 2)]) == INVAL        # partly overlapping stages
    # the streamed entry: a null descriptor, one without ready flags, an unknown gate mode, the spinning form without a workspace
    assert _rs(streamed=None) == INVAL and _rs(streamed=K.PermuteStream()) == INVAL
    st = K.PermuteStream()
    st.layer_ready_flags[0] = 0x3000
    st.gate_mode = 7
    assert _rs(streamed=st) == INVAL
    st.gate_mode = K.GATE_SPIN
    assert _rs(streamed=st) == INVAL
    # the routed scatter keeps rejecting 24 -> 64 (the anypage table's count is the same; the pages are what it rejects)
    assert _rs(routed=True, units=(0x7000, n)) == INVAL


def test_gather_argument_checks_before_any_cuda_call():
    assert _rg(seqs=[]) == 0 and _rg(seqs=[(9, 9, 1), (70, 70, 2)]) == 0 and _rg(lb=3, le=3) == 0
    for seqs in ([(0, 64, 1), (70, 130, 0)], [(0, 64, 0b101)], [(0, 64, 1 << 31)], [(0, 64, 1), (9, 9, 0)], [(0, 64, 1), (9, 9, 4)]):
        assert _rg(seqs=seqs) == INVAL and _rg(seqs=seqs, units=(0x7000, 999)) == INVAL
    # two overlapping windows of one stage in one mask
    assert _rg(seqs=[(0, 64, 0b11)]) == INVAL and _rg(seqs=[(0, 64, 0b01), (70, 130, 0b11)]) == INVAL
    sixteen = [_s(2, 4, 0, 0, 2, 0, 0, 4, ids=0x3000 + 0x100 * i, base=0x4000 + 0x100 * i) for i in range(16)]
    assert _rg(srcs=sixteen, seqs=[(0, 64, 1 << 16)], units=(0x7000, 1)) == INVAL
    n = _n(GATHER_SEQS, 24, 64, K.repage_route_anypage_units)
    assert _rg(seqs=[(0, 64, 1), (9, 8, 1)], units=(0x7000, 2)) == INVAL
    assert _rg(units=(0x7000, n + 1)) == INVAL and _rg(units=(0, n)) == INVAL
    arr = (K.StageSource * 2)(*SOURCES)
    assert K.lib().kvbm_kernels_paged_stage_repage_gather_routed_anypage(arr, 2, 24, C.byref(_side(2, 4, 64)), 2, 64, None, 2, 0x7000, n, 0, 4,
                                                                        ROW, 0, None, None, 0, None, 0, None) == INVAL
    small = 600
    big = _bound_pair(small)
    for a, b in ((small, big), (big, small)):
        for x, y, want in ((a, b, 0), (a + (a == big), b + (b == big), INVAL)):
            assert _rg(srcs=[_s(2, 4, 0, 0, 2, 0, 0, 4, page=x)], seqs=[(0, 5, 1)], ps=x, pd=y, units=(0x7000, 1), lb=2, le=2) == want
    assert _rg(lb=3, le=2) == INVAL and _rg(le=5) == INVAL
    assert _rg(srcs=[]) == INVAL and _rg(srcs=[SOURCES[0]] * 17, seqs=[(0, 64, 1)]) == INVAL
    assert _rg(cast=3) == INVAL and _rg(scales=0x5000) == INVAL
    assert _rg(srcs=[_s(2, 4, 0, 0, 2, 0, 0, 2)], seqs=[(0, 64, 1)]) == INVAL       # layers 2..4 uncovered
    # the streamed entry: ready flags only for the routed sources
    assert _rg(streamed=None) == INVAL and _rg(streamed=K.PermuteStream()) == INVAL
    st = K.PermuteStream()
    st.layer_ready_flags[0] = 0x9000
    st.gate_mode = K.GATE_SPIN
    assert _rg(seqs=[(0, 64, 0b01)], streamed=st) == INVAL                           # no workspace for the spinning form
    st.sync_workspace = 0x9100
    assert _rg(seqs=[(0, 64, 0b10)], streamed=st) == INVAL                           # routed source 1 has no flags
    st.gate_mode = 99
    assert _rg(seqs=[(0, 64, 0b01)], streamed=st) == INVAL
    assert _rg(routed=True, units=(0x7000, n)) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# the manager on host memory: the routed entries' codes and texts, and a 24 -> 64 push and pull
# ---------------------------------------------------------------------------------------------------------------------
def _err(fn):
    with pytest.raises(KvbmError) as e:
        fn()
    return e.value


def _pools(mgr, specs):
    bufs, hs = [], []
    for nl, nh, page in specs:
        cfg = LayoutConfig(8, nl, 2, page, nh * 64, dtype_width_bytes=2, num_heads=nh)
        b = np.zeros(cfg.required_bytes(), dtype=np.uint8)
        h = mgr.register_fully_contiguous(cfg, b.ctypes.data, b.size, StorageKind.System, 0)
        mgr.set_kv_block_layout(h, KV.OperationalNHD)
        bufs.append(b)
        hs.append(h)
    return bufs, hs


@pytest.fixture()
def scatter_pools():
    """a: the source, 6 layers, 4 heads, 16-token pages; b, c: 4 layers, 2 heads, 64; d: 2 layers, 2 heads, 64; e: 2 layers, 2 heads,
    32; f: a source like a with 24-token pages."""
    mgr = TransferManager(device=-1, worker_id=21)
    bufs, hs = _pools(mgr, ((6, 4, 16), (4, 2, 64), (4, 2, 64), (2, 2, 64), (2, 2, 32), (6, 4, 24)))
    yield mgr, hs
    mgr.close()


SPLAN = [ScatterWindow(0, 0, 0, 4, 0, 0, 2), ScatterWindow(1, 0, 0, 4, 2, 0, 2), ScatterWindow(2, 4, 0, 2, 0, 0, 2)]


def _sq(tokens=range(0, 64), src=(0, 1, 2, 3), **dst):
    return (tokens, list(src), {int(k[1:]): v for k, v in dst.items()})


SCATTER_CASES = [
    ([_sq(d0=[5]), _sq(range(64, 128), (4, 5, 6, 7))], (1, 2, 3), SPLAN, dict(ready_flags=0)),     # the stream's shape
    ([_sq(d0=[5]), _sq(range(64, 128), (4, 5, 6, 7))], (1, 1, 3), SPLAN, {}),                      # the windows first
    ([_sq(d0=[5]), _sq(range(64, 128), (4, 5, 6, 7))], (1, 2, 3), SPLAN[:2] + [ScatterWindow(3, 4, 0, 2, 0, 0, 2)], {}),
    ([_sq(d0=[5]), _sq(range(64, 128), (4, 5, 6, 7))], (1, 2, 3), SPLAN, {}),                      # routed to no destination
    ([_sq(d0=[5]), _sq(range(70, 64), (), d3=[])], (1, 2, 3, 4), SPLAN, {}),                       # no window writes it
    ([_sq(range(70, 64), (), d0=[]), _sq(d1=[5], d3=[5])], (1, 2, 3), SPLAN, {}),                  # past the destinations
    ([_sq(range(70, 64), (), d0=[]), _sq(src=(0, 1, 2), d0=[5])], (1, 2, 3), SPLAN, {}),           # the token range
    ([_sq(range(9, 9), (), d0=[]), _sq(src=(0, 1, 2), d0=[5])], (1, 2, 3), SPLAN, {}),             # the id counts
    ([_sq(d0=[5]), _sq(src=(0, 1, 2), d0=[5])], (1, 2, 3), SPLAN, {}),                             # the strategy first
    ([_sq(d0=[8])], (1, 2, 3), SPLAN, {}),                                                          # a routed id out of range
    ([_sq(d0=[5], d1=[9]), _sq(range(64, 128), (4, 5, 6, 7), d1=[5], d0=[9])], (1, 2, 3), SPLAN, {}),
    ([_sq(d0=[5]), _sq(range(64, 128), (4, 5, 6, 7), d0=[5])], (1, 2, 3), SPLAN, {}),
    ([_sq(d0=[5])], (1, 2, 4), SPLAN, {}),                                                          # destinations of two pages
]


@pytest.mark.parametrize("case", range(len(SCATTER_CASES)))
def test_manager_scatter_rejections_are_the_routed_scatters(scatter_pools, case):
    mgr, hs = scatter_pools
    seqs, dsts, plan, kw = SCATTER_CASES[case]
    handles = [hs[i] if i < len(hs) else 999 for i in dsts]
    routed = _err(lambda: mgr.execute_repage_scatter_routed(hs[0], handles, seqs, plan, **kw))
    anypage = _err(lambda: mgr.execute_repage_scatter_routed_anypage(hs[0], handles, seqs, plan, **kw))
    assert (anypage.code, anypage.msg) == (routed.code, routed.msg)


def test_manager_scatter_more_than_32_destinations_and_nothing_to_move(scatter_pools):
    mgr, hs = scatter_pools
    many = [hs[1], hs[2], hs[3]] + [10_000 + i for i in range(30)]
    for fn in (mgr.execute_repage_scatter_routed, mgr.execute_repage_scatter_routed_anypage):
        e = _err(lambda: fn(hs[0], many, [_sq(d0=[5])], SPLAN))
        assert e.code == ErrorCode.UNSUPPORTED and "at most 32 destinations" in e.msg
    go = lambda seqs, o=None: mgr.execute_repage_scatter_routed_anypage(hs[0], [hs[1], hs[2], hs[3]], seqs, SPLAN, o)  # noqa: E731
    assert go([]) is not None and go([_sq(range(9, 9), (), d0=[]), _sq(range(70, 70), (), d2=[])]) is not None
    assert go([_sq(d0=[5])], TransferOptions(layer_range=range(4, 4))) is not None


def test_manager_takes_a_24_to_64_routed_push(scatter_pools):
    """f has 24-token pages, the destinations 64: the routed scatter rejects the pair, the new entry gets to the strategy."""
    mgr, hs = scatter_pools
    dsts = [hs[1], hs[2], hs[3]]
    seqs = [(range(10, 70), [0, 1, 2], {0: [5, 6], 2: [5, 6]}), (range(100, 130), [3, 4], {1: [2]})]
    x = _err(lambda: mgr.execute_repage_scatter_routed(hs[5], dsts, seqs, SPLAN))
    assert x.code == ErrorCode.INCOMPATIBLE and "one page size to divide the other" in x.msg
    x = _err(lambda: mgr.execute_repage_scatter_routed_anypage(hs[5], dsts, seqs, SPLAN))
    assert x.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in x.msg
    # the id counts follow each side's own page, for routed destinations
    x = _err(lambda: mgr.execute_repage_scatter_routed_anypage(hs[5], dsts, [(range(10, 70), [0, 1], {0: [5, 6]})], SPLAN))
    assert x.code == ErrorCode.LENGTH_MISMATCH and "span 3 source and 2 destination blocks" in x.msg
    # the anypage scatter (unrouted) takes the pair too, and the other scatter entries keep rejecting it
    x = _err(lambda: mgr.execute_repage_scatter_anypage(hs[5], dsts, [(range(10, 70), [0, 1, 2], [[5, 6]] * 3)], SPLAN))
    assert x.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in x.msg
    x = _err(lambda: mgr.execute_repage_scatter_batch(hs[5], dsts, [(range(10, 70), [0, 1, 2], [[5, 6]] * 3)], SPLAN))
    assert x.code == ErrorCode.INCOMPATIBLE


def test_manager_exactness_bound():
    """The first accepted and the first rejected pair of a 40000-token small page, both directions, push and pull: the anypage
    gather's text."""
    mgr = TransferManager(device=-1, worker_id=22)
    small = 40000
    big = _bound_pair(small)
    try:
        bufs, (s, ok, past) = _pools(mgr, ((1, 1, small), (1, 1, big), (1, 1, big + 1)))
        for src, dst, want in ((s, ok, CUDA_ONLY), (ok, s, CUDA_ONLY), (s, past, "exactness bound"), (past, s, "exactness bound")):
            x = _err(lambda: mgr.execute_repage_scatter_routed_anypage(src, [dst], [(range(0, 10), [0], {0: [1]})],
                                                                       [ScatterWindow(0, 0, 0, 1, 0, 0, 1)]))
            assert x.code == ErrorCode.UNSUPPORTED and want in x.msg
            y = _err(lambda: mgr.execute_repage_batch_routed_anypage({0: src}, dst, [(range(0, 10), {0: [0]}, [1])],
                                                                     [ShardWindow(0, 0, 0, 1, 0, 0, 1)]))
            assert (y.code, y.msg) == (x.code, x.msg)
            z = _err(lambda: mgr.execute_repage_anypage({0: src}, dst, [(range(0, 10), {0: [0]}, [1])], [ShardWindow(0, 0, 0, 1, 0, 0, 1)]))
            assert (z.code, z.msg) == (x.code, x.msg)
    finally:
        mgr.close()


@pytest.fixture()
def gather_pools():
    """a, b, c: sources, 4 layers, 2 heads, 16-token pages; d: the destination, 4 layers, 2 heads, 64; e: like d; f: a source like a
    with 24-token pages."""
    mgr = TransferManager(device=-1, worker_id=23)
    bufs, hs = _pools(mgr, ((4, 2, 16), (4, 2, 16), (4, 2, 16), (4, 2, 64), (4, 2, 64), (4, 2, 24)))
    yield mgr, hs
    mgr.close()


GPLAN = [ShardWindow(0, 0, 0, 4, 0, 0, 2), ShardWindow(1, 0, 0, 4, 0, 0, 2)]
STAGED = [ShardWindow(0, 0, 0, 2, 0, 0, 2), ShardWindow(1, 0, 2, 2, 0, 0, 2)]


def _c_gather(entry, mgr, hs, seqs, plan=GPLAN, num_srcs=2, ls=None, dst=3, null_list=False):
    """A routed gather C entry with explicit masks and NULL lists: seqs are (tb, te, {src: ids}, dst_ids, mask)."""
    keep = []
    cs = (P._CRepageRouteSeq * max(1, len(seqs)))()
    for c, (tb, te, ids, dids, mask) in zip(cs, seqs):
        arrs = {r: (C.c_size_t * max(1, len(x)))(*x) for r, x in ids.items()}
        sp = (C.c_void_p * max(1, num_srcs))(*[C.addressof(arrs[r]) if r in arrs else None for r in range(num_srcs)])
        d = (C.c_size_t * max(1, len(dids)))(*dids)
        keep += [arrs, sp, d]
        n_src = len(next(iter(ids.values()))) if ids else 0
        c.token_begin, c.token_end, c.src_ids, c.n_src, c.dst_ids, c.n_dst, c.src_mask = tb, te, C.addressof(sp), n_src, C.addressof(d), len(dids), mask
    ws = (P._CShardWindow * len(plan))(*[P._CShardWindow(w.src_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin,
                                                          w.dst_head_begin, w.head_count) for w in plan])
    srcs = (C.c_uint64 * max(1, num_srcs))(*[hs[i] if i < 3 else 10_000 + i for i in range(num_srcs)])
    o, tok = TransferOptions()._c(), C.c_uint64()
    rc = entry(mgr._h, num_srcs, srcs, hs[dst], None if null_list else cs, len(seqs), ws, len(plan), ls, C.byref(o), C.byref(tok))
    return rc, P.lib().kvbm_last_error().decode() if rc else ""


S0 = (0, 64, {0: [0, 1, 2, 3]}, [5], 0b01)
S1 = (64, 128, {1: [4, 5, 6, 7]}, [6], 0b10)
ZERO = (64, 128, {}, [6], 0)
GATHER_CASES = [
    ([S0, ZERO], GPLAN + [ShardWindow(2, 0, 0, 4, 0, 0, 2)], 2, {}),
    ([S0], [ShardWindow(0, 0, 0, 4, 0, 0, 2), ShardWindow(1, 0, 1, 3, 0, 0, 2)], 2, {}),
    ([S0, ZERO], GPLAN, 2, dict(null_list=True)),
    ([S0, ZERO], GPLAN, 33, {}),
    ([S0, ZERO], GPLAN, 2, {}),
    ([S0, (64, 128, {}, [6], 0b100)], GPLAN, 2, {}),
    ([S0, (64, 128, {2: [4, 5, 6, 7]}, [6], 0b100)], GPLAN, 3, {}),
    ([S0, (64, 128, {0: [4, 5, 6, 7], 1: [4, 5, 6, 7]}, [6], 0b11)], GPLAN, 2, {}),
    ([(0, 64, {0: [0, 1, 2, 3], 1: [0, 1, 2, 3]}, [5], 0b11), S0], STAGED, 2, {}),
    ([(0, 64, {0: [0, 1, 2]}, [5], 0b01), ZERO], GPLAN, 2, {}),
    ([(0, 64, {0: [0, 1, 2]}, [5], 0b01), S1], GPLAN, 2, {}),
    ([S0, S1], GPLAN, 2, {}),
    ([(0, 64, {0: [0, 1, 2, 9]}, [5], 0b01)], GPLAN, 2, {}),
    ([(0, 64, {0: [0, 1, 2, 3]}, [5], 0b11)], STAGED, 2, {}),
    ([(0, 64, {0: [0, 1, 2, 3]}, [5], 0b10)], GPLAN, 2, {}),
    ([S0, (64, 128, {1: [4, 5, 6, 7]}, [5], 0b10)], GPLAN, 2, {}),                # a destination block named twice
]


@pytest.mark.parametrize("case", range(len(GATHER_CASES)))
def test_manager_gather_rejections_are_the_routed_gathers(gather_pools, case):
    mgr, hs = gather_pools
    seqs, plan, num_srcs, kw = GATHER_CASES[case]
    routed = _c_gather(P.lib().kvbm_manager_execute_repage_batch_routed, mgr, hs, seqs, plan, num_srcs, **kw)
    anypage = _c_gather(P.lib().kvbm_manager_execute_repage_batch_routed_anypage, mgr, hs, seqs, plan, num_srcs, **kw)
    assert routed[0] != 0 and anypage == routed


def test_manager_gather_stream_shape_and_nothing_to_move(gather_pools):
    mgr, hs = gather_pools
    ls = P._CLayerStream(None, 2, None)
    for entry in (P.lib().kvbm_manager_execute_repage_batch_routed, P.lib().kvbm_manager_execute_repage_batch_routed_anypage):
        rc, msg = _c_gather(entry, mgr, hs, [S0, ZERO], ls=C.byref(ls))
        assert rc == ErrorCode.ERR and "ready flags" in msg
    srcs = {0: hs[0], 1: hs[1]}
    assert mgr.execute_repage_batch_routed_anypage(srcs, hs[3], [], GPLAN) is not None
    assert mgr.execute_repage_batch_routed_anypage(srcs, hs[3], [(range(9, 9), {0: []}, []), (range(70, 70), {1: []}, [])], GPLAN) is not None


def test_manager_takes_a_24_to_64_routed_pull(gather_pools):
    """f has 24-token pages, the destination 64: the routed gather rejects the pair, the new entry gets to the strategy."""
    mgr, hs = gather_pools
    plan = [ShardWindow(0, 0, 0, 4, 0, 0, 2), ShardWindow(1, 0, 0, 4, 0, 0, 2)]
    srcs = {0: hs[5], 1: hs[5]}
    seqs = [(range(10, 70), {0: [0, 1, 2]}, [5, 6]), (range(100, 130), {1: [3, 4]}, [2])]
    x = _err(lambda: mgr.execute_repage_batch_routed(srcs, hs[3], seqs, plan))
    assert x.code == ErrorCode.INCOMPATIBLE and "one page size to divide the other" in x.msg
    x = _err(lambda: mgr.execute_repage_batch_routed_anypage(srcs, hs[3], seqs, plan))
    assert x.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in x.msg
    x = _err(lambda: mgr.execute_repage_batch_routed_anypage(srcs, hs[3], [(range(10, 70), {0: [0, 1]}, [5, 6])], plan))
    assert x.code == ErrorCode.LENGTH_MISMATCH


# ---------------------------------------------------------------------------------------------------------------------
# the instantiations in the built library
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s, pp) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True)) for pp in (True, False)}
NEW = ("kvbm_paged_repage_collect_kernel", "kvbm_gated_repage_collect_kernel", "kvbm_paged_repage_deal_kernel", "kvbm_gated_repage_deal_kernel")
TAKEN = ("route", "fanin", "anypage", "phased", "batch", "scatter", "push_seqs", "_stage_", "paged_copy")
FAMILIES = ("kvbm_paged_permute_kernel", "kvbm_paged_gather_kernel", "kvbm_gated_gather_kernel", "kvbm_paged_repage_kernel",
            "kvbm_paged_repage_gather_kernel", "kvbm_gated_repage_gather_kernel", "kvbm_permute_table_kernel", "kvbm_permute_kernel",
            "kvbm_gated_repage_push_kernel", "kvbm_paged_repage_scatter_kernel")


def test_the_collect_and_deal_instantiations_are_what_the_library_contains():
    """80 kernels: the 20 walks of with_repage_kernel for each of the four families; tests/test_gpu_route_anypage.py reaches each.
    No new name contains a substring other tests filter the library's kernels by, nor equals a family they count."""
    so = os.path.join(ROOT, "dynamo_b200", "libkvbm_kernels.so")
    tool = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
    if not os.path.exists(so) or tool is None:
        pytest.skip("needs the built libkvbm_kernels.so and cuobjdump")
    txt = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    found = set()
    for name in re.findall(r"Function : (\S+)", txt):
        m = re.search(r"(kvbm_[a-z0-9_]+?_kernel)I((?:L[ib]\d+E)+)E", name)
        if m and ("collect" in m.group(1) or "deal" in m.group(1)):
            assert m.group(1) in NEW
            c, p, s, pp = (int(v) if t == "i" else v == "1" for t, v in re.findall(r"L([ib])(\d+)E", m.group(2)))
            found.add((m.group(1), c, p, s, pp))
    assert len(WALKS) == 20 and found == {(k,) + w for k in NEW for w in WALKS}
    assert not any(s in k for k in NEW for s in TAKEN)
    assert not set(NEW) & set(FAMILIES)

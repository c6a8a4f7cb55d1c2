"""CPU checks of the re-paging scatter between pages that need not divide (kvbm_kernels_paged_repage_scatter_anypage and
TransferManager.execute_repage_scatter_anypage): the exported symbols, the unit table the push takes, the kernel entries' argument
checks that return before any CUDA call, the manager's rejections on a host-only manager against the batch scatter's, a 24 -> 64
push only the new entry takes, and the 40 instantiations in the built library.  The GPU cases are in
tests/test_gpu_scatter_anypage.py."""
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
from dynamo_b200.physical import ErrorCode, LayoutConfig, ScatterWindow, StorageKind, TransferManager, TransferOptions
from tests.test_repage_anypage_host import anypage_units
from tests.test_repage_scatter_host import OK, PLAN, ROW, _side, _t
from tests.test_scatter_batch_seqs_host import CUDA_ONLY, EMPTY, GOOD, REJECTED, _err

KV = K.KvBlockLayout
INVAL = K.CUDA_ERROR_INVALID_VALUE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_anypage_scatter_symbols_are_exported_and_listed():
    for name in ("kvbm_kernels_paged_repage_scatter_anypage", "kvbm_kernels_paged_repage_scatter_anypage_streamed"):
        assert name in K.EXPORTED_SYMBOLS and callable(getattr(K.lib(), name))
    assert "kvbm_manager_execute_repage_scatter_anypage" in P.EXPORTED_SYMBOLS
    assert callable(P.lib().kvbm_manager_execute_repage_scatter_anypage)


@pytest.mark.parametrize("ps,pd", [(544, 64), (48, 64), (24, 16), (3, 5), (5, 3)], ids=str)
def test_the_push_takes_the_anypage_table(ps, pd):
    """The table one anypage scatter launch reads for every target, against its definition: each big block's small_k and phase put
    every token of a prefill batch in the small block and slot that hold its position."""
    seqs = [(7, 7), (1, 3 * max(ps, pd) + 2), (max(ps, pd) - 1, max(ps, pd)), (40, 1000)]
    got = K.repage_anypage_units(seqs, ps, pd)
    want = anypage_units(seqs, ps, pd)
    assert np.array_equal(got[0], want[0]) and got[1:] == want[1:]
    assert (got[0][:, 3] % math.gcd(ps, pd) == 0).all() and (got[0][:, 3] < min(ps, pd)).all()


# ---------------------------------------------------------------------------------------------------------------------
# the kernel entries' argument checks (descriptors no check dereferences)
# ---------------------------------------------------------------------------------------------------------------------
SEQS = [(0, 64), (70, 130), (9, 9)]


def _units(seqs, ps=24, pd=64):
    u = K.repage_anypage_units(seqs, ps, pd)
    return (0x7000, len(u[0])) if u is not None else (0x7000, 0)


def _as(targets=OK, seqs=SEQS, src_nh=4, src_nl=6, ps=24, pd=64, lb=0, le=6, cast=0, scales=None, src=None, units=None, streamed=False):
    addr, n = units if units is not None else _units(seqs, ps, pd)
    s = src or _side(src_nh, src_nl, ps)
    if streamed is not False:
        return K.paged_repage_scatter_anypage_streamed(s, src_nh, ps, targets, pd, seqs, addr, n, lb, le, ROW, cast, scales, streamed)
    return K.paged_repage_scatter_anypage(s, src_nh, ps, targets, pd, seqs, addr, n, lb, le, ROW, cast, scales)


def _bound_pair(small):
    """The largest big page the exactness bound takes with `small`."""
    big = (1 << 32) // small
    while (big + small - math.gcd(big, small)) * small >= (1 << 32):
        big -= 1
    return big


def test_anypage_scatter_argument_checks_before_any_cuda_call():
    # nothing to move signals (nothing to signal here): no sequences, only empty ranges, an empty layer range
    assert _as(seqs=[]) == 0 and _as(seqs=[(9, 9), (70, 70)]) == 0 and _as(lb=3, le=3) == 0
    # the batch's own rules: a reversed range, a unit count other than the helper's, a null unit table, a null seqs
    assert _as(seqs=[(0, 64), (9, 8)], units=(0x7000, 2)) == INVAL
    n = _units(SEQS)[1]
    assert _as(units=(0x7000, n + 1)) == INVAL and _as(units=(0x7000, n - 1)) == INVAL
    assert _as(units=(0, n)) == INVAL
    arr = (K.ScatterTarget * 3)(*OK)
    assert K.lib().kvbm_kernels_paged_repage_scatter_anypage(C.byref(_side(4, 6, 24)), 4, 24, arr, 3, 64, None, 2, 0x7000, n, 0, 6, ROW, 0,
                                                            None, 0, None, 0, None) == INVAL
    # a range whose last big block ends at 2^32 tokens, next to its accepted neighbour
    top = (1 << 32) - 64
    assert K.repage_anypage_units([(top - 64, top)], 24, 64) is not None and K.repage_anypage_units([(top, top + 1)], 24, 64) is None
    assert _as(seqs=[(0, 64), (top, top + 1)], units=(0x7000, 2)) == INVAL
    # pages just past the exactness bound, in both directions; the pair just inside it passes the page check (an empty layer range
    # then moves nothing and returns before any CUDA call), the one past it does not
    small = 600
    big = _bound_pair(small)
    for a, b in ((small, big), (big, small)):
        for x, y, want in ((a, b, 0), (a + (a == big), b + (b == big), INVAL)):
            tg = [_t(2, 4, 0, 0, 2, 0, 0, 4, page=y)]
            assert _as(targets=tg, seqs=[(0, 5)], ps=x, pd=y, src=_side(4, 6, x), units=(0x7000, 1), lb=2, le=2) == want
    assert _as(ps=0, src=_side(4, 6, 24), units=(0x7000, 3)) == INVAL
    # the single scatter's rules
    assert _as(lb=4, le=3) == INVAL
    assert _as(targets=[]) == INVAL and _as(targets=[OK[0]] * 17) == INVAL           # 0 or 17 targets
    assert _as(cast=3) == INVAL
    assert _as(scales=0x5000) == INVAL                                               # scales without a cast
    assert _as(src=_side(4, 6, 32)) == INVAL                                         # a source region other than Ps * heads * row
    assert _as(le=7) == INVAL
    assert _as(targets=OK[:2] + [_t(2, 2, 0, 0, 2, 4, 0, 2, page=48)]) == INVAL      # a target region other than Pd * heads * row
    assert _as(targets=OK[:2] + [_t(2, 2, 0, 0, 0, 4, 0, 2)]) == INVAL               # an empty head window
    assert _as(targets=OK[:2] + [_t(2, 2, 0, 0, 2, 5, 0, 2)]) == INVAL               # past the source's 6 layers
    assert _as(targets=OK[:2] + [_t(2, 2, 0, 0, 2, 3, 0, 2)]) == INVAL               # partly overlapping stages
    assert _as(targets=OK[:2]) == INVAL                                              # source layers 4..6 uncovered
    assert _as(targets=[OK[0], _t(2, 4, 2, 1, 1, 0, 0, 4, ids=0x2100), OK[1], OK[2]]) == INVAL
    # the streamed entry: a null stream descriptor, a descriptor without ready flags, an unknown gate mode
    assert _as(streamed=None) == INVAL and _as(streamed=K.PermuteStream()) == INVAL
    st = K.PermuteStream()
    st.layer_ready_flags[0] = 0x3000
    st.gate_mode = 7
    assert _as(streamed=st) == INVAL
    st.gate_mode = K.GATE_SPIN
    assert _as(streamed=st) == INVAL                                                 # the spinning form without a workspace
    # the existing scatter entries keep rejecting the same pages
    addr, n = _units(SEQS)
    assert K.paged_repage_scatter_batch(_side(4, 6, 24), 4, 24, OK, 64, SEQS, addr, n, 0, 6, ROW) == INVAL
    assert K.paged_repage_scatter(_side(4, 6, 24), 4, 24, OK, 64, 0, 64, 0, 6, ROW) == INVAL


def test_the_unit_bound_is_rejected_at_2_pow_31():
    """num_units * layers * outer_dim of 2^31: 2^29 big blocks (8192 sequences of 2^22 tokens, 24 -> 64-token pages) over 2 layers
    and 2 outer indices."""
    seqs = [(0, 64 * 65536)] * 8192
    n, a, b = C.c_size_t(), C.c_size_t(), C.c_size_t()
    arr = K._repage_seqs(seqs)
    assert K.lib().kvbm_kernels_repage_anypage_units(C.cast(arr, C.c_void_p), len(seqs), 24, 64, None, 0, C.byref(n), C.byref(a),
                                                     C.byref(b)) == 0
    assert n.value == 1 << 29
    tg = [K.ScatterTarget(_side(4, 2, 64, ids=0x2100), 4, 0, 0, 4, 0, 0, 2, None)]
    assert K.paged_repage_scatter_anypage(_side(4, 2, 24), 4, 24, tg, 64, seqs, 0x7000, n.value, 0, 2, ROW) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_repage_scatter_anypage on host memory
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def host_pools():
    """tests/test_scatter_batch_seqs_host.py's pools (a: the source, 6 layers, 4 heads, 16-token pages; b, c: 4 layers, 2 heads,
    64; d: 2 layers, 2 heads, 64; e: 2 layers, 2 heads, 32) and f: a source like a with 24-token pages."""
    mgr = TransferManager(device=-1, worker_id=16)
    no, hd = 2, 64
    bufs, hs = [], []
    for nl, nh, page in ((6, 4, 16), (4, 2, 64), (4, 2, 64), (2, 2, 64), (2, 2, 32), (6, 4, 24)):
        cfg = LayoutConfig(8, nl, no, page, nh * hd, dtype_width_bytes=2, num_heads=nh)
        b = np.zeros(cfg.required_bytes(), dtype=np.uint8)
        h = mgr.register_fully_contiguous(cfg, b.ctypes.data, b.size, StorageKind.System, 0)
        mgr.set_kv_block_layout(h, KV.OperationalNHD)
        bufs.append(b)
        hs.append(h)
    yield mgr, hs
    mgr.close()


def _both(mgr, hs, plan, seqs, o=None, dsts=(1, 2, 3), src=0, **kw):
    """(code, text) of execute_repage_scatter_batch and execute_repage_scatter_anypage on the same arguments."""
    handles = [hs[i] if i < len(hs) else 999 for i in dsts]
    out = []
    for fn in (mgr.execute_repage_scatter_batch, mgr.execute_repage_scatter_anypage):
        x = _err(lambda: fn(hs[src], handles, seqs, plan, o, **kw))
        out.append((x.code, x.msg))
    return out


@pytest.mark.parametrize("case", range(len(REJECTED)))
def test_manager_rejections_are_the_batch_scatters(host_pools, case):
    """With dividing pages every rejection of the batch scatter, its code and text, alone and behind an empty sequence."""
    mgr, hs = host_pools
    seq, o, dsts, plan, code, text = REJECTED[case]
    for seqs in ([seq], [EMPTY, seq]):
        batch, anypage = _both(mgr, hs, plan, seqs, o, dsts)
        assert anypage == batch and batch[0] == code and text in batch[1]


def test_manager_rejection_order_is_the_batch_scatters(host_pools):
    mgr, hs = host_pools
    cases = [([(range(70, 64), [0], [[5], [5], [5]])], None, (1, 2, 3), {}),                        # the range before the id counts
             ([(range(0, 64), [0, 1, 2], [[5], [8], [5]])], None, (1, 2, 3), {}),                   # the id counts before the ids
             ([EMPTY, (range(0, 64), [0, 1, 2], [[5], [5], [5]]), (range(70, 64), [], [[], [], []])], None, (1, 2, 3), {}),
             ([GOOD, (range(0, 64), [0, 1, 2], [[5], [5], [5]])], None, (1, 2, 3), {}),             # the strategy first
             ([], None, (1, 1, 3), {}),                                                             # the windows, without sequences
             ([], None, (1, 2, 3), dict(ready_flags=0)),                                            # the layer stream's shape
             ([(range(0, 128), list(range(8)), [[5, 6], [5, 7], [5, 6]]), (range(200, 264), [0, 1, 2, 3], [[6], [1], [2]])], None,
              (1, 2, 3), {})]                                                                       # a block named twice
    seen = set()
    for seqs, o, dsts, kw in cases:
        batch, anypage = _both(mgr, hs, PLAN, seqs, o, dsts, **kw)
        assert anypage == batch
        seen.add(batch[0])
    assert {ErrorCode.RANGE, ErrorCode.LENGTH_MISMATCH, ErrorCode.UNSUPPORTED, ErrorCode.OVERLAP, ErrorCode.ERR} <= seen
    e = _err(lambda: mgr.execute_repage_scatter_anypage(hs[0], [hs[1], hs[2], hs[3]], [], []))
    assert e.code == ErrorCode.ERR and "at least one destination" in e.msg
    # nothing to move: no sequences, only empty ones, an empty layer range
    go = lambda seqs, o=None: mgr.execute_repage_scatter_anypage(hs[0], [hs[1], hs[2], hs[3]], seqs, PLAN, o)  # noqa: E731
    assert go([]) is not None and go([EMPTY, EMPTY]) is not None
    assert go([GOOD], TransferOptions(layer_range=range(4, 4))) is not None


def test_manager_takes_a_24_to_64_push(host_pools):
    """f has 24-token pages, the destinations 64: the batch scatter rejects the pair, the anypage scatter gets to the strategy."""
    mgr, hs = host_pools
    dsts = [hs[1], hs[2], hs[3]]
    seqs = [(range(10, 70), [0, 1, 2], [[5, 6], [5, 6], [5, 6]]), (range(100, 130), [3, 4], [[2], [2], [2]])]
    x = _err(lambda: mgr.execute_repage_scatter_batch(hs[5], dsts, seqs, PLAN))
    assert x.code == ErrorCode.INCOMPATIBLE and "one page size to divide the other" in x.msg
    x = _err(lambda: mgr.execute_repage_scatter_anypage(hs[5], dsts, seqs, PLAN))
    assert x.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in x.msg
    # the id counts follow each side's own page
    x = _err(lambda: mgr.execute_repage_scatter_anypage(hs[5], dsts, [(range(10, 70), [0, 1], [[5, 6], [5, 6], [5, 6]])], PLAN))
    assert x.code == ErrorCode.LENGTH_MISMATCH and "span 3 source and 2 destination blocks" in x.msg
    # destinations of two page sizes stay rejected, after the pair checks
    x = _err(lambda: mgr.execute_repage_scatter_anypage(hs[5], [hs[1], hs[2], hs[4]], seqs, PLAN))
    assert x.code == ErrorCode.INCOMPATIBLE and "one page size" in x.msg
    # every other scatter entry keeps rejecting the pair
    x = _err(lambda: mgr.execute_repage_scatter(hs[5], [0, 1, 2], dsts, [[5, 6], [5, 6], [5, 6]], PLAN, range(10, 70)))
    assert x.code == ErrorCode.INCOMPATIBLE and "one page size to divide the other" in x.msg
    x = _err(lambda: mgr.execute_repage_scatter_routed(hs[5], dsts, [(range(10, 70), [0, 1, 2], {0: [5, 6], 1: [5, 6], 2: [5, 6]})], PLAN))
    assert x.code == ErrorCode.INCOMPATIBLE and "one page size to divide the other" in x.msg


def test_manager_exactness_bound():
    """The first accepted and the first rejected pair of a 40000-token small page, in both directions."""
    mgr = TransferManager(device=-1, worker_id=18)
    small = 40000
    big = _bound_pair(small)
    bufs = []

    def pool(page):
        cfg = LayoutConfig(2, 1, 1, page, 8, dtype_width_bytes=2, num_heads=1)
        buf = np.zeros(cfg.required_bytes(), dtype=np.uint8)
        h = mgr.register_fully_contiguous(cfg, buf.ctypes.data, buf.size, StorageKind.System, 0)
        mgr.set_kv_block_layout(h, KV.OperationalNHD)
        bufs.append(buf)
        return h

    try:
        s, ok, past = pool(small), pool(big), pool(big + 1)
        plan = [ScatterWindow(0, 0, 0, 1, 0, 0, 1)]
        for src, dst in ((s, ok), (ok, s)):
            x = _err(lambda: mgr.execute_repage_scatter_anypage(src, [dst], [(range(0, 10), [0], [[1]])], plan))
            assert x.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in x.msg
        for src, dst in ((s, past), (past, s)):
            x = _err(lambda: mgr.execute_repage_scatter_anypage(src, [dst], [(range(0, 10), [0], [[1]])], plan))
            assert x.code == ErrorCode.UNSUPPORTED and "exactness bound" in x.msg
            # the anypage gather's text for the same pair
            y = _err(lambda: mgr.execute_repage_anypage({0: src}, dst, [(range(0, 10), {0: [0]}, [1])],
                                                        [P.ShardWindow(0, 0, 0, 1, 0, 0, 1)]))
            assert (y.code, y.msg) == (x.code, x.msg)
    finally:
        mgr.close()


# ---------------------------------------------------------------------------------------------------------------------
# the instantiations in the built library
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s, pp) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True)) for pp in (True, False)}
NEW = ("kvbm_paged_repage_phased_push_kernel", "kvbm_gated_repage_phased_push_kernel")
TAKEN = ("scatter", "batch", "push_seqs", "route", "fanin", "anypage", "_stage_")
FAMILIES = ("kvbm_paged_permute_kernel", "kvbm_paged_gather_kernel", "kvbm_gated_gather_kernel", "kvbm_paged_repage_kernel",
            "kvbm_paged_repage_gather_kernel", "kvbm_gated_repage_gather_kernel", "kvbm_permute_table_kernel", "kvbm_permute_kernel",
            "kvbm_gated_repage_push_kernel", "kvbm_paged_repage_scatter_kernel")


def test_the_phased_push_instantiations_are_what_the_library_contains():
    """40 kernels: the 20 walks of with_repage_kernel for each of the two families; tests/test_gpu_scatter_anypage.py reaches each.
    No new name contains a substring other tests filter the library's kernels by, nor equals a family they count."""
    so = os.path.join(ROOT, "dynamo_b200", "libkvbm_kernels.so")
    tool = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
    if not os.path.exists(so) or tool is None:
        pytest.skip("needs the built libkvbm_kernels.so and cuobjdump")
    txt = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    found = set()
    for name in re.findall(r"Function : (\S+)", txt):
        m = re.search(r"(kvbm_[a-z0-9_]+?_kernel)I((?:L[ib]\d+E)+)E", name)
        if m and "phased" in m.group(1):
            assert m.group(1) in NEW
            c, p, s, pp = (int(v) if t == "i" else v == "1" for t, v in re.findall(r"L([ib])(\d+)E", m.group(2)))
            found.add((m.group(1), c, p, s, pp))
    assert len(WALKS) == 20 and found == {(k,) + w for k in NEW for w in WALKS}
    assert not any(s in k for k in NEW for s in TAKEN)
    assert not set(NEW) & set(FAMILIES)

"""CPU checks of re-paging between pages that need not divide (kvbm_kernels_paged_stage_repage_gather_anypage and
TransferManager.execute_repage_anypage): the exported symbols and the C layout of kvbm_repage_anypage_unit, the unit table of
kvbm_kernels_repage_anypage_units against a restatement from its definition, the exactness bound at its edge, the kernel entries'
argument checks that return before any CUDA call, the manager's rejections on a host-only manager against the batch entry's, and
the 40 instantiations in the built library.  The GPU cases are in tests/test_gpu_repage_anypage.py."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, ShardWindow, TransferOptions
from tests.repage_batch_oracle import repage_batch_units
from tests.test_stage_repage_host import CUDA_ONLY, PLAN, ROW, _err, _side, _ss, host_pools  # noqa: F401  (host_pools is a fixture)

INVAL = K.CUDA_ERROR_INVALID_VALUE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_anypage_symbols_are_exported_and_listed():
    for name in ("kvbm_kernels_repage_anypage_units", "kvbm_kernels_paged_stage_repage_gather_anypage",
                 "kvbm_kernels_paged_stage_repage_gather_anypage_streamed"):
        assert name in K.EXPORTED_SYMBOLS and callable(getattr(K.lib(), name))
    assert "kvbm_manager_execute_repage_anypage" in P.EXPORTED_SYMBOLS and callable(P.lib().kvbm_manager_execute_repage_anypage)


def test_the_anypage_unit_mirror_matches_the_c_struct():
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("needs a C compiler")
    names = ["q0", "tokens", "small_k", "phase"]
    assert [f[0] for f in K.RepageAnypageUnit._fields_] == names
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "kvbm_kernels.h"', "int main(void) {"]
    lines += [f'  printf("%zu\\n", offsetof(kvbm_repage_anypage_unit, {f}));' for f in names]
    lines += ['  printf("%zu\\n", sizeof(kvbm_repage_anypage_unit));', "  return 0;", "}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "s.c"), os.path.join(d, "s")
        with open(src, "w") as f:
            f.write("\n".join(lines))
        subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", "-o", exe, src], check=True)
        got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert got[:-1] == [getattr(K.RepageAnypageUnit, f).offset for f in names] == [0, 4, 8, 12]
    assert got[-1] == C.sizeof(K.RepageAnypageUnit) == 16


# ---------------------------------------------------------------------------------------------------------------------
# the unit table
# ---------------------------------------------------------------------------------------------------------------------
def anypage_units(seqs, ps, pd):
    """The table from its definition: per non-empty sequence, one record per block j of the larger page it touches; F = j * big is
    the position of the block's slot 0, small_k the concatenated small table's entry of the small block holding F (mod 2^32), and
    the phase F's slot in that block."""
    big, small = max(ps, pd), min(ps, pd)
    rows, small_off, n_big = [], 0, 0
    for tb, te in seqs:
        if tb == te:
            continue
        for j in range(tb // big, -(-te // big)):
            F = j * big
            lo, hi = max(tb, F), min(te, F + big)
            rows.append([lo - F, hi - lo, (small_off + F // small - tb // small) % (1 << 32), F % small])
            n_big += 1
        small_off += -(-te // small) - tb // small
    units = np.array(rows, dtype=np.uint32).reshape(-1, 4)
    return units, (small_off if ps < pd else n_big), (n_big if ps < pd else small_off)


def _random_batch(rng, big, small):
    seqs = []
    for _ in range(int(rng.integers(1, 30))):
        kind = int(rng.integers(0, 6))
        tb = int(rng.integers(0, 5 * big + 7))
        te = tb if kind == 0 else tb + (1 if kind == 1 else int(rng.integers(1, 3 * big + 9)))   # empty, one token, or longer
        if kind == 2:
            tb -= tb % big                 # starts on a big block
        if kind == 3:
            te += -te % small              # ends on a small block
        seqs.append((tb, max(tb, te)))
    return seqs


NAMED = [(24, 16), (16, 24), (48, 64), (64, 48), (544, 64), (64, 544), (3, 5), (5, 3), (1, 7), (7, 1), (16, 16), (600, 599), (16, 64), (64, 16)]


def _pairs():
    rng = np.random.default_rng(7)
    return NAMED + [(int(a), int(b)) for a, b in rng.integers(1, 601, size=(20, 2))]


@pytest.mark.parametrize("ps,pd", _pairs(), ids=lambda p: str(p))
def test_unit_table_against_its_definition(ps, pd):
    rng = np.random.default_rng(1000 * ps + pd)
    big, small = max(ps, pd), min(ps, pd)
    for _ in range(12):
        seqs = _random_batch(rng, big, small)
        got = K.repage_anypage_units(seqs, ps, pd)
        want = anypage_units(seqs, ps, pd)
        assert got is not None
        assert np.array_equal(got[0], want[0]) and got[1:] == want[1:]
        assert (got[0][:, 3] % math.gcd(ps, pd) == 0).all() and (got[0][:, 3] < small).all()
        # every token of the range lands in the small block and slot that hold its position
        off = 0
        units = iter(got[0].tolist())
        for tb, te in seqs:
            if tb == te:
                continue
            for j in range(tb // big, -(-te // big)):
                q0, tokens, small_k, phase = next(units)
                for q in (q0, q0 + tokens - 1):
                    p = j * big + q
                    assert (small_k + (phase + q) // small) % (1 << 32) == off + p // small - tb // small
                    assert (phase + q) % small == p % small
            off += -(-te // small) - tb // small
        if big % small == 0:            # dividing pages: the batch helper's records with phase 0 in place of seq
            batch = K.repage_batch_units(seqs, ps, pd)
            assert batch[1:] == got[1:] and np.array_equal(batch[0][:, :3], got[0][:, :3]) and not got[0][:, 3].any()
            assert np.array_equal(repage_batch_units(seqs, ps, pd)[0][:, :3], got[0][:, :3])


def test_unit_table_of_24_and_16_token_pages():
    """Tokens 30..100 from 16-token pages into 24-token pages: big blocks 1..4 start at positions 24, 48, 72 and 96, in small blocks 1,
    3, 4 and 6 at slots 8, 0, 8 and 0; the range starts in small block 1, so small_k counts from there."""
    units, n_src, n_dst = K.repage_anypage_units([(30, 100)], 16, 24)
    assert units.tolist() == [[6, 18, 0, 8], [0, 24, 2, 0], [0, 24, 3, 8], [0, 4, 5, 0]]
    assert (n_src, n_dst) == (7 - 1, 5 - 1)
    same = K.repage_anypage_units([(30, 100)], 24, 16)
    assert np.array_equal(same[0], units) and same[1:] == (n_dst, n_src)


def _accepts(big, small):
    return K.repage_anypage_units([], big, small) is not None


def _bound(big, small):
    return (big + small - math.gcd(big, small)) * small < (1 << 32)


def test_the_exactness_bound_at_its_edge():
    for small in (3, 7, 600, 40000, 65535):
        big = (1 << 32) // small        # the largest big page the bound can take is below this
        while not _bound(big, small):
            big -= 1
        assert _accepts(big, small) and _accepts(small, big)                     # the first accepted pair, both directions
        assert not _accepts(big + 1, small) and not _accepts(small, big + 1)     # the first rejected one
        for b in range(big - 50, big + 50):
            assert _accepts(b, small) == _bound(b, small)
    # dividing pages: the bound is the batch helper's big * small < 2^32, so both accept and reject the same pairs
    for small, big in ((16, (1 << 28) - 16), (16, 1 << 28), (255, 255 * 66050), (255, 255 * 66051), (1 << 15, 1 << 17)):
        assert _accepts(big, small) == (K.repage_batch_units([], big, small) is not None) == (big * small < (1 << 32))
    assert not _accepts(1 << 16, 1 << 16) and not _accepts((1 << 16) + 1, 1 << 16)    # a small page of 2^16 fails, gcd or not
    assert not _accepts(0, 16) and not _accepts(16, 0)


def test_unit_table_rejections_and_sizing():
    assert K.repage_anypage_units([(5, 3)], 24, 16) is None                # reversed
    assert K.repage_anypage_units([(0, (1 << 32) - 3)], 16, 24) is None    # the last big block ends at 2^32
    last = (1 << 32) // 24 * 24                                            # the last block of 24 that ends below 2^32
    assert K.repage_anypage_units([(last - 30, last)], 16, 24) is not None
    assert K.repage_anypage_units([(last - 30, last + 1)], 16, 24) is None
    units, ns, nd = K.repage_anypage_units([], 24, 16)
    assert len(units) == 0 and (ns, nd) == (0, 0)
    # a capacity below the count writes that many records and still reports the counts
    seqs = (K.RepageSeq * 2)(K.RepageSeq(3, 200), K.RepageSeq(70, 300))
    out = (K.RepageAnypageUnit * 2)()
    n, a, b = C.c_size_t(), C.c_size_t(), C.c_size_t()
    assert K.lib().kvbm_kernels_repage_anypage_units(C.cast(seqs, C.c_void_p), 2, 48, 64, C.cast(out, C.c_void_p), 2, C.byref(n), C.byref(a),
                                                     C.byref(b)) == 0
    full = K.repage_anypage_units([(3, 200), (70, 300)], 48, 64)
    assert (n.value, a.value, b.value) == (len(full[0]),) + full[1:] and n.value > 2
    assert [[u.q0, u.tokens, u.small_k, u.phase] for u in out] == full[0][:2].tolist()
    assert K.lib().kvbm_kernels_repage_anypage_units(None, 1, 48, 64, None, 0, C.byref(n), C.byref(a), C.byref(b)) != 0


# ---------------------------------------------------------------------------------------------------------------------
# the kernel entries' argument checks (descriptors no check dereferences)
# ---------------------------------------------------------------------------------------------------------------------
OK = [_ss(2, 4, 0, 0, 2, 0, 0, 4, page=24), _ss(2, 4, 0, 2, 2, 0, 0, 4, page=24), _ss(2, 4, 0, 0, 2, 0, 4, 4, page=24),
      _ss(2, 4, 0, 2, 2, 0, 4, 4, page=24)]
SEQS = [(5, 100), (64, 70), (9, 9)]


def _any(srcs=OK, seqs=SEQS, units=0x5000, num_units=None, ps=24, pd=64, dst_nh=4, dst_nl=8, lb=0, le=8, cast=0, scales=None, st=False):
    if num_units is None:
        t = K.repage_anypage_units(seqs, ps, pd)
        num_units = len(t[0]) if t else 0
    args = (srcs, ps, _side(dst_nh, dst_nl, pd), dst_nh, pd, seqs, units, num_units, lb, le, ROW, cast, scales)
    if st is not False:
        return K.paged_stage_repage_gather_anypage_streamed(*args, st)
    return K.paged_stage_repage_gather_anypage(*args)


def test_anypage_argument_checks_before_any_cuda_call():
    # nothing to move signals (nothing to signal here): no sequences, only empty ranges, an empty layer range
    assert _any(seqs=[]) == 0 and _any(seqs=[(9, 9), (0, 0)]) == 0 and _any(lb=3, le=3) == 0
    assert _any(seqs=[(5, 100), (9, 8)]) == INVAL                           # a reversed range, also behind a good one
    assert _any(num_units=1) == INVAL and _any(num_units=5) == INVAL        # not the helper's count
    assert _any(units=0) == INVAL                                           # units to read and no table
    assert _any(seqs=[(0, (1 << 32) - 3)]) == INVAL                         # a last big block that ends at 2^32
    assert _any(ps=0) == INVAL
    # pages past the exactness bound: the first rejected pair of a 600-token small page
    big = (1 << 32) // 600
    while not _bound(big, 600):
        big -= 1
    assert _any(ps=600, pd=big + 1, srcs=[_ss(2, 4, 0, 0, 2, 0, 0, 4, page=600)], num_units=1, seqs=[(0, 5)]) == INVAL
    # the batch's rules, each on an otherwise well-formed batch
    assert _any(srcs=[]) == INVAL and _any(srcs=[OK[0]] * 17) == INVAL
    assert _any(srcs=OK[:2]) == INVAL                                       # layers 4..8 in no window
    assert _any(srcs=[OK[0], _ss(2, 4, 0, 1, 2, 0, 0, 4, page=24), OK[2], OK[3]]) == INVAL    # head overlap within a stage
    assert _any(srcs=OK[:3] + [_ss(2, 4, 0, 2, 2, 0, 4, 4, page=32)]) == INVAL                # a region that is not page * heads * row
    assert _any(le=9) == INVAL and _any(lb=3, le=2) == INVAL
    assert _any(cast=3) == INVAL and _any(scales=0x6000) == INVAL           # an unknown cast; scales without a cast
    # 2^31 units: 2^27 big blocks of 1 <- 3-token pages over 8 layers and 2 outer indices
    one = [_ss(2, 4, 0, 0, 2, 0, 0, 4, page=1), _ss(2, 4, 0, 2, 2, 0, 0, 4, page=1), _ss(2, 4, 0, 0, 2, 0, 4, 4, page=1),
           _ss(2, 4, 0, 2, 2, 0, 4, 4, page=1)]
    assert _any(ps=1, pd=3, seqs=[(0, 3 << 27)], srcs=one, num_units=1 << 27) == INVAL
    # the streamed entry: the gate's rules first
    assert _any(st=None) == INVAL
    st = K.PermuteStream()
    for j in range(4):
        st.layer_ready_flags[j] = 0x3000 + 64 * j
    st.gate_mode = 7
    assert _any(st=st) == INVAL
    st.gate_mode = K.GATE_SPIN
    assert _any(st=st) == INVAL                                             # the spinning form without a workspace
    st.sync_workspace = 0x4000
    st.layer_ready_flags[3] = 0
    assert _any(st=st) == INVAL
    # the existing entries keep rejecting the same pages
    u = K.repage_anypage_units(SEQS, 24, 64)
    assert K.paged_stage_repage_gather_batch(OK, 24, _side(4, 8, 64), 4, 64, SEQS, 0x5000, len(u[0]), 0, 8, ROW) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_repage_anypage on host memory
# ---------------------------------------------------------------------------------------------------------------------
def _seq(tokens=range(0, 64), n_src=4, dst_ids=(5,), first=0):
    return tokens, {r: list(range(first + r, first + r + n_src)) for r in range(3)}, list(dst_ids)


def _both(mgr, hs, plan, seqs, o=None, third=2, **kw):
    """(code, text) of execute_repage_batch and execute_repage_anypage on the same arguments."""
    a, b, c, d, e, f = hs
    srcs = {0: a, 1: b, 2: (a, b, c, d, e, f)[third]}
    out = []
    for fn in (mgr.execute_repage_batch, mgr.execute_repage_anypage):
        x = _err(lambda: fn(srcs, d, seqs, plan, o, **kw))
        out.append((x.code, x.msg))
    return out


def test_manager_rejections_are_the_batch_entrys(host_pools):  # noqa: F811
    """With dividing pages every rejection, its code, text and order, is the batch entry's."""
    mgr, hs = host_pools
    two = [_seq(dst_ids=(5,)), _seq(tokens=range(40, 70), n_src=3, dst_ids=(2, 3))]
    empty = _seq(tokens=range(9, 9), n_src=0, dst_ids=())
    cases = [(PLAN, two, None, {}), (PLAN, two, TransferOptions(layer_range=range(2, 6)), {}),
             ([PLAN[0], ShardWindow(1, 0, 0, 3, 0, 1, 2)] + PLAN[2:], two, None, {}), (PLAN[:2], two, None, {}),
             ([ShardWindow(0, 0, 0, 3, 1, 0, 2)] + PLAN[1:], two, None, {}), (PLAN, two, TransferOptions(layer_range=range(0, 9)), {}),
             (PLAN, two, TransferOptions(head_window=(0, 0, 1)), {}), (PLAN, two, None, dict(third=4)),
             (PLAN, two, None, dict(ready_flags={0: 0, 1: 0, 2: 0}))]
    cases += [(PLAN, [empty, bad, _seq(tokens=range(3, 2))], None, {}) for bad in (
        _seq(tokens=range(70, 64)), _seq(n_src=3), (range(0, 64), {r: [7, 8, 1, 2] for r in range(3)}, [5]), _seq(dst_ids=(8,)),
        _seq(tokens=range(0, 128), n_src=8, dst_ids=(5, 5)))]
    seen = set()
    for plan, seqs, o, kw in cases:
        batch, anypage = _both(mgr, hs, plan, seqs, o, **kw)
        assert anypage == batch
        seen.add(batch[0])
    assert {ErrorCode.UNSUPPORTED, ErrorCode.OVERLAP, ErrorCode.RANGE, ErrorCode.LENGTH_MISMATCH, ErrorCode.DUPLICATE_DST} <= seen


def test_manager_takes_pages_that_do_not_divide(host_pools):  # noqa: F811
    """f has 24-token pages, the destination d 64: the batch entry rejects the pair, the anypage entry gets to the strategy."""
    mgr, hs = host_pools
    a, b, c, d, e, f = hs
    plan = [ShardWindow(0, 0, 0, 5, 0, 0, 2), ShardWindow(0, 0, 0, 5, 0, 2, 2)]
    o = TransferOptions(layer_range=range(0, 5))
    seqs = [(range(10, 70), {0: [0, 1, 2]}, [5, 6]), (range(100, 130), {0: [3, 4]}, [2, 3])]   # 24-token blocks 0..2 and 4..5
    x = _err(lambda: mgr.execute_repage_batch({0: f}, d, seqs, plan, o))
    assert x.code == ErrorCode.INCOMPATIBLE and "one page size to divide the other" in x.msg
    x = _err(lambda: mgr.execute_repage_anypage({0: f}, d, seqs, plan, o))
    assert x.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in x.msg
    # the id counts follow each side's own page
    x = _err(lambda: mgr.execute_repage_anypage({0: f}, d, [(range(10, 70), {0: [0, 1]}, [5, 6])], plan, o))
    assert x.code == ErrorCode.LENGTH_MISMATCH and "span 3 source and 2 destination blocks" in x.msg
    # sources of two page sizes stay rejected, after the pair checks
    x = _err(lambda: mgr.execute_repage_anypage({0: a, 1: b, 2: f}, d, [_seq()], PLAN))
    assert x.code == ErrorCode.INCOMPATIBLE and "need one page size" in x.msg
    # nothing to move
    assert mgr.execute_repage_anypage({0: f}, d, [], plan, o) is not None


def test_manager_exactness_bound(host_pools):  # noqa: F811
    """The first accepted and the first rejected pair of a 40000-token small page, registered as host pools."""
    mgr, _ = host_pools
    small = 40000
    big = (1 << 32) // small
    while not _bound(big, small):
        big -= 1
    bufs = []

    def pool(page):
        cfg = P.LayoutConfig(2, 1, 1, page, 8, dtype_width_bytes=2, num_heads=1)
        buf = np.zeros(cfg.required_bytes(), dtype=np.uint8)
        h = mgr.register_fully_contiguous(cfg, buf.ctypes.data, buf.size, P.StorageKind.System, 0)
        mgr.set_kv_block_layout(h, K.KvBlockLayout.OperationalNHD)
        bufs.append(buf)
        return h

    s, ok, past = pool(small), pool(big), pool(big + 1)
    plan = [ShardWindow(0, 0, 0, 1, 0, 0, 1)]
    for src, dst in ((s, ok), (ok, s)):
        x = _err(lambda: mgr.execute_repage_anypage({0: src}, dst, [(range(0, 10), {0: [0]}, [1])], plan))
        assert x.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in x.msg
    for src, dst in ((s, past), (past, s)):
        x = _err(lambda: mgr.execute_repage_anypage({0: src}, dst, [(range(0, 10), {0: [0]}, [1])], plan))
        assert x.code == ErrorCode.UNSUPPORTED and "exactness bound" in x.msg


# ---------------------------------------------------------------------------------------------------------------------
# the instantiations in the built library
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s, pp) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True)) for pp in (True, False)}
NEW = ("kvbm_paged_repage_anypage_kernel", "kvbm_gated_repage_anypage_kernel")
TAKEN = ("batch", "route", "scatter", "push_seqs", "_stage_", "fanin")
MATRIX_FAMILIES = ("kvbm_paged_permute_kernel", "kvbm_paged_gather_kernel", "kvbm_gated_gather_kernel", "kvbm_paged_repage_kernel",
                   "kvbm_paged_repage_gather_kernel", "kvbm_gated_repage_gather_kernel", "kvbm_permute_table_kernel", "kvbm_permute_kernel")


def test_the_anypage_instantiations_are_what_the_library_contains():
    """40 kernels: the 20 walks of with_repage_kernel for each of the two families; tests/test_gpu_repage_anypage.py reaches each.
    No new name contains a substring other tests filter the library's kernels by, nor equals a family they count."""
    so = os.path.join(ROOT, "dynamo_b200", "libkvbm_kernels.so")
    tool = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
    if not os.path.exists(so) or tool is None:
        pytest.skip("needs the built libkvbm_kernels.so and cuobjdump")
    txt = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    found = set()
    for name in re.findall(r"Function : (\S+)", txt):
        m = re.search(r"(kvbm_[a-z0-9_]+?_kernel)I((?:L[ib]\d+E)+)E", name)
        if m and "anypage" in m.group(1):
            assert m.group(1) in NEW
            c, p, s, pp = (int(v) if t == "i" else v == "1" for t, v in re.findall(r"L([ib])(\d+)E", m.group(2)))
            found.add((m.group(1), c, p, s, pp))
    assert len(WALKS) == 20 and found == {(k,) + w for k in NEW for w in WALKS}
    assert not any(s in k for k in NEW for s in TAKEN)
    assert not set(NEW) & set(MATRIX_FAMILIES)

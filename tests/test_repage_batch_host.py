"""CPU checks of a batch of sequences in one re-paging launch: the exported symbols and the ctypes mirrors' sizes, the unit table
of kvbm_kernels_repage_batch_units against a numpy restatement over randomised batches, the batch entries' argument checks that
return before any CUDA call, the new instantiations in the built library, and kvbm_manager_execute_repage_batch's rejections on a
host-only manager against what the single entry returns for the same sequence."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, HeadWindow, KvbmError, ShardWindow, TransferOptions
from tests.repage_batch_oracle import repage_batch_units
from tests.test_stage_repage_host import PLAN, ROW, _err, _side, _ss, host_pools  # noqa: F401  (host_pools is a fixture)

INVAL = K.CUDA_ERROR_INVALID_VALUE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAGES = [1, 16, 48, 64, 256]


def test_batch_symbols_and_mirrors():
    for name in ("kvbm_kernels_repage_batch_units", "kvbm_kernels_paged_stage_repage_gather_batch",
                 "kvbm_kernels_paged_stage_repage_gather_batch_streamed"):
        assert name in K.EXPORTED_SYMBOLS and callable(getattr(K.lib(), name))
    assert "kvbm_manager_execute_repage_batch" in P.EXPORTED_SYMBOLS and callable(P.lib().kvbm_manager_execute_repage_batch)
    assert C.sizeof(K.RepageUnit) == 16 and C.sizeof(K.RepageSeq) == 8
    assert C.sizeof(P._CRepageBatchSeq) == 6 * C.sizeof(C.c_size_t)


# ---------------------------------------------------------------------------------------------------------------------
# the unit table
# ---------------------------------------------------------------------------------------------------------------------
def _random_batch(rng, big):
    seqs = []
    for _ in range(int(rng.integers(1, 40))):
        kind = rng.integers(0, 5)
        tb = int(rng.integers(0, 6 * big + 7))
        te = tb if kind == 0 else tb + int(rng.integers(1, 4 * big + 9))      # kind 0: an empty sequence
        if kind == 1:
            tb -= tb % big                                                      # starts on a block boundary
        if kind == 2:
            te += -te % big                                                     # ends on one
        seqs.append((tb, max(te, tb)))
    return seqs


@pytest.mark.parametrize("ps,pd", [(a, b) for a in PAGES for b in PAGES if max(a, b) % min(a, b) == 0])
def test_unit_table_against_numpy(ps, pd):
    rng = np.random.default_rng(1000 * ps + pd)
    for _ in range(25):
        seqs = _random_batch(rng, max(ps, pd))
        got = K.repage_batch_units(seqs, ps, pd)
        want = repage_batch_units(seqs, ps, pd)
        assert got is not None
        assert np.array_equal(got[0], want[0]) and got[1:] == want[1:]
        # the table lengths are the single entries' id counts, summed
        blocks = lambda p: sum(0 if b == e else -(-e // p) - b // p for b, e in seqs)  # noqa: E731
        assert got[1:] == (blocks(ps), blocks(pd))


def test_unit_table_of_a_range_whose_first_small_blocks_precede_it():
    """Tokens 40..70 with 16 <-> 64-token pages: big block 0 starts at small block 0, the range at small block 2, so the first
    sequence's small_k is -2 in uint32; the second sequence's counts on from the first's 3 small blocks."""
    units, n_src, n_dst = K.repage_batch_units([(40, 70), (100, 130)], 16, 64)
    assert units.tolist() == [[40, 24, (1 << 32) - 2, 0], [0, 6, 2, 0], [36, 28, 3 + 4 - 6, 1], [0, 2, 3 + 8 - 6, 1]]
    assert (n_src, n_dst) == (3 + 3, 2 + 2)
    # every token's small block, as the kernel indexes it: (small_k + q // small) mod 2^32 lands inside the sequence's run
    for (q0, tokens, small_k, seq), lo in zip(units.tolist(), (0, 0, 3, 3)):
        for q in (q0, q0 + tokens - 1):
            assert lo <= (small_k + q // 16) % (1 << 32) < lo + 3
    same = K.repage_batch_units([(40, 70), (100, 130)], 64, 16)           # the other direction: the same table, the counts swapped
    assert np.array_equal(same[0], units) and same[1:] == (n_dst, n_src)


def test_unit_table_rejections_and_sizing():
    assert K.repage_batch_units([(5, 3)], 16, 64) is None                  # reversed
    assert K.repage_batch_units([(0, 4)], 0, 16) is None and K.repage_batch_units([(0, 4)], 16, 0) is None
    assert K.repage_batch_units([(0, 4)], 48, 64) is None                  # neither divides the other
    assert K.repage_batch_units([(0, 4)], 1 << 16, 1 << 16) is None        # big_page * small_page reaches 2^32
    assert K.repage_batch_units([(0, (1 << 32) - 3)], 16, 64) is None      # the last big block ends at 2^32
    assert K.repage_batch_units([((1 << 32) - 3, (1 << 32) - 3)], 16, 64)[1:] == (0, 0)   # an empty sequence has no block to end
    units, ns, nd = K.repage_batch_units([], 16, 64)
    assert len(units) == 0 and (ns, nd) == (0, 0)
    # a capacity below the count writes that many records and still reports the counts
    seqs = (K.RepageSeq * 2)(K.RepageSeq(3, 200), K.RepageSeq(70, 300))
    out = (K.RepageUnit * 2)()
    n, a, b = C.c_size_t(), C.c_size_t(), C.c_size_t()
    assert K.lib().kvbm_kernels_repage_batch_units(C.cast(seqs, C.c_void_p), 2, 16, 64, C.cast(out, C.c_void_p), 2, C.byref(n), C.byref(a),
                                                   C.byref(b)) == 0
    full = K.repage_batch_units([(3, 200), (70, 300)], 16, 64)
    assert (n.value, a.value, b.value) == (len(full[0]),) + full[1:] and n.value > 2
    assert [[u.q0, u.tokens, u.small_k, u.seq] for u in out] == full[0][:2].tolist()


# ---------------------------------------------------------------------------------------------------------------------
# the batch entries' argument checks (descriptors no check dereferences)
# ---------------------------------------------------------------------------------------------------------------------
OK = [_ss(2, 4, 0, 0, 2, 0, 0, 4), _ss(2, 4, 0, 2, 2, 0, 0, 4), _ss(2, 4, 0, 0, 2, 0, 4, 4), _ss(2, 4, 0, 2, 2, 0, 4, 4)]
SEQS = [(5, 100), (64, 70), (9, 9)]


def _batch(srcs=OK, seqs=SEQS, units=0x5000, num_units=None, ps=16, pd=64, dst_nh=4, dst_nl=8, lb=0, le=8, cast=0, scales=None):
    if num_units is None:
        t = K.repage_batch_units(seqs, ps, pd)
        num_units = len(t[0]) if t else 0
    return K.paged_stage_repage_gather_batch(srcs, ps, _side(dst_nh, dst_nl, pd), dst_nh, pd, seqs, units, num_units, lb, le, ROW, cast, scales)


def test_batch_argument_checks_before_any_cuda_call():
    # nothing to move signals (nothing to signal here): no sequences, only empty ranges, an empty layer range
    assert _batch(seqs=[]) == 0 and _batch(seqs=[(9, 9), (0, 0)]) == 0 and _batch(lb=3, le=3) == 0
    assert _batch(seqs=[(5, 100), (9, 8)]) == INVAL                         # a reversed range, also behind a good one
    assert _batch(lb=3, le=3, seqs=[(9, 8)]) == INVAL                       # ... and with nothing else to move
    assert _batch(num_units=1) == INVAL and _batch(num_units=4) == INVAL    # not the helper's count (3)
    assert _batch(units=0) == INVAL                                         # units to read and no table
    assert _batch(seqs=[(0, (1 << 32) - 3)]) == INVAL                       # a last big block that ends at 2^32
    assert _batch(ps=24, srcs=[_ss(2, 4, 0, 0, 2, 0, 0, 4, page=24)] * 1) == INVAL   # pages where neither divides the other
    assert _batch(ps=0) == INVAL
    # 2^31 units: 2^25 big blocks of one-token pages over 8 layers and 2 outer indices x 4
    assert _batch(ps=1, pd=1, seqs=[(0, 1 << 27)], srcs=[_ss(2, 4, 0, 0, 2, 0, 0, 4, page=1), _ss(2, 4, 0, 2, 2, 0, 0, 4, page=1),
                                                         _ss(2, 4, 0, 0, 2, 0, 4, 4, page=1), _ss(2, 4, 0, 2, 2, 0, 4, 4, page=1)]) == INVAL
    # the single entry's rules, each on an otherwise well-formed batch
    assert _batch(srcs=[]) == INVAL and _batch(srcs=[OK[0]] * 17) == INVAL
    assert _batch(srcs=OK[:2]) == INVAL                                     # layers 4..8 in no window
    assert _batch(srcs=[OK[0], _ss(2, 4, 0, 1, 2, 0, 0, 4), OK[2], OK[3]]) == INVAL    # head overlap within a stage
    assert _batch(srcs=OK[:3] + [_ss(2, 4, 0, 2, 2, 0, 4, 4, page=32)]) == INVAL        # a region that is not page * heads * row
    assert _batch(le=9) == INVAL
    assert _batch(cast=3) == INVAL and _batch(scales=0x6000) == INVAL       # an unknown cast; scales without a cast
    # the streamed entry: the gate's rules first
    units = K.repage_batch_units(SEQS, 16, 64)[0]
    stream = lambda st: K.paged_stage_repage_gather_batch_streamed(OK, 16, _side(4, 8, 64), 4, 64, SEQS, 0x5000, len(units), 0, 8, ROW, 0,  # noqa: E731
                                                                   None, st)
    assert stream(None) == INVAL
    st = K.PermuteStream()
    for j in range(4):
        st.layer_ready_flags[j] = 0x3000 + 64 * j
    st.gate_mode = 7
    assert stream(st) == INVAL
    st.gate_mode = K.GATE_SPIN
    assert stream(st) == INVAL                                              # the spinning form without a workspace
    st.sync_workspace = 0x4000
    st.layer_ready_flags[3] = 0
    assert stream(st) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# the instantiations the library contains
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True))}
BATCH_FAMILIES = ("kvbm_paged_batch_repage_gather_kernel", "kvbm_gated_batch_repage_gather_kernel")
EXPECTED = {(f, w + (pp,)) for f in BATCH_FAMILIES for w in WALKS for pp in (True, False)}


def test_the_batch_instantiations_are_what_the_library_contains():
    """40 kernels: both families over <cast, row pow2, scaled, small page pow2>; tests/test_gpu_repage_batch.py reaches each."""
    assert len(EXPECTED) == 40
    so = os.path.join(ROOT, "dynamo_b200", "libkvbm_kernels.so")
    tool = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
    if not os.path.exists(so) or tool is None:
        pytest.skip("needs the built libkvbm_kernels.so and cuobjdump")
    txt = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    found = set()
    for name in re.findall(r"Function : (\S+)", txt):
        m = re.search(r"(kvbm_[a-z0-9_]+?_kernel)I((?:L[ib]\d+E)+)E", name)
        if m and "batch" in m.group(1):
            found.add((m.group(1), tuple(int(v) if t == "i" else v == "1" for t, v in re.findall(r"L([ib])(\d+)E", m.group(2)))))
    assert found == EXPECTED


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_repage_batch on host memory: the single entry's codes and texts, sequence by sequence
# ---------------------------------------------------------------------------------------------------------------------
def _seq(tokens=range(0, 64), n_src=4, dst_ids=(5,), first=0):
    return tokens, {r: list(range(first + r, first + r + n_src)) for r in range(3)}, list(dst_ids)


def _single(mgr, hs, plan, seq, o=None, third=2, **kw):
    a, b, c, d, e, f = hs
    tokens, src, dst_ids = seq
    return mgr.execute_stage_repage_gather({0: (a, src[0]), 1: (b, src[1]), 2: ((a, b, c, d, e, f)[third], src[2])}, d, dst_ids, plan, tokens,
                                           o, **kw)


def _many(mgr, hs, plan, seqs, o=None, third=2, **kw):
    a, b, c, d, e, f = hs
    return mgr.execute_repage_batch({0: a, 1: b, 2: (a, b, c, d, e, f)[third]}, d, seqs, plan, o, **kw)


GOOD = _seq()
BAD = {
    "a reversed range": _seq(tokens=range(70, 64)),
    "id counts": _seq(n_src=3),
    "a source id out of range": _seq(first=6),
    "a destination id out of range": _seq(dst_ids=(8,)),
    "a duplicate destination id": _seq(tokens=range(0, 128), n_src=8, dst_ids=(5, 5)),
}


@pytest.mark.parametrize("what", list(BAD))
@pytest.mark.parametrize("at", [0, 2])
def test_manager_batch_first_rejected_sequence(host_pools, what, at):  # noqa: F811
    """The first rejected sequence returns what the single call returns for it, wherever it sits, also behind an empty sequence."""
    mgr, hs = host_pools
    bad = BAD[what]
    if what == "a source id out of range":
        bad = (bad[0], {r: [7, 8, 1, 2] for r in range(3)}, bad[2])
    want = _err(lambda: _single(mgr, hs, PLAN, bad))
    # on host memory a well-formed sequence that moves bytes is itself rejected (at the strategy), so only empty ones come first
    seqs = [_seq(tokens=range(9, 9), n_src=0, dst_ids=())] * at + [bad, _seq(tokens=range(3, 2))]
    got = _err(lambda: _many(mgr, hs, PLAN, seqs))
    assert (got.code, got.msg) == (want.code, want.msg)
    assert want.code in (ErrorCode.RANGE, ErrorCode.LENGTH_MISMATCH, ErrorCode.DUPLICATE_DST)


def test_manager_batch_rejections(host_pools):  # noqa: F811
    mgr, hs = host_pools
    many = lambda *a, **kw: _many(mgr, hs, *a, **kw)  # noqa: E731
    single = lambda *a, **kw: _single(mgr, hs, *a, **kw)  # noqa: E731
    two = [_seq(dst_ids=(5,)), _seq(tokens=range(40, 70), n_src=3, dst_ids=(2, 3))]
    # a well-formed batch passes every check down to the strategy, as the single entry on host memory
    for o in (None, TransferOptions(layer_range=range(2, 6))):
        e, w = _err(lambda: many(PLAN, two, o)), _err(lambda: single(PLAN, two[0], o))
        assert (e.code, e.msg) == (w.code, w.msg) and e.code == ErrorCode.UNSUPPORTED and "direct CUDA strategy only" in e.msg
    # the plan's and the options' rejections are the single entry's, with or without sequences
    for plan, o, kw in (([PLAN[0], ShardWindow(1, 0, 0, 3, 0, 1, 2)] + PLAN[2:], None, {}),
                        (PLAN[:2], None, {}),
                        ([ShardWindow(0, 0, 0, 3, 1, 0, 2)] + PLAN[1:], None, {}),
                        (PLAN, TransferOptions(layer_range=range(0, 9)), {}),
                        (PLAN, TransferOptions(head_window=(0, 0, 1)), {}),
                        (PLAN, None, dict(third=4)),
                        (PLAN, None, dict(third=5)),
                        (PLAN, None, dict(ready_flags={0: 0, 1: 0, 2: 0}))):
        e, w = _err(lambda: many(plan, two, o, **kw)), _err(lambda: single(plan, two[0], o, **kw))
        assert (e.code, e.msg) == (w.code, w.msg)
    e = _err(lambda: many([PLAN[0], ShardWindow(1, 0, 0, 3, 0, 1, 2)] + PLAN[2:], []))
    assert e.code == ErrorCode.OVERLAP                                       # the windows are checked without sequences too
    # nothing to move: no sequences, only empty ranges, an empty layer range
    assert many(PLAN, []) is not None
    assert many(PLAN, [_seq(tokens=range(9, 9), n_src=0, dst_ids=())] * 2) is not None
    assert many(PLAN, two, TransferOptions(layer_range=range(4, 4))) is not None
    # (a destination block named by two sequences passes each sequence's checks and needs a device to get past the strategy:
    # tests/test_gpu_repage_batch.py)
    # a HeadWindow plan is the PP1 plan over the destination's layers, and needs their count
    with pytest.raises(ValueError):
        many([HeadWindow(0, 0, 0, 2)], two)
    e = _err(lambda: many([HeadWindow(0, 0, 0, 2), HeadWindow(1, 0, 2, 2)], two, num_layers=8))   # a and b hold 3 layers, not 8
    assert e.code == ErrorCode.RANGE and "source's num_layers" in e.msg
    with pytest.raises(ValueError):
        many(PLAN, [(range(0, 64, 2),) + two[0][1:]])
    with pytest.raises(KvbmError):
        many(PLAN, [(two[0][0], {0: [0, 1, 2, 3], 1: [1, 2, 3], 2: [2, 3, 4, 5]}, [5])])

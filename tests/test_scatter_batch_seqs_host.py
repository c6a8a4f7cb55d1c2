"""CPU checks of the batch re-paging scatter (a prefill batch's sequences pushed to every decode rank in one launch): the exported
symbols and the ctypes mirror of kvbm_scatter_batch_seq, the oracle against n single-scatter oracles, the kernel entries' argument
checks that return before any CUDA call, the manager's rejections on a host-only manager with the first rejection pinned, and the
40 instantiations in the built library.  The GPU cases are in tests/test_gpu_scatter_seqs.py."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, KvbmError, LayoutConfig, ScatterWindow, StorageKind, TransferManager, TransferOptions
from tests.cast_oracle import CAST_NONE
from tests.scatter_batch_oracle import repage_scatter_batch, table_len
from tests.scatter_oracle import repage_scatter
from tests.test_repage_scatter_host import OK, PLAN, ROW, _side, _t

KV = K.KvBlockLayout
INVAL = K.CUDA_ERROR_INVALID_VALUE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_batch_scatter_symbols_are_exported_and_listed():
    for name in ("kvbm_kernels_paged_repage_scatter_batch", "kvbm_kernels_paged_repage_scatter_batch_streamed"):
        assert name in K.EXPORTED_SYMBOLS and callable(getattr(K.lib(), name))
    assert "kvbm_manager_execute_repage_scatter_batch" in P.EXPORTED_SYMBOLS
    assert callable(P.lib().kvbm_manager_execute_repage_scatter_batch)


def test_the_batch_seq_mirror_matches_the_c_struct():
    """kvbm_scatter_batch_seq: two size_t, a pointer, a size_t, a pointer, a size_t, as the C compiler lays it out."""
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("needs a C compiler")
    fields = [f[0] for f in P._CScatterBatchSeq._fields_]
    assert fields == ["token_begin", "token_end", "src_ids", "n_src", "dst_ids", "n_dst"]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "kvbm_physical.h"', "int main(void) {"]
    lines += [f'  printf("%zu\\n", offsetof(kvbm_scatter_batch_seq, {f}));' for f in fields]
    lines += ['  printf("%zu\\n", sizeof(kvbm_scatter_batch_seq));', "  return 0;", "}"]
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "s.c"), os.path.join(d, "s")
        with open(src, "w") as f:
            f.write("\n".join(lines))
        subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", "-o", exe, src], check=True)
        got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert got[:-1] == [getattr(P._CScatterBatchSeq, f).offset for f in fields]
    assert got[-1] == C.sizeof(P._CScatterBatchSeq) == 6 * C.sizeof(C.c_size_t)


# ---------------------------------------------------------------------------------------------------------------------
# the oracle: n single-scatter oracles over the slices of the concatenated tables
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ps,pd", [(4, 8), (8, 4), (4, 4), (1, 4)])
def test_the_batch_oracle_is_n_single_oracles(ps, pd):
    rng = np.random.default_rng(ps * 10 + pd)
    nl, no, nh, hd = 2, 1, 2, 16
    seqs = [(3, 17), (9, 9), (0, 5), (6, 30)]
    ns = sum(table_len(tb, te, ps) for tb, te in seqs)
    nd = sum(table_len(tb, te, pd) for tb, te in seqs)
    s_block, d_block = nl * no * ps * nh * hd, nl * no * pd * nh * hd
    src = rng.integers(0, 256, (ns // 2 + 2, s_block), dtype=np.uint8)
    sids = rng.integers(0, len(src), ns)                       # sequences share source blocks
    pools = [rng.integers(0, 256, (nd + 3, d_block), dtype=np.uint8) for _ in range(2)]
    dids = [rng.permutation(nd + 3)[:nd] for _ in pools]
    windows = [(0, 0, 2, 0, 0, 1), (0, 0, 2, 1, 1, 1)]
    targets = [(p, dids[p], int(KV.OperationalNHD), nh, nl, windows[p]) for p in range(2)]
    got = [p.copy() for p in pools]
    repage_scatter_batch((src, sids, int(KV.OperationalHND), nh, nl), targets, got, no, ps, pd, hd, seqs)
    want = [p.copy() for p in pools]
    so = do = 0
    for tb, te in seqs:
        a, b = table_len(tb, te, ps), table_len(tb, te, pd)
        if a:
            repage_scatter(([src[x] for x in sids[so:so + a]], int(KV.OperationalHND), nh, nl),
                           [(p, dids[p][do:do + b], int(KV.OperationalNHD), nh, nl, windows[p]) for p in range(2)], want, no, ps, pd, hd, tb, te,
                           CAST_NONE)
        so, do = so + a, do + b
    assert all(np.array_equal(g, w) for g, w in zip(got, want))
    assert not all(np.array_equal(g, p) for g, p in zip(got, pools))


# ---------------------------------------------------------------------------------------------------------------------
# the kernel entries' argument checks (descriptors no check dereferences)
# ---------------------------------------------------------------------------------------------------------------------
SEQS = [(0, 64), (70, 130)]


def _units(seqs, ps=16, pd=64):
    u = K.repage_batch_units(seqs, ps, pd)
    return (0x7000, len(u[0])) if u is not None else (0x7000, 0)


def _bs(targets, seqs=SEQS, src_nh=4, src_nl=6, ps=16, pd=64, lb=0, le=6, cast=0, scales=None, src=None, units=None, streamed=None):
    addr, n = units if units is not None else _units(seqs, ps, pd)
    s = src or _side(src_nh, src_nl, ps)
    if streamed is not None:
        return K.paged_repage_scatter_batch_streamed(s, src_nh, ps, targets, pd, seqs, addr, n, lb, le, ROW, cast, scales, streamed)
    return K.paged_repage_scatter_batch(s, src_nh, ps, targets, pd, seqs, addr, n, lb, le, ROW, cast, scales)


def test_batch_argument_checks_before_any_cuda_call():
    # nothing to move signals (nothing to signal here): no sequences, only empty ranges, an empty layer range
    assert _bs(OK, seqs=[]) == 0 and _bs(OK, seqs=[(9, 9), (70, 70)]) == 0 and _bs(OK, lb=3, le=3) == 0
    # the batch's own rules: a reversed range, a unit count other than the helper's, a null unit table, a null seqs
    assert _bs(OK, seqs=[(0, 64), (9, 8)], units=(0x7000, 2)) == INVAL
    assert _bs(OK, units=(0x7000, 4)) == INVAL and _bs(OK, units=(0x7000, 2)) == INVAL
    assert _bs(OK, units=(0, 3)) == INVAL
    arr = (K.ScatterTarget * 3)(*OK)
    assert K.lib().kvbm_kernels_paged_repage_scatter_batch(C.byref(_side(4, 6, 16)), 4, 16, arr, 3, 64, None, 2, 0x7000, 3, 0, 6, ROW, 0, None,
                                                          0, None, 0, None) == INVAL
    # a range whose last big block ends at 2^32 tokens, next to its accepted neighbour's unit count
    top = (1 << 32) - 64
    assert K.repage_batch_units([(top - 64, top)], 16, 64) is not None and K.repage_batch_units([(top, top + 1)], 16, 64) is None
    assert _bs(OK, seqs=[(0, 64), (top, top + 1)], units=(0x7000, 2)) == INVAL
    # the single scatter's rules
    assert _bs(OK, lb=4, le=3) == INVAL
    assert _bs([]) == INVAL and _bs([OK[0]] * 17) == INVAL
    assert _bs(OK, cast=3) == INVAL
    assert _bs(OK, scales=0x5000) == INVAL                                          # scales without a cast
    assert _bs([_t(2, 4, 0, 0, 2, 0, 0, 4, page=24), _t(2, 4, 2, 0, 2, 0, 0, 4, page=24, ids=9), _t(2, 2, 0, 0, 2, 4, 0, 2, page=24)],
               pd=24, units=(0x7000, 9)) == INVAL                                    # pages where neither divides the other
    assert _bs(OK, ps=0, src=_side(4, 6, 16), units=(0x7000, 3)) == INVAL
    assert _bs(OK, src=_side(4, 6, 32)) == INVAL                                    # a source region other than Ps * heads * row
    assert _bs(OK, le=7) == INVAL
    assert _bs(OK[:2] + [_t(2, 2, 0, 0, 2, 4, 0, 2, page=32)]) == INVAL
    assert _bs(OK[:2] + [_t(2, 2, 0, 0, 0, 4, 0, 2)]) == INVAL                      # an empty head window
    assert _bs(OK[:2] + [_t(2, 2, 0, 0, 2, 5, 0, 2)]) == INVAL                      # past the source's 6 layers
    assert _bs(OK[:2] + [_t(2, 2, 0, 0, 2, 3, 0, 2)]) == INVAL                      # partly overlapping stages
    assert _bs(OK[:2]) == INVAL                                                     # source layers 4..6 uncovered
    assert _bs([OK[0], _t(2, 4, 2, 1, 1, 0, 0, 4, ids=0x2100), OK[1], OK[2]]) == INVAL
    # the streamed entry: a null stream descriptor, a descriptor without ready flags
    assert K.paged_repage_scatter_batch_streamed(_side(4, 6, 16), 4, 16, OK, 64, SEQS, *_units(SEQS), 0, 6, ROW, 0, None, None) == INVAL
    assert _bs(OK, streamed=K.PermuteStream()) == INVAL


def test_the_unit_bound_is_rejected_at_2_pow_31():
    """num_units * layers * outer_dim of 2^31: 2^29 big blocks (8192 sequences of 2^22 tokens) over 2 layers and 2 outer indices."""
    seqs = [(0, 64 * 65536)] * 8192
    n, a, b = C.c_size_t(), C.c_size_t(), C.c_size_t()
    arr = K._repage_seqs(seqs)
    assert K.lib().kvbm_kernels_repage_batch_units(C.cast(arr, C.c_void_p), len(seqs), 16, 64, None, 0, C.byref(n), C.byref(a),
                                                   C.byref(b)) == 0
    assert n.value == 1 << 29
    tg = [K.ScatterTarget(_side(4, 2, 64, ids=0x2100), 4, 0, 0, 4, 0, 0, 2, None)]
    assert K.paged_repage_scatter_batch(_side(4, 2, 16), 4, 16, tg, 64, seqs, 0x7000, n.value, 0, 2, ROW) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_repage_scatter_batch on host memory: its rejections, with codes and texts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def host_pools():
    """a: the source, 6 layers, 4 heads, 16-token pages; b, c: 4 layers, 2 heads, 64; d: 2 layers, 2 heads, 64; e: 2 layers,
    2 heads, 32-token pages."""
    mgr = TransferManager(device=-1, worker_id=15)
    no, hd = 2, 64
    bufs, hs = [], []
    for nl, nh, page in ((6, 4, 16), (4, 2, 64), (4, 2, 64), (2, 2, 64), (2, 2, 32)):
        cfg = LayoutConfig(8, nl, no, page, nh * hd, dtype_width_bytes=2, num_heads=nh)
        b = np.zeros(cfg.required_bytes(), dtype=np.uint8)
        h = mgr.register_fully_contiguous(cfg, b.ctypes.data, b.size, StorageKind.System, 0)
        mgr.set_kv_block_layout(h, KV.OperationalNHD)
        bufs.append(b)
        hs.append(h)
    yield mgr, hs
    mgr.close()


def _err(fn):
    with pytest.raises(KvbmError) as e:
        fn()
    return e.value


CUDA_ONLY = "direct CUDA strategy only"
EMPTY = (range(9, 9), [], [[], [], []])
GOOD = (range(0, 64), [0, 1, 2, 3], [[5], [5], [5]])


def _single(mgr, hs, plan, seq, o=None, dsts=(1, 2, 3)):
    tokens, s, d = seq
    return mgr.execute_repage_scatter(hs[0], s, [hs[i] if i < len(hs) else 999 for i in dsts], d, plan, tokens, o)


def _batch(mgr, hs, plan, seqs, o=None, dsts=(1, 2, 3), **kw):
    return mgr.execute_repage_scatter_batch(hs[0], [hs[i] if i < len(hs) else 999 for i in dsts], seqs, plan, o, **kw)


# (sequence, options, destinations) that the single scatter rejects, each with the code and a piece of its text
REJECTED = [
    (GOOD, None, (1, 2, 3), PLAN[:2] + [ScatterWindow(3, 4, 0, 2, 0, 0, 2)], ErrorCode.RANGE, "names destination 3"),
    (GOOD, None, (1, 2, 9), PLAN, ErrorCode.HANDLE, "destination handle"),
    (GOOD, None, (1, 2, 3), PLAN[:2], ErrorCode.RANGE, "source layer 4"),
    (GOOD, None, (1, 2, 4), PLAN, ErrorCode.INCOMPATIBLE, "one page size"),
    (GOOD, TransferOptions(layer_done_flags=0x100), (1, 2, 3), PLAN, ErrorCode.UNSUPPORTED, "layer streaming"),
    ((range(70, 64), [], [[], [], []]), None, (1, 2, 3), PLAN, ErrorCode.RANGE, "Token range"),
    (GOOD, TransferOptions(layer_range=range(0, 7)), (1, 2, 3), PLAN, ErrorCode.RANGE, "exceeds num_layers 6"),
    ((range(0, 64), [0, 1, 2], [[5], [5], [5]]), None, (1, 2, 3), PLAN, ErrorCode.LENGTH_MISMATCH, "span 4 source and 1 destination"),
    ((range(0, 128), list(range(8)), [[5, 6], [5, 5], [5, 6]]), None, (1, 2, 3), PLAN, ErrorCode.DUPLICATE_DST, ""),
    ((range(0, 64), [0, 1, 2, 3], [[5], [8], [5]]), None, (1, 2, 3), PLAN, ErrorCode.RANGE, "out of range for destination"),
    (GOOD, None, (1, 2, 3), PLAN, ErrorCode.UNSUPPORTED, CUDA_ONLY),
]


@pytest.mark.parametrize("case", range(len(REJECTED)))
def test_a_batch_rejects_what_the_single_call_rejects(host_pools, case):
    """Each rejection of the single scatter, as the batch's only sequence and as its second after an empty one: the same code and
    text."""
    mgr, hs = host_pools
    seq, o, dsts, plan, code, text = REJECTED[case]
    single = _err(lambda: _single(mgr, hs, plan, seq, o, dsts))
    assert single.code == code and text in single.msg
    for seqs in ([seq], [EMPTY, seq]):
        e = _err(lambda: _batch(mgr, hs, plan, seqs, o, dsts))
        assert (e.code, e.msg) == (single.code, single.msg)


def test_the_first_rejected_sequence_wins(host_pools):
    mgr, hs = host_pools
    go = lambda seqs, **kw: _batch(mgr, hs, PLAN, seqs, **kw)  # noqa: E731
    # a sequence that fails two checks reports the earlier one: the token range before the id counts
    e = _err(lambda: go([(range(70, 64), [0], [[5], [5], [5]])]))
    assert e.code == ErrorCode.RANGE and "Token range" in e.msg
    # the id counts before the block ids
    e = _err(lambda: go([(range(0, 64), [0, 1, 2], [[5], [8], [5]])]))
    assert e.code == ErrorCode.LENGTH_MISMATCH
    # the second sequence's rejection after an empty first one; the first non-empty sequence's strategy before a later id count
    e = _err(lambda: go([EMPTY, (range(0, 64), [0, 1, 2], [[5], [5], [5]]), (range(70, 64), [], [[], [], []])]))
    assert e.code == ErrorCode.LENGTH_MISMATCH
    e = _err(lambda: go([GOOD, (range(0, 64), [0, 1, 2], [[5], [5], [5]])]))
    assert e.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in e.msg
    # the windows come first, also for a batch without sequences
    e = _err(lambda: go([], dsts=(1, 1, 3)))
    assert e.code == ErrorCode.OVERLAP and "one layout" in e.msg
    e = _err(lambda: _batch(mgr, hs, [], []))
    assert e.code == ErrorCode.ERR and "at least one destination" in e.msg
    # with a layer stream, its shape before everything else
    e = _err(lambda: _batch(mgr, hs, [], [], ready_flags=0))
    assert e.code == ErrorCode.ERR and "ready flags" in e.msg
    # nothing to move: no sequences, only empty ones, an empty layer range
    assert go([]) is not None and go([EMPTY, EMPTY]) is not None
    assert go([GOOD], o=TransferOptions(layer_range=range(4, 4))) is not None


# ---------------------------------------------------------------------------------------------------------------------
# the instantiations in the built library
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s, pp) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True)) for pp in (True, False)}
NEW = ("kvbm_paged_repage_push_seqs_kernel", "kvbm_gated_repage_push_seqs_kernel")


def test_the_batch_push_instantiations_are_what_the_library_contains():
    """40 kernels: the 20 walks of with_repage_kernel for each of the two families; tests/test_gpu_scatter_seqs.py reaches each."""
    so = os.path.join(ROOT, "dynamo_b200", "libkvbm_kernels.so")
    tool = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
    if not os.path.exists(so) or tool is None:
        pytest.skip("needs the built libkvbm_kernels.so and cuobjdump")
    txt = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    found = set()
    for name in re.findall(r"Function : (\S+)", txt):
        m = re.search(r"(kvbm_[a-z0-9_]+?_kernel)I((?:L[ib]\d+E)+)E", name)
        if m and "push_seqs" in m.group(1):
            assert m.group(1) in NEW
            c, p, s, pp = (int(v) if t == "i" else v == "1" for t, v in re.findall(r"L([ib])(\d+)E", m.group(2)))
            found.add((m.group(1), c, p, s, pp))
    assert len(WALKS) == 20 and found == {(k,) + w for k in NEW for w in WALKS}

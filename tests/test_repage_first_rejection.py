"""The first rejection of the staged re-paging gather, its streamed form and a batch of sequences, on a host-only manager.
tests/test_stage_repage_host.py and tests/test_repage_batch_host.py fault these entries one check at a time; the requests here
fail two or more, so they pin the order in which each entry makes its checks: each case names the code and a fragment of the
text the first failing check reports.  A batch reports its first rejected sequence with the single entry's code and text."""
import ctypes as C

import numpy as np
import pytest

from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, KvbmError, ShardWindow, TransferOptions
from tests.test_stage_repage_host import PLAN, host_pools  # noqa: F401  (host_pools is a fixture)

BAD = 0xDEAD
PP = C.POINTER(C.c_size_t)
OVERLAP = [PLAN[0], ShardWindow(1, 0, 0, 3, 0, 1, 2)] + PLAN[2:]          # heads 1-2 of stage 0 written twice


def _first(fn, code, fragment):
    with pytest.raises(KvbmError) as e:
        fn()
    assert (e.value.code, fragment in e.value.msg) == (code, True), (e.value.code, e.value.msg)
    return e.value


def _c_first(rc, code, fragment):
    msg = P.lib().kvbm_last_error().decode()
    assert (rc, fragment in msg) == (code, True), (rc, msg)


def _seq(tokens=range(0, 64), n_src=4, dst_ids=(5,), first=0):
    """One sequence as execute_repage_batch takes it: tokens 0..64 are 4 source blocks (16-token pages) and 1 destination block."""
    return tokens, {r: list(range(first + r, first + r + n_src)) for r in range(3)}, list(dst_ids)


EMPTY = _seq(tokens=range(9, 9), n_src=0, dst_ids=())
COUNTS = _seq(n_src=3)                                                       # 3 source ids for a range that spans 4
DST_PAST = _seq(dst_ids=(8,))                                                # past the destination's 8 blocks
REVERSED = _seq(tokens=range(70, 64))


def _sources(hs, third, seq):
    a, b, c, d, e, f = hs
    return {0: (a, seq[1][0]), 1: (b, seq[1][1]), 2: ((a, b, c, d, e, f)[third], seq[1][2])}


def _single(mgr, hs, plan, seq, o=None, third=2, dst=None, **kw):
    return mgr.execute_stage_repage_gather(_sources(hs, third, seq), hs[3] if dst is None else dst, seq[2], plan, seq[0], o, **kw)


def _batch(mgr, hs, plan, seqs, o=None, third=2, dst=None, **kw):
    a, b, c, d, e, f = hs
    return mgr.execute_repage_batch({0: a, 1: b, 2: (a, b, c, d, e, f)[third]}, d if dst is None else dst, seqs, plan, o, **kw)


def _c_windows(plan):
    return (P._CShardWindow * len(plan))(*[P._CShardWindow(w.src_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin,
                                                          w.dst_head_begin, w.head_count) for w in plan])


# ---------------------------------------------------------------------------------------------------------------------
# execute_stage_repage_gather
# ---------------------------------------------------------------------------------------------------------------------
def test_stage_repage_gather_first_rejection(host_pools):  # noqa: F811
    mgr, hs = host_pools
    go = lambda plan=PLAN, seq=_seq(), o=None, **kw: lambda: _single(mgr, hs, plan, seq, o, **kw)  # noqa: E731
    # overlapping windows and an invalid destination handle: the windows before any handle
    _first(go(OVERLAP, dst=BAD), ErrorCode.OVERLAP, "overlap in the destination")
    # a window past its source's layers and an invalid destination handle: the destination is looked up first
    _first(go([ShardWindow(0, 1, 0, 3, 0, 0, 2)] + PLAN[1:], dst=BAD), ErrorCode.HANDLE, "invalid destination handle")
    # stage 1 past the destination's layers, its source the destination itself: the layer windows before any pair
    _first(go(PLAN[:2] + [ShardWindow(2, 0, 4, 5, 0, 0, 2), ShardWindow(2, 0, 4, 5, 0, 2, 2)], third=3, dst=hs[3]), ErrorCode.RANGE,
           "destination's num_layers")
    # a head window past a's heads and a third source with another page size: the pair, in window order
    _first(go([ShardWindow(0, 0, 0, 3, 1, 0, 2)] + PLAN[1:], third=4), ErrorCode.RANGE, "Head window")
    # a reversed range, ids that do not match it and a layer range past the destination's layers: the token range first
    _first(go(seq=_seq(tokens=range(70, 64), n_src=3), o=TransferOptions(layer_range=range(0, 9))), ErrorCode.RANGE, "Token range")
    # ids that do not match the range and a destination id past its blocks: the counts first
    _first(go(seq=_seq(n_src=3, dst_ids=(8,))), ErrorCode.LENGTH_MISMATCH, "span 4 source and 1 destination blocks")
    # a destination id past its blocks and pools whose strategy is Memcpy: the ids first
    _first(go(seq=DST_PAST), ErrorCode.RANGE, "out of range for destination")
    # scales without a cast on host pools: the scales' rule before the strategy
    _first(go(o=TransferOptions(cast_scales=np.ones(16, np.float32))), ErrorCode.ERR, "need a cast_mode")


def test_stage_repage_gather_null_lists_first_rejection(host_pools):  # noqa: F811
    mgr, hs = host_pools
    a, b, c, d = hs[:4]
    handles = (C.c_uint64 * 3)(a, b, c)
    ws = _c_windows(PLAN)
    go = lambda src_ids, dst, dst_ids, n_src=4: P.lib().kvbm_manager_execute_stage_repage_gather(  # noqa: E731
        mgr._h, 3, handles, src_ids, n_src, dst, dst_ids, 1, 0, 64, ws, len(PLAN), None, C.byref(P._COptions()), None)
    ids = (C.c_size_t * 1)(9)
    # null id lists and an invalid destination handle: the handle first
    _c_first(go(None, BAD, None), ErrorCode.HANDLE, "invalid destination handle")
    # null id lists and counts that do not match the range: the counts first
    _c_first(go(None, d, None, n_src=3), ErrorCode.LENGTH_MISMATCH, "span 4 source and 1 destination blocks")
    # null source lists and a destination id past its blocks: the null list first
    _c_first(go((PP * 3)(None, None, None), d, ids), ErrorCode.ERR, "null block id list")


def test_stage_repage_gather_streamed_first_rejection(host_pools):  # noqa: F811
    mgr, hs = host_pools
    flags = np.zeros(16, np.uint32)
    f = flags.ctypes.data
    go = lambda plan=PLAN, ready=None, seq=_seq(), o=None, **kw: lambda: _single(mgr, hs, plan, seq, o, ready_flags=ready or {0: f, 1: f, 2: f},  # noqa: E731
                                                                                  **kw)
    # a source without ready flags and overlapping windows: the stream's shape first
    _first(go(OVERLAP, {0: f, 1: f}), ErrorCode.ERR, "no layer ready flags")
    # a source without ready flags and an invalid destination handle
    _first(go(ready={1: f, 2: f}, dst=BAD), ErrorCode.ERR, "no layer ready flags")
    # flags in the options and overlapping windows: the windows' checks, then the pairs'
    _first(go(OVERLAP, o=TransferOptions(layer_ready_flags=f)), ErrorCode.OVERLAP, "overlap in the destination")
    _first(go(o=TransferOptions(layer_ready_flags=f)), ErrorCode.UNSUPPORTED, "re-paging transfer takes no")
    # ids that do not match the range, and pageable flags: the counts first
    _first(go(seq=COUNTS), ErrorCode.LENGTH_MISMATCH, "span 4 source and 1 destination blocks")
    # pageable flags on host pools: the strategy before the flags
    _first(go(), ErrorCode.UNSUPPORTED, "direct CUDA strategy")
    # a stream naming 2 sources for a request with 3, and overlapping windows
    fl = (C.c_void_p * 2)(f, f)
    ls = P._CLayerStream(C.cast(fl, C.c_void_p), 2, None)
    a, b, c, d = hs[:4]
    rc = P.lib().kvbm_manager_execute_stage_repage_gather(mgr._h, 3, (C.c_uint64 * 3)(a, b, c), None, 0, d, None, 0, 9, 9, _c_windows(OVERLAP),
                                                          len(OVERLAP), C.byref(ls), C.byref(P._COptions()), None)
    _c_first(rc, ErrorCode.LENGTH_MISMATCH, "names 2 sources' ready flags")


# ---------------------------------------------------------------------------------------------------------------------
# execute_repage_batch
# ---------------------------------------------------------------------------------------------------------------------
def test_batch_first_and_third_sequences_fail(host_pools):  # noqa: F811
    mgr, hs = host_pools
    for first, third in ((COUNTS, DST_PAST), (DST_PAST, COUNTS), (REVERSED, COUNTS)):
        want = _first(lambda: _single(mgr, hs, PLAN, first), *_code_and_fragment(first))
        got = _first(lambda: _batch(mgr, hs, PLAN, [first, EMPTY, third]), *_code_and_fragment(first))
        assert got.msg == want.msg


def _code_and_fragment(seq):
    return {id(COUNTS): (ErrorCode.LENGTH_MISMATCH, "span 4 source and 1 destination blocks"), id(DST_PAST): (ErrorCode.RANGE, "out of range for destination"),
            id(REVERSED): (ErrorCode.RANGE, "Token range")}[id(seq)]


def test_batch_fails_a_window_check_and_a_sequence_check(host_pools):  # noqa: F811
    mgr, hs = host_pools
    _first(lambda: _batch(mgr, hs, OVERLAP, [COUNTS]), ErrorCode.OVERLAP, "overlap in the destination")
    _first(lambda: _batch(mgr, hs, [ShardWindow(0, 0, 0, 1, 0, 0, 1)] * 17, [COUNTS]), ErrorCode.UNSUPPORTED, "at most 16")
    # the stream's shape before the windows, and before every sequence
    _first(lambda: _batch(mgr, hs, OVERLAP, [COUNTS], ready_flags={0: 0, 1: 0, 2: 0}), ErrorCode.ERR, "no layer ready flags")
    # windows past the destination's layers, then the sequence: the stage layers are checked with the first sequence
    _first(lambda: _batch(mgr, hs, PLAN[:2], [COUNTS]), ErrorCode.RANGE, "destination layer 3")
    # a third source with another page size behind a bad sequence: the page size is the sequence's pair check, before its ids
    _first(lambda: _batch(mgr, hs, PLAN, [COUNTS], third=4), ErrorCode.INCOMPATIBLE, "one page size")
    # a layer range past the destination's layers fails with the first sequence, before its counts
    _first(lambda: _batch(mgr, hs, PLAN, [COUNTS], TransferOptions(layer_range=range(0, 9))), ErrorCode.RANGE, "exceeds num_layers 8")


def test_empty_batch_first_rejection(host_pools):  # noqa: F811
    mgr, hs = host_pools
    a, b, c, d = hs[:4]
    handles = (C.c_uint64 * 3)(a, b, c)
    go = lambda plan, seqs, num_seqs, dst=d: P.lib().kvbm_manager_execute_repage_batch(  # noqa: E731
        mgr._h, 3, handles, dst, seqs, num_seqs, _c_windows(plan), len(plan), None, C.byref(P._COptions()), None)
    # a null list of two sequences and overlapping windows: the windows first
    _c_first(go(OVERLAP, None, 2), ErrorCode.OVERLAP, "overlap in the destination")
    _c_first(go(PLAN, None, 2), ErrorCode.ERR, "null sequence list")
    # no sequences: the windows and the stream are checked, nothing that needs a sequence is
    _first(lambda: _batch(mgr, hs, OVERLAP, []), ErrorCode.OVERLAP, "overlap in the destination")
    _first(lambda: _batch(mgr, hs, PLAN, [], ready_flags={0: 0, 1: 0, 2: 0}), ErrorCode.ERR, "no layer ready flags")
    assert go(PLAN, None, 0) == ErrorCode.OK
    assert _batch(mgr, hs, PLAN, [], dst=BAD) is not None
    assert _batch(mgr, hs, PLAN, [], TransferOptions(layer_range=range(0, 9))) is not None


def test_batch_whose_only_nonempty_sequence_is_rejected(host_pools):  # noqa: F811
    mgr, hs = host_pools
    for bad in (COUNTS, DST_PAST, REVERSED):
        want = _first(lambda: _single(mgr, hs, PLAN, bad), *_code_and_fragment(bad))
        for seqs in ([EMPTY, bad], [EMPTY, bad, EMPTY], [bad, EMPTY]):
            got = _first(lambda: _batch(mgr, hs, PLAN, seqs), *_code_and_fragment(bad))
            assert got.msg == want.msg
    # the one non-empty sequence well-formed: the strategy rejects it, as the single entry does
    want = _first(lambda: _single(mgr, hs, PLAN, _seq()), ErrorCode.UNSUPPORTED, "direct CUDA strategy")
    got = _first(lambda: _batch(mgr, hs, PLAN, [EMPTY, _seq(), EMPTY]), ErrorCode.UNSUPPORTED, "direct CUDA strategy")
    assert got.msg == want.msg
    # an empty sequence still takes the single entry's checks: an invalid destination handle rejects it
    _first(lambda: _batch(mgr, hs, PLAN, [EMPTY], dst=BAD), ErrorCode.HANDLE, "invalid destination handle")

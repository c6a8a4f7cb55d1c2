"""CPU checks of the TP re-shard: the head-window oracle (tests/reshard_oracle.py) and kvbm_tp_reshard_plan."""
import itertools

import numpy as np
import pytest

from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, HeadWindow, KvbmError
from oracle import oracle as O
from tests.reshard_oracle import rank_heads, reshard_block, reshard_plan

ALL = [O.KV_UNIVERSAL_TP, O.KV_UNIVERSAL_PP, O.KV_OPERATIONAL_HND, O.KV_OPERATIONAL_NHD]
HEADS = [1, 2, 4, 8, 16, 64]


def _tps(H):
    """Every TP degree up to 16 the ownership rule allows for H heads."""
    return [tp for tp in range(1, 17) if H % tp == 0 or tp % H == 0]


@pytest.mark.parametrize("H", HEADS)
def test_plan_covers_every_head_of_every_decode_rank_once(H):
    for src_tp, dst_tp in itertools.product(_tps(H), _tps(H)):
        for rank in range(dst_tp):
            plan = P.tp_reshard_plan(H, src_tp, dst_tp, rank)
            want = rank_heads(H, dst_tp, rank)
            got = []
            for w in plan:
                assert 0 <= w.src_rank < src_tp and w.head_count >= 1
                src_heads = rank_heads(H, src_tp, w.src_rank)
                assert w.src_head_begin + w.head_count <= len(src_heads)          # inside the source rank's heads
                for j in range(w.head_count):                                     # ... and the same global heads on both sides
                    assert src_heads[w.src_head_begin + j] == want[w.dst_head_begin + j]
                got += range(w.dst_head_begin, w.dst_head_begin + w.head_count)
            assert got == list(range(len(want))), (H, src_tp, dst_tp, rank)       # ascending, each head exactly once
            for a, b in zip(plan, plan[1:]):                                       # merged: no two adjacent windows could be one
                assert not (a.src_rank == b.src_rank and a.src_head_begin + a.head_count == b.src_head_begin)


@pytest.mark.parametrize("H", HEADS)
def test_c_plan_equals_the_python_rule(H):
    for src_tp, dst_tp in itertools.product(_tps(H), _tps(H)):
        for rank in range(dst_tp):
            got = [(w.src_rank, w.src_head_begin, w.dst_head_begin, w.head_count) for w in P.tp_reshard_plan(H, src_tp, dst_tp, rank)]
            assert got == reshard_plan(H, src_tp, dst_tp, rank), (H, src_tp, dst_tp, rank)


def test_plan_examples_and_replicas():
    # Llama-3-70B, 8 KV heads: TP4 prefill -> TP2 decode, rank 1 takes 2 heads from each of prefill ranks 2 and 3
    assert P.tp_reshard_plan(8, 4, 2, 1) == [HeadWindow(2, 0, 0, 2), HeadWindow(3, 0, 2, 2)]
    # TP2 -> TP8: rank 5 is global head 5, head 1 of prefill rank 1
    assert P.tp_reshard_plan(8, 2, 8, 5) == [HeadWindow(1, 1, 0, 1)]
    # TP1 -> TP2 is one window: every head of the one source is adjacent
    assert P.tp_reshard_plan(8, 1, 2, 1) == [HeadWindow(0, 4, 0, 4)]
    # replicated sources (TP16 over 8 heads): head g lives on ranks 2g, 2g+1; decode rank r reads replica r % 2
    assert [w.src_rank for w in P.tp_reshard_plan(8, 16, 2, 0)] == [0, 2, 4, 6]
    assert [w.src_rank for w in P.tp_reshard_plan(8, 16, 2, 1)] == [9, 11, 13, 15]
    # MLA: one latent head, every decode rank reads it from source rank dst_rank % src_tp
    for src_tp, dst_tp in ((1, 8), (4, 8), (8, 4), (2, 2)):
        for r in range(dst_tp):
            assert P.tp_reshard_plan(1, src_tp, dst_tp, r) == [HeadWindow(r % src_tp, 0, 0, 1)]


def test_plan_error_codes():
    def code(*args):
        with pytest.raises(KvbmError) as e:
            P.tp_reshard_plan(*args)
        return e.value.code
    assert code(8, 3, 2, 0) == ErrorCode.CONFIG           # neither divides the other
    assert code(8, 2, 12, 0) == ErrorCode.CONFIG
    assert code(6, 4, 2, 0) == ErrorCode.CONFIG
    assert code(0, 1, 1, 0) == ErrorCode.CONFIG
    assert code(8, 0, 2, 0) == ErrorCode.CONFIG
    assert code(8, 2, 0, 0) == ErrorCode.CONFIG
    assert code(8, 4, 2, 2) == ErrorCode.RANGE            # no decode rank 2 at TP2
    assert code(1, 1, 4, 4) == ErrorCode.RANGE


def test_plan_buffer_rules():
    import ctypes as C
    L = P.lib()
    n = C.c_size_t(99)
    assert L.kvbm_tp_reshard_plan(8, 8, 1, 0, None, 0, C.byref(n)) == 0 and n.value == 8   # out == NULL counts
    buf = (P._CHeadWindow * 4)()
    assert L.kvbm_tp_reshard_plan(8, 8, 1, 0, buf, 4, C.byref(n)) == ErrorCode.ERR          # cap below the count
    assert L.kvbm_tp_reshard_plan(8, 8, 1, 0, buf, 4, None) == ErrorCode.ERR                 # no n_out


@pytest.mark.parametrize("src_kv,dst_kv", list(itertools.product(ALL, ALL)))
def test_split_into_tp_windows_and_reassemble_is_the_identity(src_kv, dst_kv):
    """A TP1 block (8 heads, src_kv) split into TP2 / TP4 / TP8 blocks (dst_kv) by the plan, then re-assembled into a TP1 block
    (src_kv) with the plan of the other direction, equals the original; every split block equals the oracle's slice."""
    nl, no, nt, H, row = 3, 2, 4, 8, 32
    rng = np.random.default_rng(int(src_kv) * 10 + int(dst_kv))
    block = rng.integers(0, 256, nl * no * nt * H * row, dtype=np.uint8)
    tp1 = O.kv_layout_permute(block, src_kv, O.KV_UNIVERSAL_TP, nl, no, nt, H, row).reshape(H, -1)
    for tp in (2, 4, 8):
        k = H // tp
        shards = []
        for r in range(tp):
            blk = np.full(nl * no * nt * k * row, 0xEE, dtype=np.uint8)
            for w in P.tp_reshard_plan(H, 1, tp, r):
                blk = reshard_block(block, blk, src_kv, dst_kv, nl, no, nt, H, k, row, 0, w.src_head_begin, w.dst_head_begin, w.head_count)
            uni = O.kv_layout_permute(blk, dst_kv, O.KV_UNIVERSAL_TP, nl, no, nt, k, row).reshape(k, -1)
            assert np.array_equal(uni, tp1[r * k:(r + 1) * k])
            shards.append(blk)
        back = np.full(block.size, 0x11, dtype=np.uint8)
        for w in P.tp_reshard_plan(H, tp, 1, 0):
            back = reshard_block(shards[w.src_rank], back, dst_kv, src_kv, nl, no, nt, k, H, row, 0, w.src_head_begin, w.dst_head_begin,
                                 w.head_count)
        assert np.array_equal(back, block), tp


def test_oracle_window_leaves_other_heads_and_layers_alone():
    nl, no, nt, row = 4, 2, 3, 16
    rng = np.random.default_rng(5)
    src = rng.integers(0, 256, nl * no * nt * 4 * row, dtype=np.uint8)
    old = rng.integers(0, 256, nl * no * nt * 6 * row, dtype=np.uint8)
    out = reshard_block(src, old, O.KV_OPERATIONAL_NHD, O.KV_UNIVERSAL_PP, nl, no, nt, 4, 6, row, 0, 1, 3, 2, layers=range(1, 3))
    s = O.kv_layout_permute(src, O.KV_OPERATIONAL_NHD, O.KV_UNIVERSAL_TP, nl, no, nt, 4, row).reshape(4, nl, -1)
    o = O.kv_layout_permute(old, O.KV_UNIVERSAL_PP, O.KV_UNIVERSAL_TP, nl, no, nt, 6, row).reshape(6, nl, -1)
    g = O.kv_layout_permute(out, O.KV_UNIVERSAL_PP, O.KV_UNIVERSAL_TP, nl, no, nt, 6, row).reshape(6, nl, -1)
    want = o.copy()
    want[3:5, 1:3] = s[1:3, 1:3]
    assert np.array_equal(g, want)

"""Oracle of the head-window transform (kvbm_kernels_paged_permute_heads, and TransferManager transfers with a head window):
both blocks are brought to UniversalTP with oracle.kv_layout_permute, where heads are the outermost dimension; source heads
[sb, sb + k) are cast with the oracle's cast and written over destination heads [db, db + k); the result goes back to the
destination format.  The re-shard has no reference implementation (kv_block_layout.rs:41-46 names the use and builds nothing):
its oracle is this definition over the dim_order one.  Also the head ownership rule kvbm_tp_reshard_plan follows, restated."""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np

from oracle import oracle as O
from tests.cast_oracle import cast_bytes, dst_row_bytes


def reshard_block(src_block: np.ndarray, dst_old: np.ndarray, src_kv: int, dst_kv: int, nl: int, no: int, nt: int, src_nh: int, dst_nh: int,
                  src_row_bytes: int, cast_mode: int, src_head_begin: int, dst_head_begin: int, head_count: int,
                  layers: Optional[range] = None) -> np.ndarray:
    """The destination block (uint8[nl*no*nt*dst_nh*dst_row]) after heads [src_head_begin, +head_count) of the source block
    (uint8[nl*no*nt*src_nh*src_row_bytes]) land as heads [dst_head_begin, +head_count), in `layers` only (all when None)."""
    d_row = dst_row_bytes(src_row_bytes, cast_mode)
    s = O.kv_layout_permute(src_block, src_kv, O.KV_UNIVERSAL_TP, nl, no, nt, src_nh, src_row_bytes).reshape(src_nh, nl, no, nt, src_row_bytes)
    d = O.kv_layout_permute(dst_old, dst_kv, O.KV_UNIVERSAL_TP, nl, no, nt, dst_nh, d_row).reshape(dst_nh, nl, no, nt, d_row).copy()
    win = cast_bytes(s[src_head_begin:src_head_begin + head_count].reshape(-1), cast_mode).reshape(head_count, nl, no, nt, d_row)
    lsel = slice(None) if layers is None else slice(layers.start, layers.stop)
    d[dst_head_begin:dst_head_begin + head_count, lsel] = win[:, lsel]
    return O.kv_layout_permute(d.reshape(-1), O.KV_UNIVERSAL_TP, dst_kv, nl, no, nt, dst_nh, d_row)


def rank_heads(num_kv_heads: int, tp: int, rank: int) -> range:
    """vLLM's head ownership: rank r of tp holds [r*H/tp, r*H/tp + max(1, H/tp)) (replicated over tp/H ranks when tp > H)."""
    first = rank * num_kv_heads // tp
    return range(first, first + max(1, num_kv_heads // tp))


def reshard_plan(num_kv_heads: int, src_tp: int, dst_tp: int, dst_rank: int) -> List[Tuple[int, int, int, int]]:
    """(src_rank, src_head_begin, dst_head_begin, head_count) per window, the rule kvbm_tp_reshard_plan implements: every head
    of the decode rank from the source rank that holds it -- replica dst_rank % (src_tp / H) of a replicated one --, adjacent
    heads of one source merged."""
    H = num_kv_heads
    out: List[list] = []
    for j, g in enumerate(rank_heads(H, dst_tp, dst_rank)):
        holders = [r for r in range(src_tp) if g in rank_heads(H, src_tp, r)]
        r = holders[dst_rank % len(holders)]
        local = g - rank_heads(H, src_tp, r).start
        if out and out[-1][0] == r and out[-1][1] + out[-1][3] == local:
            out[-1][3] += 1
        else:
            out.append([r, local, j, 1])
    return [tuple(w) for w in out]

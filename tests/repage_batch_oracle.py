"""Oracle of a batch of sequences in one re-paging launch (kvbm_kernels_paged_stage_repage_gather_batch,
TransferManager.execute_repage_batch), written from the semantics alone: a batch is its sequences moved one after the other, each
as tests/stage_repage_oracle.py moves one sequence, into one destination image.  No two sequences share a destination block, so
the order does not matter; two sequences may read the same source blocks.

`repage_batch_units` restates the unit table of include/kvbm_kernels.h (kvbm_repage_unit) in numpy arithmetic, from the
definition of its four words rather than from the helper's loop."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

from tests.cast_oracle import CAST_NONE
from tests.stage_repage_oracle import stage_repage_gather


def repage_batch(src_pools: Sequence[Tuple[np.ndarray, int, int, int]], windows: Sequence[Tuple[int, int, int, int, int, int, int]],
                 dst_pool: np.ndarray, dst_kv: int, dst_nh: int, dst_nl: int, no: int, src_page: int, dst_page: int, src_row_bytes: int,
                 seqs: Sequence[Tuple[int, int, Sequence[Sequence[int]], Sequence[int]]], cast_mode: int = CAST_NONE,
                 scales: Optional[np.ndarray] = None, layers: Optional[range] = None) -> np.ndarray:
    """src_pools: (pool bytes [num_blocks, block_bytes], kv, num_heads, num_layers) per source; dst_pool: the destination pool's bytes
    before the transfer; seqs: (token_begin, token_end, per-source block ids, destination block ids) per sequence, the ids being
    what the single entry takes for that range.  Returns the destination pool after the transfer."""
    out = np.array(dst_pool, dtype=np.uint8, copy=True)
    for tb, te, sids, dids in seqs:
        sources = [([pool[b] for b in sids[s]], kv, nh, nl) for s, (pool, kv, nh, nl) in enumerate(src_pools)]
        new = stage_repage_gather(sources, windows, [out[b] for b in dids], dst_kv, dst_nh, dst_nl, no, src_page, dst_page, src_row_bytes,
                                  tb, te, cast_mode, scales, layers)
        for b, blk in zip(dids, new):
            out[b] = blk
    return out


def repage_batch_units(seqs: Sequence[Tuple[int, int]], src_page: int, dst_page: int):
    """(units uint32 [n, 4], source table length, destination table length) of a batch of (token_begin, token_end) ranges."""
    big, small = max(src_page, dst_page), min(src_page, dst_page)
    rows, small_off = [], 0
    for i, (tb, te) in enumerate(seqs):
        if tb == te:
            continue
        bigs = np.arange(tb // big, -(-te // big), dtype=np.int64)          # the sequence's big blocks
        lo, hi = np.maximum(bigs * big, tb), np.minimum((bigs + 1) * big, te)   # each clipped to the range
        first_small = bigs * (big // small) - tb // small + small_off      # entry of the concatenated small table, may be < 0
        rows.append(np.stack([lo - bigs * big, hi - lo, first_small % (1 << 32), np.full_like(bigs, i)], axis=1))
        small_off += -(-te // small) - tb // small
    units = np.concatenate(rows).astype(np.uint32) if rows else np.zeros((0, 4), np.uint32)
    n_big, n_small = len(units), small_off
    return units, (n_small if src_page < dst_page else n_big), (n_big if src_page < dst_page else n_small)

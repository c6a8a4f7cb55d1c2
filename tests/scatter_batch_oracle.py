"""Oracle of a batch of sequences in one re-paging scatter launch (kvbm_kernels_paged_repage_scatter_batch,
TransferManager.execute_repage_scatter_batch), written from the semantics alone: a batch is its sequences pushed one after the
other, each as tests/scatter_oracle.repage_scatter pushes one sequence, over its range and its slices of the concatenated tables.
Within one destination pool no two sequences share a block, so the order does not matter; two sequences may read the same source
blocks."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

from tests.cast_oracle import CAST_NONE
from tests.scatter_oracle import repage_scatter


def table_len(tb: int, te: int, page: int) -> int:
    """The entries a sequence [tb, te) contributes to a concatenated table of page `page`: none when its range is empty."""
    return 0 if tb == te else -(-te // page) - tb // page


def repage_scatter_batch(src: Tuple[np.ndarray, Sequence[int], int, int, int], targets: Sequence[tuple], pools: Sequence[np.ndarray],
                         no: int, src_page: int, dst_page: int, src_row_bytes: int, seqs: Sequence[Tuple[int, int]],
                         cast_mode: int = CAST_NONE, scales: Optional[np.ndarray] = None, layers: Optional[range] = None) -> None:
    """src: (pool bytes [num_blocks, block], concatenated ids, kv, num_heads, num_layers); targets: (pool index, concatenated ids,
    kv, num_heads, num_layers, (sl, dl, c, sb, db, k)) as tests/scatter_oracle.repage_scatter takes them, but with every table the
    concatenation in batch order of the per-sequence tables; seqs: the (token_begin, token_end) ranges.  Updates pools in place."""
    pool, sids, kv, nh, nl = src
    so = do = 0
    for tb, te in seqs:
        ns, nd = table_len(tb, te, src_page), table_len(tb, te, dst_page)
        if ns == 0:
            continue
        blocks = [pool[b] for b in sids[so:so + ns]]
        tg = [(p, ids[do:do + nd], d_kv, d_nh, d_nl, w) for p, ids, d_kv, d_nh, d_nl, w in targets]
        repage_scatter((blocks, kv, nh, nl), tg, pools, no, src_page, dst_page, src_row_bytes, tb, te, cast_mode, scales, layers)
        so, do = so + ns, do + nd

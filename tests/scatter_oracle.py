"""Oracle of the re-paging scatter (kvbm_kernels_paged_repage_scatter, TransferManager.execute_repage_scatter), defined as its
header defines it: one tests/stage_repage_oracle.stage_repage_gather call per target, in target order, each with the source as
its one stage source under the target's windows, over the destination image of the source layer range, with the source's scales
re-indexed to destination layers."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

from tests.cast_oracle import CAST_NONE
from tests.stage_repage_oracle import stage_repage_gather


def dst_layers(window: Tuple[int, int, int, int, int, int], src_layers: range) -> range:
    """The destination layers a target's window (sl, dl, c, sb, db, k) writes for source layers `src_layers`."""
    sl, dl, c = window[:3]
    lo, hi = max(sl, src_layers.start), min(sl + c, src_layers.stop)
    return range(lo - sl + dl, max(lo, hi) - sl + dl)


def dst_scales(window, src_scales: Optional[np.ndarray], dst_nl: int, no: int) -> Optional[np.ndarray]:
    """The source's float[src_nl * no] scales as a destination's float[dst_nl * no] array under the window (1 outside it)."""
    if src_scales is None:
        return None
    sl, dl, c = window[:3]
    out = np.ones(dst_nl * no, dtype=np.float32)
    out[dl * no:(dl + c) * no] = src_scales[sl * no:(sl + c) * no]
    return out


def repage_scatter(src: Tuple[Sequence[np.ndarray], int, int, int], targets: Sequence[tuple], pools: Sequence[np.ndarray], no: int,
                   src_page: int, dst_page: int, src_row_bytes: int, token_begin: int, token_end: int, cast_mode: int = CAST_NONE,
                   scales: Optional[np.ndarray] = None, layers: Optional[range] = None) -> None:
    """src: (blocks, kv, num_heads, num_layers), blocks being the source's table[token_begin // Ps .. ceil(token_end / Ps)) (uint8,
    in kv, over its own layers); targets: (pool index, ids, kv, num_heads, num_layers, (sl, dl, c, sb, db, k)), ids being the
    target's table[token_begin // Pd .. ceil(token_end / Pd)) in pools[pool] (uint8 [num_blocks, block]), updated in place;
    scales: the source's float[src num_layers * no]; layers: the SOURCE layer range (all when None)."""
    blocks, kv, nh, nl = src
    rng = range(nl) if layers is None else layers
    for pool, ids, d_kv, d_nh, d_nl, w in targets:
        img = dst_layers(w, rng)
        if len(img) == 0:
            continue
        p = pools[pool]
        new = stage_repage_gather([(blocks, kv, nh, nl)], [(0,) + tuple(w)], [p[b] for b in ids], d_kv, d_nh, d_nl, no, src_page, dst_page,
                                  src_row_bytes, token_begin, token_end, cast_mode, dst_scales(w, scales, d_nl, no), img)
        for b, blk in zip(ids, new):
            p[b] = blk

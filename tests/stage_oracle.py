"""Oracle of the staged gather (kvbm_kernels_paged_stage_gather, TransferManager.execute_stage_gather) and of the PP x TP
re-shard plan (kvbm_tp_pp_reshard_plan).  A window moves source layers [sl, sl + c) to destination layers [dl, dl + c): both
blocks are brought to UniversalTP over their own layer counts, the two layer slices are cut out as c-layer UniversalTP blocks,
tests/reshard_oracle.reshard_block (or its scaled twin, with the destination layers' scales) moves the head window between
them, and the destination slice goes back.  The plan is the TP plan of tests/reshard_oracle per pair of stages that share
layers."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from oracle import oracle as O
from tests.cast_oracle import dst_row_bytes
from tests.reshard_oracle import reshard_block, reshard_plan
from tests.scaled_cast_oracle import reshard_block_scaled

UTP = O.KV_UNIVERSAL_TP


def stage_block(src_block: np.ndarray, dst_old: np.ndarray, src_kv: int, dst_kv: int, src_nl: int, dst_nl: int, no: int, nt: int,
                src_nh: int, dst_nh: int, src_row_bytes: int, cast_mode: int, window: Tuple[int, int, int, int, int, int],
                layers: Optional[range] = None, scales: Optional[np.ndarray] = None) -> np.ndarray:
    """The destination block (dst_nl layers) after `window` = (src_layer_begin, dst_layer_begin, layer_count, src_head_begin,
    dst_head_begin, head_count) of the source block (src_nl layers) landed, at the destination layers of `layers` only (all
    when None).  scales: float[dst_nl * no], by the destination layer."""
    sl, dl, c, sb, db, k = window
    d_row = dst_row_bytes(src_row_bytes, cast_mode)
    s = O.kv_layout_permute(src_block, src_kv, UTP, src_nl, no, nt, src_nh, src_row_bytes).reshape(src_nh, src_nl, no, nt, src_row_bytes)
    d = O.kv_layout_permute(dst_old, dst_kv, UTP, dst_nl, no, nt, dst_nh, d_row).reshape(dst_nh, dst_nl, no, nt, d_row).copy()
    lo, hi = dl, dl + c
    if layers is not None:
        lo, hi = max(lo, layers.start), min(hi, layers.stop)
    if hi > lo:
        sub_s = np.ascontiguousarray(s[:, sl:sl + c]).reshape(-1)
        sub_d = np.ascontiguousarray(d[:, dl:dl + c]).reshape(-1)
        sub_layers = range(lo - dl, hi - dl)
        if scales is None:
            out = reshard_block(sub_s, sub_d, UTP, UTP, c, no, nt, src_nh, dst_nh, src_row_bytes, cast_mode, sb, db, k, layers=sub_layers)
        else:
            out = reshard_block_scaled(sub_s, sub_d, UTP, UTP, c, no, nt, src_nh, dst_nh, src_row_bytes, cast_mode,
                                       np.asarray(scales)[dl * no:(dl + c) * no], sb, db, k, layers=sub_layers)
        d[:, dl:dl + c] = out.reshape(dst_nh, c, no, nt, d_row)
    return O.kv_layout_permute(d.reshape(-1), UTP, dst_kv, dst_nl, no, nt, dst_nh, d_row)


def stage_bounds(num_layers: int, pp: int, parts: Optional[Sequence[int]] = None) -> List[int]:
    """First layer of every stage, then num_layers."""
    parts = list(parts) if parts is not None else [num_layers // pp] * pp
    out = [0]
    for c in parts:
        out.append(out[-1] + c)
    return out


def stage_plan(num_kv_heads: int, num_layers: int, src_tp: int, src_pp: int, dst_tp: int, dst_pp: int, dst_rank: int,
               src_parts: Optional[Sequence[int]] = None, dst_parts: Optional[Sequence[int]] = None) -> List[tuple]:
    """(src_rank, src_layer_begin, dst_layer_begin, layer_count, src_head_begin, dst_head_begin, head_count) per window: for each
    source stage meeting the decode rank's stage, the TP plan of the two TP degrees over the shared layers, stage-local layers,
    ranks pp_rank * tp + tp_rank."""
    sb, db = stage_bounds(num_layers, src_pp, src_parts), stage_bounds(num_layers, dst_pp, dst_parts)
    d0, d1 = db[dst_rank // dst_tp], db[dst_rank // dst_tp + 1]
    heads = reshard_plan(num_kv_heads, src_tp, dst_tp, dst_rank % dst_tp)
    out = []
    for p in range(src_pp):
        lo, hi = max(d0, sb[p]), min(d1, sb[p + 1])
        if lo < hi:
            out += [(p * src_tp + r, lo - sb[p], lo - d0, hi - lo, shb, dhb, k) for r, shb, dhb, k in heads]
    return out

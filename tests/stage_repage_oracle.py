"""Oracle of the staged re-paging gather (kvbm_kernels_paged_stage_repage_gather, TransferManager.execute_stage_repage_gather),
written from the semantics alone: sequence token p sits in slot p % P of block table[p // P] on a side of page P, and window
(source, sl, dl, c, sb, db, k) moves heads [sb, sb + k) of source layers [sl, sl + c) to heads [db, db + k) of destination layers
[dl, dl + c).

1. every listed block of each source is brought to a UniversalTP sequence view over ITS OWN layer count
   (tests/repage_oracle._sequence), and so is the destination over its own;
2. per window and destination layer l of the range inside the window, the source's heads at layer l - dl + sl are cast over the
   token range (tests/cast_oracle.py, or tests/scaled_cast_oracle.py with the destination layer's scale);
3. they are written over the destination's heads and tokens at layer l;
4. the destination view is split back into pages and brought back to the destination's format."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

from oracle import oracle as O
from tests.cast_oracle import CAST_NONE, cast_bytes, dst_row_bytes
from tests.repage_oracle import _sequence
from tests.scaled_cast_oracle import cast_bytes_scaled


def stage_repage_gather(sources: Sequence[Tuple[Sequence[np.ndarray], int, int, int]],
                        windows: Sequence[Tuple[int, int, int, int, int, int, int]], dst_blocks: Sequence[np.ndarray], dst_kv: int,
                        dst_nh: int, dst_nl: int, no: int, src_page: int, dst_page: int, src_row_bytes: int, token_begin: int,
                        token_end: int, cast_mode: int = CAST_NONE, scales: Optional[np.ndarray] = None,
                        layers: Optional[range] = None) -> list:
    """sources: (blocks, kv, num_heads, num_layers) per source, blocks being its logical blocks table[token_begin // Ps ..
    ceil(token_end / Ps)) (uint8, in kv, over its own layers); windows: (source index, src_layer_begin, dst_layer_begin,
    layer_count, src_head_begin, dst_head_begin, head_count); dst_blocks: the destination blocks table[token_begin // Pd ..
    ceil(token_end / Pd)) before the transfer; scales: float[dst_nl * no], by the destination layer; layers: the destination
    layer range (all when None).  Returns those destination blocks after the transfer."""
    d_row = dst_row_bytes(src_row_bytes, cast_mode)
    if token_begin == token_end:
        return [np.array(b, dtype=np.uint8, copy=True) for b in dst_blocks]
    seqs = [_sequence(blocks, kv, nl, no, src_page, nh, src_row_bytes) for blocks, kv, nh, nl in sources]
    d = _sequence(dst_blocks, dst_kv, dst_nl, no, dst_page, dst_nh, d_row).copy()
    s0, d0 = token_begin // src_page * src_page, token_begin // dst_page * dst_page
    n = token_end - token_begin
    rng = range(dst_nl) if layers is None else layers
    for src, sl, dl, c, sb, db, k in windows:
        s = seqs[src]
        for l in range(max(dl, rng.start), min(dl + c, rng.stop)):
            for o in range(no):
                part = np.ascontiguousarray(s[sb:sb + k, l - dl + sl, o, token_begin - s0:token_end - s0]).reshape(-1)
                cast = cast_bytes(part, cast_mode) if scales is None else cast_bytes_scaled(part, cast_mode, float(scales[l * no + o]))
                d[db:db + k, l, o, token_begin - d0:token_end - d0] = cast.reshape(k, n, d_row)
    out = []
    for i in range(len(dst_blocks)):
        blk = np.ascontiguousarray(d[:, :, :, i * dst_page:(i + 1) * dst_page]).reshape(-1)
        out.append(O.kv_layout_permute(blk, O.KV_UNIVERSAL_TP, dst_kv, dst_nl, no, dst_page, dst_nh, d_row))
    return out

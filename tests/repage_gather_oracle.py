"""Oracle of re-paging with the gather's head windows (kvbm_kernels_paged_repage_gather, TransferManager.execute_repage_gather),
built from tests/repage_oracle.py and tests/reshard_oracle.py and written from the semantics alone: sequence token p sits in slot
p % P of block table[p // P] on a side of page P, and window (source, sb, db, k) moves source heads [sb, sb + k) to destination
heads [db, db + k).

1. every listed block of each source, and of the destination, is brought to a UniversalTP sequence view ([nh, nl, no, tokens,
   row], starting at (token_begin // P) * P);
2. each window's heads of its source are cast over the token range (tests/cast_oracle.py, or tests/scaled_cast_oracle.py with one
   scale per (layer, outer));
3. they are written over the destination's heads and tokens, for the layers of the range only;
4. the destination view is split back into pages and brought back to the destination's format."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

from oracle import oracle as O
from tests.cast_oracle import CAST_NONE, cast_bytes, dst_row_bytes
from tests.repage_oracle import _sequence
from tests.scaled_cast_oracle import cast_bytes_scaled


def repage_gather(sources: Sequence[Tuple[Sequence[np.ndarray], int, int]], windows: Sequence[Tuple[int, int, int, int]],
                  dst_blocks: Sequence[np.ndarray], dst_kv: int, dst_nh: int, nl: int, no: int, src_page: int, dst_page: int,
                  src_row_bytes: int, token_begin: int, token_end: int, cast_mode: int = CAST_NONE, scales: Optional[np.ndarray] = None,
                  layers: Optional[range] = None) -> list:
    """sources: (blocks, kv, num_heads) per source, blocks being its logical blocks table[token_begin // Ps .. ceil(token_end / Ps))
    (uint8, in kv); windows: (source index, src_head_begin, dst_head_begin, head_count); dst_blocks: the destination blocks
    table[token_begin // Pd .. ceil(token_end / Pd)) before the transfer.  Returns those destination blocks after it."""
    d_row = dst_row_bytes(src_row_bytes, cast_mode)
    if token_begin == token_end:
        return [np.array(b, dtype=np.uint8, copy=True) for b in dst_blocks]
    seqs = [_sequence(blocks, kv, nl, no, src_page, nh, src_row_bytes) for blocks, kv, nh in sources]
    d = _sequence(dst_blocks, dst_kv, nl, no, dst_page, dst_nh, d_row).copy()
    s0, d0 = token_begin // src_page * src_page, token_begin // dst_page * dst_page
    n = token_end - token_begin
    for src, sb, db, k in windows:
        s = seqs[src]
        for l in (range(nl) if layers is None else layers):
            for o in range(no):
                part = np.ascontiguousarray(s[sb:sb + k, l, o, token_begin - s0:token_end - s0]).reshape(-1)
                cast = cast_bytes(part, cast_mode) if scales is None else cast_bytes_scaled(part, cast_mode, float(scales[l * no + o]))
                d[db:db + k, l, o, token_begin - d0:token_end - d0] = cast.reshape(k, n, d_row)
    out = []
    for i in range(len(dst_blocks)):
        blk = np.ascontiguousarray(d[:, :, :, i * dst_page:(i + 1) * dst_page]).reshape(-1)
        out.append(O.kv_layout_permute(blk, O.KV_UNIVERSAL_TP, dst_kv, nl, no, dst_page, dst_nh, d_row))
    return out


def split_heads(blocks: Sequence[np.ndarray], kv: int, nl: int, no: int, page: int, nh: int, row: int, heads: range, out_kv: int) -> list:
    """The blocks of one TP rank holding `heads` of a sequence's blocks (nh heads, format kv), in format out_kv."""
    out = []
    for b in blocks:
        u = O.kv_layout_permute(b, kv, O.KV_UNIVERSAL_TP, nl, no, page, nh, row).reshape(nh, nl, no, page, row)
        part = np.ascontiguousarray(u[heads.start:heads.stop]).reshape(-1)
        out.append(O.kv_layout_permute(part, O.KV_UNIVERSAL_TP, out_kv, nl, no, page, len(heads), row))
    return out

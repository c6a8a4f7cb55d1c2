"""Oracle of re-paging (kvbm_kernels_paged_repage, TransferManager.execute_repage), written from the semantics alone: sequence token
p sits in slot p % P of block table[p // P] on a side of page P.

1. every listed block of each side is brought to UniversalTP ([nh, nl, no, page, row]) with oracle.kv_layout_permute;
2. the blocks are concatenated along the token axis: the sequence view of that side, starting at (token_begin // P) * P;
3. the source's tokens [token_begin, token_end) are cast (tests/cast_oracle.py, or tests/scaled_cast_oracle.py with one scale
   per (layer, outer));
4. they are written over the destination's sequence view, for the layers of the range only;
5. the destination view is split back into pages and brought back to the destination's format."""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from oracle import oracle as O
from tests.cast_oracle import CAST_NONE, cast_bytes, dst_row_bytes
from tests.scaled_cast_oracle import cast_bytes_scaled


def _sequence(blocks: Sequence[np.ndarray], kv: int, nl: int, no: int, page: int, nh: int, row: int) -> np.ndarray:
    """Logical blocks of one side -> [nh, nl, no, len(blocks) * page, row]."""
    uni = [O.kv_layout_permute(b, kv, O.KV_UNIVERSAL_TP, nl, no, page, nh, row).reshape(nh, nl, no, page, row) for b in blocks]
    return np.concatenate(uni, axis=3)


def repage(src_blocks: Sequence[np.ndarray], dst_blocks: Sequence[np.ndarray], src_kv: int, dst_kv: int, nl: int, no: int, nh: int,
           src_page: int, dst_page: int, src_row_bytes: int, token_begin: int, token_end: int, cast_mode: int = CAST_NONE,
           scales: Optional[np.ndarray] = None, layers: Optional[range] = None) -> list:
    """src_blocks: the logical source blocks src_table[token_begin // Ps .. ceil(token_end / Ps)) (uint8, in src_kv); dst_blocks: the
    destination blocks dst_table[token_begin // Pd .. ceil(token_end / Pd)) before the transfer.  Returns those destination
    blocks after it."""
    d_row = dst_row_bytes(src_row_bytes, cast_mode)
    if token_begin == token_end:
        return [np.array(b, dtype=np.uint8, copy=True) for b in dst_blocks]
    s = _sequence(src_blocks, src_kv, nl, no, src_page, nh, src_row_bytes)
    d = _sequence(dst_blocks, dst_kv, nl, no, dst_page, nh, d_row).copy()
    s0, d0 = token_begin // src_page * src_page, token_begin // dst_page * dst_page
    n = token_end - token_begin
    for l in (range(nl) if layers is None else layers):
        for o in range(no):
            part = np.ascontiguousarray(s[:, l, o, token_begin - s0:token_end - s0]).reshape(-1)
            cast = cast_bytes(part, cast_mode) if scales is None else cast_bytes_scaled(part, cast_mode, float(scales[l * no + o]))
            d[:, l, o, token_begin - d0:token_end - d0] = cast.reshape(nh, n, d_row)
    out = []
    for i in range(len(dst_blocks)):
        blk = np.ascontiguousarray(d[:, :, :, i * dst_page:(i + 1) * dst_page]).reshape(-1)
        out.append(O.kv_layout_permute(blk, O.KV_UNIVERSAL_TP, dst_kv, nl, no, dst_page, nh, d_row))
    return out


def table_slice(table: Sequence[int], token_begin: int, token_end: int, page: int) -> list:
    """The ids a call takes for one side: table[token_begin // page .. ceil(token_end / page))."""
    if token_begin == token_end:
        return []
    return [int(x) for x in table[token_begin // page:-(-token_end // page)]]

"""Oracle of the layout transform with the fused fp8 e4m3 <-> bf16 cast (kvbm_kernels_paged_permute_cast): the oracle's cast
(oracle.cast_e4m3_to_bf16 / cast_bf16_to_e4m3) of every element of a block, then oracle.kv_layout_permute with the
destination row.  The cast has no reference implementation (parity unpinned, DESIGN §5); it is pinned to the torch tables
under tests/golden by tests/test_oracle_permute_cast.py."""
from __future__ import annotations

from typing import Optional

import numpy as np

from oracle import oracle as O

CAST_NONE, CAST_FP8_TO_BF16, CAST_BF16_TO_FP8 = 0, 1, 2


def cast_bytes(data: np.ndarray, cast_mode: int) -> np.ndarray:
    """uint8 bytes of fp8 codes / bf16 patterns -> the uint8 bytes of the cast elements."""
    data = np.ascontiguousarray(data, dtype=np.uint8)
    if cast_mode == CAST_FP8_TO_BF16:
        return O.cast_e4m3_to_bf16(data).view(np.uint8)
    if cast_mode == CAST_BF16_TO_FP8:
        return O.cast_bf16_to_e4m3(data.view(np.uint16))
    return data


def dst_row_bytes(src_row_bytes: int, cast_mode: int) -> int:
    return {CAST_NONE: src_row_bytes, CAST_FP8_TO_BF16: 2 * src_row_bytes, CAST_BF16_TO_FP8: src_row_bytes // 2}[cast_mode]


def kv_layout_permute_cast(block: np.ndarray, src_kv: int, dst_kv: int, nl: int, no: int, nt: int, nh: int, src_row_bytes: int,
                           cast_mode: int, layers: Optional[range] = None, dst_old: Optional[np.ndarray] = None) -> np.ndarray:
    """One contiguous source block (uint8[nl*no*nt*nh*src_row_bytes]) cast element by element and re-ordered from `src_kv` to
    `dst_kv`.  With `layers`, only those layers move; every other byte keeps `dst_old`'s value (in the destination dtype)."""
    return O.kv_layout_permute(cast_bytes(block, cast_mode), src_kv, dst_kv, nl, no, nt, nh, dst_row_bytes(src_row_bytes, cast_mode),
                               layers=layers, dst_old=dst_old)

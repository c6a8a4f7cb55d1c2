"""Oracle of the scaled fp8 e4m3 <-> bf16 cast (kvbm_paged_copy_opts.cast_scales, kvbm_kernels_paged_permute_heads_scaled,
kvbm_kernels_paged_permute_gather_scaled): an engine's fp8 KV cache stores x / s and dequantises fp8 * s, with s the fp32 scale of
the fp8 side for one (layer, outer index).

    fp8 -> bf16   bf16_rne(fp32_rn(float(code) * s))          NaN codes -> 0x7fc0
    bf16 -> fp8   e4m3_satfinite_rne(fp32_rn(float(x) / s))   NaN -> 0x7f | sign of x

Both are numpy restatements in fp32 (IEEE products and quotients), pinned to torch CPU by the tables under tests/golden
(make_scaled_cast_tables.py); where torch overflows to NaN the oracle saturates to +-448, as the unscaled cast does.  With s = 1
both equal the unscaled oracle (oracle.cast_e4m3_to_bf16 / cast_bf16_to_e4m3)."""
from __future__ import annotations

from typing import Optional

import numpy as np

from oracle import oracle as O
from tests.cast_oracle import CAST_BF16_TO_FP8, CAST_FP8_TO_BF16, CAST_NONE, dst_row_bytes


def fp32_to_bf16_rne(f: np.ndarray) -> np.ndarray:
    """float32 -> bf16 bit patterns, round to nearest even; NaN -> 0x7fc0."""
    u = np.ascontiguousarray(f, dtype=np.float32).view(np.uint32).astype(np.uint64)
    out = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(f), np.uint16(0x7FC0), out)


def fp32_to_e4m3_satfinite_rne(q: np.ndarray) -> np.ndarray:
    """float32 -> e4m3fn codes, round to nearest even, saturating to +-448 (infinities included); NaN -> 0x7f | sign."""
    q = np.asarray(q, dtype=np.float32)
    a = np.minimum(np.abs(q.astype(np.float64)), 1e4)       # past 464 every value saturates; keeps frexp finite
    a = np.where(np.isnan(a), 0.0, a)
    _, ex = np.frexp(a)
    e = np.where(a < 2.0**-6, -6, ex - 1)                    # below the smallest normal: the subnormal step 2^-9
    k = np.rint(np.ldexp(a, 3 - e))                          # significand in steps of 2^(e-3), ties to even (exact scaling)
    code = np.minimum((e + 7) * 8 + (k - 8), 0x7E).astype(np.uint8)
    sign = (np.signbit(q).astype(np.uint8) << 7).astype(np.uint8)
    return np.where(np.isnan(q), np.uint8(0x7F), code) | sign


def e4m3_to_bf16_scaled(codes: np.ndarray, s: float) -> np.ndarray:
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    with np.errstate(over="ignore", invalid="ignore"):
        f = (O.cast_e4m3_to_bf16(codes).astype(np.uint32) << 16).view(np.float32) * np.float32(s)
    return np.where((codes & 0x7F) == 0x7F, np.uint16(0x7FC0), fp32_to_bf16_rne(f))


def bf16_to_e4m3_scaled(bits: np.ndarray, s: float) -> np.ndarray:
    bits = np.ascontiguousarray(bits, dtype=np.uint16)
    x = (bits.astype(np.uint32) << 16).view(np.float32)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        out = fp32_to_e4m3_satfinite_rne(x / np.float32(s))
    return np.where(np.isnan(x), np.uint8(0x7F) | ((bits >> 8).astype(np.uint8) & 0x80), out)


def cast_bytes_scaled(data: np.ndarray, cast_mode: int, s: float) -> np.ndarray:
    """uint8 bytes of fp8 codes / bf16 patterns -> the uint8 bytes of the scaled cast."""
    data = np.ascontiguousarray(data, dtype=np.uint8)
    if cast_mode == CAST_FP8_TO_BF16:
        return e4m3_to_bf16_scaled(data, s).view(np.uint8)
    if cast_mode == CAST_BF16_TO_FP8:
        return bf16_to_e4m3_scaled(data.view(np.uint16), s)
    assert cast_mode == CAST_NONE
    return data


def kv_layout_permute_cast_scaled(block: np.ndarray, src_kv: int, dst_kv: int, nl: int, no: int, nt: int, nh: int, src_row_bytes: int,
                                  cast_mode: int, scales: np.ndarray, layers: Optional[range] = None,
                                  dst_old: Optional[np.ndarray] = None) -> np.ndarray:
    """tests.cast_oracle.kv_layout_permute_cast with the scaled cast: every element of (layer l, outer o) is cast with
    scales[l * no + o] before the re-ordering."""
    block = np.ascontiguousarray(block, dtype=np.uint8)
    ein, eout = {CAST_FP8_TO_BF16: (1, 2), CAST_BF16_TO_FP8: (2, 1)}[cast_mode]
    n = block.size // ein
    # cast the block once per (layer, outer) scale and keep, per element, the result of its own (layer, outer)
    tags = _element_tags(src_kv, nl, no, nt, nh, src_row_bytes // ein)
    out = np.empty(n * eout, dtype=np.uint8)
    for lo in np.unique(tags):
        sel = tags == lo
        cast = cast_bytes_scaled(block, cast_mode, float(scales[lo])).reshape(n, eout)
        out.reshape(n, eout)[sel] = cast[sel]
    return O.kv_layout_permute(out, src_kv, dst_kv, nl, no, nt, nh, dst_row_bytes(src_row_bytes, cast_mode), layers=layers,
                               dst_old=dst_old)


def _element_tags(kv: int, nl: int, no: int, nt: int, nh: int, hd: int) -> np.ndarray:
    """l * no + o of every element of one block stored in format `kv` (element order of the block's bytes)."""
    shape = {1: (nh, nl, no, nt, hd), 2: (nl, nh, no, nt, hd), 3: (nl, no, nh, nt, hd), 4: (nl, no, nt, nh, hd)}[kv]
    axes = {1: (1, 2), 2: (0, 2), 3: (0, 1), 4: (0, 1)}[kv]
    idx = np.indices(shape, dtype=np.int64)
    return (idx[axes[0]] * no + idx[axes[1]]).reshape(-1)


def reshard_block_scaled(src_block: np.ndarray, dst_old: np.ndarray, src_kv: int, dst_kv: int, nl: int, no: int, nt: int, src_nh: int,
                         dst_nh: int, src_row_bytes: int, cast_mode: int, scales: np.ndarray, src_head_begin: int, dst_head_begin: int,
                         head_count: int, layers: Optional[range] = None) -> np.ndarray:
    """tests.reshard_oracle.reshard_block with the scaled cast: the window's elements of (layer l, outer o) are cast with
    scales[l * no + o]."""
    d_row = dst_row_bytes(src_row_bytes, cast_mode)
    s = O.kv_layout_permute(src_block, src_kv, O.KV_UNIVERSAL_TP, nl, no, nt, src_nh, src_row_bytes).reshape(src_nh, nl, no, nt, src_row_bytes)
    d = O.kv_layout_permute(dst_old, dst_kv, O.KV_UNIVERSAL_TP, nl, no, nt, dst_nh, d_row).reshape(dst_nh, nl, no, nt, d_row).copy()
    win = s[src_head_begin:src_head_begin + head_count]
    lrange = range(nl) if layers is None else layers
    for l in lrange:
        for o in range(no):
            part = np.ascontiguousarray(win[:, l, o]).reshape(-1)
            d[dst_head_begin:dst_head_begin + head_count, l, o] = cast_bytes_scaled(part, cast_mode, float(scales[l * no + o])).reshape(
                head_count, nt, d_row)
    return O.kv_layout_permute(d.reshape(-1), O.KV_UNIVERSAL_TP, dst_kv, nl, no, nt, dst_nh, d_row)

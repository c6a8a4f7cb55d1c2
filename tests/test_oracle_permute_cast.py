"""CPU checks of the oracle of the layout transform with the fused fp8 <-> bf16 cast (tests/cast_oracle.py): casting and
re-ordering commute for every ordered pair of KvBlockLayouts, and the composition carries the torch-generated cast tables
(tests/golden) through unchanged -- all 256 fp8 codes and all 65 536 bf16 patterns."""
import itertools
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests.cast_oracle import CAST_BF16_TO_FP8, CAST_FP8_TO_BF16, cast_bytes, kv_layout_permute_cast

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KVS = [O.KV_UNIVERSAL_TP, O.KV_UNIVERSAL_PP, O.KV_OPERATIONAL_HND, O.KV_OPERATIONAL_NHD]
SIZE_OF = {"h": "nh", "l": "nl", "o": "no", "t": "nt"}


def _splice(full: np.ndarray, old: np.ndarray, dst_kv: int, dims: dict, row: int, layers: range) -> np.ndarray:
    """`old` with the elements of `layers` taken from `full` (both destination blocks in dst_kv order)."""
    order = O.KV_DIM_ORDER[dst_kv]
    shape = [dims[SIZE_OF[c]] for c in order] + [row]
    out = old.reshape(shape).copy()
    sel = [slice(None)] * 5
    sel[order.index("l")] = slice(layers.start, layers.stop)
    out[tuple(sel)] = full.reshape(shape)[tuple(sel)]
    return out.reshape(-1)


@pytest.mark.parametrize("cast", [CAST_FP8_TO_BF16, CAST_BF16_TO_FP8], ids=["fp8_to_bf16", "bf16_to_fp8"])
@pytest.mark.parametrize("layers", [None, range(1, 3)], ids=["all_layers", "layers_1_3"])
def test_cast_then_permute_equals_permute_then_cast(cast, layers):
    dims = dict(nl=3, no=2, nt=5, nh=3)
    hd = 32
    src_elem, dst_elem = (1, 2) if cast == CAST_FP8_TO_BF16 else (2, 1)
    src_row, dst_row = hd * src_elem, hd * dst_elem
    n = dims["nl"] * dims["no"] * dims["nt"] * dims["nh"]
    rng = np.random.default_rng(5 + cast)
    for src_kv, dst_kv in itertools.product(KVS, KVS):
        block = rng.integers(0, 256, n * src_row, dtype=np.uint8)
        old = rng.integers(0, 256, n * dst_row, dtype=np.uint8)
        got = kv_layout_permute_cast(block, src_kv, dst_kv, dims["nl"], dims["no"], dims["nt"], dims["nh"], src_row, cast,
                                     layers=layers, dst_old=old)
        want = cast_bytes(O.kv_layout_permute(block, src_kv, dst_kv, dims["nl"], dims["no"], dims["nt"], dims["nh"], src_row), cast)
        if layers is not None:
            want = _splice(want, old, dst_kv, dims, dst_row, layers)
        assert np.array_equal(got, want), (src_kv, dst_kv)


def test_every_fp8_code_matches_the_torch_table():
    table = np.load(os.path.join(GOLD, "fp8_e4m3_to_bf16_torch.npy"))
    nl, no, nt, nh, hd = 2, 2, 4, 2, 16                       # 512 elements: every code twice
    codes = np.random.default_rng(1).permutation(np.arange(512) % 256).astype(np.uint8)
    for src_kv, dst_kv in ((O.KV_OPERATIONAL_NHD, O.KV_UNIVERSAL_TP), (O.KV_UNIVERSAL_PP, O.KV_OPERATIONAL_HND)):
        got = kv_layout_permute_cast(codes, src_kv, dst_kv, nl, no, nt, nh, hd, CAST_FP8_TO_BF16)
        want = O.kv_layout_permute(table[codes].view(np.uint8), src_kv, dst_kv, nl, no, nt, nh, 2 * hd)
        assert np.array_equal(got, want)


def test_every_bf16_pattern_matches_the_torch_table_up_to_saturation():
    """torch turns |x| > 464 into NaN; the cast saturates to +-448 (0x7e with the sign), as the paged copy's cast does."""
    table = np.load(os.path.join(GOLD, "bf16_to_fp8_e4m3_torch.npy"))
    bits = np.arange(65536, dtype=np.uint16)
    mag = bits & 0x7FFF
    overflow = ((table & 0x7F) == 0x7F) & ~(mag > 0x7F80)
    expect = table.copy()
    expect[overflow] = 0x7E | ((bits[overflow] >> 8) & 0x80).astype(np.uint8)
    nl, no, nt, nh, hd = 2, 2, 32, 8, 64                      # 65 536 elements
    pats = np.random.default_rng(2).permutation(bits)
    for src_kv, dst_kv in ((O.KV_UNIVERSAL_TP, O.KV_OPERATIONAL_NHD), (O.KV_OPERATIONAL_HND, O.KV_UNIVERSAL_PP)):
        got = kv_layout_permute_cast(pats.view(np.uint8), src_kv, dst_kv, nl, no, nt, nh, 2 * hd, CAST_BF16_TO_FP8)
        want = O.kv_layout_permute(expect[pats], src_kv, dst_kv, nl, no, nt, nh, hd)
        assert np.array_equal(got, want)

"""CPU checks of the scaled fp8 <-> bf16 cast: the oracle (tests/scaled_cast_oracle.py) against the torch tables under
tests/golden, its s = 1 case against the unscaled oracle, its commutation with the layout transform and head windows, the
ctypes mirrors of the two option structs, the exported symbols, and the argument checks that return before any CUDA call."""
import ctypes as C
import itertools
import os
import shutil
import subprocess

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, KvbmError, LayoutConfig, StorageKind, TransferManager, TransferOptions
from oracle import oracle as O
from tests.cast_oracle import CAST_BF16_TO_FP8, CAST_FP8_TO_BF16, kv_layout_permute_cast
from tests.golden.make_scaled_cast_tables import SCALES
from tests.scaled_cast_oracle import (_element_tags, bf16_to_e4m3_scaled, cast_bytes_scaled, e4m3_to_bf16_scaled,
                                      kv_layout_permute_cast_scaled, reshard_block_scaled)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
KVS = [O.KV_UNIVERSAL_TP, O.KV_UNIVERSAL_PP, O.KV_OPERATIONAL_HND, O.KV_OPERATIONAL_NHD]
CODES = np.arange(256, dtype=np.uint8)
BITS = np.arange(65536, dtype=np.uint16)


@pytest.mark.parametrize("i", range(len(SCALES)), ids=[f"s={s:g}" for s in SCALES])
def test_oracle_equals_the_torch_tables(i):
    s = float(SCALES[i])
    up = np.load(os.path.join(GOLD, "scaled_fp8_e4m3_to_bf16_torch.npy"))[i]
    got = e4m3_to_bf16_scaled(CODES, s)
    nan = (CODES & 0x7F) == 0x7F
    assert np.array_equal(got[~nan], up[~nan]) and (got[nan] == 0x7FC0).all()
    down = np.load(os.path.join(GOLD, "scaled_bf16_to_fp8_e4m3_torch.npy"))[i]
    x = (BITS.astype(np.uint32) << 16).view(np.float32)
    overflow = ((down & 0x7F) == 0x7F) & ~np.isnan(x)      # torch: NaN past 464; the cast saturates to +-448
    want = down.copy()
    want[overflow] = 0x7E | ((BITS[overflow] >> 8) & 0x80).astype(np.uint8)
    assert np.array_equal(bf16_to_e4m3_scaled(BITS, s), want)


def test_tables_cover_overflow_and_subnormals():
    down = np.load(os.path.join(GOLD, "scaled_bf16_to_fp8_e4m3_torch.npy"))
    finite = ~np.isnan((BITS.astype(np.uint32) << 16).view(np.float32)) & ((BITS & 0x7F80) != 0x7F80)
    sat = [int((((d & 0x7F) == 0x7F) & finite).sum()) for d in down]
    sub = [int((((d & 0x78) == 0) & ((d & 0x7) != 0)).sum()) for d in down]
    assert sat[list(SCALES).index(np.float32(2.0**-12))] > sat[0]       # the small scale overflows e4m3 for more of the range
    assert sub[list(SCALES).index(np.float32(600.0))] > sub[0]          # the large one lands more of it in the subnormals


def test_scale_one_is_the_unscaled_cast():
    assert np.array_equal(e4m3_to_bf16_scaled(CODES, 1.0), O.cast_e4m3_to_bf16(CODES))
    assert np.array_equal(bf16_to_e4m3_scaled(BITS, 1.0), O.cast_bf16_to_e4m3(BITS))


@pytest.mark.parametrize("cast", [CAST_FP8_TO_BF16, CAST_BF16_TO_FP8], ids=["fp8_to_bf16", "bf16_to_fp8"])
def test_scaled_cast_commutes_with_permute_and_head_windows(cast):
    nl, no, nt, nh, hd = 3, 2, 4, 3, 16
    ein, eout = (1, 2) if cast == CAST_FP8_TO_BF16 else (2, 1)
    n = nl * no * nt * nh
    rng = np.random.default_rng(7 + cast)
    scales = rng.uniform(0.01, 4, nl * no).astype(np.float32)
    for src_kv, dst_kv in itertools.product(KVS, KVS):
        block = rng.integers(0, 256, n * hd * ein, dtype=np.uint8)
        got = kv_layout_permute_cast_scaled(block, src_kv, dst_kv, nl, no, nt, nh, hd * ein, cast, scales)
        # permute first, then cast every element with the scale of its own (layer, outer)
        moved = O.kv_layout_permute(block, src_kv, dst_kv, nl, no, nt, nh, hd * ein).reshape(-1, ein)
        tags = _element_tags(dst_kv, nl, no, nt, nh, hd)
        want = np.empty((n * hd, eout), dtype=np.uint8)
        for lo in range(nl * no):
            want[tags == lo] = cast_bytes_scaled(moved[tags == lo].reshape(-1), cast, float(scales[lo])).reshape(-1, eout)
        assert np.array_equal(got, want.reshape(-1)), (src_kv, dst_kv)
        # a head window of the scaled transform is the same window of the full transform; other heads keep their bytes
        old = rng.integers(0, 256, n * hd * eout, dtype=np.uint8)
        win = reshard_block_scaled(block, old, src_kv, dst_kv, nl, no, nt, nh, nh, hd * ein, cast, scales, 1, 0, 2, layers=range(1, 3))
        tp = lambda b: O.kv_layout_permute(b, dst_kv, O.KV_UNIVERSAL_TP, nl, no, nt, nh, hd * eout).reshape(nh, nl, no, nt, -1)  # noqa: E731
        full, w, o = tp(got), tp(win), tp(old)
        assert np.array_equal(w[0:2, 1:3], full[1:3, 1:3]) and np.array_equal(w[2], o[2]) and np.array_equal(w[:, 0], o[:, 0])
    # s = 1 everywhere is the unscaled composition
    block = rng.integers(0, 256, n * hd * ein, dtype=np.uint8)
    ones = np.ones(nl * no, np.float32)
    assert np.array_equal(kv_layout_permute_cast_scaled(block, KVS[0], KVS[3], nl, no, nt, nh, hd * ein, cast, ones),
                          kv_layout_permute_cast(block, KVS[0], KVS[3], nl, no, nt, nh, hd * ein, cast))


def test_scaled_symbols_are_exported_and_listed():
    for s in ("kvbm_kernels_paged_permute_heads_scaled", "kvbm_kernels_paged_permute_gather_scaled"):
        assert s in K.EXPORTED_SYMBOLS and callable(getattr(K.lib(), s))


def test_option_structs_mirror_the_headers(tmp_path):
    gcc = shutil.which("gcc")
    cuda_inc = "/usr/local/cuda/include"
    if not gcc or not os.path.exists(os.path.join(cuda_inc, "cuda_runtime_api.h")):
        pytest.skip("gcc or the CUDA headers are not installed")
    structs = {"kvbm_paged_copy_opts": K.PagedCopyOpts, "kvbm_transfer_options": P._COptions}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "kvbm_kernels.h"', '#include "kvbm_physical.h"', "int main(void) {"]
    for cname, mirror in structs.items():
        lines.append(f'  printf("{cname} sizeof %zu\\n", sizeof({cname}));')
        for fname, _ in mirror._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    r = subprocess.run([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), "-I", cuda_inc, "-o", str(exe), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    c = {(a, b): int(v) for a, b, v in (ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True,
                                                                               check=True).stdout.splitlines())}
    for cname, mirror in structs.items():
        assert C.sizeof(mirror) == c[(cname, "sizeof")], cname
        for fname, _ in mirror._fields_:
            assert getattr(mirror, fname).offset == c[(cname, fname)], f"{cname}.{fname}"
    assert K.PagedCopyOpts._fields_[-1][0] == "cast_scales" and P._COptions._fields_[-1][0] == "num_cast_scales"


def test_scaled_entries_reject_scales_without_a_cast_before_any_cuda_call():
    """Host descriptors no check dereferences; every call returns before touching the GPU (this machine may have none)."""
    inval = K.CUDA_ERROR_INVALID_VALUE
    side = K.PermuteSide(K.PagedLayout(0x1000, 4096, 2048, 2048, 2, 2, 4), 0x2000, int(K.KvBlockLayout.OperationalNHD))
    fake = 0x3000
    assert K.paged_permute_heads(side, side, 1, 0, 2, 1, 0, 1, 0, 1, 16, 128, 0, cast_scales=fake) == inval
    assert K.paged_permute_heads(side, side, 0, 0, 2, 1, 0, 1, 0, 1, 16, 128, 0, cast_scales=fake) == inval   # even with nothing to move
    src = K.PermuteSource(side, 1, 0, 0, 1)
    assert K.paged_permute_gather([src], side, 1, 1, 0, 2, 16, 128, 0, cast_scales=fake) == inval
    assert K.paged_permute_gather([src], side, 1, 0, 0, 2, 16, 128, 0, cast_scales=fake) == inval
    lay = K.PagedLayout(0x1000, 4096, 2048, 2048, 2, 2, 4)
    dst = K.PagedDst(lay, 0x2000, 0x2000, 0, 0)
    assert K.paged_copy(lay, [dst], 1, 0, 2, 0, K.PagedCopyOpts(cast_scales=fake)) == inval
    assert K.paged_copy(lay, [dst], 0, 0, 2, 0, K.PagedCopyOpts(cast_scales=fake)) == inval
    # too many layers to pack the outer index above the layer of an item
    big = K.PagedLayout(0x1000, 4096, 2048, 2048, 70000, 2, 4)
    assert K.paged_copy(big, [K.PagedDst(K.PagedLayout(0x1000, 8192, 4096, 4096, 70000, 2, 4), 0x2000, 0x2000, 0, 0)], 1, 0, 1,
                        int(K.CastMode.FP8E4M3_TO_BF16), K.PagedCopyOpts(cast_scales=fake)) == inval


def test_manager_rejects_scales_without_a_cast_and_short_arrays():
    mgr = TransferManager(device=-1, worker_id=21)
    try:
        nl, no = 3, 2
        hs, bufs = [], []
        for w in (2, 1, 2):
            cfg = LayoutConfig(4, nl, no, 16, 64, dtype_width_bytes=w, allow_fp8=(w == 1))
            b = np.zeros(cfg.required_bytes(), dtype=np.uint8)
            bufs.append(b)
            hs.append(mgr.register_fully_contiguous(cfg, b.ctypes.data, b.size, StorageKind.System, 0))
        scales = np.ones(nl * no, dtype=np.float32)
        with pytest.raises(KvbmError) as e:
            mgr.execute_transfer(hs[0], [0], hs[2], [1], TransferOptions(cast_scales=scales))
        assert e.value.code == ErrorCode.ERR and "need a cast_mode" in e.value.msg
        with pytest.raises(KvbmError) as e:
            mgr.execute_transfer(hs[0], [0], hs[1], [1], TransferOptions(cast_mode=K.CastMode.BF16_TO_FP8E4M3, cast_scales=scales[:-1]))
        assert e.value.code == ErrorCode.RANGE and "num_layers * outer_dim = 6" in e.value.msg
        with pytest.raises(TypeError):
            TransferOptions(cast_scales=0x1000)._c()
        # host pools take the Memcpy strategy, whose rejection of the cast keeps its text
        with pytest.raises(KvbmError) as e:
            mgr.execute_transfer(hs[0], [0], hs[1], [1], TransferOptions(cast_mode=K.CastMode.BF16_TO_FP8E4M3, cast_scales=scales))
        assert e.value.code == ErrorCode.UNSUPPORTED and "CUDA strategies" in e.value.msg
    finally:
        mgr.close()

"""CPU checks of the re-shard gather (kvbm_kernels_paged_permute_gather, kvbm_manager_execute_gather): exported symbols, the
ctypes mirrors, the argument checks that return before any CUDA call, and the window bound over every plan."""
import ctypes as C
import itertools
import os
import shutil
import subprocess

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, HeadWindow, KvbmError, LayoutConfig, StorageKind, TransferManager, TransferOptions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KV = K.KvBlockLayout
INVAL = K.CUDA_ERROR_INVALID_VALUE


def test_gather_symbols_are_exported_and_listed():
    assert "kvbm_kernels_paged_permute_gather" in K.EXPORTED_SYMBOLS
    assert "kvbm_manager_execute_gather" in P.EXPORTED_SYMBOLS
    assert callable(K.lib().kvbm_kernels_paged_permute_gather) and callable(P.lib().kvbm_manager_execute_gather)


def test_permute_source_and_head_window_mirror_the_headers(tmp_path):
    gcc = shutil.which("gcc")
    cuda_inc = "/usr/local/cuda/include"
    if not gcc or not os.path.exists(os.path.join(cuda_inc, "cuda_runtime_api.h")):
        pytest.skip("gcc or the CUDA headers are not installed")
    structs = {"kvbm_permute_source": K.PermuteSource, "kvbm_permute_side": K.PermuteSide, "kvbm_head_window": P._CHeadWindow}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "kvbm_kernels.h"', '#include "kvbm_physical.h"', "int main(void) {",
             '  printf("max sources %d\\n", KVBM_GATHER_MAX_SOURCES);', '  printf("max heads %d\\n", KVBM_GATHER_MAX_HEADS);']
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
    assert c[("max", "sources")] == K.GATHER_MAX_SOURCES and c[("max", "heads")] == K.GATHER_MAX_HEADS
    for cname, mirror in structs.items():
        assert C.sizeof(mirror) == c[(cname, "sizeof")], cname
        for fname, _ in mirror._fields_:
            assert getattr(mirror, fname).offset == c[(cname, fname)], f"{cname}.{fname}"


# Host-side descriptors that no check ever dereferences: 2 layers x 2 outer, 16-token pages, head_dim 64 bf16 (128 B rows),
# NHD regions of nh heads.  Every call below is refused by the entry's argument checks before any CUDA call.
NL, NO, NT, ROW = 2, 2, 16, 128


def _side(nh, kv=KV.OperationalNHD, nl=NL, no=NO, row=ROW, ids=0x2000, base=0x1000):
    reg = NT * nh * row
    return K.PermuteSide(K.PagedLayout(base, reg, 8 * reg, reg, nl, no, 8), ids, int(kv))


def _src(nh, sb, db, k, **kw):
    return K.PermuteSource(_side(nh, **kw), nh, sb, db, k)


def _gather(srcs, dst=None, dst_nh=4, n=1, lb=0, le=NL, row=ROW, cast=0):
    return K.paged_permute_gather(srcs, _side(dst_nh) if dst is None else dst, dst_nh, n, lb, le, NT, row, cast)


def test_gather_argument_checks_before_any_cuda_call():
    two = [_src(2, 0, 0, 2), _src(2, 0, 2, 2)]
    # counts, ranges and cast mode
    assert _gather([]) == INVAL
    assert _gather([_src(2, 0, 0, 1)] * 17) == INVAL
    assert _gather(two, n=-1) == INVAL
    assert _gather(two, lb=1, le=0) == INVAL
    assert _gather(two, cast=3) == INVAL
    assert K.lib().kvbm_kernels_paged_permute_gather(None, 1, C.byref(_side(4)), 4, 1, 0, NL, NT, ROW, 0, None, 0, None, 0, None) == INVAL
    # the zero-count early return (no flags: nothing to launch)
    assert _gather(two, n=0) == 0 and _gather(two, lb=1, le=1) == 0
    # null sides and tables
    assert _gather(two, dst=_side(4, ids=0)) == INVAL
    assert _gather(two, dst=_side(4, base=0)) == INVAL
    assert _gather([_src(2, 0, 0, 2, ids=0), _src(2, 0, 2, 2)]) == INVAL
    assert _gather([_src(2, 0, 0, 2), _src(2, 0, 2, 2, base=0)]) == INVAL
    # windows: empty, past the source's heads, past the destination's heads, overlapping in the destination
    assert _gather([_src(2, 0, 0, 0), _src(2, 0, 2, 2)]) == INVAL
    assert _gather([_src(2, 1, 0, 2), _src(2, 0, 2, 2)]) == INVAL
    assert _gather([_src(2, 0, 0, 2), _src(2, 0, 3, 2)]) == INVAL
    assert _gather([_src(2, 2**32 - 1, 0, 2)]) == INVAL
    assert _gather([_src(2, 0, 0, 2), _src(2, 0, 1, 2)]) == INVAL
    assert _gather([_src(4, 0, 0, 3), _src(2, 0, 2, 2)]) == INVAL   # overlap is in the destination, whatever the sources
    # a source whose layers / outer dim differ from the destination
    assert _gather([_src(2, 0, 0, 2, nl=NL + 1), _src(2, 0, 2, 2)]) == INVAL
    assert _gather([_src(2, 0, 0, 2), _src(2, 0, 2, 2, no=1)]) == INVAL
    assert _gather(two, le=NL + 1) == INVAL
    # region = page * that side's heads * row, on each side
    assert _gather([K.PermuteSource(_side(2), 3, 0, 0, 2), _src(2, 0, 2, 2)]) == INVAL
    assert _gather(two, dst=_side(8)) == INVAL
    # the row and cast rules of paged_permute_heads: 8 B rows, 65 KiB rows, an odd bf16 row
    assert _gather([_src(2, 0, 0, 2, row=8)], row=8) == INVAL
    assert _gather(two, row=ROW + 8) == INVAL
    assert _gather(two, row=ROW + 1, cast=int(K.CastMode.BF16_TO_FP8E4M3)) == INVAL
    # strides that are not whole 16 B vectors, and a format without a kernel
    assert _gather([_src(2, 0, 0, 2, kv=KV.Custom), _src(2, 0, 2, 2)]) == INVAL
    assert _gather(two, dst=_side(4, kv=KV.Unknown)) == INVAL
    # more than KVBM_GATHER_MAX_HEADS destination heads covered
    assert _gather([_src(300, 0, 0, 257)], dst=_side(300), dst_nh=300) == INVAL


def _tps(H):
    return [tp for tp in range(1, 17) if H % tp == 0 or tp % H == 0]


@pytest.mark.parametrize("H", [1, 2, 4, 8, 16, 64])
def test_every_plan_fits_one_gather(H):
    """Every plan kvbm_tp_reshard_plan makes for TP degrees up to 16 fits one gather: at most 16 windows, disjoint in the
    destination, and no more covered heads than the kernel's map holds."""
    worst = 0
    for src_tp, dst_tp in itertools.product(_tps(H), _tps(H)):
        for rank in range(dst_tp):
            plan = P.tp_reshard_plan(H, src_tp, dst_tp, rank)
            worst = max(worst, len(plan))
            assert len(plan) <= K.GATHER_MAX_SOURCES, (H, src_tp, dst_tp, rank)
            assert sum(w.head_count for w in plan) <= K.GATHER_MAX_HEADS
            heads = [h for w in plan for h in range(w.dst_head_begin, w.dst_head_begin + w.head_count)]
            assert len(heads) == len(set(heads))
    assert worst == min(H, 16)   # TP16 -> TP1 (or H heads, one per source rank, when H < 16) is the widest plan


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_gather on host memory: the gather's own rejections, and the Memcpy strategy's
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def host_pools():
    mgr = TransferManager(device=-1, worker_id=11)
    nl, no, nt, hd = 2, 2, 16, 64
    bufs, hs = [], []
    for nh in (2, 2, 4):
        cfg = LayoutConfig(4, nl, no, nt, nh * hd, dtype_width_bytes=2, num_heads=nh)
        b = np.zeros(cfg.required_bytes(), dtype=np.uint8)
        h = mgr.register_fully_contiguous(cfg, b.ctypes.data, b.size, StorageKind.System, 0)
        mgr.set_kv_block_layout(h, KV.OperationalNHD)
        bufs.append(b)
        hs.append(h)
    yield mgr, hs
    mgr.close()


def _code(fn):
    with pytest.raises(KvbmError) as e:
        fn()
    return e.value


def test_manager_gather_rejections(host_pools):
    mgr, (a, b, d) = host_pools
    src = {0: (a, [0, 1]), 1: (b, [2, 3])}
    plan = [HeadWindow(0, 0, 0, 2), HeadWindow(1, 0, 2, 2)]
    e = _code(lambda: mgr.execute_gather(src, d, [1, 2], [HeadWindow(0, 0, 0, 2), HeadWindow(1, 0, 1, 2)]))
    assert e.code == ErrorCode.OVERLAP
    e = _code(lambda: mgr.execute_gather(src, d, [1, 2], [HeadWindow(0, 0, 0, 1)] * 17))
    assert e.code == ErrorCode.UNSUPPORTED and "at most 16" in e.msg
    e = _code(lambda: mgr.execute_gather(src, d, [1, 2], plan, TransferOptions(head_window=(0, 0, 2))))
    assert e.code == ErrorCode.ERR and "head_count" in e.msg
    e = _code(lambda: mgr.execute_gather(src, d, [1, 2], [HeadWindow(0, 0, 0, 0)]))
    assert e.code == ErrorCode.RANGE
    e = _code(lambda: mgr.execute_gather(src, d, [1, 2], [HeadWindow(0, 1, 0, 2)]))       # past source 0's heads
    assert e.code == ErrorCode.RANGE and "Head window" in e.msg
    # src_rank indexes the sources array (the Python wrapper packs the ranks the plan names)
    L = P.lib()
    hs = (C.c_uint64 * 1)(a)
    ids = (C.c_size_t * 2)(0, 1)
    sp = (C.POINTER(C.c_size_t) * 1)(C.cast(ids, C.POINTER(C.c_size_t)))
    w = (P._CHeadWindow * 1)(P._CHeadWindow(1, 0, 0, 2))
    tok = C.c_uint64()
    assert L.kvbm_manager_execute_gather(mgr._h, 1, hs, sp, d, ids, 2, w, 1, C.byref(P._COptions()), C.byref(tok)) == ErrorCode.RANGE
    # host pools take the Memcpy strategy, which has no permuting launch: the windowed transfer's text
    e = _code(lambda: mgr.execute_gather(src, d, [1, 2], plan))
    assert e.code == ErrorCode.UNSUPPORTED and "CUDA strategies" in e.msg
    e = _code(lambda: mgr.execute_gather({0: (a, [0]), 1: (b, [2, 3])}, d, [1, 2], plan))
    assert e.code == ErrorCode.LENGTH_MISMATCH

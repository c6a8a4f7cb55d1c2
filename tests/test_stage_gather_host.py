"""CPU checks of the staged gather (a PP x TP re-shard): kvbm_tp_pp_reshard_plan against tests/stage_oracle over every small
PP x TP group, the exported symbols and ctypes mirrors, the kernel entry's argument checks that return before any CUDA call,
and the manager's rejections on a host-only manager."""
import ctypes as C
import itertools
import os
import shutil
import subprocess

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, KvbmError, LayoutConfig, ShardWindow, StorageKind, TransferManager, TransferOptions
from tests.reshard_oracle import rank_heads
from tests.stage_oracle import stage_bounds, stage_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KV = K.KvBlockLayout
INVAL = K.CUDA_ERROR_INVALID_VALUE


def test_stage_symbols_are_exported_and_listed():
    for name in ("kvbm_kernels_paged_stage_gather", "kvbm_kernels_paged_stage_gather_streamed"):
        assert name in K.EXPORTED_SYMBOLS and callable(getattr(K.lib(), name))
    for name in ("kvbm_tp_pp_reshard_plan", "kvbm_manager_execute_stage_gather"):
        assert name in P.EXPORTED_SYMBOLS and callable(getattr(P.lib(), name))


def test_stage_source_and_shard_window_mirror_the_headers(tmp_path):
    gcc = shutil.which("gcc")
    cuda_inc = "/usr/local/cuda/include"
    if not gcc or not os.path.exists(os.path.join(cuda_inc, "cuda_runtime_api.h")):
        pytest.skip("gcc or the CUDA headers are not installed")
    structs = {"kvbm_stage_source": K.StageSource, "kvbm_shard_window": P._CShardWindow, "kvbm_permute_source": K.PermuteSource}
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


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_tp_pp_reshard_plan
# ---------------------------------------------------------------------------------------------------------------------
def _groups():
    return [(tp, pp) for tp in (1, 2, 4, 8) for pp in (1, 2, 3, 4) if tp * pp <= 8]


def _uneven(L, pp):
    """A partition of L layers over pp stages that is not the even split where one exists (the last stage one layer short)."""
    if pp == 1 or L < pp + 1:
        return None
    base = [L // pp] * pp
    base[-1] += L % pp
    base[0] += 1
    base[-1] -= 1
    return base if all(base) else None


def _as_tuples(plan):
    return [(w.src_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan]


def _tiles_once(H, L, src_tp, src_pp, sp, dst_tp, dst_pp, dp, rank, plan):
    """The windows cover the decode rank's (layer, head) cells exactly once, each from a source rank that holds that layer and
    head."""
    sb, db = stage_bounds(L, src_pp, sp), stage_bounds(L, dst_pp, dp)
    d0, d1 = db[rank // dst_tp], db[rank // dst_tp + 1]
    mine = rank_heads(H, dst_tp, rank % dst_tp)
    seen = np.zeros((d1 - d0, len(mine)), dtype=np.int64)
    for r, sl, dl, c, shb, dhb, k in plan:
        p, t = divmod(r, src_tp)
        assert p < src_pp and sl + c <= sb[p + 1] - sb[p] and dl + c <= d1 - d0
        assert sb[p] + sl == d0 + dl                    # the same global layers on both sides
        held = rank_heads(H, src_tp, t)
        for j in range(k):
            assert held.start + shb + j in held and held.start + shb + j == mine.start + dhb + j
        seen[dl:dl + c, dhb:dhb + k] += 1
    assert (seen == 1).all()


@pytest.mark.parametrize("H", [1, 2, 8, 16])
@pytest.mark.parametrize("L", [1, 7, 32, 80])
def test_plan_equals_the_oracle_and_tiles_every_decode_rank(H, L):
    checked = 0
    for (src_tp, src_pp), (dst_tp, dst_pp) in itertools.product(_groups(), _groups()):
        if (H % src_tp and src_tp % H) or (H % dst_tp and dst_tp % H):
            continue
        for sp, dp in itertools.product({None, tuple(_uneven(L, src_pp) or ()) or None}, {None, tuple(_uneven(L, dst_pp) or ()) or None}):
            if (sp is None and L % src_pp) or (dp is None and L % dst_pp) or src_pp > L or dst_pp > L:
                continue
            for rank in range(dst_tp * dst_pp):
                plan = _as_tuples(P.tp_pp_reshard_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, sp, dp))
                assert plan == stage_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, sp, dp), (src_tp, src_pp, sp, dst_tp, dst_pp, dp, rank)
                _tiles_once(H, L, src_tp, src_pp, sp, dst_tp, dst_pp, dp, rank, plan)
                assert len(plan) <= K.GATHER_MAX_SOURCES and sum(w[6] for w in plan) <= K.GATHER_MAX_HEADS * src_pp
                checked += 1
    assert checked > 0


@pytest.mark.parametrize("H,src_tp,dst_tp", [(8, 4, 2), (8, 1, 8), (2, 4, 1), (16, 2, 4)])
def test_pp1_on_both_sides_is_the_tp_plan_over_every_layer(H, src_tp, dst_tp):
    for rank in range(dst_tp):
        tp = P.tp_reshard_plan(H, src_tp, dst_tp, rank)
        pp = P.tp_pp_reshard_plan(H, 80, src_tp, 1, dst_tp, 1, rank)
        assert pp == [ShardWindow(w.src_rank, 0, 0, 80, w.src_head_begin, w.dst_head_begin, w.head_count) for w in tp]


def _plan_code(*args, **kw):
    with pytest.raises(KvbmError) as e:
        P.tp_pp_reshard_plan(*args, **kw)
    return e.value.code


def test_plan_errors():
    assert _plan_code(8, 7, 1, 2, 1, 1, 0) == ErrorCode.CONFIG                       # uneven split without a partition
    assert _plan_code(8, 8, 1, 1, 1, 3, 0) == ErrorCode.CONFIG
    assert _plan_code(8, 16, 1, 2, 1, 1, 0, src_stage_layers=[7, 8]) == ErrorCode.CONFIG   # does not sum to num_layers
    assert _plan_code(8, 16, 1, 2, 1, 1, 0, src_stage_layers=[16, 0]) == ErrorCode.CONFIG  # a zero stage
    assert _plan_code(8, 16, 1, 1, 1, 2, 0, dst_stage_layers=[10, 7]) == ErrorCode.CONFIG
    for zero in range(6):
        args = [8, 16, 1, 1, 1, 1]
        args[zero] = 0
        assert _plan_code(*args, 0) == ErrorCode.CONFIG
    assert _plan_code(8, 16, 3, 1, 1, 1, 0) == ErrorCode.CONFIG                      # 8 heads over TP 3
    assert _plan_code(8, 16, 1, 1, 2, 2, 4) == ErrorCode.RANGE                       # dst_rank past PP2 x TP2
    n = C.c_size_t()
    L = P.lib()
    assert L.kvbm_tp_pp_reshard_plan(8, 16, 2, 1, None, 1, 1, None, 0, None, 0, None) == ErrorCode.ERR
    assert L.kvbm_tp_pp_reshard_plan(8, 16, 2, 2, None, 1, 1, None, 0, None, 0, C.byref(n)) == 0 and n.value == 4
    out = (P._CShardWindow * 4)()
    assert L.kvbm_tp_pp_reshard_plan(8, 16, 2, 2, None, 1, 1, None, 0, out, 3, C.byref(n)) == ErrorCode.ERR


# ---------------------------------------------------------------------------------------------------------------------
# the kernel entry's argument checks (descriptors no check dereferences)
# ---------------------------------------------------------------------------------------------------------------------
NO, NT, ROW = 2, 16, 128


def _side(nh, nl, kv=KV.OperationalNHD, no=NO, ids=0x2000, base=0x1000):
    reg = NT * nh * ROW
    return K.PermuteSide(K.PagedLayout(base, reg, 8 * reg, reg, nl, no, 8), ids, int(kv))


def _ss(nh, nl, hb, db, k, sl, dl, c, **kw):
    return K.StageSource(K.PermuteSource(_side(nh, nl, **kw), nh, hb, db, k), sl, dl, c)


def _stage(srcs, dst_nh=4, dst_nl=8, n=1, lb=0, le=8):
    return K.paged_stage_gather(srcs, _side(dst_nh, dst_nl), dst_nh, n, lb, le, NT, ROW)


def test_stage_argument_checks_before_any_cuda_call():
    # two stages of two TP sources each: PP2 x TP2 -> TP1 over 8 layers
    ok = [_ss(2, 4, 0, 0, 2, 0, 0, 4), _ss(2, 4, 0, 2, 2, 0, 0, 4), _ss(2, 4, 0, 0, 2, 0, 4, 4), _ss(2, 4, 0, 2, 2, 0, 4, 4)]
    assert _stage(ok, n=0) == 0 and _stage(ok, lb=3, le=3) == 0          # empty ranges signal (nothing to signal here)
    assert _stage([]) == INVAL
    assert _stage([ok[0]] * 17) == INVAL
    # a partial layer overlap
    assert _stage([_ss(2, 4, 0, 0, 2, 0, 0, 4), _ss(2, 4, 0, 2, 2, 0, 0, 4), _ss(2, 4, 0, 0, 2, 0, 3, 4), _ss(2, 4, 0, 2, 2, 0, 4, 4)]) == INVAL
    # windows past the source's layers and past the destination's
    assert _stage(ok[:3] + [_ss(2, 4, 0, 2, 2, 1, 4, 4)]) == INVAL
    assert _stage(ok[:3] + [_ss(2, 8, 0, 2, 2, 0, 5, 4)]) == INVAL
    assert _stage([_ss(2, 4, 0, 0, 2, 0, 0, 0)] + ok[1:]) == INVAL        # no layers
    # an untiled range: layers 4..8 uncovered
    assert _stage(ok[:2]) == INVAL
    assert _stage(ok[:2], lb=2, le=5) == INVAL
    # head overlap within a stage (across stages the same heads are the point)
    assert _stage([ok[0], _ss(2, 4, 0, 1, 2, 0, 0, 4), ok[2], ok[3]]) == INVAL
    # 257 covered heads summed over stages, each stage within the limit
    big = [_ss(300, 4, 0, 0, 129, 0, 0, 4), _ss(300, 4, 0, 0, 128, 0, 4, 4)]
    assert K.paged_stage_gather(big, _side(300, 8), 300, 1, 0, 8, NT, ROW) == INVAL
    # a differing outer_dim
    assert _stage(ok[:3] + [_ss(2, 4, 0, 2, 2, 0, 4, 4, no=1)]) == INVAL
    # the streamed entry: its gate's rules first
    assert K.paged_stage_gather_streamed(ok, _side(4, 8), 4, 1, 0, 8, NT, ROW, 0, None, None) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_stage_gather on host memory: its own rejections, with codes and texts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def host_pools():
    mgr = TransferManager(device=-1, worker_id=12)
    no, nt, hd = 2, 16, 64
    bufs, hs = [], []
    for nl, nh in ((3, 2), (3, 2), (5, 2), (8, 4)):
        cfg = LayoutConfig(4, nl, no, nt, nh * hd, dtype_width_bytes=2, num_heads=nh)
        b = np.zeros(cfg.required_bytes(), dtype=np.uint8)
        h = mgr.register_fully_contiguous(cfg, b.ctypes.data, b.size, StorageKind.System, 0)
        mgr.set_kv_block_layout(h, KV.OperationalNHD)
        bufs.append(b)
        hs.append(h)
    yield mgr, hs
    mgr.close()


def _err(fn):
    with pytest.raises(KvbmError) as e:
        fn()
    return e.value


def test_manager_stage_gather_rejections(host_pools):
    mgr, (a, b, c, d) = host_pools
    src = {0: (a, [0, 1]), 1: (b, [2, 3]), 2: (c, [1, 0])}
    # stage 0: layers 0..3 of a and b (heads 0-1 and 2-3); stage 1: layers 0..5 of c as destination layers 3..8, both head pairs
    plan = [ShardWindow(0, 0, 0, 3, 0, 0, 2), ShardWindow(1, 0, 0, 3, 0, 2, 2), ShardWindow(2, 0, 3, 5, 0, 0, 2), ShardWindow(2, 0, 3, 5, 0, 2, 2)]
    go = lambda p, o=None, **kw: mgr.execute_stage_gather(src, d, [1, 2], p, o, **kw)  # noqa: E731
    e = _err(lambda: go([plan[0], ShardWindow(1, 0, 0, 3, 0, 1, 2)] + plan[2:]))
    assert e.code == ErrorCode.OVERLAP and "overlap in the destination" in e.msg
    e = _err(lambda: go(plan[:2] + [ShardWindow(2, 0, 2, 5, 0, 0, 2), plan[3]]))
    assert e.code == ErrorCode.OVERLAP and "partly overlap" in e.msg
    e = _err(lambda: go(plan[:2] + [ShardWindow(2, 0, 3, 0, 0, 0, 2)]))
    assert e.code == ErrorCode.RANGE and "no layers" in e.msg
    e = _err(lambda: go([ShardWindow(0, 0, 0, 1, 0, 0, 1)] * 17))
    assert e.code == ErrorCode.UNSUPPORTED and "at most 16" in e.msg
    e = _err(lambda: go(plan, TransferOptions(head_window=(0, 0, 2))))
    assert e.code == ErrorCode.ERR and "head_count" in e.msg
    e = _err(lambda: go(plan[:2] + [ShardWindow(2, 1, 3, 5, 0, 0, 2), plan[3]]))           # past c's 5 layers
    assert e.code == ErrorCode.RANGE and "source's num_layers" in e.msg
    e = _err(lambda: go(plan[:2] + [ShardWindow(2, 0, 4, 5, 0, 0, 2), ShardWindow(2, 0, 4, 5, 0, 2, 2)]))   # past the destination's 8
    assert e.code == ErrorCode.RANGE and "destination's num_layers" in e.msg
    e = _err(lambda: go(plan[:2]))                                                          # layers 3..8 untiled
    assert e.code == ErrorCode.RANGE and "destination layer 3" in e.msg
    e = _err(lambda: go(plan, TransferOptions(layer_range=range(0, 9))))
    assert e.code == ErrorCode.RANGE and "exceeds num_layers 8" in e.msg
    e = _err(lambda: go([ShardWindow(0, 1, 0, 3, 0, 0, 2)] + plan[1:]))                    # past a's 3 layers
    assert e.code == ErrorCode.RANGE
    e = _err(lambda: go([ShardWindow(0, 0, 0, 3, 1, 0, 2)] + plan[1:]))                    # past a's heads: the pair's own check
    assert e.code == ErrorCode.RANGE and "Head window" in e.msg
    e = _err(lambda: go(plan, ready_flags={0: 0, 1: 0, 2: 0}))
    assert e.code == ErrorCode.ERR and "no layer ready flags" in e.msg
    # a sub-range inside stage 0 needs no other stage; host pools then take the Memcpy strategy, the windowed transfer's text
    e = _err(lambda: go(plan[:2], TransferOptions(layer_range=range(0, 3))))
    assert e.code == ErrorCode.UNSUPPORTED and "CUDA strategies" in e.msg
    e = _err(lambda: go(plan))
    assert e.code == ErrorCode.UNSUPPORTED and "CUDA strategies" in e.msg
    # an empty range moves nothing
    assert go(plan, TransferOptions(layer_range=range(4, 4))) is not None

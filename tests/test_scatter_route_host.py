"""CPU checks of the routed re-paging scatter (each sequence of a prefill batch pushed to its own decode workers in one launch): the
exported symbols and the C layouts of kvbm_route_seq, kvbm_route_unit and kvbm_scatter_route_seq, the routed unit table against the
batch's, the kernel entries' argument checks that return before any CUDA call, the manager's rejections on a host-only manager in
their order, the plan helper, and the 40 instantiations in the built library.  The GPU cases are in tests/test_gpu_scatter_route.py."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import (ErrorCode, KvbmError, LayoutConfig, ScatterWindow, StorageKind, TransferManager, TransferOptions,
                                  tile_scatter_plan, tp_pp_scatter_plan)

KV = K.KvBlockLayout
INVAL = K.CUDA_ERROR_INVALID_VALUE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO, ROW = 2, 128


def test_routed_symbols_are_exported_and_listed():
    for name in ("kvbm_kernels_repage_route_units", "kvbm_kernels_paged_repage_scatter_routed",
                 "kvbm_kernels_paged_repage_scatter_routed_streamed"):
        assert name in K.EXPORTED_SYMBOLS and callable(getattr(K.lib(), name))
    assert "kvbm_manager_execute_repage_scatter_routed" in P.EXPORTED_SYMBOLS
    assert callable(P.lib().kvbm_manager_execute_repage_scatter_routed)


def _c_layout(header, struct, fields):
    """offsetof every field and sizeof the struct, as the C compiler lays it out."""
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("needs a C compiler")
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{header}"', "int main(void) {"]
    lines += [f'  printf("%zu\\n", offsetof({struct}, {f}));' for f in fields]
    lines += [f'  printf("%zu\\n", sizeof({struct}));', "  return 0;", "}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "s.c"), os.path.join(d, "s")
        with open(src, "w") as f:
            f.write("\n".join(lines))
        subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", "-o", exe, src], check=True)
        return [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]


@pytest.mark.parametrize("header,struct,mirror,names", [
    ("kvbm_kernels.h", "kvbm_route_seq", K.RouteSeq, ["token_begin", "token_end", "targets"]),
    ("kvbm_kernels.h", "kvbm_route_unit", K.RouteUnit, ["q0", "tokens", "small_k", "targets"]),
    ("kvbm_physical.h", "kvbm_scatter_route_seq", P._CScatterRouteSeq,
     ["token_begin", "token_end", "src_ids", "n_src", "dst_ids", "n_dst", "dst_mask"]),
], ids=["route_seq", "route_unit", "scatter_route_seq"])
def test_the_struct_mirrors_match_the_c_structs(header, struct, mirror, names):
    assert [f[0] for f in mirror._fields_] == names
    got = _c_layout(header, struct, names)
    assert got[:-1] == [getattr(mirror, f).offset for f in names]
    assert got[-1] == C.sizeof(mirror)
    assert C.sizeof(K.RouteUnit) == C.sizeof(K.RepageUnit) == 16


# ---------------------------------------------------------------------------------------------------------------------
# the routed unit table: the batch's with the fourth word replaced
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (16, 16), (1, 16), (48, 96), (96, 48), (64, 64)], ids=str)
def test_route_units_are_batch_units_with_the_last_word_replaced(ps, pd):
    rng = np.random.default_rng(ps * 1000 + pd)
    for trial in range(20):
        n = int(rng.integers(0, 40))
        seqs = []
        for _ in range(n):
            tb = int(rng.integers(0, 5000))
            seqs.append((tb, tb + int(rng.integers(0, 3000)) * int(rng.integers(0, 2))))
        masks = [int(rng.integers(1, 1 << 16)) for _ in seqs]
        want = K.repage_batch_units(seqs, ps, pd)
        got = K.repage_route_units([(b, e, m) for (b, e), m in zip(seqs, masks)], ps, pd)
        assert want is not None and got is not None
        assert got[1:] == want[1:]
        assert np.array_equal(got[0][:, :3], want[0][:, :3])
        assert got[0][:, 3].tolist() == [masks[s] for s in want[0][:, 3]]


def test_route_units_share_the_batch_rules():
    top = (1 << 32) - 64
    for seqs, ps, pd in (([(9, 8)], 16, 64), ([(0, 64)], 0, 64), ([(0, 64)], 48, 64), ([(top, top + 1)], 16, 64)):
        assert K.repage_batch_units(seqs, ps, pd) is None
        assert K.repage_route_units([s + (1,) for s in seqs], ps, pd) is None
    n, a, b = C.c_size_t(), C.c_size_t(), C.c_size_t()
    assert K.lib().kvbm_kernels_repage_route_units(None, 2, 16, 64, None, 0, C.byref(n), C.byref(a), C.byref(b)) != 0
    # capacity below the count: counted, min(count, cap) written
    seqs = [(3, 200, 5), (7, 90, 2)]
    full = K.repage_route_units(seqs, 16, 64)[0]
    out = np.full((2, 4), 0xDEAD, dtype=np.uint32)
    arr = K._route_seqs(seqs)
    assert K.lib().kvbm_kernels_repage_route_units(C.cast(arr, C.c_void_p), 2, 16, 64, out.ctypes.data, 2, C.byref(n), C.byref(a),
                                                   C.byref(b)) == 0
    assert n.value == len(full) > 2 and np.array_equal(out, full[:2])


# ---------------------------------------------------------------------------------------------------------------------
# the kernel entries' argument checks (descriptors no check dereferences)
# ---------------------------------------------------------------------------------------------------------------------
def _side(nh, nl, page, no=NO, ids=0x2000, base=0x1000):
    reg = page * nh * ROW
    return K.PermuteSide(K.PagedLayout(base, reg, 8 * reg, reg, nl, no, 8), ids, int(KV.OperationalNHD))


def _t(nh, nl, sb, db, k, sl, dl, c, page=64, **kw):
    return K.ScatterTarget(_side(nh, nl, page, **kw), nh, sb, db, k, sl, dl, c, None)


# stage 0: source layers 0..4 to two decode ranks (heads 0-1 and 2-3); stage 1: layers 4..6 to a third
OK = [_t(2, 4, 0, 0, 2, 0, 0, 4, ids=0x2100), _t(2, 4, 2, 0, 2, 0, 0, 4, ids=0x2200, base=0x1100), _t(2, 2, 0, 0, 2, 4, 0, 2, base=0x1200)]
SEQS = [(0, 64, 0b011), (70, 130, 0b100)]


def _rs(targets=OK, seqs=SEQS, ps=16, pd=64, lb=0, le=6, cast=0, scales=None, units=None, streamed=None):
    if units is None:
        u = K.repage_route_units(seqs, ps, pd)
        units = (0x7000, len(u[0]) if u is not None else 0)
    s = _side(4, 6, ps)
    if streamed is not None:
        return K.paged_repage_scatter_routed_streamed(s, 4, ps, targets, pd, seqs, *units, lb, le, ROW, cast, scales, streamed)
    return K.paged_repage_scatter_routed(s, 4, ps, targets, pd, seqs, *units, lb, le, ROW, cast, scales)


def test_routed_argument_checks_before_any_cuda_call():
    # nothing to move signals (nothing to signal here): no sequences, only empty ranges, an empty layer range
    assert _rs(seqs=[]) == 0 and _rs(seqs=[(9, 9, 1), (70, 70, 4)]) == 0 and _rs(lb=3, le=3) == 0
    # the routing: a mask of 0, a bit at num_targets (3) or above, also on an empty sequence
    assert _rs(seqs=[(0, 64, 0b011), (70, 130, 0)]) == INVAL
    assert _rs(seqs=[(0, 64, 0b1011), (70, 130, 1)]) == INVAL
    assert _rs(seqs=[(0, 64, 1 << 31), (70, 130, 1)]) == INVAL
    assert _rs(seqs=[(0, 64, 1), (9, 9, 0)]) == INVAL
    assert _rs(seqs=[(0, 64, 1), (9, 9, 8)]) == INVAL
    # sixteen targets take bit 15, not bit 16
    sixteen = [_t(2, 6, 0, 0, 2, 0, 0, 6, ids=0x3000 + 0x100 * i, base=0x4000 + 0x100 * i) for i in range(16)]
    assert _rs(targets=sixteen, seqs=[(0, 64, 1 << 16)]) == INVAL
    # the batch's own rules: a reversed range, a unit count other than the helper's, a null unit table, a null seqs
    assert _rs(seqs=[(0, 64, 1), (9, 8, 1)], units=(0x7000, 2)) == INVAL
    assert _rs(units=(0x7000, 4)) == INVAL and _rs(units=(0x7000, 2)) == INVAL
    assert _rs(units=(0, 3)) == INVAL
    arr = (K.ScatterTarget * 3)(*OK)
    assert K.lib().kvbm_kernels_paged_repage_scatter_routed(C.byref(_side(4, 6, 16)), 4, 16, arr, 3, 64, None, 2, 0x7000, 3, 0, 6, ROW, 0,
                                                           None, 0, None, 0, None) == INVAL
    # the single scatter's rules
    assert _rs(lb=4, le=3) == INVAL
    assert _rs(targets=[]) == INVAL and _rs(targets=[OK[0]] * 17, seqs=[(0, 64, 1)]) == INVAL
    assert _rs(cast=3) == INVAL
    assert _rs(scales=0x5000) == INVAL                                       # scales without a cast
    assert _rs(le=7) == INVAL
    assert _rs(targets=OK[:2], seqs=[(0, 64, 1)]) == INVAL                   # source layers 4..6 uncovered
    assert _rs(targets=OK[:2] + [_t(2, 2, 0, 0, 2, 3, 0, 2)]) == INVAL      # partly overlapping stages
    # the streamed entry: a null stream descriptor, a descriptor without ready flags
    u = K.repage_route_units(SEQS, 16, 64)
    assert K.paged_repage_scatter_routed_streamed(_side(4, 6, 16), 4, 16, OK, 64, SEQS, 0x7000, len(u[0]), 0, 6, ROW, 0, None, None) == INVAL
    assert _rs(streamed=K.PermuteStream()) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# the plan helper
# ---------------------------------------------------------------------------------------------------------------------
def test_tile_scatter_plan():
    one = tp_pp_scatter_plan(8, 4, 2, 1, 4, 1, 0)       # prefill TP2 rank 0 -> one TP4 decode worker: ranks 0 and 1
    ranks = 4
    plan = tile_scatter_plan(one, 3, ranks)
    assert len(plan) == 3 * len(one)
    for w in range(3):
        for a, b in zip(one, plan[w * len(one):(w + 1) * len(one)]):
            assert b.dst_rank == a.dst_rank + w * ranks and (b.src_layer_begin, b.head_count) == (a.src_layer_begin, a.head_count)
    with pytest.raises(ValueError):
        tile_scatter_plan(one, 2, 1)
    with pytest.raises(ValueError):
        tile_scatter_plan(one, 0, ranks)


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_repage_scatter_routed on host memory: its rejections in order, with codes and texts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def host_pools():
    """a: the source, 6 layers, 4 heads, 16-token pages; b, c: 4 layers, 2 heads, 64; d: 2 layers, 2 heads, 64; e: 2 layers,
    2 heads, 32-token pages; f: like b."""
    mgr = TransferManager(device=-1, worker_id=17)
    no, hd = 2, 64
    bufs, hs = [], []
    for nl, nh, page in ((6, 4, 16), (4, 2, 64), (4, 2, 64), (2, 2, 64), (2, 2, 32), (4, 2, 64)):
        cfg = LayoutConfig(8, nl, no, page, nh * hd, dtype_width_bytes=2, num_heads=nh)
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


# the source's layers 0..4 to destinations 0 and 1 (heads 0-1, 2-3), layers 4..6 to destination 2
PLAN = [ScatterWindow(0, 0, 0, 4, 0, 0, 2), ScatterWindow(1, 0, 0, 4, 2, 0, 2), ScatterWindow(2, 4, 0, 2, 0, 0, 2)]
CUDA_ONLY = "direct CUDA strategy only"


def _routed(mgr, hs, plan, seqs, o=None, dsts=(1, 2, 3), **kw):
    return mgr.execute_repage_scatter_routed(hs[0], [hs[i] if i < len(hs) else 999 for i in dsts], seqs, plan, o, **kw)


def _seq(tokens=range(0, 64), src=(0, 1, 2, 3), **dst):
    return (tokens, list(src), {int(k[1:]): v for k, v in dst.items()})


def test_the_routing_rejections_in_order(host_pools):
    mgr, hs = host_pools
    go = lambda seqs, plan=PLAN, **kw: _routed(mgr, hs, plan, seqs, **kw)  # noqa: E731
    bad_mask = [_seq(d0=[5]), _seq(range(64, 128), (4, 5, 6, 7))]               # the second sequence goes nowhere
    # with a layer stream, its shape first; then the windows' checks, even when a sequence is also misrouted
    e = _err(lambda: go(bad_mask, ready_flags=0))
    assert e.code == ErrorCode.ERR and "ready flags" in e.msg
    e = _err(lambda: go(bad_mask, dsts=(1, 1, 3)))
    assert e.code == ErrorCode.OVERLAP and "one layout" in e.msg
    e = _err(lambda: go(bad_mask, plan=PLAN[:2] + [ScatterWindow(3, 4, 0, 2, 0, 0, 2)]))
    assert e.code == ErrorCode.RANGE and "names destination 3" in e.msg
    # then more than 32 destinations
    e = _err(lambda: go(bad_mask, dsts=(1, 2, 3) + (5,) * 30))
    assert e.code == ErrorCode.OVERLAP                                           # the windows' duplicate-handle check comes first
    many = [hs[1], hs[2], hs[3]] + [10_000 + i for i in range(30)]                # distinct handles, never looked up
    e = _err(lambda: mgr.execute_repage_scatter_routed(hs[0], many, [_seq(d0=[5])], PLAN))
    assert e.code == ErrorCode.UNSUPPORTED and "at most 32 destinations" in e.msg
    # then, sequence by sequence, the routing, before the second sequence's token range
    e = _err(lambda: go(bad_mask))
    assert e.code == ErrorCode.RANGE and "sequence 1 is routed to no destination" in e.msg
    e = _err(lambda: go([_seq(d0=[5]), _seq(range(70, 64), (), d3=[])], dsts=(1, 2, 3, 4)))
    assert e.code == ErrorCode.RANGE and "sequence 1 is routed to a destination no window writes" in e.msg
    e = _err(lambda: go([_seq(range(70, 64), (), d0=[]), _seq(d1=[5], d3=[5])]))
    assert e.code == ErrorCode.RANGE and "sequence 1 is routed past the 3 destinations" in e.msg
    # then the single scatter's checks, sequence by sequence: the token range before the second one's id counts
    e = _err(lambda: go([_seq(range(70, 64), (), d0=[]), _seq(src=(0, 1, 2), d0=[5])]))
    assert e.code == ErrorCode.RANGE and "Token range" in e.msg
    e = _err(lambda: go([_seq(range(9, 9), (), d0=[]), _seq(src=(0, 1, 2), d0=[5])]))
    assert e.code == ErrorCode.LENGTH_MISMATCH
    e = _err(lambda: go([_seq(d0=[5]), _seq(src=(0, 1, 2), d0=[5])]))            # a non-empty sequence's strategy comes first
    assert e.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in e.msg
    # a routed destination's id list is range-checked, an unrouted one's is not read
    e = _err(lambda: go([_seq(d0=[8])]))
    assert e.code == ErrorCode.RANGE and "out of range for destination" in e.msg
    assert "direct CUDA" in _err(lambda: go([_seq(d0=[5], d1=[5])])).msg


def test_unrouted_id_lists_are_not_read(host_pools):
    """A NULL id list for an unrouted destination is accepted: the request gets as far as the strategy (a host-only manager has
    no direct CUDA one)."""
    mgr, hs = host_pools
    cs = (P._CScatterRouteSeq * 1)()
    src = (C.c_size_t * 4)(0, 1, 2, 3)
    d0 = (C.c_size_t * 1)(5)
    dp = (C.POINTER(C.c_size_t) * 3)(C.cast(d0, C.POINTER(C.c_size_t)), None, None)
    cs[0].token_begin, cs[0].token_end, cs[0].src_ids, cs[0].n_src = 0, 64, C.addressof(src), 4
    cs[0].dst_ids, cs[0].n_dst, cs[0].dst_mask = C.addressof(dp), 1, 0b001
    ws = (P._CScatterWindow * 3)(*[P._CScatterWindow(w.dst_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin,
                                                      w.dst_head_begin, w.head_count) for w in PLAN])
    hsa = (C.c_uint64 * 3)(hs[1], hs[2], hs[3])
    o, tok = TransferOptions()._c(), C.c_uint64()
    rc = P.lib().kvbm_manager_execute_repage_scatter_routed(mgr._h, hs[0], 3, hsa, cs, 1, ws, 3, None, C.byref(o), C.byref(tok))
    assert rc == ErrorCode.UNSUPPORTED and CUDA_ONLY in P.lib().kvbm_last_error().decode()
    # the same call routed to destination 1, whose list is NULL: rejected as a null list
    cs[0].dst_mask = 0b011
    rc = P.lib().kvbm_manager_execute_repage_scatter_routed(mgr._h, hs[0], 3, hsa, cs, 1, ws, 3, None, C.byref(o), C.byref(tok))
    assert rc == ErrorCode.ERR and "null block id list" in P.lib().kvbm_last_error().decode()


def test_duplicates_count_over_routed_sequences_only(host_pools):
    """Destination block 5 in two sequences routed to different destinations is accepted (the call reaches the strategy); in two
    sequences routed to one destination it is KVBM_ERR_DUPLICATE_DST, after every per-sequence check."""
    mgr, hs = host_pools
    go = lambda seqs: _routed(mgr, hs, PLAN, seqs)  # noqa: E731
    two = (range(64, 128), (4, 5, 6, 7))
    e = _err(lambda: go([_seq(d0=[5], d1=[9]), _seq(*two, d1=[5], d0=[9])]))
    assert e.code == ErrorCode.RANGE                                              # 9 is past the 8 blocks: the per-sequence check
    e = _err(lambda: go([_seq(d0=[5]), _seq(*two, d1=[5])]))
    assert e.code == ErrorCode.UNSUPPORTED and CUDA_ONLY in e.msg
    e = _err(lambda: go([_seq(d0=[5]), _seq(*two, d0=[5])]))
    assert e.code == ErrorCode.UNSUPPORTED                                        # the strategy of a non-empty sequence comes first


def test_nothing_to_move_returns_at_once(host_pools):
    mgr, hs = host_pools
    go = lambda seqs, **kw: _routed(mgr, hs, PLAN, seqs, **kw)  # noqa: E731
    assert go([]) is not None
    assert go([_seq(range(9, 9), (), d0=[]), _seq(range(70, 70), (), d2=[])]) is not None
    assert go([_seq(d0=[5])], o=TransferOptions(layer_range=range(4, 4))) is not None


def test_python_rejects_indices_past_a_32_bit_mask(host_pools):
    mgr, hs = host_pools
    with pytest.raises(ValueError):
        _routed(mgr, hs, PLAN, [_seq(d32=[5])])


# ---------------------------------------------------------------------------------------------------------------------
# the instantiations in the built library
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s, pp) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True)) for pp in (True, False)}
NEW = ("kvbm_paged_repage_route_kernel", "kvbm_gated_repage_route_kernel")


def test_the_route_instantiations_are_what_the_library_contains():
    """40 kernels: the 20 walks of with_repage_kernel for each of the two families; tests/test_gpu_scatter_route.py reaches each.
    No new name contains 'scatter', 'batch', 'push_seqs' or '_stage_'."""
    so = os.path.join(ROOT, "dynamo_b200", "libkvbm_kernels.so")
    tool = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
    if not os.path.exists(so) or tool is None:
        pytest.skip("needs the built libkvbm_kernels.so and cuobjdump")
    txt = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    found = set()
    for name in re.findall(r"Function : (\S+)", txt):
        m = re.search(r"(kvbm_[a-z0-9_]+?_kernel)I((?:L[ib]\d+E)+)E", name)
        if m and "route" in m.group(1):
            assert m.group(1) in NEW
            c, p, s, pp = (int(v) if t == "i" else v == "1" for t, v in re.findall(r"L([ib])(\d+)E", m.group(2)))
            found.add((m.group(1), c, p, s, pp))
    assert len(WALKS) == 20 and found == {(k,) + w for k in NEW for w in WALKS}
    assert not any(s in k for k in NEW for s in ("scatter", "batch", "push_seqs", "_stage_"))

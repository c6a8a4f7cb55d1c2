"""CPU checks of layer streaming on the layout-transforming hand-offs (kvbm_kernels_paged_permute_gather_streamed,
kvbm_kernels_paged_repage_gather_streamed, kvbm_manager_execute_gather_streamed, kvbm_manager_execute_repage_gather_streamed):
the exported symbols, the ctypes mirrors against the C layout, the gate's argument checks that return before any CUDA call, and
the manager's rejection table on a host-only manager, where every check runs before the missing device is reported."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, HeadWindow, KvbmError, TransferOptions, tp_reshard_plan
from tests.test_repage_host import host_mgr  # noqa: F401  (the host-only manager fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KV = K.KvBlockLayout
INVAL = K.CUDA_ERROR_INVALID_VALUE


def test_streamed_symbols_are_exported_and_listed():
    for name in ("kvbm_kernels_paged_permute_gather_streamed", "kvbm_kernels_paged_repage_gather_streamed"):
        assert name in K.EXPORTED_SYMBOLS and callable(getattr(K.lib(), name))
    for name in ("kvbm_manager_execute_gather_streamed", "kvbm_manager_execute_repage_gather_streamed"):
        assert name in P.EXPORTED_SYMBOLS and callable(getattr(P.lib(), name))


def test_stream_structs_mirror_the_headers(tmp_path):
    gcc = shutil.which("gcc")
    cuda_inc = "/usr/local/cuda/include"
    if not gcc or not os.path.exists(os.path.join(cuda_inc, "cuda_runtime_api.h")):
        pytest.skip("gcc or the CUDA headers are not installed")
    structs = {"kvbm_permute_stream": K.PermuteStream, "kvbm_layer_stream": P._CLayerStream}
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
        assert c[(cname, "sizeof")] == C.sizeof(mirror), cname
        for fname, _ in mirror._fields_:
            assert c[(cname, fname)] == getattr(mirror, fname).offset, (cname, fname)


# ---------------------------------------------------------------------------------------------------------------------
# the kernel entries: the gate's own checks, then the twin's, all before any CUDA call
# ---------------------------------------------------------------------------------------------------------------------
NL, NO, ROW = 2, 2, 128


def _side(page, nh, kv=KV.OperationalNHD, row=ROW, ids=0x2000, base=0x1000):
    reg = page * nh * row
    return K.PermuteSide(K.PagedLayout(base, reg, 8 * reg, reg, NL, NO, 8), ids, int(kv))


def _src(page=16, nh=2, sb=0, db=0, k=2, **kw):
    return K.PermuteSource(_side(page, nh, **kw), nh, sb, db, k)


def _st(n=2, mode=K.GATE_STREAM_WAIT, ws=0x3000, null=None):
    st = K.PermuteStream()
    for s in range(n):
        st.layer_ready_flags[s] = None if s == null else 0x5000 + 64 * s
    st.sync_workspace = ws or None
    st.gate_mode = mode
    return st


def _g(srcs, st, dnh=4, nb=4, lb=0, le=NL, page=16, cast=0, scales=None, dst=None):
    return K.paged_permute_gather_streamed(srcs, _side(page, dnh) if dst is None else dst, dnh, nb, lb, le, page, ROW, cast, scales, st)


def _rg(srcs, st, dnh=4, ps=16, pd=64, tb=0, te=32, lb=0, le=NL, cast=0, dst=None):
    return K.paged_repage_gather_streamed(srcs, ps, _side(pd, dnh) if dst is None else dst, dnh, pd, tb, te, lb, le, ROW, cast, None, st)


@pytest.mark.parametrize("entry", ["gather", "repage_gather"])
def test_gate_argument_checks_before_any_cuda_call(entry):
    two = [_src(db=0), _src(db=2)]
    call = _g if entry == "gather" else _rg
    assert call(two, None) == INVAL                                 # no descriptor
    assert call(two, _st(null=1)) == INVAL                          # a used source without ready flags
    assert call(two, _st(mode=3)) == INVAL and call(two, _st(mode=-1)) == INVAL
    assert call(two, _st(mode=K.GATE_SPIN, ws=0)) == INVAL          # the spinning form without a workspace
    # a ready-flag array past the used sources is not looked at: the twin's empty-range return (nothing to signal) succeeds
    st = _st(n=2)
    assert call(two, st, lb=1, le=1) == 0


def test_gather_twin_checks_through_the_streamed_entry():
    two = [_src(db=0), _src(db=2)]
    st = _st()
    assert _g(two, st, lb=1, le=0) == INVAL
    assert _g(two, st, cast=3) == INVAL
    assert _g(two, st, scales=0x4000) == INVAL                      # scales without a cast
    assert _g([], _st(n=0)) == INVAL
    assert _g([_src(db=i % 4, k=1) for i in range(17)], _st(n=16)) == INVAL
    assert _g([_src(), _src(db=1)], st) == INVAL                    # overlapping windows
    assert _g([_src(k=0), _src(db=2)], st) == INVAL
    assert _g(two, st, le=NL + 1) == INVAL
    assert _g(two, st, dst=_side(16, 4, ids=0)) == INVAL
    # the gather's 256 covered heads apply to one source too (the unstreamed one-source entry has no such limit)
    wide = [K.PermuteSource(_side(16, 260), 260, 0, 0, 260)]
    assert _g(wide, _st(n=1), dnh=260, dst=_side(16, 260)) == INVAL


def test_repage_gather_twin_checks_through_the_streamed_entry():
    two = [_src(db=0), _src(db=2)]
    st = _st()
    assert _rg(two, st, tb=5, te=4) == INVAL
    assert _rg(two, st, ps=0) == INVAL
    assert _rg([_src(page=48), _src(page=48, db=2)], st, ps=48) == INVAL   # pages that do not divide
    assert _rg(two, st, dst=_side(32, 4)) == INVAL                  # the destination's region at its page
    assert _rg(two, st, tb=2**32 - 70, te=2**32 - 1) == INVAL


# ---------------------------------------------------------------------------------------------------------------------
# the manager entries on a host-only manager
# ---------------------------------------------------------------------------------------------------------------------
def _err(fn):
    with pytest.raises(KvbmError) as e:
        fn()
    return e.value


def test_manager_streamed_rejections(host_mgr):  # noqa: F811
    mgr, reg = host_mgr
    s0, s1, d = reg(16, nh=2), reg(16, nh=2), reg(16, nh=4)
    plan = tp_reshard_plan(4, 2, 1, 0)
    flags = {0: 0x5000, 1: 0x6000}
    sources = {0: (s0, [0, 1]), 1: (s1, [2, 3])}

    def gather(**kw):
        a = dict(sources=sources, dst=d, dst_block_ids=[4, 5], plan=plan, ready_flags=flags, options=None)
        a.update(kw)
        return lambda: mgr.execute_gather_streamed(a["sources"], a["dst"], a["dst_block_ids"], a["plan"], a["ready_flags"], a["options"])

    # new: a source without flags
    e = _err(gather(ready_flags={0: 0x5000}))
    assert e.code == ErrorCode.ERR and "source 1 has no layer ready flags" in e.msg
    # the twin's checks, with its codes and texts
    e = _err(gather(plan=[]))
    assert e.code == ErrorCode.ERR and "at least one source and one window" in e.msg
    e = _err(gather(plan=[HeadWindow(0, 0, 0, 2), HeadWindow(1, 0, 1, 2)]))
    assert e.code == ErrorCode.OVERLAP
    for o in (TransferOptions(layer_ready_flags=0x1000), TransferOptions(layer_done_flags=0x1000), TransferOptions(multicast=1)):
        e = _err(gather(options=o))
        assert e.code == ErrorCode.UNSUPPORTED and "layer streaming / multicast are not available" in e.msg
    e = _err(gather(plan=[HeadWindow(0, 1, 0, 2)]))
    assert e.code == ErrorCode.RANGE and "Head window" in e.msg
    assert _err(gather(dst=0xDEAD)).code == ErrorCode.HANDLE
    # CUDA: a host-only manager, after every other check
    e = _err(gather())
    assert e.code == ErrorCode.CUDA and "without a CUDA device" in e.msg

    rsources = {0: (s0, [0, 1, 2]), 1: (s1, [3, 4, 5])}
    rd = reg(64, nh=4)

    def repage(**kw):
        a = dict(sources=rsources, dst=rd, dst_block_ids=[3], plan=plan, tokens=range(5, 40), ready_flags=flags, options=None)
        a.update(kw)
        return lambda: mgr.execute_repage_gather_streamed(a["sources"], a["dst"], a["dst_block_ids"], a["plan"], a["tokens"],
                                                          a["ready_flags"], a["options"])

    e = _err(repage(ready_flags={1: 0x6000}))
    assert e.code == ErrorCode.ERR and "source 0 has no layer ready flags" in e.msg
    e = _err(repage(options=TransferOptions(layer_ready_flags=0x1000)))
    assert e.code == ErrorCode.UNSUPPORTED and "re-paging transfer takes no" in e.msg
    e = _err(repage(sources={0: (s0, [0, 1, 2]), 1: (reg(32, nh=2), [3, 4, 5])}))
    assert e.code == ErrorCode.INCOMPATIBLE and "one page size" in e.msg
    e = _err(repage(sources={0: (s0, [0, 1]), 1: (s1, [3, 4])}))
    assert e.code == ErrorCode.LENGTH_MISMATCH
    # empty ranges: accepted before the strategy, as the twin
    assert mgr.execute_repage_gather_streamed({0: (s0, []), 1: (s1, [])}, rd, [], plan, range(7, 7), flags).is_complete()
    e = _err(repage())
    assert e.code == ErrorCode.CUDA and "without a CUDA device" in e.msg
    assert mgr.bytes_moved() == 0 and mgr.h2d_bytes() == 0


def test_manager_streamed_layer_stream_shape(host_mgr):  # noqa: F811
    """The kvbm_layer_stream itself, through the C entries: NULL, a NULL table, a source count that differs, a NULL entry."""
    mgr, reg = host_mgr
    s0, d = reg(16, nh=2), reg(16, nh=2)
    hs = (C.c_uint64 * 1)(s0)
    ws = (P._CHeadWindow * 1)(P._CHeadWindow(0, 0, 0, 2))
    PP = C.POINTER(C.c_size_t)
    ids = (C.c_size_t * 1)(0)
    sp = (PP * 1)(C.cast(ids, PP))
    did = (C.c_size_t * 1)(1)
    o = P._COptions()
    L = P.lib()
    flags = (C.c_void_p * 1)(0x5000)
    null_entry = (C.c_void_p * 1)(None)
    cases = [(None, ErrorCode.ERR, b"kvbm_layer_stream"),
             (P._CLayerStream(None, 1, None), ErrorCode.ERR, b"kvbm_layer_stream"),
             (P._CLayerStream(C.cast(flags, C.c_void_p), 2, None), ErrorCode.LENGTH_MISMATCH, b"names 2 sources"),
             (P._CLayerStream(C.cast(null_entry, C.c_void_p), 1, None), ErrorCode.ERR, b"source 0 has no layer ready flags")]
    for ls, code, text in cases:
        arg = C.byref(ls) if ls is not None else None
        rc = L.kvbm_manager_execute_gather_streamed(mgr._h, 1, hs, sp, d, did, 1, ws, 1, arg, C.byref(o), None)
        assert rc == code and text in L.kvbm_last_error()
        rc = L.kvbm_manager_execute_repage_gather_streamed(mgr._h, 1, hs, sp, 1, d, did, 1, 0, 16, ws, 1, arg, C.byref(o), None)
        assert rc == code and text in L.kvbm_last_error()
    good = P._CLayerStream(C.cast(flags, C.c_void_p), 1, None)
    rc = L.kvbm_manager_execute_gather_streamed(mgr._h, 1, hs, sp, d, did, 1, ws, 1, C.byref(good), C.byref(o), None)
    assert rc == ErrorCode.CUDA                                      # every check passed: the missing device is reported

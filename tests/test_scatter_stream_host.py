"""CPU checks of the streamed re-paging scatter: the exported symbols, every rejection of the kernel entry before any CUDA call
(the gate's own rules and a sample of the scatter's reached through the streamed entry), the manager's rejections on a host-only
manager with the first rejection pinned and codes and texts equal to execute_repage_scatter's, and the gated push kernel's
instantiations in the built library.  The accepted calls launch on the GPU in tests/test_gpu_scatter_stream.py."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from dynamo_b200 import kernels as K
from dynamo_b200 import physical as P
from dynamo_b200.physical import ErrorCode, ScatterWindow, TransferOptions
from tests.test_repage_scatter_host import OK, PLAN, ROOT, _err, _go, _side, _t, host_pools  # noqa: F401

INVAL = K.CUDA_ERROR_INVALID_VALUE


def test_streamed_scatter_symbols_are_exported_and_listed():
    assert "kvbm_kernels_paged_repage_scatter_streamed" in K.EXPORTED_SYMBOLS
    assert callable(K.lib().kvbm_kernels_paged_repage_scatter_streamed)
    assert "kvbm_manager_execute_repage_scatter_streamed" in P.EXPORTED_SYMBOLS
    assert callable(P.lib().kvbm_manager_execute_repage_scatter_streamed)


def _st(ready=0x3000, gate_mode=K.GATE_SPIN, ws=0x4000):
    st = K.PermuteStream()
    st.layer_ready_flags[0] = ready or None
    st.gate_mode = gate_mode
    st.sync_workspace = ws or None
    st.epoch = 1
    return st


def _ss(targets=OK, st="default", ps=16, pd=64, tb=0, te=64, lb=0, le=6, cast=0, scales=None, row=128):
    st = _st() if st == "default" else st
    return K.paged_repage_scatter_streamed(_side(4, 6, ps), 4, ps, targets, pd, tb, te, lb, le, row, cast, scales, st)


def test_the_gate_rules_come_before_any_cuda_call():
    assert _ss(st=None) == INVAL                                   # no descriptor
    assert _ss(st=_st(ready=0)) == INVAL                           # the source's ready flags
    assert _ss(st=_st(gate_mode=-1)) == INVAL                      # gate mode out of range
    assert _ss(st=_st(gate_mode=K.GATE_STREAM_WAIT + 1)) == INVAL
    assert _ss(st=_st(ws=0)) == INVAL                              # the spinning form without a workspace
    # the gate's rules win over the scatter's own: a bad descriptor with an empty range still fails
    assert _ss(st=None, tb=9, te=9) == INVAL
    # the other ready-flag entries are not read
    st = _st()
    st.layer_ready_flags[1] = None
    assert _ss(st=st, tb=9, te=9) == 0


def test_the_scatters_own_rules_through_the_streamed_entry():
    for gate in (K.GATE_SPIN, K.GATE_STREAM_WAIT, K.GATE_AUTO):
        st = _st(gate_mode=gate)
        assert _ss(st=st, tb=9, te=9) == 0 and _ss(st=st, lb=3, le=3) == 0     # empty ranges signal (nothing to signal here)
        assert _ss(st=st, tb=9, te=8) == INVAL
        assert _ss(st=st, lb=4, le=3) == INVAL
        assert _ss([], st=st) == INVAL
        assert _ss([OK[0]] * 17, st=st) == INVAL
        assert _ss(st=st, cast=3) == INVAL
        assert _ss(st=st, scales=0x5000) == INVAL                  # scales without a cast
        assert _ss(st=st, row=120) == INVAL                        # not whole 16 B vectors
        assert _ss(st=st, le=7) == INVAL                           # past the source's layers
        assert _ss(OK[:2], st=st) == INVAL                         # source layers 4..6 uncovered
        assert _ss(OK[:2] + [_t(2, 2, 0, 0, 2, 3, 0, 2)], st=st) == INVAL    # stages that overlap partly
        assert _ss(OK[:2] + [_t(2, 2, 0, 1, 2, 4, 0, 2)], st=st) == INVAL    # past the destination's heads


# ---------------------------------------------------------------------------------------------------------------------
# kvbm_manager_execute_repage_scatter_streamed on host memory
# ---------------------------------------------------------------------------------------------------------------------
def _go_streamed(mgr, hs, plan, o=None, tokens=range(0, 64), n_src=4, dsts=(1, 2, 3), dst_ids=None, ready=0x3000):
    """test_repage_scatter_host._go's request through the streamed entry."""
    ids = dst_ids if dst_ids is not None else [[5]] * len(dsts)
    return mgr.execute_repage_scatter_streamed(hs[0], list(range(n_src)), [hs[i] if i < len(hs) else 999 for i in dsts], ids, plan, tokens,
                                               ready, o)


def _raw(mgr, hs, ls):
    """The C entry with a hand-made layer stream over the PLAN request."""
    ids = (C.c_size_t * 4)(0, 1, 2, 3)
    d = (C.c_size_t * 1)(5)
    dp = (C.POINTER(C.c_size_t) * 3)(*[C.cast(d, C.POINTER(C.c_size_t))] * 3)
    dh = (C.c_uint64 * 3)(hs[1], hs[2], hs[3])
    ws = (P._CScatterWindow * 3)(*[P._CScatterWindow(w.dst_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin,
                                                     w.dst_head_begin, w.head_count) for w in PLAN])
    o = TransferOptions()._c()
    tok = C.c_uint64()
    rc = P.lib().kvbm_manager_execute_repage_scatter_streamed(mgr._h, hs[0], ids, 4, 3, dh, dp, 1, 0, 64, ws, 3, ls, C.byref(o), C.byref(tok))
    return rc, P.lib().kvbm_last_error().decode() if rc else ""


def test_manager_layer_stream_shape_comes_first(host_pools):
    mgr, hs = host_pools
    assert _raw(mgr, hs, None)[0] == ErrorCode.ERR
    ls = P.TransferManager._layer_stream([0], {}, 0)              # a null entry
    rc, msg = _raw(mgr, hs, C.byref(ls))
    assert rc == ErrorCode.ERR and "source 0 has no layer ready flags" in msg
    ls = P.TransferManager._layer_stream([0, 1], {0: 0x3000, 1: 0x3000}, 0)
    rc, msg = _raw(mgr, hs, C.byref(ls))
    assert rc == ErrorCode.LENGTH_MISMATCH and "names 2 sources" in msg
    ls = P.TransferManager._layer_stream([0], {0: 0x3000}, 0)
    ls.src_layer_ready_flags = None
    assert _raw(mgr, hs, C.byref(ls))[0] == ErrorCode.ERR
    # the shape before the request's own first rule (an empty plan)
    e = _err(lambda: mgr.execute_repage_scatter_streamed(hs[0], [0], [hs[1]], [[5]], [], range(0, 64), 0))
    assert e.code == ErrorCode.ERR and "no layer ready flags" in e.msg


BAD = [
    dict(plan=[]),
    dict(o=TransferOptions(head_window=(0, 0, 1))),
    dict(plan=[ScatterWindow(0, 0, 0, 1, 0, 0, 1)] * 17),
    dict(plan=PLAN[:2] + [ScatterWindow(3, 4, 0, 2, 0, 0, 2)]),
    dict(plan=PLAN[:2] + [ScatterWindow(2, 4, 0, 2, 0, 0, 0)]),
    dict(plan=PLAN[:2] + [ScatterWindow(2, 4, 0, 0, 0, 0, 2)]),
    dict(plan=PLAN[:2] + [ScatterWindow(2, 3, 0, 2, 0, 0, 2)]),
    dict(plan=PLAN + [ScatterWindow(0, 0, 0, 4, 3, 1, 1)]),
    dict(dsts=(1, 1, 3)),
    dict(dsts=(1, 2, 9)),
    dict(plan=PLAN[:2] + [ScatterWindow(2, 4, 0, 3, 0, 0, 2)]),
    dict(plan=PLAN[:2] + [ScatterWindow(2, 4, 1, 2, 0, 0, 2)]),
    dict(plan=PLAN[:2]),
    dict(plan=[ScatterWindow(0, 0, 0, 4, 3, 0, 2)] + PLAN[1:]),
    dict(dsts=(1, 2, 4)),
    dict(o=TransferOptions(layer_done_flags=0x100)),
    dict(o=TransferOptions(layer_ready_flags=0x100)),
    dict(o=TransferOptions(multicast=1)),
    dict(tokens=range(70, 64)),
    dict(o=TransferOptions(layer_range=range(0, 7))),
    dict(n_src=3),
    dict(tokens=range(0, 128), n_src=8, dst_ids=[[5, 6], [5, 5], [5, 6]]),
    dict(dst_ids=[[5], [8], [5]]),
    # two checks failing at once: the earlier one wins, as in execute_repage_scatter
    dict(plan=PLAN + [ScatterWindow(0, 0, 0, 4, 3, 1, 1)], dsts=(1, 2, 9)),
    dict(plan=PLAN[:2], dsts=(1, 2, 9)),
    dict(plan=[ScatterWindow(0, 0, 0, 4, 3, 0, 2), PLAN[1]]),
    dict(plan=PLAN[:2] + [ScatterWindow(2, 4, 0, 2, 3, 0, 2)], dsts=(1, 2, 4)),
    dict(tokens=range(70, 64), dsts=(1, 2, 4)),
    dict(o=TransferOptions(layer_range=range(0, 7)), tokens=range(70, 64)),
    dict(o=TransferOptions(layer_range=range(0, 7)), n_src=3),
]


def test_manager_rejections_equal_the_unstreamed_entrys(host_pools):
    """Every bad request gives the streamed entry the code and text execute_repage_scatter gives it."""
    mgr, hs = host_pools
    for bad in BAD:
        kw = dict(bad)
        plan, o = kw.pop("plan", PLAN), kw.pop("o", None)
        want = _err(lambda: _go(mgr, hs, plan, o, **kw))
        got = _err(lambda: _go_streamed(mgr, hs, plan, o, **kw))
        assert (got.code, got.msg) == (want.code, want.msg), bad


def test_manager_a_well_formed_request_reaches_the_strategy(host_pools):
    """Past every request check, the host-only manager refuses the CUDA strategy, streamed or not; empty ranges move nothing."""
    mgr, hs = host_pools
    for o in (None, TransferOptions(per_dst_done_flags=[0, 0, 0], done_flag=0, gate_mode=K.GATE_SPIN, max_ctas=3)):
        e = _err(lambda: _go_streamed(mgr, hs, PLAN, o))
        assert e.code == ErrorCode.UNSUPPORTED and "direct CUDA strategy only" in e.msg
    assert _go_streamed(mgr, hs, PLAN, tokens=range(9, 9), n_src=0, dst_ids=[[], [], []]) is not None
    assert _go_streamed(mgr, hs, PLAN, TransferOptions(layer_range=range(4, 4))) is not None


# ---------------------------------------------------------------------------------------------------------------------
# the instantiations in the built library
# ---------------------------------------------------------------------------------------------------------------------
EXPECTED = {(c, p, s, pp) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True)) for pp in (True, False)}


def test_the_push_instantiations_are_what_the_library_contains():
    """20 kernels: the walks of with_walk_kernel x the small page's split; tests/test_gpu_scatter_stream.py reaches each."""
    assert len(EXPECTED) == 20
    so = os.path.join(ROOT, "dynamo_b200", "libkvbm_kernels.so")
    tool = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
    if not os.path.exists(so) or tool is None:
        pytest.skip("needs the built libkvbm_kernels.so and cuobjdump")
    txt = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    found = set()
    for name in re.findall(r"Function : (\S+)", txt):
        m = re.search(r"(kvbm_[a-z0-9_]+?_kernel)I((?:L[ib]\d+E)+)E", name)
        if m and m.group(1) == "kvbm_gated_repage_push_kernel":
            c, p, s, pp = (int(v) if t == "i" else v == "1" for t, v in re.findall(r"L([ib])(\d+)E", m.group(2)))
            found.add((c, p, s, pp))
    assert found == EXPECTED

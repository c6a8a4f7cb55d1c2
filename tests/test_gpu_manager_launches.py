"""What each layout-transforming manager entry launches, for each request shape: the kernels and copies the CUDA profiler
records for one call, in order, with the call's bytes_moved and h2d_bytes deltas.  Every case also compares the whole
destination pool, byte for byte, with the oracle of its rig (tests/test_gpu_stage_gather.py's for the permuting entries,
tests/test_gpu_repage_batch.py's for the re-paging ones).  The streamed forms run behind flags already released, in both
gate modes."""
import warnings

import pytest
import torch
from torch.autograd import DeviceType

from dynamo_b200 import kernels as K
from dynamo_b200.physical import HeadWindow, ShardWindow, TransferManager, TransferOptions, tp_pp_reshard_plan, tp_reshard_plan
from tests.test_gpu_repage_batch import BatchRig
from tests.test_gpu_stage_gather import StageRig, _register

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
EPOCH = 4


def _windows(plan, ranks):
    return [(ranks.index(w.src_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
            for w in plan]


def _shard(plan, L):
    """A HeadWindow plan as ShardWindows over every layer (a PP1 plan)."""
    return [w if isinstance(w, ShardWindow) else ShardWindow(w.src_rank, 0, 0, L, w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan]


def _stage_rig(mgr, plan, H, L, src_tp, src_pp, dst_tp, dst_pp, rank, src_nh=None):
    """A permuting rig (one page size) of the plan, its pools registered: UniversalTP sources, an OperationalNHD destination."""
    ranks = sorted({w.src_rank for w in plan})
    srcs = [(L // src_pp, src_nh or max(1, H // src_tp), KV.UniversalTP) for _ in ranks]
    r = StageRig(srcs, _windows(_shard(plan, L // src_pp), ranks), L // dst_pp, max(1, H // dst_tp), KV.OperationalNHD, seed=len(plan) + H)
    return r, ranks, [_register(mgr, p, KV.UniversalTP) for p in r.srcs], _register(mgr, r.dst, KV.OperationalNHD)


def _batch_rig(mgr, plan, H, L, src_tp, src_pp, dst_tp, dst_pp, rank, seqs):
    """A re-paging rig (16-token source pages, 64-token destination pages) of the plan over `seqs`, its pools registered."""
    ranks = sorted({w.src_rank for w in plan})
    srcs = [(L // src_pp, max(1, H // src_tp), KV.UniversalTP) for _ in ranks]
    r = BatchRig(srcs, _windows(_shard(plan, L // src_pp), ranks), L // dst_pp, max(1, H // dst_tp), KV.OperationalNHD, seqs, seed=len(seqs) + H)
    return r, ranks, [_register(mgr, p, KV.UniversalTP) for p in r.srcs], _register(mgr, r.dst, KV.OperationalNHD)


def _ids(x):
    return [int(v) for v in x]


def _stream_kw(r, ranks):
    for p in r.srcs:
        p.ready.fill_(EPOCH)
    torch.cuda.synchronize()
    return dict(ready_flags={rk: r.srcs[i].ready.data_ptr() for i, rk in enumerate(ranks)}, layer_done_flags=r.layer_done.data_ptr())


def _opts(gate=None):
    return TransferOptions(epoch=EPOCH, gate_mode=gate) if gate is not None else TransferOptions(epoch=EPOCH)


TP4_TP2 = (8, 2, 4, 1, 2, 1, 0)          # H, L, src_tp, src_pp, dst_tp, dst_pp, rank
PP2TP4_TP2 = (8, 4, 4, 2, 2, 1, 1)
PP2TP2_TP1 = (4, 4, 2, 2, 1, 1, 0)
ONE = (4, 2, 1, 1, 1, 1, 0)              # one source over every head and layer
SEQS3 = [(5, 150), (40, 41), (96, 200)]


def _plan(shape):
    H, L, stp, spp, dtp, dpp, rank = shape
    return tp_reshard_plan(H, stp, dtp, rank) if spp == dpp == 1 else tp_pp_reshard_plan(H, L, stp, spp, dtp, dpp, rank)


# every case builds its rig on the manager and returns it (its check() is the oracle's) with the call; `gate`: None, or the
# streamed form's gate mode
def _repage(mgr):
    r, ranks, hs, dh = _batch_rig(mgr, [HeadWindow(0, 0, 0, 4)], *ONE, [(21, 170)])
    return r, lambda: mgr.execute_repage(hs[0], _ids(r.sids[0][0]), dh, _ids(r.dids[0]), range(21, 170), _opts())


def _repage_gather(shape, gate=None):
    def case(mgr):
        plan = _plan(shape)
        r, ranks, hs, dh = _batch_rig(mgr, plan, *shape, [(21, 170)])
        src = {rk: (hs[i], _ids(r.sids[i][0])) for i, rk in enumerate(ranks)}
        if gate is None:
            return r, lambda: mgr.execute_repage_gather(src, dh, _ids(r.dids[0]), plan, range(21, 170), _opts())
        kw = _stream_kw(r, ranks)
        return r, lambda: mgr.execute_repage_gather_streamed(src, dh, _ids(r.dids[0]), plan, range(21, 170), kw["ready_flags"], _opts(gate),
                                                             kw["layer_done_flags"])
    return case


def _stage_repage(gate=None):
    def case(mgr):
        plan = _plan(PP2TP2_TP1)
        r, ranks, hs, dh = _batch_rig(mgr, plan, *PP2TP2_TP1, [(21, 170)])
        src = {rk: (hs[i], _ids(r.sids[i][0])) for i, rk in enumerate(ranks)}
        kw = _stream_kw(r, ranks) if gate is not None else {}
        return r, lambda: mgr.execute_stage_repage_gather(src, dh, _ids(r.dids[0]), plan, range(21, 170), _opts(gate), **kw)
    return case


def _batch(seqs, gate=None):
    def case(mgr):
        plan = _plan(PP2TP2_TP1)
        r, ranks, hs, dh = _batch_rig(mgr, plan, *PP2TP2_TP1, seqs)
        reqs = [(range(tb, te), {rk: _ids(r.sids[i][q]) for i, rk in enumerate(ranks)}, _ids(r.dids[q])) for q, (tb, te) in enumerate(r.seqs)]
        kw = _stream_kw(r, ranks) if gate is not None else {}
        return r, lambda: mgr.execute_repage_batch(dict(zip(ranks, hs)), dh, reqs, plan, _opts(gate), **kw)
    return case


def _gather(shape, gate=None, src_nh=None):
    def case(mgr):
        plan = [HeadWindow(0, 0, 0, src_nh)] if src_nh else _plan(shape)
        r, ranks, hs, dh = _stage_rig(mgr, plan, *shape, src_nh=src_nh)
        src = {rk: (hs[i], _ids(r.sids[i])) for i, rk in enumerate(ranks)}
        if gate is None:
            return r, lambda: mgr.execute_gather(src, dh, _ids(r.dids), plan, _opts())
        kw = _stream_kw(r, ranks)
        return r, lambda: mgr.execute_gather_streamed(src, dh, _ids(r.dids), plan, kw["ready_flags"], _opts(gate), kw["layer_done_flags"])
    return case


def _transfer_320_heads(mgr):
    r, ranks, hs, dh = _stage_rig(mgr, [HeadWindow(0, 0, 0, 320)], 320, 2, 1, 1, 1, 1, 0, src_nh=320)
    return r, lambda: mgr.execute_transfer(hs[0], _ids(r.sids[0]), dh, _ids(r.dids), _opts())


def _stage_gather(gate=None):
    def case(mgr):
        plan = _plan(PP2TP4_TP2)
        r, ranks, hs, dh = _stage_rig(mgr, plan, *PP2TP4_TP2)
        src = {rk: (hs[i], _ids(r.sids[i])) for i, rk in enumerate(ranks)}
        kw = _stream_kw(r, ranks) if gate is not None else {}
        return r, lambda: mgr.execute_stage_gather(src, dh, _ids(r.dids), plan, _opts(gate), **kw)
    return case


SPIN, WAIT = K.GATE_SPIN, K.GATE_STREAM_WAIT
CASES = {
    "repage": _repage,
    "repage_gather_one_window": _repage_gather(ONE),
    "repage_gather_tp": _repage_gather(TP4_TP2),
    "gather_tp": _gather(TP4_TP2),
    "gather_one_window_320_heads": _gather((320, 2, 1, 1, 1, 1, 0), src_nh=320),
    "transfer_320_heads": _transfer_320_heads,
    "stage_gather": _stage_gather(),
    "stage_repage_gather": _stage_repage(),
    "batch_1": _batch([(21, 170)]),
    "batch_3": _batch(SEQS3),
}
for _g, _n in ((SPIN, "spin"), (WAIT, "stream_wait")):
    CASES["gather_streamed_" + _n] = _gather(TP4_TP2, _g)
    CASES["stage_gather_streamed_" + _n] = _stage_gather(_g)
    CASES["repage_gather_streamed_" + _n] = _repage_gather(TP4_TP2, _g)
    CASES["stage_repage_gather_streamed_" + _n] = _stage_repage(_g)
    CASES["batch_3_streamed_" + _n] = _batch(SEQS3, _g)


ENQUEUE = ("cudaMemcpyAsync", "cudaLaunchKernel")
WINDOWS = 4      # profile windows one case may take before a complete one


def _window(events):
    """The copies and kernels a profile window holds, in enqueue order, or None when the window is incomplete.  The order is that
    of the window's cudaMemcpyAsync / cudaLaunchKernel runtime records (their correlation ids); a kernel is named by the device
    record of the same correlation id, and a device record of a call made outside the window is not this call's.  CUPTI has been
    seen to drop records in two ways, with the library's bytes right each time:
    - in a process whose earlier profiler sessions ran many launches, the device record of every staged pinned -> device copy,
      window after window, while keeping its cudaMemcpyAsync record: a copy is therefore named by its call (H2D), and by its
      device record when there is one, which must then be that direction;
    - now and then, every record of a window: a window with no enqueue call, or with a kernel launch whose device record is
      missing, is incomplete."""
    calls = sorted((e for e in events if e.device_type() != DeviceType.CUDA and e.name() in ENQUEUE), key=lambda e: e.correlation_id())
    device = {e.correlation_id(): e.name() for e in events if e.device_type() == DeviceType.CUDA}
    if not calls or any(c.name() == "cudaLaunchKernel" and c.correlation_id() not in device for c in calls):
        return None
    names = []
    for c in calls:
        d = device.get(c.correlation_id())
        if c.name() == "cudaMemcpyAsync":
            names.append(H2D if d is None or d.startswith(H2D) else d)
        else:
            names.append(d.split("(")[0].removeprefix("void ").removeprefix("kvbm::").strip())
    return names


def _describe(events):
    return "; ".join(f"{'gpu' if e.device_type() == DeviceType.CUDA else 'cpu'} {e.name()[:48]} c{e.correlation_id()}"
                     for e in sorted(events, key=lambda e: e.correlation_id()) if e.device_type() == DeviceType.CUDA or e.name() in ENQUEUE)


def run_case(mgr, name):
    """One call of the case under the profiler: (the copies and kernels it enqueued, in order, bytes_moved delta, h2d_bytes delta),
    after the destination pool was compared with the oracle.  A window the profiler delivered incomplete (_window) is reported as
    a warning with its records and the call runs again in a new window, up to WINDOWS windows; every run is checked against the
    oracle and must move the same bytes."""
    from torch.profiler import ProfilerActivity, profile
    r, call = CASES[name](mgr)
    seen = []
    for _ in range(WINDOWS):
        torch.cuda.synchronize()
        moved, h2d = mgr.bytes_moved(), mgr.h2d_bytes()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call().wait(30.0)
            torch.cuda.synchronize()
        moved, h2d = mgr.bytes_moved() - moved, mgr.h2d_bytes() - h2d
        if isinstance(r, BatchRig):
            r.check(singles=False)
        else:
            r.check()
        events = prof.profiler.kineto_results.events()
        names = _window(events)
        if names is not None:
            return names, moved, h2d
        seen.append(_describe(events))
        warnings.warn(f"{name}: incomplete profile window {len(seen)}: {seen[-1]}")
    pytest.fail(f"{name}: no complete profile window in {WINDOWS}: " + " | ".join(seen))


@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=17)
    yield m
    torch.cuda.synchronize()
    m.close()


# the kernels and copies of each case (bf16, 128 B rows, 16-token source pages and 64-token destination pages when re-paging):
# the staged copy of the tables, the transfer's kernel, then the signal; a streamed call gated in the kernel, or per layer
# with the stream-wait gate, each layer's launch followed by its layer signal
H2D, SIG, LSIG = "Memcpy HtoD", "kvbm_signal_kernel", "kvbm_layer_signal_kernel"
PERMUTE, GATHER, GATED = "kvbm_paged_permute_kernel<0, true, false>", "kvbm_paged_gather_kernel<0, true, false>", "kvbm_gated_gather_kernel<0, true, false>"
REPAGE, REPAGE_GATHER = "kvbm_paged_repage_kernel<0, true, false, true>", "kvbm_paged_repage_gather_kernel<0, true, false, true>"
GATED_REPAGE = "kvbm_gated_repage_gather_kernel<0, true, false, true>"
BATCH, GATED_BATCH = "kvbm_paged_batch_repage_gather_kernel<0, true, false, true>", "kvbm_gated_batch_repage_gather_kernel<0, true, false, true>"
EXPECTED = {
    "repage": ([H2D, REPAGE, SIG], 305152, 52),
    "repage_gather_one_window": ([H2D, REPAGE, SIG], 305152, 52),
    "repage_gather_tp": ([H2D, REPAGE_GATHER, SIG], 305152, 92),
    "gather_tp": ([H2D, GATHER, SIG], 98304, 36),
    "gather_one_window_320_heads": ([H2D, PERMUTE, SIG], 7864320, 24),
    "transfer_320_heads": ([H2D, PERMUTE, SIG], 7864320, 24),
    "stage_gather": ([H2D, GATHER, SIG], 196608, 60),
    "stage_repage_gather": ([H2D, REPAGE_GATHER, SIG], 610304, 172),
    "batch_1": ([H2D, BATCH, SIG], 610304, 224),
    "batch_3": ([H2D, BATCH, SIG], 1024000, 432),
    "gather_streamed_spin": ([H2D, GATED], 98304, 36),
    "stage_gather_streamed_spin": ([H2D, GATED], 196608, 60),
    "repage_gather_streamed_spin": ([H2D, GATED_REPAGE], 305152, 92),
    "stage_repage_gather_streamed_spin": ([H2D, GATED_REPAGE], 610304, 172),
    "batch_3_streamed_spin": ([H2D, GATED_BATCH], 1024000, 432),
    "gather_streamed_stream_wait": ([H2D] + [GATHER, LSIG] * 2, 98304, 36),
    "stage_gather_streamed_stream_wait": ([H2D] + [GATHER, LSIG] * 4, 196608, 60),
    "repage_gather_streamed_stream_wait": ([H2D] + [REPAGE_GATHER, LSIG] * 2, 305152, 92),
    "stage_repage_gather_streamed_stream_wait": ([H2D] + [REPAGE_GATHER, LSIG] * 4, 610304, 172),
    "batch_3_streamed_stream_wait": ([H2D] + [BATCH, LSIG] * 4, 1024000, 432),
}


@pytest.mark.parametrize("name", list(CASES))
def test_manager_launches(mgr, name):
    names, moved, h2d = run_case(mgr, name)
    assert (names, moved, h2d) == EXPECTED[name]

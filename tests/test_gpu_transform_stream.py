"""Layer streaming of the layout-transforming hand-offs against producers that write the sources after the launch.

kvbm_kernels_paged_permute_gather_streamed and kvbm_kernels_paged_repage_gather_streamed read layer l of source s only after
that source's ready flag l has reached the epoch, and publish the destination's layer_done_flags[l] once layer l landed.  The
discipline is tests/test_gpu_layer_stream.py's:

  * every source pool starts as poison (its final bytes XOR 0xA5) and has its own ready flags and producer stream;
  * the streamed launch is enqueued first, on its own stream, with few CTAs; each producer then sleeps, writes one layer's final
    bytes and releases its flag, layer by layer;
  * the oracle (tests/repage_gather_oracle.py, which is also the gather's over whole blocks) runs on the final bytes, so a gate
    that lets a read through early moves poison, and whole destination pools (guard blocks included) are compared;
  * state is observed only through a checker stream that waits for a flag; every host wait has a deadline; a `finally` releases
    every ready flag; every torch kernel runs once before the first launch.

Sources are in operational formats, so one layer of a block is one contiguous run the producer can write; destinations take
every format."""
import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import ErrorCode, KvbmError, TransferManager, TransferOptions
from tests.gpu_util import stream_ptr
from tests.repage_gather_oracle import repage_gather
from tests.test_gpu_layer_stream import _finish
from tests.test_gpu_repage_gather import ELEMS, _Managed

pytestmark = pytest.mark.gpu

KV = K.KvBlockLayout
CM = K.CastMode
MASK = 0xFFFFFFFF
GATES = [K.GATE_SPIN, K.GATE_STREAM_WAIT]
GATE_IDS = ["spin", "stream_wait"]
LAYER_SLEEP = 300_000     # cycles a producer sleeps before each layer (~0.15 ms)
CHECKER_SLEEP = 2_000_000  # ~1 ms
MAX_CTAS = 4


def _i32(v):
    v &= MASK
    return v - (1 << 32) if v >= 1 << 31 else v


class Pool:
    """A fully contiguous device pool of nb blocks [nl, no, region] (any format inside a block), with its host bytes."""

    def __init__(self, nb, nl, no, page, nh, row, kv, seed, poison=False):
        self.nb, self.nl, self.no, self.page, self.nh, self.row, self.kv = nb, nl, no, page, nh, row, int(kv)
        self.region = page * nh * row
        self.block = nl * no * self.region
        rng = np.random.default_rng(seed)
        self.final_np = rng.integers(0, 256, (nb, self.block), dtype=np.uint8)
        self.final = torch.from_numpy(self.final_np).cuda()
        self.poison = torch.from_numpy(self.final_np ^ 0xA5).cuda()
        self.buf = (self.poison if poison else self.final).clone()
        base = self.buf.data_ptr()
        self.layer_base = torch.tensor([base + l * no * self.region for l in range(nl)], dtype=torch.int64, device="cuda")
        self.ready = torch.zeros(nl, dtype=torch.int32, device="cuda")
        self.stream = torch.cuda.Stream()

    def side(self, ids):
        return K.PermuteSide(K.PagedLayout(self.layer_base.data_ptr(), self.block, self.region, self.region, self.nl, self.no, self.nb),
                             ids.data_ptr(), self.kv)

    def layer(self, t, l):
        return t.view(self.nb, self.nl, -1)[:, l]

    def produce(self, layers, epoch):
        """On this source's producer stream: per layer sleep, write its final bytes, release its flag."""
        with torch.cuda.stream(self.stream):
            for l in layers:
                torch.cuda._sleep(LAYER_SLEEP)
                self.layer(self.buf, l).copy_(self.layer(self.final, l))
                K.check(K.set_flags(self.ready.data_ptr(), l, 1, epoch, stream_ptr(self.stream)), "set_flags")


class Rig:
    """srcs: (nh, kv) per source; windows (source, src_head_begin, dst_head_begin, head_count); ps == pd with tokens None is the
    gather over n whole blocks, else the re-paging gather over tokens [tb, te)."""

    def __init__(self, srcs, windows, dst_nh, dst_kv, ps=16, pd=16, tokens=None, n=5, nl=4, no=2, hd=64, cast=CM.NONE, scaled=False,
                 layers=None, seed=0, max_ctas=MAX_CTAS):
        se, de = ELEMS[cast]
        self.max_ctas = max_ctas
        self.row, self.d_row = hd * se, hd * de
        self.ps, self.pd, self.nl, self.no, self.cast, self.windows = ps, pd, nl, no, int(cast), windows
        self.repage = tokens is not None
        self.tb, self.te = tokens if self.repage else (0, n * ps)
        self.lb, self.le = (layers.start, layers.stop) if layers else (0, nl)
        ns = -(-self.te // ps) - self.tb // ps
        nd = -(-self.te // pd) - self.tb // pd
        self.srcs = [Pool(ns + 2, nl, no, ps, nh, self.row, kv, seed + 10 + s, poison=True) for s, (nh, kv) in enumerate(srcs)]
        self.dst = Pool(nd + 2, nl, no, pd, dst_nh, self.d_row, dst_kv, seed + 1)
        self.dst_nh = dst_nh
        rng = np.random.default_rng(seed + 2)
        self.sids = [rng.permutation(ns + 2)[:ns].astype(np.int32) for _ in srcs]
        self.dids = rng.permutation(nd + 2)[:nd].astype(np.int32)
        self.sids_t = [torch.from_numpy(x).cuda() for x in self.sids]
        self.dids_t = torch.from_numpy(self.dids).cuda()
        self.initial = self.dst.buf.clone()
        self.scales_np = (rng.uniform(0.1, 4.0, nl * no) * (1 + np.arange(nl * no) * 1e-2)).astype(np.float32) if scaled else None
        self.scales = torch.from_numpy(self.scales_np).cuda() if scaled else None
        self.layer_done = torch.zeros(nl, dtype=torch.int32, device="cuda")
        self.done = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.completion = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.ws = torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device="cuda")
        self.side_stream, self.checker = torch.cuda.Stream(), torch.cuda.Stream()

    def expected(self, layers=None):
        srcs = [([p.final_np[b] for b in self.sids[s]], p.kv, p.nh) for s, p in enumerate(self.srcs)]
        init = self.initial.cpu().numpy()
        out = repage_gather(srcs, self.windows, [init[b] for b in self.dids], self.dst.kv, self.dst_nh, self.nl, self.no, self.ps, self.pd,
                            self.row, self.tb, self.te, self.cast, self.scales_np, layers if layers is not None else range(self.lb, self.le))
        for b, blk in zip(self.dids, out):
            init[b] = blk
        return init

    def warm(self):
        """Every torch kernel of the producers and the checker once, then the poison back and the destination reset."""
        for p in self.srcs:
            for s in (p.stream, self.checker):
                with torch.cuda.stream(s):
                    torch.cuda._sleep(100)
                    for l in range(self.nl):
                        p.layer(p.buf, l).copy_(p.layer(p.final, l))
                    self.dst.buf.copy_(self.initial)
        with torch.cuda.stream(self.checker):
            torch.cuda._sleep(100)
            self.snap_t = self.dst.buf.clone()
            self.snap_flags = self.layer_done.clone()
            self.snap_done = self.done.clone()
            self.snap_flags.copy_(self.layer_done)
            self.snap_done.copy_(self.done)
            self.snap_t.copy_(self.dst.buf)
        torch.cuda.synchronize()
        self.reset()

    def reset(self):
        for p in self.srcs:
            p.buf.copy_(p.poison)
        self.dst.buf.copy_(self.initial)
        torch.cuda.synchronize()

    def stream_desc(self, epoch, gate_mode, value):
        st = K.PermuteStream()
        for j, (s, *_r) in enumerate(self.windows):
            st.layer_ready_flags[j] = self.srcs[s].ready.data_ptr()
        st.layer_done_flags = self.layer_done.data_ptr()
        st.done_flag = self.done.data_ptr()
        st.epoch = epoch & MASK
        st.sync_workspace = self.ws.data_ptr()
        st.completion_flag = self.completion.data_ptr()
        st.completion_value = value
        st.gate_mode = gate_mode
        st.gate_timeout_ms = 10000
        st.max_ctas = self.max_ctas
        return st

    def launch(self, epoch, gate_mode, value):
        dside = self.dst.side(self.dids_t)
        srcs = [K.PermuteSource(self.srcs[s].side(self.sids_t[s]), self.srcs[s].nh, sb, db, k) for s, sb, db, k in self.windows]
        st = self.stream_desc(epoch, gate_mode, value)
        sp = stream_ptr(self.side_stream)
        if self.repage:
            rc = K.paged_repage_gather_streamed(srcs, self.ps, dside, self.dst_nh, self.pd, self.tb, self.te, self.lb, self.le, self.row,
                                                self.cast, self.scales, st, sp)
        else:
            rc = K.paged_permute_gather_streamed(srcs, dside, self.dst_nh, len(self.dids), self.lb, self.le, self.ps, self.row, self.cast,
                                                 self.scales, st, sp)
        K.check(rc, "streamed launch")

    def rescue(self, epoch):
        """Release every source's flags from a fresh stream and let the launch and the checker drain."""
        s = torch.cuda.Stream()
        for p in self.srcs:
            K.set_flags(p.ready.data_ptr(), 0, self.nl, epoch & MASK, stream_ptr(s))
        assert _finish(s) and _finish(self.side_stream), "a streamed launch is still waiting"
        for p in self.srcs:
            assert _finish(p.stream)
        if not _finish(self.checker, 2.0):
            K.set_flags(self.layer_done.data_ptr(), 0, self.nl, epoch & MASK, stream_ptr(s))
            assert _finish(self.checker), "the checker is still waiting"
        torch.cuda.synchronize()

    def check_end(self, epoch, value):
        assert np.array_equal(self.dst.buf.cpu().numpy(), self.expected())
        want = [_i32(epoch) if self.lb <= l < self.le else 0 for l in range(self.nl)]
        assert [_i32(v) for v in self.layer_done.tolist()] == want
        assert self.done.item() == _i32(epoch) and self.completion.item() == _i32(value)
        assert not self.ws.any().item(), "the workspace must be left zeroed"

    def produce_skewed(self, epoch, lag):
        """Every source's layers on ONE producer stream, source s lagging lag[s] layers: at step t, source s writes layer t - lag[s]
        and releases its own flag.  (Eight producer streams next to the launch's would outnumber the device's hardware queues,
        and the stream-wait form's cuStreamWaitValue32 would then hold the producer stream that shares its queue.)"""
        p0 = self.srcs[0]
        with torch.cuda.stream(p0.stream):
            for t in range(self.nl + max(lag)):
                torch.cuda._sleep(LAYER_SLEEP)
                for s, p in enumerate(self.srcs):
                    l = t - lag[s]
                    if 0 <= l < self.nl:
                        p.layer(p.buf, l).copy_(p.layer(p.final, l))
                        K.check(K.set_flags(p.ready.data_ptr(), l, 1, epoch, stream_ptr(p0.stream)), "set_flags")

    def run(self, epoch, gate_mode, value, lag=None):
        """The whole transfer against producers that start after the launch; lag[s]: source s runs that many layers late."""
        try:
            self.launch(epoch, gate_mode, value)
            if lag:
                self.produce_skewed(epoch & MASK, lag)
            else:
                for p in self.srcs:
                    p.produce(range(self.nl), epoch & MASK)
            ok = _finish(self.side_stream) and all(_finish(p.stream) for p in self.srcs)
            assert ok, "the streamed transfer did not finish"
        finally:
            self.rescue(epoch)


CASES = {
    # a format change: one source, every head
    "format_nhd_to_universal_tp": dict(srcs=[(4, KV.OperationalNHD)], windows=[(0, 0, 0, 4)], dst_nh=4, dst_kv=KV.UniversalTP),
    # one TP re-shard window
    "reshard_window": dict(srcs=[(8, KV.OperationalHND)], windows=[(0, 2, 1, 4)], dst_nh=6, dst_kv=KV.OperationalNHD),
    # TP4 -> TP2 (8 heads), decode rank 0, fp8 -> bf16 with scales
    "tp4_tp2_fp8_to_bf16_scaled": dict(srcs=[(2, KV.OperationalNHD), (2, KV.OperationalHND)], windows=[(0, 0, 0, 2), (1, 0, 2, 2)],
                                       dst_nh=4, dst_kv=KV.UniversalPP, cast=CM.FP8E4M3_TO_BF16, scaled=True),
    # a re-page 1 -> 16 over a range that starts and ends inside pages
    "repage_1_to_16": dict(srcs=[(4, KV.OperationalNHD)], windows=[(0, 0, 0, 4)], dst_nh=4, dst_kv=KV.OperationalHND, ps=1, pd=16,
                           tokens=(5, 70)),
    # a re-paging gather TP4 page 64 -> TP2 page 16, bf16 -> fp8
    "repage_gather_tp4_tp2_64_to_16_bf16_to_fp8": dict(srcs=[(2, KV.OperationalHND), (2, KV.OperationalNHD)],
                                                       windows=[(0, 0, 0, 2), (1, 0, 2, 2)], dst_nh=4, dst_kv=KV.UniversalTP, ps=64, pd=16,
                                                       tokens=(10, 150), cast=CM.BF16_TO_FP8E4M3),
    # an inner layer range
    "inner_layers": dict(srcs=[(2, KV.OperationalNHD), (2, KV.OperationalNHD)], windows=[(1, 0, 0, 2), (0, 0, 2, 2)], dst_nh=4,
                         dst_kv=KV.OperationalHND, layers=range(1, 3)),
}
TP8 = dict(srcs=[(1, KV.OperationalNHD if s % 2 else KV.OperationalHND) for s in range(8)], windows=[(s, 0, s, 1) for s in range(8)],
           dst_nh=8, dst_kv=KV.UniversalTP)


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("name", list(CASES))
def test_layers_written_after_the_launch_arrive_whole(gate_mode, name):
    r = Rig(**CASES[name], seed=len(name))
    r.warm()
    r.run(5, gate_mode, 77)
    r.check_end(5, 77)


@pytest.mark.parametrize("name", ["tp4_tp2_fp8_to_bf16_scaled", "repage_gather_tp4_tp2_64_to_16_bf16_to_fp8"])
def test_default_grid_leaves_the_producer_room(name):
    """The spinning form at its default grid (max_ctas 0: half the SMs) next to a producer on the same GPU: enough units that the
    grid is the whole default, and the producer's per-layer kernels (a sleep, a multi-CTA copy) must still run while it spins."""
    big = dict(CASES[name], nl=6, seed=51)
    if "tokens" in big:
        big["tokens"] = (10, 40 * 64 - 3)
    else:
        big["n"] = 48
    r = Rig(**big, max_ctas=0)
    per_layer = (len(r.dids) if not r.repage else -(-r.te // max(r.ps, r.pd)) - r.tb // max(r.ps, r.pd)) * r.no
    assert per_layer >= torch.cuda.get_device_properties(0).multi_processor_count // 2
    r.warm()
    r.run(6, K.GATE_SPIN, 61)
    r.check_end(6, 61)


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_tp8_to_tp1_eight_producers_on_skewed_schedules(gate_mode):
    """Each of 8 source ranks has its own bytes, flags and release schedule; source s lags s layers, so source 7 releases last."""
    r = Rig(**TP8, nl=6, seed=8)
    r.warm()
    r.run(3, gate_mode, 9, lag=list(range(8)))
    r.check_end(3, 9)


def _partial(r, gate_mode, k, per_source):
    """Release per_source[s] layers of each source, observe the destination once layer_done[lb + k - 1] appears, then release
    the rest.  Returns the snapshot (pool, layer flags, done flag)."""
    epoch = 7
    try:
        r.launch(epoch, gate_mode, 1)
        for s, p in enumerate(r.srcs):
            p.produce(range(r.lb, r.lb + per_source[s]), epoch)
        with torch.cuda.stream(r.checker):
            K.check(K.wait_flag(r.layer_done.data_ptr() + 4 * (r.lb + k - 1), epoch, stream_ptr(r.checker)), "wait_flag")
            torch.cuda._sleep(CHECKER_SLEEP)
            r.snap_flags.copy_(r.layer_done)
            r.snap_done.copy_(r.done)
            r.snap_t.copy_(r.dst.buf)
        assert _finish(r.checker), "layer_done of the released layers did not appear"
        snap = (r.snap_t.cpu().numpy(), [_i32(v) for v in r.snap_flags.tolist()], r.snap_done.item())
        for s, p in enumerate(r.srcs):
            p.produce(range(r.lb + per_source[s], r.le), epoch)
        assert _finish(r.side_stream) and all(_finish(p.stream) for p in r.srcs)
    finally:
        r.rescue(epoch)
    r.check_end(epoch, 1)
    return snap


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("how", ["every_source_k", "one_source_all"])
def test_only_released_layers_move(gate_mode, how):
    r = Rig(**CASES["tp4_tp2_fp8_to_bf16_scaled"], seed=21)
    r.warm()
    k = 2
    per_source = [k, k] if how == "every_source_k" else [r.nl, k]
    pool, flags, done = _partial(r, gate_mode, k, per_source)
    assert np.array_equal(pool, r.expected(range(0, k)))
    assert flags == [7 if l < k else 0 for l in range(r.nl)]
    assert done == 0


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_a_repaged_layer_has_landed_when_its_flag_appears(gate_mode):
    """The checker waits on layer_done[l] and copies layer l: it equals the oracle (an operational destination, so a layer of a
    block is one contiguous run)."""
    r = Rig(**dict(CASES["repage_gather_tp4_tp2_64_to_16_bf16_to_fp8"], dst_kv=KV.OperationalNHD), seed=31)
    r.warm()
    want = r.expected()
    epoch = 12
    snaps = [r.dst.buf.clone() for _ in range(r.nl)]
    with torch.cuda.stream(r.checker):   # warm the copies into the snapshots
        for t in snaps:
            t.copy_(r.dst.buf)
    torch.cuda.synchronize()
    try:
        r.launch(epoch, gate_mode, 2)
        for p in r.srcs:
            p.produce(range(r.nl), epoch)
        with torch.cuda.stream(r.checker):
            for l in range(r.nl):
                K.check(K.wait_flag(r.layer_done.data_ptr() + 4 * l, epoch, stream_ptr(r.checker)), "wait_flag")
                snaps[l].copy_(r.dst.buf)
        assert _finish(r.checker) and _finish(r.side_stream)
    finally:
        r.rescue(epoch)
    lay = r.dst.no * r.dst.region
    for l in range(r.nl):
        got = snaps[l].cpu().numpy()
        assert np.array_equal(got[:, l * lay:(l + 1) * lay], want[:, l * lay:(l + 1) * lay]), f"layer {l}"
    r.check_end(epoch, 2)


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("start,epochs", [(0, [1, 2, 3]), (0xFFFFFFFD, [0xFFFFFFFE, 0xFFFFFFFF, 0, 1])], ids=["1_2_3", "wrap"])
def test_rounds_of_epochs_on_the_same_flags(gate_mode, start, epochs):
    r = Rig(**CASES["inner_layers"], seed=41)
    r.warm()
    for p in r.srcs:
        p.ready.fill_(_i32(start))
    r.layer_done.fill_(_i32(start))
    r.done.fill_(_i32(start))
    torch.cuda.synchronize()
    for i, e in enumerate(epochs):
        r.reset()
        r.run(e, gate_mode, 100 + i)
        assert np.array_equal(r.dst.buf.cpu().numpy(), r.expected())
        want = [_i32(e) if r.lb <= l < r.le else _i32(start) for l in range(r.nl)]
        assert [_i32(v) for v in r.layer_done.tolist()] == want
        assert r.done.item() == _i32(e) and r.completion.item() == 100 + i
        assert not r.ws.any().item(), "the workspace must be left zeroed"


# ---------------------------------------------------------------------------------------------------------------------
# TransferManager.execute_gather_streamed / execute_repage_gather_streamed against the unstreamed entries
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=43)
    yield m
    torch.cuda.synchronize()
    m.close()


def _flags(c, nl, epoch):
    return {r: torch.full((nl,), _i32(epoch), dtype=torch.int32, device="cuda") for r in c.ranks}


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("kind", ["gather", "repage_gather"])
@pytest.mark.parametrize("how", ["manager_stream", "caller_stream"])
def test_manager_streamed_equals_unstreamed(mgr, gate_mode, kind, how):
    tp, cast = ((8, 1), CM.NONE) if kind == "gather" else ((4, 2), CM.FP8E4M3_TO_BF16)
    ps, pd = (16, 16) if kind == "gather" else (64, 16)
    tb, te = (0, 5 * 16) if kind == "gather" else (9, 140)
    geom = (8, 3, 2, 64)
    a = _Managed(mgr, tp, ps, pd, te, cast, KV.OperationalNHD, KV.UniversalTP, geom=geom)
    b = _Managed(mgr, tp, ps, pd, te, cast, KV.OperationalNHD, KV.UniversalTP, geom=geom)
    ready = _flags(b, geom[1], 21)
    layer_done = torch.zeros(geom[1], dtype=torch.int32, device="cuda")
    done_a, done_b = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    extra = dict(cuda_stream=int(s.cuda_stream)) if how == "caller_stream" else {}
    oa = TransferOptions(cast_mode=int(cast), done_flag=done_a.data_ptr(), epoch=21, **extra)
    ob = TransferOptions(cast_mode=int(cast), done_flag=done_b.data_ptr(), epoch=21, gate_mode=gate_mode, max_ctas=MAX_CTAS, **extra)
    if kind == "gather":
        na = mgr.execute_gather(a.sources(tb, te), a.dst.h, a.dids(tb, te), a.plan, oa)
        na.wait(20.0)
        torch.cuda.synchronize()
        b0 = mgr.bytes_moved()
        nb = mgr.execute_gather_streamed(b.sources(tb, te), b.dst.h, b.dids(tb, te), b.plan, {r: t.data_ptr() for r, t in ready.items()}, ob,
                                         layer_done_flags=layer_done.data_ptr())
    else:
        na = mgr.execute_repage_gather(a.sources(tb, te), a.dst.h, a.dids(tb, te), a.plan, range(tb, te), oa)
        na.wait(20.0)
        torch.cuda.synchronize()
        b0 = mgr.bytes_moved()
        nb = mgr.execute_repage_gather_streamed(b.sources(tb, te), b.dst.h, b.dids(tb, te), b.plan, range(tb, te),
                                                {r: t.data_ptr() for r, t in ready.items()}, ob, layer_done_flags=layer_done.data_ptr())
    moved = mgr.bytes_moved() - b0
    if how == "caller_stream":
        assert nb.is_complete()
        assert _finish(s)
    else:
        nb.wait(20.0)
    torch.cuda.synchronize()
    assert done_a.item() == 21 and done_b.item() == 21
    assert layer_done.tolist() == [21] * geom[1]
    covered = sum(w.head_count for w in b.plan)
    assert moved == (te - tb) * geom[1] * geom[2] * covered * geom[3] * ELEMS[cast][1]
    a.dst.download()
    b.dst.download()
    for x, y in zip(a.dst.twin.buffers, b.dst.twin.buffers):
        assert np.array_equal(x, y)
    b.expect(tb, te)
    b.check()


def test_manager_rejects_flags_the_device_cannot_reach(mgr):
    """Pageable host memory as ready or layer-done flags is rejected before any launch, with no bytes moved."""
    c = _Managed(mgr, (4, 2), 16, 16, 64, CM.NONE, KV.OperationalNHD, KV.OperationalHND)
    ready = {r: torch.zeros(c.nl, dtype=torch.int32, device="cuda") for r in c.ranks}
    pageable = np.zeros(c.nl, dtype=np.uint32)
    b0 = mgr.bytes_moved()
    for flags, done in (({**{r: t.data_ptr() for r, t in ready.items()}, c.ranks[0]: pageable.ctypes.data}, 0),
                        ({r: t.data_ptr() for r, t in ready.items()}, pageable.ctypes.data)):
        with pytest.raises(KvbmError) as e:
            mgr.execute_gather_streamed(c.sources(0, 64), c.dst.h, c.dids(0, 64), c.plan, flags, TransferOptions(epoch=1),
                                        layer_done_flags=done)
        assert e.value.code == ErrorCode.ERR and "not reachable" in e.value.msg
    assert mgr.bytes_moved() == b0


@pytest.mark.multigpu
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_manager_streamed_repage_gather_across_gpus(gate_mode):
    """The decode GPU pulls every source rank's heads, and polls their ready flags, on the other GPU over NVLink."""
    m = TransferManager(device=1, worker_id=44)
    probe = torch.zeros(4, dtype=torch.int32, device="cuda:0")
    c0 = _Managed(m, (4, 2), 16, 16, 64, CM.NONE, KV.OperationalNHD, KV.OperationalHND, device=(1, 1))
    with pytest.raises(KvbmError) as e:   # device 0's memory before peer access is enabled
        m.execute_gather_streamed(c0.sources(0, 64), c0.dst.h, c0.dids(0, 64), c0.plan, {r: probe.data_ptr() for r in c0.ranks})
    assert e.value.code == ErrorCode.ERR and "not reachable" in e.value.msg
    m.enable_peer_access(0)
    tb, te = 3, 150
    c = _Managed(m, (4, 2), 16, 64, te, CM.NONE, KV.OperationalNHD, KV.OperationalHND, device=(0, 1))
    ready = {r: torch.full((c.nl,), 5, dtype=torch.int32, device="cuda:0") for r in c.ranks}
    o = TransferOptions(epoch=5, gate_mode=gate_mode, max_ctas=MAX_CTAS)
    m.execute_repage_gather_streamed(c.sources(tb, te), c.dst.h, c.dids(tb, te), c.plan, range(tb, te),
                                     {r: t.data_ptr() for r, t in ready.items()}, o).wait(20.0)
    torch.cuda.synchronize(0)
    torch.cuda.synchronize(1)
    c.expect(tb, te)
    c.check()
    m.close()

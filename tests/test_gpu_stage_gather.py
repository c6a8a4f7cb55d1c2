"""GPU parity of the staged gather (a PP x TP re-shard): kvbm_kernels_paged_stage_gather, its streamed form and
TransferManager.execute_stage_gather, against tests/stage_oracle over whole destination pools (guard blocks and the heads no
window covers included).  Source pools hold only their stage's layers, so their layer counts differ from the destination's.
The streamed cases follow tests/test_gpu_transform_stream.py's discipline: poisoned sources, the launch first, per-layer writes
and flag releases on one producer stream after it, the checker's state read once the launch finished, every flag released in
a `finally`."""
import re

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import TransferManager, TransferOptions, tp_pp_reshard_plan
from tests.gpu_util import stream_ptr
from tests.stage_oracle import stage_block
from tests.test_gpu_layer_stream import _finish
from tests.test_gpu_transform_stream import LAYER_SLEEP, Pool, _i32

KV = K.KvBlockLayout
CM = K.CastMode
ALL = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]
ELEMS = {CM.NONE: (2, 2), CM.FP8E4M3_TO_BF16: (1, 2), CM.BF16_TO_FP8E4M3: (2, 1)}
GATES = [K.GATE_SPIN, K.GATE_STREAM_WAIT]
GATE_IDS = ["spin", "stream_wait"]
GUARD = 8                       # u32 words after every source's ready flags


class StageRig:
    """srcs: (num_layers, num_heads, kv) per source pool; windows: (source, src_layer_begin, dst_layer_begin, layer_count,
    src_head_begin, dst_head_begin, head_count), one kernel source each."""

    def __init__(self, srcs, windows, dst_nl, dst_nh, dst_kv, n=3, no=2, page=16, hd=64, cast=CM.NONE, scaled=False, layers=None,
                 seed=0, poison=False, max_ctas=4):
        se, de = ELEMS[cast]
        self.row, self.cast, self.windows, self.no, self.page, self.max_ctas = hd * se, int(cast), windows, no, page, max_ctas
        self.lb, self.le = (layers.start, layers.stop) if layers else (0, dst_nl)
        self.srcs = [Pool(n + 2, nl, no, page, nh, hd * se, kv, seed + 10 + s, poison=poison) for s, (nl, nh, kv) in enumerate(srcs)]
        for p in self.srcs:               # ready flags followed by guard words that stay 0
            p.ready_all = torch.zeros(p.nl + GUARD, dtype=torch.int32, device="cuda")
            p.ready = p.ready_all[:p.nl]
        self.dst = Pool(n + 2, dst_nl, no, page, dst_nh, hd * de, dst_kv, seed + 1)
        rng = np.random.default_rng(seed + 2)
        self.sids = [rng.permutation(n + 2)[:n].astype(np.int32) for _ in srcs]
        self.dids = rng.permutation(n + 2)[:n].astype(np.int32)
        self.sids_t = [torch.from_numpy(x).cuda() for x in self.sids]
        self.dids_t = torch.from_numpy(self.dids).cuda()
        self.initial = self.dst.buf.clone()
        self.scales_np = (rng.uniform(0.1, 4.0, dst_nl * no) * (1 + np.arange(dst_nl * no) * 1e-2)).astype(np.float32) if scaled else None
        self.scales = torch.from_numpy(self.scales_np).cuda() if scaled else None
        self.layer_done = torch.zeros(dst_nl, dtype=torch.int32, device="cuda")
        self.done = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.completion = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.ws = torch.zeros(K.sync_workspace_words(dst_nl), dtype=torch.int32, device="cuda")
        self.side_stream = torch.cuda.Stream()

    def sources(self):
        return [K.StageSource(K.PermuteSource(self.srcs[s].side(self.sids_t[s]), self.srcs[s].nh, sb, db, k), sl, dl, c)
                for s, sl, dl, c, sb, db, k in self.windows]

    def expected(self):
        init = self.initial.cpu().numpy()
        d = self.dst
        for i, b in enumerate(self.dids):
            blk = init[b]
            for s, sl, dl, c, sb, db, k in self.windows:
                p = self.srcs[s]
                blk = stage_block(p.final_np[self.sids[s][i]], blk, p.kv, d.kv, p.nl, d.nl, self.no, self.page, p.nh, d.nh, self.row, self.cast,
                                  (sl, dl, c, sb, db, k), layers=range(self.lb, self.le), scales=self.scales_np)
            init[b] = blk
        return init

    def run(self):
        rc = K.paged_stage_gather(self.sources(), self.dst.side(self.dids_t), self.dst.nh, len(self.dids), self.lb, self.le, self.page, self.row,
                                  self.cast, self.scales, self.done.data_ptr(), 5, self.completion.data_ptr(), 6, stream_ptr())
        torch.cuda.synchronize()
        return rc

    def check(self):
        assert np.array_equal(self.dst.buf.cpu().numpy(), self.expected())

    # ---- streamed ----
    def stream_desc(self, epoch, gate_mode, timeout_ms):
        st = K.PermuteStream()
        for j, w in enumerate(self.windows):
            st.layer_ready_flags[j] = self.srcs[w[0]].ready.data_ptr()
        st.layer_done_flags = self.layer_done.data_ptr()
        st.done_flag = self.done.data_ptr()
        st.epoch = epoch
        st.sync_workspace = self.ws.data_ptr()
        st.completion_flag = self.completion.data_ptr()
        st.completion_value = epoch + 1
        st.gate_mode = gate_mode
        st.gate_timeout_ms = timeout_ms
        st.max_ctas = self.max_ctas
        return st

    def produce(self, epoch):
        """One producer stream, stage by stage (sources ordered by their first destination layer), each source's layers by its own
        layer numbers: sleep, write the final bytes, release the flag."""
        first = {}
        for s, sl, dl, *_r in self.windows:
            first[s] = min(first.get(s, 1 << 30), dl)
        p0 = self.srcs[0]
        with torch.cuda.stream(p0.stream):
            for s in sorted(first, key=lambda x: first[x]):
                p = self.srcs[s]
                for l in range(p.nl):
                    torch.cuda._sleep(LAYER_SLEEP)
                    p.layer(p.buf, l).copy_(p.layer(p.final, l))
                    K.check(K.set_flags(p.ready.data_ptr(), l, 1, epoch, stream_ptr(p0.stream)), "set_flags")

    def run_streamed(self, epoch, gate_mode, timeout_ms=10000):
        p0 = self.srcs[0].stream
        for p in self.srcs:        # every torch kernel of the producer once, then the poison back
            with torch.cuda.stream(p0):
                torch.cuda._sleep(100)
                p.layer(p.buf, 0).copy_(p.layer(p.final, 0))
        torch.cuda.synchronize()
        for p in self.srcs:
            p.buf.copy_(p.poison)
            if gate_mode == K.GATE_STREAM_WAIT:     # the stream-wait form has no timeout: its guards stay released
                p.ready_all[p.nl:].fill_(epoch)
        torch.cuda.synchronize()
        try:
            st = self.stream_desc(epoch, gate_mode, timeout_ms)
            K.check(K.paged_stage_gather_streamed(self.sources(), self.dst.side(self.dids_t), self.dst.nh, len(self.dids), self.lb, self.le,
                                                  self.page, self.row, self.cast, self.scales, st, stream_ptr(self.side_stream)), "launch")
            self.produce(epoch)
            assert _finish(self.side_stream) and _finish(p0), "the streamed transfer did not finish"
        finally:
            s = torch.cuda.Stream()
            for p in self.srcs:
                K.set_flags(p.ready.data_ptr(), 0, p.nl, epoch, stream_ptr(s))
            assert _finish(s) and _finish(self.side_stream)
            torch.cuda.synchronize()
        self.check()
        assert [_i32(v) for v in self.layer_done.tolist()] == [epoch if self.lb <= l < self.le else 0 for l in range(self.dst.nl)]
        assert self.done.item() == epoch and self.completion.item() == epoch + 1
        assert not self.ws.any().item(), "the workspace must be left zeroed"


def _plan_rig(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, src_parts=None, dst_parts=None, src_kv=KV.OperationalNHD, dst_kv=KV.OperationalNHD,
              **kw):
    """A rig of the plan's windows: one pool per source rank it names, holding that rank's stage of layers and its heads."""
    plan = tp_pp_reshard_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, src_parts, dst_parts)
    sparts = list(src_parts) if src_parts else [L // src_pp] * src_pp
    dparts = list(dst_parts) if dst_parts else [L // dst_pp] * dst_pp
    ranks = sorted({w.src_rank for w in plan})
    srcs = [(sparts[r // src_tp], max(1, H // src_tp), src_kv) for r in ranks]
    windows = [(ranks.index(w.src_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
               for w in plan]
    return StageRig(srcs, windows, dparts[rank // dst_tp], max(1, H // dst_tp), dst_kv, **kw)


PLANS = {
    "pp2tp4_to_tp2_rank0": (8, 8, 4, 2, 2, 1, 0),
    "pp2tp4_to_tp2_rank1": (8, 8, 4, 2, 2, 1, 1),
    "pp1tp8_to_pp2tp1_rank0": (8, 8, 8, 1, 1, 2, 0),
    "pp1tp8_to_pp2tp1_rank1": (8, 8, 8, 1, 1, 2, 1),
    "h2_replicated_pp2tp4_to_tp1": (2, 6, 4, 2, 1, 1, 0),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PLANS))
def test_plans(name):
    r = _plan_rig(*PLANS[name], src_kv=KV.OperationalHND, dst_kv=KV.UniversalTP, seed=len(name))
    assert r.run() == 0
    r.check()
    assert r.done.item() == 5 and r.completion.item() == 6


@pytest.mark.gpu
@pytest.mark.parametrize("rank", range(4))
def test_uneven_partitions(rank):
    r = _plan_rig(4, 16, 1, 2, 1, 4, rank, [7, 9], [4, 4, 4, 4], seed=rank)
    assert r.run() == 0
    r.check()


@pytest.mark.gpu
@pytest.mark.parametrize("dst_kv", ALL, ids=lambda k: k.name)
@pytest.mark.parametrize("src_kv", ALL, ids=lambda k: k.name)
def test_every_format_pair(src_kv, dst_kv):
    """PP2 x TP2 -> TP1 over 6 layers with 4-head sources of 3 layers each: universal pools whose layer count is not the
    destination's, which a shifted layer_base view of them cannot express."""
    r = _plan_rig(4, 6, 2, 2, 1, 1, 0, src_kv=src_kv, dst_kv=dst_kv, seed=10 * int(src_kv) + int(dst_kv))
    assert r.run() == 0
    r.check()


@pytest.mark.gpu
@pytest.mark.parametrize("scaled", [False, True], ids=["unscaled", "scaled"])
@pytest.mark.parametrize("cast", [CM.FP8E4M3_TO_BF16, CM.BF16_TO_FP8E4M3], ids=lambda c: c.name)
def test_casts_scales_and_a_layer_sub_range(cast, scaled):
    for layers in (None, range(2, 5)):
        r = _plan_rig(8, 8, 4, 2, 2, 1, 1, src_kv=KV.OperationalNHD, dst_kv=KV.UniversalPP, cast=cast, scaled=scaled, layers=layers, hd=80,
                      seed=int(cast) + 3 * scaled)
        assert r.run() == 0
        r.check()


@pytest.mark.gpu
def test_a_pp1_plan_is_the_gather():
    """Identity layer windows over pools of the destination's layer count take the gather's launch, with its bytes."""
    a = _plan_rig(8, 4, 4, 1, 2, 1, 0, seed=3)
    b = _plan_rig(8, 4, 4, 1, 2, 1, 0, seed=3)
    assert a.run() == 0
    srcs = [x.src for x in b.sources()]
    K.check(K.paged_permute_gather(srcs, b.dst.side(b.dids_t), b.dst.nh, len(b.dids), 0, 4, b.page, b.row, stream=stream_ptr()), "gather")
    torch.cuda.synchronize()
    assert torch.equal(a.dst.buf, b.dst.buf)
    a.check()


# ---------------------------------------------------------------------------------------------------------------------
# every instantiation of the two families, reached under the profiler
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True))}
EXPECTED = {(f, w) for f in ("paged", "gated") for w in WALKS}


@pytest.mark.gpu
def test_staged_plans_reach_every_gather_instantiation():
    from torch.profiler import ProfilerActivity, profile
    rigs = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c, p, s in sorted(WALKS):
            cast = CM(c)
            for gated in (False, True):
                r = _plan_rig(8, 8, 4, 2, 2, 1, 0, dst_kv=KV.UniversalTP, cast=cast, scaled=s, hd=64 if p else 80, seed=c + 2 * p + 4 * s)
                if gated:
                    for q in r.srcs:
                        q.ready.fill_(9)
                    torch.cuda.synchronize()
                    st = r.stream_desc(9, K.GATE_SPIN, 10000)
                    K.check(K.paged_stage_gather_streamed(r.sources(), r.dst.side(r.dids_t), r.dst.nh, len(r.dids), 0, 8, r.page, r.row, r.cast,
                                                          r.scales, st, stream_ptr()), "gated")
                    torch.cuda.synchronize()
                else:
                    assert r.run() == 0
                r.check()
                rigs.append(r)
    names = {e.name for e in prof.events()}
    found = set()
    for n in names:
        for m in re.finditer(r"kvbm_(paged|gated)_gather_kernel<([^<>]*)>", n):
            c, p, s = (a.strip().replace("(int)", "") for a in m.group(2).split(","))
            found.add((m.group(1), (int(c), p == "true", s == "true")))
    assert found == EXPECTED, sorted(names)[:20]


# ---------------------------------------------------------------------------------------------------------------------
# streamed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("name", ["pp2tp4_to_tp2_rank0", "pp1tp8_to_pp2tp1_rank1"])
def test_streamed_stage_by_stage(gate_mode, name):
    """The producer releases stage 0's layers, then stage 1's, each source by its own layer numbers.  The sources' flag arrays
    are followed by guard words below the epoch: a spinning gate that read a destination-layer index past a source's array
    would time out (0xFFFFFFFF completion), not hang."""
    r = _plan_rig(*PLANS[name], src_kv=KV.OperationalHND, dst_kv=KV.UniversalTP, seed=7, poison=True, cast=CM.FP8E4M3_TO_BF16, scaled=True)
    r.run_streamed(3, gate_mode, timeout_ms=3000)


@pytest.mark.gpu
@pytest.mark.parametrize("ctas", [1, 2, 3])
def test_spinning_batches_cross_a_stage_boundary(ctas):
    """7 units per layer (7 blocks, one outer index): at 1-3 CTAs a batch is 4 or 2 units, so batches span layers and one crosses
    from stage 0 (layers 0-2) into stage 1 at unit 21."""
    r = _plan_rig(4, 6, 2, 2, 1, 1, 0, n=7, no=1, seed=ctas, poison=True, max_ctas=ctas)
    r.run_streamed(5, K.GATE_SPIN, timeout_ms=3000)


@pytest.mark.gpu
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_streamed_layer_sub_range_and_uneven_stages(gate_mode):
    r = _plan_rig(4, 16, 2, 2, 2, 1, 1, [7, 9], None, seed=11, poison=True, layers=range(3, 12))
    r.run_streamed(7, gate_mode, timeout_ms=3000)


# ---------------------------------------------------------------------------------------------------------------------
# through the TransferManager
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=9)
    yield m
    torch.cuda.synchronize()
    m.close()


def _register(mgr, p, kv):
    from dynamo_b200.physical import LayoutConfig, StorageKind
    cfg = LayoutConfig(p.nb, p.nl, p.no, p.page, p.nh * (p.row // 2), dtype_width_bytes=2, num_heads=p.nh)
    h = mgr.register_fully_contiguous(cfg, p.buf.data_ptr(), p.buf.numel(), StorageKind.Device, 0)
    mgr.set_kv_block_layout(h, kv)
    return h


@pytest.mark.gpu
@pytest.mark.parametrize("streamed", [False, True], ids=["unstreamed", "streamed"])
def test_manager_stage_gather(mgr, streamed):
    """PP2 x TP4 -> TP2 decode rank 1 through execute_stage_gather: one launch, one notification, the oracle's bytes, bytes_moved
    over every window; streamed with every flag already released (the stream-wait form)."""
    H, L = 8, 8
    plan = tp_pp_reshard_plan(H, L, 4, 2, 2, 1, 1)
    r = _plan_rig(H, L, 4, 2, 2, 1, 1, src_kv=KV.UniversalTP, dst_kv=KV.OperationalNHD, seed=21)
    ranks = sorted({w.src_rank for w in plan})
    hs = {rk: _register(mgr, r.srcs[i], KV.UniversalTP) for i, rk in enumerate(ranks)}
    dh = _register(mgr, r.dst, KV.OperationalNHD)
    sources = {rk: (hs[rk], [int(x) for x in r.sids[i]]) for i, rk in enumerate(ranks)}
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    moved0 = mgr.bytes_moved()
    o = TransferOptions(done_flag=flag.data_ptr(), epoch=4)
    if streamed:
        for p in r.srcs:
            p.ready.fill_(4)
        torch.cuda.synchronize()
        o = TransferOptions(done_flag=flag.data_ptr(), epoch=4, gate_mode=K.GATE_STREAM_WAIT)
        note = mgr.execute_stage_gather(sources, dh, [int(x) for x in r.dids], plan, o,
                                        ready_flags={rk: r.srcs[i].ready.data_ptr() for i, rk in enumerate(ranks)},
                                        layer_done_flags=r.layer_done.data_ptr())
    else:
        note = mgr.execute_stage_gather(sources, dh, [int(x) for x in r.dids], plan, o)
    note.wait(20.0)
    torch.cuda.synchronize()
    r.check()
    assert flag.item() == 4
    assert mgr.bytes_moved() - moved0 == sum(len(r.dids) * w.layer_count * r.no * r.page * w.head_count * r.row for w in plan)
    if streamed:
        assert r.layer_done.tolist() == [4] * L

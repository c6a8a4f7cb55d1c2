"""GPU parity of the staged re-paging gather (a PP x TP re-shard across engines with different page sizes):
kvbm_kernels_paged_stage_repage_gather, its streamed form and TransferManager.execute_stage_repage_gather, against
tests/stage_repage_oracle over whole destination pools: guard blocks no table names, heads no window of a layer's stage covers,
slots outside the token range and layers outside the layer range are all compared.  Source pools hold only their stage's
layers at page Ps; the destination holds its own layers at page Pd.  The rig is tests/test_gpu_stage_gather.py's, with block
tables over a token range; the streamed cases keep its discipline (poisoned sources, the launch first, one producer stream that
releases stage by stage, guard words after every source's flags, every flag released in a `finally`)."""
import re

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import TransferManager, TransferOptions, tp_pp_reshard_plan
from tests.gpu_util import stream_ptr
from tests.repage_oracle import table_slice
from tests.stage_repage_oracle import stage_repage_gather
from tests.test_gpu_layer_stream import _finish
from tests.test_gpu_stage_gather import ELEMS, GATE_IDS, GATES, GUARD, StageRig, _register
from tests.test_gpu_transform_stream import Pool, _i32

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
ALL = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]
PAGES = [(16, 64), (64, 16), (1, 16), (16, 1), (12, 48), (48, 6)]


def _tokens(ps, pd):
    """A range that starts and ends inside blocks of the larger page (and of the smaller, unless it is one token)."""
    big = max(ps, pd)
    return range(3, 2 * big - 5 if big > 8 else 2 * big + 3)


class StageRepageRig(StageRig):
    """StageRig's sources and windows with pages: every source at page ps over its own layers, the destination at pd; the
    tables are a sequence's, sliced to `tokens` as the entry takes them, with two blocks per pool that no table names."""

    def __init__(self, srcs, windows, dst_nl, dst_nh, dst_kv, ps=16, pd=64, tokens=None, no=2, hd=64, cast=CM.NONE, scaled=False,
                 layers=None, seed=0, poison=False, max_ctas=4):
        se, de = ELEMS[cast]
        self.row, self.cast, self.windows, self.no, self.ps, self.pd, self.max_ctas = hd * se, int(cast), windows, no, ps, pd, max_ctas
        tokens = tokens if tokens is not None else _tokens(ps, pd)
        self.tb, self.te = tokens.start, tokens.stop
        self.lb, self.le = (layers.start, layers.stop) if layers else (0, dst_nl)
        ns, nd = max(1, -(-self.te // ps)), max(1, -(-self.te // pd))
        self.srcs = [Pool(ns + 2, nl, no, ps, nh, hd * se, kv, seed + 10 + s, poison=poison) for s, (nl, nh, kv) in enumerate(srcs)]
        for p in self.srcs:
            p.ready_all = torch.zeros(p.nl + GUARD, dtype=torch.int32, device="cuda")
            p.ready = p.ready_all[:p.nl]
        self.dst = Pool(nd + 2, dst_nl, no, pd, dst_nh, hd * de, dst_kv, seed + 1)
        rng = np.random.default_rng(seed + 2)
        self.sids = [np.array(table_slice(rng.permutation(ns + 2)[:ns], self.tb, self.te, ps), dtype=np.int32) for _ in srcs]
        self.dids = np.array(table_slice(rng.permutation(nd + 2)[:nd], self.tb, self.te, pd), dtype=np.int32)
        self.sids_t = [torch.from_numpy(x if len(x) else np.zeros(1, np.int32)).cuda() for x in self.sids]
        self.dids_t = torch.from_numpy(self.dids if len(self.dids) else np.zeros(1, np.int32)).cuda()
        self.initial = self.dst.buf.clone()
        self.scales_np = (rng.uniform(0.1, 4.0, dst_nl * no) * (1 + np.arange(dst_nl * no) * 1e-2)).astype(np.float32) if scaled else None
        self.scales = torch.from_numpy(self.scales_np).cuda() if scaled else None
        self.layer_done = torch.zeros(dst_nl, dtype=torch.int32, device="cuda")
        self.done = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.completion = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.ws = torch.zeros(K.sync_workspace_words(dst_nl), dtype=torch.int32, device="cuda")
        self.side_stream = torch.cuda.Stream()

    def expected(self):
        init = self.initial.cpu().numpy()
        d = self.dst
        sources = [([p.final_np[b] for b in self.sids[s]], p.kv, p.nh, p.nl) for s, p in enumerate(self.srcs)]
        new = stage_repage_gather(sources, self.windows, [init[b] for b in self.dids], d.kv, d.nh, d.nl, self.no, self.ps, self.pd, self.row,
                                  self.tb, self.te, self.cast, self.scales_np, range(self.lb, self.le))
        for b, blk in zip(self.dids, new):
            init[b] = blk
        return init

    def args(self):
        return (self.sources(), self.ps, self.dst.side(self.dids_t), self.dst.nh, self.pd, self.tb, self.te, self.lb, self.le, self.row,
                self.cast, self.scales)

    def run(self):
        rc = K.paged_stage_repage_gather(*self.args(), self.done.data_ptr(), 5, self.completion.data_ptr(), 6, stream_ptr())
        torch.cuda.synchronize()
        return rc

    def stream_desc(self, epoch, gate_mode, timeout_ms):
        st = super().stream_desc(epoch, gate_mode, timeout_ms)
        st.completion_value = epoch          # a completion word that counts hand-offs by the producer's epoch
        return st

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
            K.check(K.paged_stage_repage_gather_streamed(*self.args(), st, stream_ptr(self.side_stream)), "launch")
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
        assert self.done.item() == epoch and self.completion.item() == epoch
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
    return StageRepageRig(srcs, windows, dparts[rank // dst_tp], max(1, H // dst_tp), dst_kv, **kw)


PLANS = {
    "pp2tp4_to_tp2_rank1": (8, 8, 4, 2, 2, 1, 1),
    "pp4tp2_to_tp1": (8, 8, 2, 4, 1, 1, 0),
    "pp2tp2_to_tp4_replicated_rank3": (2, 8, 2, 2, 4, 1, 3),
    "pp3_uneven_3_3_4_to_tp2_rank1": (4, 10, 1, 3, 2, 1, 1, [3, 3, 4]),
    "pp2tp4_to_pp2tp2_rank3": (8, 8, 4, 2, 2, 2, 3),
}


@pytest.mark.parametrize("ps,pd", PAGES, ids=lambda p: str(p))
@pytest.mark.parametrize("name", list(PLANS))
def test_plans_and_pages(name, ps, pd):
    r = _plan_rig(*PLANS[name], src_kv=KV.OperationalHND, dst_kv=KV.OperationalNHD, ps=ps, pd=pd, seed=len(name) + ps + pd)
    assert r.run() == 0
    r.check()
    assert r.done.item() == 5 and r.completion.item() == 6


@pytest.mark.parametrize("dst_kv", ALL, ids=lambda k: k.name)
@pytest.mark.parametrize("src_kv", ALL, ids=lambda k: k.name)
def test_every_format_pair(src_kv, dst_kv):
    """PP2 x TP2 -> TP1 over 6 layers, 16 <-> 64-token pages by turns."""
    ps, pd = (16, 64) if (int(src_kv) + int(dst_kv)) % 2 else (64, 16)
    r = _plan_rig(4, 6, 2, 2, 1, 1, 0, src_kv=src_kv, dst_kv=dst_kv, ps=ps, pd=pd, seed=10 * int(src_kv) + int(dst_kv))
    assert r.run() == 0
    r.check()


@pytest.mark.parametrize("hd", [64, 80, 128])
@pytest.mark.parametrize("scaled", [False, True], ids=["unscaled", "scaled"])
@pytest.mark.parametrize("cast", [CM.FP8E4M3_TO_BF16, CM.BF16_TO_FP8E4M3], ids=lambda c: c.name)
def test_casts_scales_head_dims_and_a_range_across_a_stage_boundary(cast, scaled, hd):
    """Layers 2..6 of PP2 x TP4 -> TP2 cross the stage boundary at layer 4; the scales are the destination layers'."""
    for layers, (ps, pd) in ((None, (16, 64)), (range(2, 6), (48, 6))):
        r = _plan_rig(8, 8, 4, 2, 2, 1, 1, src_kv=KV.OperationalNHD, dst_kv=KV.UniversalPP, cast=cast, scaled=scaled, layers=layers, hd=hd,
                      ps=ps, pd=pd, seed=int(cast) + 3 * scaled + hd)
        assert r.run() == 0
        r.check()


@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16], ids=lambda c: c.name)
def test_mla_one_head_pp_only(cast):
    """MLA's one 576-wide latent head: a PP4 -> PP1 plan with no head split."""
    r = _plan_rig(1, 8, 1, 4, 1, 1, 0, ps=64, pd=16, hd=576, no=1, cast=cast, seed=5)
    assert r.run() == 0
    r.check()


def _kernels(prof):
    """The library's kernels among the profiler's events, templated or not."""
    return {m.group(1) for e in prof.events() for m in re.finditer(r"(kvbm_\w+_kernel)\b", e.name)}


@pytest.mark.parametrize("tp", [(4, 2), (1, 1)], ids=["tp4_to_tp2", "tp1_full_window"])
def test_a_pp1_plan_is_the_repage_gather(tp):
    """Identity layer windows over pools of the destination's layer count give the re-paging gather's bytes and take its launch:
    kvbm_paged_repage_gather_kernel, or kvbm_paged_repage_kernel for one window over every head, then the signal kernel.
    The profiled window holds host work on both sides of the launch (the rig's set-up, the oracle's check), as every other
    profiler test here does.  A window that closes right after the launch's synchronize keeps the cudaLaunchKernel records
    but, late in a long process, mostly loses the kernels' device records (38 of 40 such sessions after the GPU suite on an
    H100, none of 40 with the host work inside)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        a = _plan_rig(8, 4, tp[0], 1, tp[1], 1, 0, seed=3)
        assert a.run() == 0
        a.check()
    want = "kvbm_paged_repage_kernel" if tp == (1, 1) else "kvbm_paged_repage_gather_kernel"
    assert _kernels(prof) == {want, "kvbm_signal_kernel"}
    b = _plan_rig(8, 4, tp[0], 1, tp[1], 1, 0, seed=3)
    srcs = [x.src for x in b.sources()]
    K.check(K.paged_repage_gather(srcs, b.ps, b.dst.side(b.dids_t), b.dst.nh, b.pd, b.tb, b.te, 0, 4, b.row, stream=stream_ptr()), "gather")
    torch.cuda.synchronize()
    assert torch.equal(a.dst.buf, b.dst.buf)


# ---------------------------------------------------------------------------------------------------------------------
# every instantiation of the two families, reached under the profiler
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True))}
EXPECTED = {(f, w + (pp,)) for f in ("paged", "gated") for w in WALKS for pp in (True, False)}


def test_staged_plans_reach_every_repage_gather_instantiation():
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c, p, s in sorted(WALKS):
            for ppow2 in (True, False):
                for gated in (False, True):
                    ps, pd = (16, 64) if ppow2 else (48, 12)
                    r = _plan_rig(8, 8, 4, 2, 2, 1, 0, dst_kv=KV.UniversalTP, cast=CM(c), scaled=s, hd=64 if p else 80, ps=ps, pd=pd,
                                  seed=c + 2 * p + 4 * s + 8 * ppow2)
                    if gated:
                        for q in r.srcs:
                            q.ready.fill_(9)
                        torch.cuda.synchronize()
                        K.check(K.paged_stage_repage_gather_streamed(*r.args(), r.stream_desc(9, K.GATE_SPIN, 10000), stream_ptr()), "gated")
                        torch.cuda.synchronize()
                    else:
                        assert r.run() == 0
                    r.check()
    found = set()
    for e in prof.events():
        for m in re.finditer(r"kvbm_(paged|gated)_repage_gather_kernel<([^<>]*)>", e.name):
            c, p, s, pp = (a.strip().replace("(int)", "") for a in m.group(2).split(","))
            found.add((m.group(1), (int(c), p == "true", s == "true", pp == "true")))
    assert found == EXPECTED


# ---------------------------------------------------------------------------------------------------------------------
# streamed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("name,ps,pd", [("pp2tp4_to_tp2_rank1", 16, 64), ("pp4tp2_to_tp1", 64, 16), ("pp3_uneven_3_3_4_to_tp2_rank1", 12, 48)])
def test_streamed_stage_by_stage(gate_mode, name, ps, pd):
    """One producer stream releases stage 0's layers, then stage 1's, each source by its own layer numbers.  The sources' flag
    arrays are followed by guard words below the epoch: a spinning gate that read a destination-layer index past a source's
    array would time out (0xFFFFFFFF completion), not hang."""
    r = _plan_rig(*PLANS[name], src_kv=KV.OperationalHND, dst_kv=KV.UniversalTP, ps=ps, pd=pd, seed=7, poison=True, cast=CM.FP8E4M3_TO_BF16,
                  scaled=True)
    r.run_streamed(3, gate_mode, timeout_ms=3000)


@pytest.mark.parametrize("ctas", [1, 2, 3])
def test_spinning_batches_cross_a_stage_boundary(ctas):
    """7 big blocks and one outer index: 7 units per layer, so at 1-3 CTAs a batch is 4 or 2 units, batches span layers and one
    crosses from stage 0 (layers 0-2) into stage 1 at unit 21."""
    per_layer, grid = 7, ctas
    batch = min(8, max(1, (per_layer + 2 * grid - 1) // (2 * grid)))
    assert any(u // per_layer == 2 and (u + batch - 1) // per_layer == 3 for u in range(0, 6 * per_layer, batch))
    r = _plan_rig(4, 6, 2, 2, 1, 1, 0, ps=16, pd=64, tokens=range(0, 7 * 64), no=1, seed=ctas, poison=True, max_ctas=ctas)
    r.run_streamed(5, K.GATE_SPIN, timeout_ms=3000)


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_sixteen_sources_over_256_heads(gate_mode):
    """PP2 x TP8 -> TP1 over 128 heads: 16 sources, 8 per stage, 128 covered heads per stage and 256 over both."""
    r = _plan_rig(128, 2, 8, 2, 1, 1, 0, ps=16, pd=64, tokens=range(5, 60), no=1, seed=16, poison=True)
    assert len(r.windows) == 16 and sum(w[6] for w in r.windows) == 256
    r.run_streamed(2, gate_mode, timeout_ms=3000)


# ---------------------------------------------------------------------------------------------------------------------
# through the TransferManager
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=10)
    yield m
    torch.cuda.synchronize()
    m.close()


@pytest.mark.parametrize("streamed", [False, True], ids=["unstreamed", "streamed"])
def test_manager_stage_repage_gather(mgr, streamed):
    """PP2 x TP4 -> TP2 decode rank 1 with 16 -> 64-token pages over layers 2..6 through execute_stage_repage_gather: one launch,
    one notification, the oracle's bytes, bytes_moved over each window's layers inside the range; streamed with every flag
    already released (the stream-wait form)."""
    H, L = 8, 8
    plan = tp_pp_reshard_plan(H, L, 4, 2, 2, 1, 1)
    r = _plan_rig(H, L, 4, 2, 2, 1, 1, src_kv=KV.UniversalTP, dst_kv=KV.OperationalNHD, ps=16, pd=64, layers=range(2, 6), seed=21)
    ranks = sorted({w.src_rank for w in plan})
    hs = {rk: _register(mgr, r.srcs[i], KV.UniversalTP) for i, rk in enumerate(ranks)}
    dh = _register(mgr, r.dst, KV.OperationalNHD)
    sources = {rk: (hs[rk], [int(x) for x in r.sids[i]]) for i, rk in enumerate(ranks)}
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    moved0 = mgr.bytes_moved()
    kw = dict(done_flag=flag.data_ptr(), epoch=4, layer_range=range(2, 6))
    tokens = range(r.tb, r.te)
    if streamed:
        for p in r.srcs:
            p.ready.fill_(4)
        torch.cuda.synchronize()
        note = mgr.execute_stage_repage_gather(sources, dh, [int(x) for x in r.dids], plan, tokens,
                                               TransferOptions(gate_mode=K.GATE_STREAM_WAIT, **kw),
                                               ready_flags={rk: r.srcs[i].ready.data_ptr() for i, rk in enumerate(ranks)},
                                               layer_done_flags=r.layer_done.data_ptr())
    else:
        note = mgr.execute_stage_repage_gather(sources, dh, [int(x) for x in r.dids], plan, tokens, TransferOptions(**kw))
    note.wait(20.0)
    torch.cuda.synchronize()
    r.check()
    assert flag.item() == 4
    inside = lambda w: max(0, min(6, w.dst_layer_begin + w.layer_count) - max(2, w.dst_layer_begin))  # noqa: E731
    assert mgr.bytes_moved() - moved0 == sum(len(tokens) * inside(w) * r.no * w.head_count * r.row for w in plan)
    if streamed:
        assert r.layer_done.tolist() == [4 if 2 <= l < 6 else 0 for l in range(L)]

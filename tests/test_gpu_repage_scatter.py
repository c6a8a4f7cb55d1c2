"""GPU parity of the re-paging scatter (one prefill rank's KV to every decode rank that needs it, in one launch):
kvbm_kernels_paged_repage_scatter and TransferManager.execute_repage_scatter, each case against tests/scatter_oracle AND against
one kvbm_kernels_paged_stage_repage_gather launch per target, over whole destination pools: guard blocks no table names, heads
and layers no target covers, and the slots of the first and last blocks outside the token range all keep their random bytes and
are compared.  Every pool lives on one GPU."""
import dataclasses
import re

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import TransferManager, TransferOptions, tp_pp_scatter_plan
from tests.gpu_util import stream_ptr
from tests.repage_oracle import table_slice
from tests.scatter_oracle import dst_layers, dst_scales, repage_scatter
from tests.test_gpu_stage_gather import ELEMS, _register
from tests.test_gpu_transform_stream import Pool

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
ALL = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]
PAGES = [(16, 64), (64, 16), (1, 16), (12, 48), (16, 16)]


def _tokens(ps, pd):
    """A range that starts and ends inside blocks of the larger page; equal pages: whole blocks but a partial last one."""
    if ps == pd:
        return range(0, 3 * ps + 5)
    big = max(ps, pd)
    return range(3, 2 * big - 5 if big > 8 else 2 * big + 3)


class ScatterRig:
    """src: (num_layers, num_heads, kv) of the source pool at page ps; dsts: (num_layers, num_heads, kv) per destination pool at
    page pd; targets: (pool, src_layer_begin, dst_layer_begin, layer_count, src_head_begin, dst_head_begin, head_count).  Every
    pool has two blocks no table names; every target of a pool takes that pool's one table."""

    def __init__(self, src, dsts, targets, ps=16, pd=64, tokens=None, no=2, hd=64, cast=CM.NONE, scaled=False, layers=None, seed=0):
        se, de = ELEMS[cast]
        self.row, self.cast, self.targets, self.no, self.ps, self.pd = hd * se, int(cast), targets, no, ps, pd
        tokens = tokens if tokens is not None else _tokens(ps, pd)
        self.tb, self.te = tokens.start, tokens.stop
        nl, nh, kv = src
        self.lb, self.le = (layers.start, layers.stop) if layers else (0, nl)
        ns, nd = max(1, -(-self.te // ps)), max(1, -(-self.te // pd))
        self.src = Pool(ns + 2, nl, no, ps, nh, hd * se, kv, seed + 10)
        self.dsts = [Pool(nd + 2, dnl, no, pd, dnh, hd * de, dkv, seed + 20 + i) for i, (dnl, dnh, dkv) in enumerate(dsts)]
        rng = np.random.default_rng(seed + 2)
        self.sids = np.array(table_slice(rng.permutation(ns + 2)[:ns], self.tb, self.te, ps), dtype=np.int32)
        self.dids = [np.array(table_slice(rng.permutation(nd + 2)[:nd], self.tb, self.te, pd), dtype=np.int32) for _ in dsts]
        as_t = lambda x: torch.from_numpy(x if len(x) else np.zeros(1, np.int32)).cuda()  # noqa: E731
        self.sids_t, self.dids_t = as_t(self.sids), [as_t(x) for x in self.dids]
        self.initial = [p.buf.clone() for p in self.dsts]
        self.scales_np = (rng.uniform(0.1, 4.0, nl * no) * (1 + np.arange(nl * no) * 1e-2)).astype(np.float32) if scaled else None
        self.scales = torch.from_numpy(self.scales_np).cuda() if scaled else None
        self.done = torch.zeros(len(targets), dtype=torch.int32, device="cuda")
        self.completion = torch.zeros(1, dtype=torch.int32, device="cuda")

    def kernel_targets(self):
        return [K.ScatterTarget(self.dsts[p].side(self.dids_t[p]), self.dsts[p].nh, sb, db, k, sl, dl, c, self.done[t:].data_ptr())
                for t, (p, sl, dl, c, sb, db, k) in enumerate(self.targets)]

    def launch(self, epoch=5, value=6, tokens=None):
        tb, te = (tokens.start, tokens.stop) if tokens is not None else (self.tb, self.te)
        return K.paged_repage_scatter(self.src.side(self.sids_t), self.src.nh, self.ps, self.kernel_targets(), self.pd, tb, te, self.lb, self.le,
                                      self.row, self.cast, self.scales, epoch, self.completion.data_ptr(), value, stream_ptr())

    def expected(self):
        pools = [x.cpu().numpy() for x in self.initial]
        s = self.src
        targets = [(p, self.dids[p], self.dsts[p].kv, self.dsts[p].nh, self.dsts[p].nl, (sl, dl, c, sb, db, k))
                   for p, sl, dl, c, sb, db, k in self.targets]
        repage_scatter(([s.final_np[b] for b in self.sids], s.kv, s.nh, s.nl), targets, pools, self.no, self.ps, self.pd, self.row, self.tb,
                       self.te, self.cast, self.scales_np, range(self.lb, self.le))
        return pools

    def gathers(self):
        """The same bytes as one kvbm_kernels_paged_stage_repage_gather launch per target, from the initial pools."""
        for p, x in zip(self.dsts, self.initial):
            p.buf.copy_(x)
        keep = []
        for p, sl, dl, c, sb, db, k in self.targets:
            img = dst_layers((sl, dl, c), range(self.lb, self.le))
            if len(img) == 0:
                continue
            d = self.dsts[p]
            sc = dst_scales((sl, dl, c), self.scales_np, d.nl, self.no)
            sc_t = torch.from_numpy(sc).cuda() if sc is not None else None
            keep.append(sc_t)
            src = [K.StageSource(K.PermuteSource(self.src.side(self.sids_t), self.src.nh, sb, db, k), sl, dl, c)]
            K.check(K.paged_stage_repage_gather(src, self.ps, d.side(self.dids_t[p]), d.nh, self.pd, self.tb, self.te, img.start, img.stop,
                                                self.row, self.cast, sc_t, stream=stream_ptr()), "stage_repage_gather")
        torch.cuda.synchronize()
        return [p.buf.clone() for p in self.dsts]

    def run_and_check(self, epoch=5, value=6):
        """The scatter against the oracle, its flags, then against the per-target gathers."""
        assert self.launch(epoch, value) == 0
        torch.cuda.synchronize()
        got = [p.buf.clone() for p in self.dsts]
        for g, want in zip(got, self.expected()):
            assert np.array_equal(g.cpu().numpy(), want)
        assert self.done.tolist() == [epoch] * len(self.targets) and self.completion.item() == value
        for g, ref in zip(got, self.gathers()):
            assert torch.equal(g, ref)


def _plan_rig(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, src_parts=None, dst_parts=None, src_kv=KV.OperationalHND, dst_kvs=(KV.OperationalNHD,),
              **kw):
    """The scatter plan of prefill rank `rank`: one source pool with its stage's layers and heads, one pool per decode rank the plan
    names (formats from dst_kvs by turns)."""
    plan = tp_pp_scatter_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, src_parts, dst_parts)
    sparts = list(src_parts) if src_parts else [L // src_pp] * src_pp
    dparts = list(dst_parts) if dst_parts else [L // dst_pp] * dst_pp
    ranks = sorted({w.dst_rank for w in plan})
    dsts = [(dparts[r // dst_tp], max(1, H // dst_tp), dst_kvs[i % len(dst_kvs)]) for i, r in enumerate(ranks)]
    targets = [(ranks.index(w.dst_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
               for w in plan]
    return ScatterRig((sparts[rank // src_tp], max(1, H // src_tp), src_kv), dsts, targets, **kw)


PLANS = {
    "tp2_to_tp4_rank0": (8, 4, 2, 1, 4, 1, 0),
    "tp1_to_tp8": (8, 4, 1, 1, 8, 1, 0),
    "h8_tp2_to_tp16_rank0": (8, 4, 2, 1, 16, 1, 0),
    "pp2tp2_rank0_to_pp3tp2": (4, 12, 2, 2, 2, 3, 0),
    "pp2tp2_rank3_to_pp3tp2": (4, 12, 2, 2, 2, 3, 3),
}


@pytest.mark.parametrize("ps,pd", PAGES, ids=lambda p: str(p))
@pytest.mark.parametrize("name", list(PLANS))
def test_plans_and_pages(name, ps, pd):
    r = _plan_rig(*PLANS[name], ps=ps, pd=pd, seed=len(name) + ps + pd)
    r.run_and_check()


def test_the_plans_shapes():
    """TP2 -> TP16 sends each of the rank's 4 heads to 2 decode ranks; a PP2 source stage splits across two PP3 decode stages."""
    r = _plan_rig(*PLANS["h8_tp2_to_tp16_rank0"])
    assert len(r.targets) == 8 and sorted(t[4] for t in r.targets) == [0, 0, 1, 1, 2, 2, 3, 3]
    r = _plan_rig(*PLANS["pp2tp2_rank0_to_pp3tp2"])
    assert sorted({(t[1], t[3]) for t in r.targets}) == [(0, 4), (4, 2)]


@pytest.mark.parametrize("ps,pd", [(64, 64), (1, 64)], ids=lambda p: str(p))
@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16], ids=lambda c: c.name)
def test_mla_latent_head_to_eight_targets(cast, ps, pd):
    """MLA's one 576-wide latent head on every decode TP rank: 8 targets, one source head, 8 pairs."""
    r = _plan_rig(1, 4, 1, 1, 8, 1, 0, ps=ps, pd=pd, hd=576, no=1, cast=cast, seed=5 + ps)
    assert len(r.targets) == 8
    r.run_and_check()


@pytest.mark.parametrize("cast,scaled", [(CM.NONE, False)] + [(c, s) for c in (CM.FP8E4M3_TO_BF16, CM.BF16_TO_FP8E4M3) for s in (False, True)],
                         ids=lambda v: v.name if isinstance(v, CM) else ("scaled" if v else "unscaled"))
def test_casts_scales_mixed_formats_and_a_layer_sub_range(cast, scaled):
    """TP1 -> TP4 into four destination formats, source layers 1..3 of 4; the scales are the source's, by source layer."""
    for layers, (ps, pd) in ((None, (16, 64)), (range(1, 3), (48, 12))):
        r = _plan_rig(8, 4, 1, 1, 4, 1, 0, src_kv=KV.OperationalNHD, dst_kvs=ALL, cast=cast, scaled=scaled, layers=layers, ps=ps, pd=pd,
                      seed=int(cast) + 3 * scaled)
        r.run_and_check()


def test_one_pool_in_two_targets():
    """Every source head twice into one pool (heads 0..3 and 4..7 of it), through the same table: disjoint rectangles."""
    r = ScatterRig((4, 4, KV.OperationalHND), [(4, 8, KV.OperationalNHD)], [(0, 0, 0, 4, 0, 0, 4), (0, 0, 0, 4, 0, 4, 4)], seed=9)
    r.run_and_check()


def test_sixteen_targets_and_256_pairs():
    """16 pools, each taking all 16 heads of the source: 16 entries of 16 pairs."""
    r = ScatterRig((2, 16, KV.OperationalNHD), [(2, 16, ALL[i % 4]) for i in range(16)], [(i, 0, 0, 2, 0, 0, 16) for i in range(16)],
                   tokens=range(5, 60), no=1, seed=16)
    assert len(r.targets) == 16 and sum(t[6] for t in r.targets) == 256
    r.run_and_check()


def test_an_empty_range_signals_every_target():
    r = _plan_rig(*PLANS["tp1_to_tp8"], seed=3)
    before = [p.buf.clone() for p in r.dsts]
    assert r.launch(7, 8, tokens=range(9, 9)) == 0
    torch.cuda.synchronize()
    assert r.done.tolist() == [7] * 8 and r.completion.item() == 8
    assert all(torch.equal(a, p.buf) for a, p in zip(before, r.dsts))


# ---------------------------------------------------------------------------------------------------------------------
# every instantiation, reached under the profiler
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True))}
EXPECTED = {w + (pp,) for w in WALKS for pp in (True, False)}


def test_every_scatter_instantiation():
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c, p, s in sorted(WALKS):
            for ppow2 in (True, False):
                ps, pd = (16, 64) if ppow2 else (48, 12)
                r = _plan_rig(8, 4, 2, 1, 4, 1, 0, dst_kvs=(KV.UniversalTP, KV.OperationalHND), cast=CM(c), scaled=s, hd=64 if p else 80,
                              ps=ps, pd=pd, seed=c + 2 * p + 4 * s + 8 * ppow2)
                r.run_and_check()
    found = set()
    for e in prof.events():
        for m in re.finditer(r"kvbm_paged_repage_scatter_kernel<([^<>]*)>", e.name):
            c, p, s, pp = (a.strip().replace("(int)", "") for a in m.group(1).split(","))
            found.add((int(c), p == "true", s == "true", pp == "true"))
    assert found == EXPECTED and len(found) == 20


# ---------------------------------------------------------------------------------------------------------------------
# through the TransferManager
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=11)
    yield m
    torch.cuda.synchronize()
    m.close()


def test_manager_repage_scatter(mgr):
    """PP2 x TP2 prefill rank 0 into the decode ranks 0 and 2 of PP3 x TP2 that need it, 16 -> 64-token pages, source layers
    [1, 5) of 6: one launch, one notification, the oracle's bytes, per-destination done flags, the done flag, and bytes_moved
    over each window's layers inside the range.  The plan's dst_rank is renumbered to index the destinations passed."""
    H, L = 4, 12
    full = tp_pp_scatter_plan(H, L, 2, 2, 2, 3, 0)
    r = _plan_rig(H, L, 2, 2, 2, 3, 0, src_kv=KV.UniversalTP, ps=16, pd=64, layers=range(1, 5), seed=21)
    ranks = sorted({w.dst_rank for w in full})
    assert ranks == [0, 2]
    plan = [dataclasses.replace(w, dst_rank=ranks.index(w.dst_rank)) for w in full]
    sh = _register(mgr, r.src, KV.UniversalTP)
    dhs = [_register(mgr, p, KV.OperationalNHD) for p in r.dsts]
    flags = torch.zeros(len(ranks) + 1, dtype=torch.int32, device="cuda")
    moved0 = mgr.bytes_moved()
    tokens = range(r.tb, r.te)
    opts = TransferOptions(done_flag=flags[len(ranks):].data_ptr(), epoch=4, layer_range=range(1, 5),
                           per_dst_done_flags=[flags[d:].data_ptr() for d in range(len(ranks))])
    note = mgr.execute_repage_scatter(sh, [int(x) for x in r.sids], dhs, [[int(x) for x in d] for d in r.dids], plan, tokens, opts)
    note.wait(20.0)
    torch.cuda.synchronize()
    for p, want in zip(r.dsts, r.expected()):
        assert np.array_equal(p.buf.cpu().numpy(), want)
    assert flags.tolist() == [4] * (len(ranks) + 1)
    inside = lambda w: max(0, min(5, w.src_layer_begin + w.layer_count) - max(1, w.src_layer_begin))  # noqa: E731
    assert mgr.bytes_moved() - moved0 == sum(len(tokens) * inside(w) * r.no * w.head_count * r.row for w in plan)

"""GPU parity of the batch re-paging scatter (a prefill batch's sequences pushed to every decode rank that needs them, in one launch):
kvbm_kernels_paged_repage_scatter_batch, its streamed form and TransferManager.execute_repage_scatter_batch.  Every case compares
whole destination pools, guard blocks included, with tests/scatter_batch_oracle.py, and the unstreamed cases also byte for byte with
one kvbm_kernels_paged_repage_scatter launch per sequence from the same initial pools.  Every sequence starts inside a block of the
larger page.  Every test ends with a device synchronize."""
import re

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import ErrorCode, KvbmError, ScatterWindow, TransferManager, TransferOptions, tp_pp_scatter_plan
from tests.gpu_util import stream_ptr
from tests.scatter_batch_oracle import repage_scatter_batch, table_len
from tests.test_gpu_scatter_stream import MAX_CTAS, StreamRig, _Layers, _finish
from tests.test_gpu_stage_gather import ELEMS, _register
from tests.test_gpu_transform_stream import GATE_IDS, GATES, MASK, Pool, _i32

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode


def _batch(n, length, first=3, step=11):
    return [(first + step * i, first + step * i + length) for i in range(n)]


def _mixed(seed=7):
    """1 to 4000 tokens, empty sequences between others."""
    rng = np.random.default_rng(seed)
    lens = [1, 4000] + [int(x) for x in rng.integers(1, 4001, 8)]
    out = []
    for i, n in enumerate(lens):
        tb = int(rng.integers(1, 300)) | 1
        out.append((tb, tb + n))
        if i % 3 == 1:
            out.append((tb + 5, tb + 5))
    return out


BATCHES = {"8x2048": _batch(8, 2048), "32x512": _batch(32, 512), "128x128": _batch(128, 128, step=5), "mixed": _mixed()}


class BatchRig:
    """src: (num_layers, num_heads, kv) of the source pool at page ps; dsts: (num_layers, num_heads, kv) per destination pool at page
    pd; targets: (pool, src_layer_begin, dst_layer_begin, layer_count, src_head_begin, dst_head_begin, head_count); seqs: the token
    ranges.  Every pool has two blocks no table names; every target of a pool takes that pool's one concatenated table.  share:
    the source table draws its blocks with repeats (sequences sharing source blocks)."""

    def __init__(self, src, dsts, targets, seqs, ps=16, pd=64, no=2, hd=64, cast=CM.NONE, scaled=False, layers=None, seed=0, share=False,
                 poison=False):
        se, de = ELEMS[cast]
        self.row, self.cast, self.targets, self.no, self.ps, self.pd, self.seqs = hd * se, int(cast), targets, no, ps, pd, list(seqs)
        nl, nh, kv = src
        self.lb, self.le = (layers.start, layers.stop) if layers else (0, nl)
        ns = sum(table_len(tb, te, ps) for tb, te in self.seqs)
        nd = sum(table_len(tb, te, pd) for tb, te in self.seqs)
        nsb = ns // 2 + 2 if share else ns + 2
        self.src = Pool(nsb, nl, no, ps, nh, hd * se, kv, seed + 10, poison=poison)
        self.dsts = [Pool(nd + 2, dnl, no, pd, dnh, hd * de, dkv, seed + 20 + i) for i, (dnl, dnh, dkv) in enumerate(dsts)]
        rng = np.random.default_rng(seed + 2)
        self.sids = (rng.integers(0, nsb, ns) if share else rng.permutation(nsb)[:ns]).astype(np.int32)
        self.dids = [rng.permutation(nd + 2)[:nd].astype(np.int32) for _ in dsts]
        u = K.repage_batch_units(self.seqs, ps, pd)
        assert u is not None and (u[1], u[2]) == (ns, nd)
        self.units_np, self.nu = u[0], len(u[0])
        as_t = lambda x: torch.from_numpy(x if len(x) else np.zeros(1, np.int32)).cuda()  # noqa: E731
        self.sids_t, self.dids_t = as_t(self.sids), [as_t(x) for x in self.dids]
        self.units_t = as_t(np.ascontiguousarray(self.units_np).view(np.int32).reshape(-1))
        self.initial = [p.buf.clone() for p in self.dsts]
        self.scales_np = (rng.uniform(0.1, 4.0, nl * no) * (1 + np.arange(nl * no) * 1e-2)).astype(np.float32) if scaled else None
        self.scales = torch.from_numpy(self.scales_np).cuda() if scaled else None
        self.done = torch.zeros(len(targets), dtype=torch.int32, device="cuda")
        self.completion = torch.zeros(1, dtype=torch.int32, device="cuda")

    def kernel_targets(self, dids_t=None):
        dids_t = dids_t or self.dids_t
        return [K.ScatterTarget(self.dsts[p].side(dids_t[p]), self.dsts[p].nh, sb, db, k, sl, dl, c, self.done[t:].data_ptr())
                for t, (p, sl, dl, c, sb, db, k) in enumerate(self.targets)]

    def launch(self, epoch=5, value=6):
        return K.paged_repage_scatter_batch(self.src.side(self.sids_t), self.src.nh, self.ps, self.kernel_targets(), self.pd, self.seqs,
                                            self.units_t.data_ptr(), self.nu, self.lb, self.le, self.row, self.cast, self.scales, epoch,
                                            self.completion.data_ptr(), value, stream_ptr())

    def expected(self):
        pools = [x.cpu().numpy() for x in self.initial]
        s = self.src
        targets = [(p, self.dids[p], self.dsts[p].kv, self.dsts[p].nh, self.dsts[p].nl, (sl, dl, c, sb, db, k))
                   for p, sl, dl, c, sb, db, k in self.targets]
        repage_scatter_batch((s.final_np, self.sids, s.kv, s.nh, s.nl), targets, pools, self.no, self.ps, self.pd, self.row, self.seqs,
                             self.cast, self.scales_np, range(self.lb, self.le))
        return pools

    def singles(self, initial=None):
        """One kvbm_kernels_paged_repage_scatter launch per sequence, from `initial` (the rig's initial pools by default)."""
        for p, x in zip(self.dsts, initial or self.initial):
            p.buf.copy_(x)
        so = do = 0
        keep = []
        for tb, te in self.seqs:
            a, b = table_len(tb, te, self.ps), table_len(tb, te, self.pd)
            if a:
                s_t = self.sids_t[so:so + a]
                d_t = [d[do:do + b] for d in self.dids_t]
                keep += [s_t, d_t]
                K.check(K.paged_repage_scatter(self.src.side(s_t), self.src.nh, self.ps, self.kernel_targets(d_t), self.pd, tb, te, self.lb,
                                               self.le, self.row, self.cast, self.scales, stream=stream_ptr()), "single scatter")
            so, do = so + a, do + b
        torch.cuda.synchronize()
        return [p.buf.clone() for p in self.dsts]

    def run_and_check(self, epoch=5, value=6, singles=True):
        assert self.launch(epoch, value) == 0
        torch.cuda.synchronize()
        got = [p.buf.clone() for p in self.dsts]
        for g, want in zip(got, self.expected()):
            assert np.array_equal(g.cpu().numpy(), want)
        assert self.done.tolist() == [epoch] * len(self.targets) and self.completion.item() == value
        if singles:
            for g, ref in zip(got, self.singles()):
                assert torch.equal(g, ref)


def _plan_rig(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, seqs, src_kv=KV.OperationalHND, dst_kvs=(KV.OperationalNHD,), **kw):
    """The scatter plan of prefill rank `rank` (equal PP stages): one source pool with its stage's layers and heads, one pool per
    decode rank the plan names."""
    plan = tp_pp_scatter_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank)
    ranks = sorted({w.dst_rank for w in plan})
    dsts = [(L // dst_pp, max(1, H // dst_tp), dst_kvs[i % len(dst_kvs)]) for i in range(len(ranks))]
    targets = [(ranks.index(w.dst_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
               for w in plan]
    return BatchRig((L // src_pp, max(1, H // src_tp), src_kv), dsts, targets, seqs, **kw)


PLANS = {
    "tp2_to_tp16": (8, 2, 2, 1, 16, 1, 0),
    "tp1_to_tp8": (8, 2, 1, 1, 8, 1, 0),
    "pp2tp2_rank0_to_pp3tp2": (4, 12, 2, 2, 2, 3, 0),
}
SMALL = [(5, 200), (40, 41), (3, 3), (17, 333)]


@pytest.mark.parametrize("batch", list(BATCHES))
def test_batches(batch):
    """TP2 -> TP16 (replicated heads: every source head to two decode ranks), 16 -> 64-token pages."""
    r = _plan_rig(*PLANS["tp2_to_tp16"], BATCHES[batch], no=1, hd=32, seed=len(batch))
    r.run_and_check()
    torch.cuda.synchronize()


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (1, 16), (16, 16), (48, 96), (96, 48)], ids=str)
def test_pages(ps, pd):
    r = _plan_rig(*PLANS["tp1_to_tp8"], BATCHES["mixed"][:7] + SMALL, ps=ps, pd=pd, no=1, hd=32, seed=ps + pd)
    r.run_and_check()
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", list(PLANS))
def test_plans(name):
    r = _plan_rig(*PLANS[name], BATCHES["32x512"][:6] + SMALL, seed=len(name))
    r.run_and_check()
    torch.cuda.synchronize()


def test_mla_latent_head():
    """MLA's one 576-wide latent head to 8 decode ranks."""
    r = _plan_rig(1, 2, 1, 1, 8, 1, 0, SMALL + _batch(4, 300), no=1, hd=576, ps=64, pd=16, seed=57)
    assert len(r.targets) == 8
    r.run_and_check()
    torch.cuda.synchronize()


@pytest.mark.parametrize("cast,scaled", [(CM.FP8E4M3_TO_BF16, False), (CM.FP8E4M3_TO_BF16, True), (CM.BF16_TO_FP8E4M3, False),
                                         (CM.BF16_TO_FP8E4M3, True)], ids=["up", "up_scaled", "down", "down_scaled"])
def test_casts_and_scales(cast, scaled):
    """TP1 -> TP4 into four destination formats, source layers 1..3 of 4."""
    r = _plan_rig(8, 4, 1, 1, 4, 1, 0, SMALL + _batch(3, 100), src_kv=KV.OperationalNHD,
                  dst_kvs=(KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD), cast=cast, scaled=scaled,
                  layers=range(1, 3), seed=int(cast) + 3 * scaled)
    r.run_and_check()
    torch.cuda.synchronize()


def test_shared_source_blocks():
    r = _plan_rig(*PLANS["tp1_to_tp8"], BATCHES["mixed"], no=1, hd=32, share=True, seed=77)
    assert len(set(r.sids.tolist())) < len(r.sids)
    r.run_and_check()
    torch.cuda.synchronize()


def test_a_batch_of_one_is_the_single_scatter():
    for seqs in ([(37, 1000)], [(64, 64)]):
        r = _plan_rig(*PLANS["tp2_to_tp16"], seqs, seed=3)
        r.run_and_check()
    torch.cuda.synchronize()


def test_a_batch_equals_n_singles_over_poisoned_pools():
    """The destination pools start as poison: every byte the batch and the n singles leave is compared, whole pools."""
    r = _plan_rig(*PLANS["tp1_to_tp8"], BATCHES["mixed"], no=1, hd=32, seed=91)
    for p in r.dsts:
        p.buf.copy_(p.poison)
    r.initial = [p.buf.clone() for p in r.dsts]
    r.run_and_check()
    torch.cuda.synchronize()


def test_empty_batches_signal():
    r = _plan_rig(*PLANS["tp1_to_tp8"], [(9, 9), (70, 70)], seed=4)
    before = [p.buf.clone() for p in r.dsts]
    for seqs in ([], [(9, 9), (70, 70)]):
        r.done.zero_()
        assert K.paged_repage_scatter_batch(r.src.side(r.sids_t), r.src.nh, 16, r.kernel_targets(), 64, seqs, 0, 0, 0, r.le, r.row, 0, None,
                                            7, r.completion.data_ptr(), 8, stream_ptr()) == 0
        torch.cuda.synchronize()
        assert r.done.tolist() == [7] * 8 and r.completion.item() == 8
    assert all(torch.equal(a, p.buf) for a, p in zip(before, r.dsts))
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# limits
# ---------------------------------------------------------------------------------------------------------------------
def test_a_sequence_at_the_32_bit_token_bound():
    """A sequence whose last 64-token block ends at 2^32 beside others; one token more is rejected before any launch."""
    top = (1 << 32) - 64
    seqs = [(top - 200, top), (5, 90), (top - 1000, top - 930)]
    r = _plan_rig(*PLANS["tp2_to_tp16"], seqs, no=1, hd=32, seed=13)
    r.run_and_check()
    bad = seqs[:2] + [(top, top + 1)]
    assert K.repage_batch_units(bad, 16, 64) is None
    before = [p.buf.clone() for p in r.dsts]
    assert K.paged_repage_scatter_batch(r.src.side(r.sids_t), r.src.nh, 16, r.kernel_targets(), 64, bad, r.units_t.data_ptr(), r.nu + 1, 0,
                                        r.le, r.row) == K.CUDA_ERROR_INVALID_VALUE
    torch.cuda.synchronize()
    assert all(torch.equal(a, p.buf) for a, p in zip(before, r.dsts))


# ---------------------------------------------------------------------------------------------------------------------
# every instantiation of both families, reached under the profiler
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True))}
EXPECTED = {w + (pp,) for w in WALKS for pp in (True, False)}
SRC_KV = dict(src_kv=KV.OperationalHND)


def _found(prof, family):
    found = set()
    for e in prof.events():
        for m in re.finditer(family + r"<([^<>]*)>", e.name):
            c, p, s, pp = (a.strip().replace("(int)", "") for a in m.group(1).split(","))
            found.add((int(c), p == "true", s == "true", pp == "true"))
    return found


def test_every_instantiation():
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c, p, sc in sorted(WALKS):
            for ppow2 in (True, False):
                ps, pd = (16, 64) if ppow2 else (48, 12)
                r = _plan_rig(8, 4, 2, 1, 4, 1, 0, SMALL, dst_kvs=(KV.UniversalTP, KV.OperationalHND), cast=CM(c), scaled=sc,
                              hd=64 if p else 80, ps=ps, pd=pd, seed=c + 2 * p + 4 * sc + 8 * ppow2, **SRC_KV)
                r.run_and_check(singles=False)
                s = StreamBatch(r)
                s.r.src.buf.copy_(s.r.src.final)   # the flags released before the launch
                s.r.src.ready.fill_(3)
                torch.cuda.synchronize()
                s.launch(3, K.GATE_SPIN, 5)
                assert _finish(s.side_stream)
                torch.cuda.synchronize()
                s.check_end(3, 5)
    assert _found(prof, "kvbm_paged_repage_push_seqs_kernel") == EXPECTED
    assert _found(prof, "kvbm_gated_repage_push_seqs_kernel") == EXPECTED
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# the streamed batch, behind a producer that writes the source after the launch (tests/test_gpu_scatter_stream.py's discipline)
# ---------------------------------------------------------------------------------------------------------------------
class StreamBatch(StreamRig):
    """StreamRig over a BatchRig: `unstreamed` is the unstreamed batch's result."""

    def launch(self, epoch, gate_mode, value):
        r = self.r
        K.check(K.paged_repage_scatter_batch_streamed(r.src.side(r.sids_t), r.src.nh, r.ps, r.kernel_targets(), r.pd, r.seqs,
                                                      r.units_t.data_ptr(), r.nu, r.lb, r.le, r.row, r.cast, r.scales,
                                                      self.stream_desc(epoch, gate_mode, value), stream_ptr(self.side_stream)),
                "streamed batch")


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("name", ["tp2_to_tp16", "pp2tp2_rank0_to_pp3tp2"])
def test_streamed_layers_written_after_the_launch(gate_mode, name):
    s = StreamBatch(_plan_rig(*PLANS[name], BATCHES["mixed"][:6] + SMALL, hd=32, seed=len(name), **SRC_KV))
    s.run(5, gate_mode, 77)
    s.check_end(5, 77)
    torch.cuda.synchronize()


@pytest.mark.parametrize("max_ctas", [1, 2, 3])
def test_spinning_batches_that_span_layers(max_ctas):
    """A handful of units per layer on 1-3 CTAs: claims of several units cross layer boundaries."""
    s = StreamBatch(_plan_rig(8, 4, 2, 1, 4, 1, 0, [(3, 70), (5, 5), (100, 180), (1, 2)], no=1, seed=90 + max_ctas, **SRC_KV),
                    max_ctas=max_ctas)
    s.run(8, K.GATE_SPIN, 5)
    s.check_end(8, 5)
    torch.cuda.synchronize()


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_only_released_layers_move(gate_mode):
    """Release k source layers, observe once layer_done[k - 1] appears: only those layers landed, for every sequence, and no done
    flag is written."""
    from tests.test_gpu_transform_stream import CHECKER_SLEEP
    s = StreamBatch(_plan_rig(8, 4, 2, 1, 16, 1, 0, SMALL + _batch(3, 200), seed=41, **SRC_KV))
    r, k, epoch = s.r, 2, 7
    snaps = [p.buf.clone() for p in r.dsts]
    flags = [s.layer_done.clone(), r.done.clone(), s.st_done.clone()]
    with torch.cuda.stream(s.checker):
        for t, p in zip(snaps, r.dsts):
            t.copy_(p.buf)
    torch.cuda.synchronize()
    try:
        s.launch(epoch, gate_mode, 1)
        r.src.produce(range(k), epoch)
        with torch.cuda.stream(s.checker):
            K.check(K.wait_flag(s.layer_done.data_ptr() + 4 * (k - 1), epoch, stream_ptr(s.checker)), "wait_flag")
            torch.cuda._sleep(CHECKER_SLEEP)
            for t, f in zip(flags, (s.layer_done, r.done, s.st_done)):
                t.copy_(f)
            for t, p in zip(snaps, r.dsts):
                t.copy_(p.buf)
        assert _finish(s.checker), "layer_done of the released layers did not appear"
        r.src.produce(range(k, s.nl), epoch)
        assert _finish(s.side_stream) and _finish(r.src.stream)
    finally:
        s.rescue(epoch)
    s.check_end(epoch, 1)
    partial = BatchRig.expected(_Layers(r, range(0, k)))
    for t, want in zip(snaps, partial):
        assert np.array_equal(t.cpu().numpy(), want)
    assert flags[0].tolist() == [epoch if l < k else 0 for l in range(s.nl)]
    assert not flags[1].any().item() and flags[2].item() == 0
    torch.cuda.synchronize()


def test_a_gate_timeout_writes_no_done_flag():
    s = StreamBatch(_plan_rig(8, 4, 2, 1, 4, 1, 0, SMALL, seed=71, **SRC_KV), timeout_ms=200)
    r, epoch = s.r, 4
    try:
        s.launch(epoch, K.GATE_SPIN, 9)
        r.src.produce(range(2), epoch)
        assert _finish(s.side_stream), "the gate did not time out"
    finally:
        s.rescue(epoch)
    assert _i32(r.completion.item()) == _i32(MASK)
    assert not r.done.any().item() and s.st_done.item() == 0
    assert not s.ws.any().item()
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# TransferManager.execute_repage_scatter_batch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=53)
    yield m
    torch.cuda.synchronize()
    m.close()


def _managed(mgr, r):
    """Register the rig's pools; the plan renumbered to index the destinations passed, and the per-sequence requests."""
    sh = _register(mgr, r.src, KV(r.src.kv))
    dhs = [_register(mgr, p, KV(p.kv)) for p in r.dsts]
    plan = [ScatterWindow(p, sl, dl, c, sb, db, k) for p, sl, dl, c, sb, db, k in r.targets]
    reqs, so, do = [], 0, 0
    for tb, te in r.seqs:
        a, b = table_len(tb, te, r.ps), table_len(tb, te, r.pd)
        reqs.append((range(tb, te), [int(x) for x in r.sids[so:so + a]], [[int(x) for x in d[do:do + b]] for d in r.dids]))
        so, do = so + a, do + b
    return sh, dhs, plan, reqs


def test_manager_batch(mgr):
    """One call: the oracle's bytes, per-destination done flags, the done flag, and bytes_moved equal to the n single calls'."""
    r = _plan_rig(*PLANS["tp1_to_tp8"], BATCHES["mixed"], no=1, hd=32, seed=101)
    sh, dhs, plan, reqs = _managed(mgr, r)
    flags = torch.zeros(len(dhs) + 1, dtype=torch.int32, device="cuda")
    m0 = mgr.bytes_moved()
    for tokens, s, d in reqs:
        mgr.execute_repage_scatter(sh, s, dhs, d, plan, tokens).wait(20.0)
    singles_bytes = mgr.bytes_moved() - m0
    torch.cuda.synchronize()
    singles = [p.buf.clone() for p in r.dsts]
    for p, x in zip(r.dsts, r.initial):
        p.buf.copy_(x)
    torch.cuda.synchronize()
    opts = TransferOptions(done_flag=flags[len(dhs):].data_ptr(), epoch=4, per_dst_done_flags=[flags[d:].data_ptr() for d in range(len(dhs))])
    m0 = mgr.bytes_moved()
    mgr.execute_repage_scatter_batch(sh, dhs, reqs, plan, opts).wait(20.0)
    torch.cuda.synchronize()
    assert mgr.bytes_moved() - m0 == singles_bytes > 0
    for p, want, ref in zip(r.dsts, r.expected(), singles):
        assert np.array_equal(p.buf.cpu().numpy(), want) and torch.equal(p.buf, ref)
    assert flags.tolist() == [4] * (len(dhs) + 1)
    torch.cuda.synchronize()


def test_manager_duplicate_destination_across_sequences(mgr):
    r = _plan_rig(*PLANS["tp1_to_tp8"], [(3, 70), (100, 180)], seed=103)
    sh, dhs, plan, reqs = _managed(mgr, r)
    reqs[1][2][3][0] = reqs[0][2][3][0]
    with pytest.raises(KvbmError) as e:
        mgr.execute_repage_scatter_batch(sh, dhs, reqs, plan)
    assert e.value.code == ErrorCode.DUPLICATE_DST
    torch.cuda.synchronize()
    assert all(torch.equal(a, p.buf) for a, p in zip(r.initial, r.dsts))


def test_manager_300_sequences_outgrow_a_staging_slot(mgr):
    r = _plan_rig(*PLANS["tp2_to_tp16"], _batch(300, 70, step=3), no=1, hd=32, seed=107)
    sh, dhs, plan, reqs = _managed(mgr, r)
    mgr.execute_repage_scatter_batch(sh, dhs, reqs, plan).wait(20.0)
    torch.cuda.synchronize()
    for p, want in zip(r.dsts, r.expected()):
        assert np.array_equal(p.buf.cpu().numpy(), want)
    torch.cuda.synchronize()


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_manager_streamed_batch(mgr, gate_mode):
    s = StreamBatch(_plan_rig(*PLANS["tp2_to_tp16"], BATCHES["mixed"][:5] + SMALL, hd=32, seed=109, **SRC_KV))
    r = s.r
    sh, dhs, plan, reqs = _managed(mgr, r)
    flags = torch.zeros(len(dhs) + 1, dtype=torch.int32, device="cuda")
    opts = TransferOptions(done_flag=flags[len(dhs):].data_ptr(), epoch=4, gate_mode=gate_mode, max_ctas=MAX_CTAS,
                           per_dst_done_flags=[flags[d:].data_ptr() for d in range(len(dhs))])
    try:
        note = mgr.execute_repage_scatter_batch(sh, dhs, reqs, plan, opts, ready_flags=r.src.ready.data_ptr(),
                                                layer_done_flags=s.layer_done.data_ptr())
        r.src.produce(range(s.nl), 4)
        note.wait(20.0)
    finally:
        s.rescue(4)
    for p, want, ref in zip(r.dsts, s.want, s.unstreamed):
        assert np.array_equal(p.buf.cpu().numpy(), want) and torch.equal(p.buf, ref)
    assert flags.tolist() == [4] * (len(dhs) + 1)
    assert s.layer_done.tolist() == [4] * s.nl
    torch.cuda.synchronize()


def test_manager_gate_timeout(mgr):
    s = StreamBatch(_plan_rig(8, 4, 2, 1, 4, 1, 0, SMALL, seed=113, **SRC_KV))
    r = s.r
    sh, dhs, plan, reqs = _managed(mgr, r)
    flags = torch.zeros(len(dhs) + 1, dtype=torch.int32, device="cuda")
    opts = TransferOptions(done_flag=flags[len(dhs):].data_ptr(), epoch=6, gate_mode=K.GATE_SPIN, max_ctas=MAX_CTAS, gate_timeout_ms=200,
                           per_dst_done_flags=[flags[d:].data_ptr() for d in range(len(dhs))])
    try:
        note = mgr.execute_repage_scatter_batch(sh, dhs, reqs, plan, opts, ready_flags=r.src.ready.data_ptr())
        r.src.produce(range(2), 6)
        with pytest.raises(KvbmError) as e:
            note.wait(20.0)
        assert e.value.code == ErrorCode.TIMEOUT
    finally:
        s.rescue(6)
    assert not flags.any().item()
    torch.cuda.synchronize()

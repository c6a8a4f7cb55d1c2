"""GPU parity of the re-paging scatter between pages that need not divide: kvbm_kernels_paged_repage_scatter_anypage, its streamed
form and TransferManager.execute_repage_scatter_anypage.  Every case compares whole destination pools, guard blocks included, with
tests/scatter_batch_oracle.py, which states the scatter by token position and needs no divisibility: the pools start as random
bytes, so every slot no sequence touches (guard blocks, the slots of a first or last block outside a range, heads no window
covers, layers outside the layer range) must survive.  With dividing pages the anypage scatter is also compared byte for byte with
the batch scatter on the same inputs.  Every test ends with a device synchronize, so a profile window never loses a launch."""
import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import TransferManager, TransferOptions, tp_pp_scatter_plan
from tests.gpu_util import ids_dev, stream_ptr
from tests.scatter_batch_oracle import repage_scatter_batch, table_len
from tests.test_gpu_scatter_seqs import BATCHES, BatchRig, _found, _managed
from tests.test_gpu_scatter_stream import StreamRig, _finish, _Layers
from tests.test_gpu_stage_gather import ELEMS
from tests.test_gpu_transform_limits import BHD, BIG_IDS, BNH, BNL, BNO, BNT, _into_big, big_pool  # noqa: F401  (big_pool: the fixture)
from tests.test_gpu_transform_stream import GATE_IDS, GATES, MASK, Pool, _i32

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
NHD, HND, UTP, UPP = KV.OperationalNHD, KV.OperationalHND, KV.UniversalTP, KV.UniversalPP


def _sync():
    torch.cuda.synchronize()


def _divides(ps, pd):
    return max(ps, pd) % min(ps, pd) == 0


class AnyRig(BatchRig):
    """BatchRig over the anypage scatter: the tables are sized at each side's own page and the unit table is
    kvbm_kernels_repage_anypage_units'.  With dividing pages the batch helper's table is kept too, for the batch scatter."""

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
        u = K.repage_anypage_units(self.seqs, ps, pd)
        assert u is not None and (u[1], u[2]) == (ns, nd)
        self.units_np, self.nu = u[0], len(u[0])
        as_t = lambda x: torch.from_numpy(x if len(x) else np.zeros(1, np.int32)).cuda()  # noqa: E731
        self.sids_t, self.dids_t = as_t(self.sids), [as_t(x) for x in self.dids]
        self.units_t = as_t(np.ascontiguousarray(self.units_np).view(np.int32).reshape(-1))
        if _divides(ps, pd):
            self.batch_units_t = as_t(np.ascontiguousarray(K.repage_batch_units(self.seqs, ps, pd)[0]).view(np.int32).reshape(-1))
        self.initial = [p.buf.clone() for p in self.dsts]
        self.scales_np = (rng.uniform(0.1, 4.0, nl * no) * (1 + np.arange(nl * no) * 1e-2)).astype(np.float32) if scaled else None
        self.scales = torch.from_numpy(self.scales_np).cuda() if scaled else None
        self.done = torch.zeros(len(targets), dtype=torch.int32, device="cuda")
        self.completion = torch.zeros(1, dtype=torch.int32, device="cuda")

    def launch(self, epoch=5, value=6):
        return K.paged_repage_scatter_anypage(self.src.side(self.sids_t), self.src.nh, self.ps, self.kernel_targets(), self.pd, self.seqs,
                                              self.units_t.data_ptr(), self.nu, self.lb, self.le, self.row, self.cast, self.scales, epoch,
                                              self.completion.data_ptr(), value, stream_ptr())

    def run_and_check(self, epoch=5, value=6, singles=False):
        """The oracle's pools, every target's done flag and the completion word (singles: the single scatter takes dividing pages
        only, so it is not the reference here)."""
        assert not singles
        super().run_and_check(epoch, value, singles=False)

    def batch_scatter(self):
        """The batch scatter's pools from the initial ones, on the same inputs (dividing pages)."""
        for p, x in zip(self.dsts, self.initial):
            p.buf.copy_(x)
        K.check(K.paged_repage_scatter_batch(self.src.side(self.sids_t), self.src.nh, self.ps, self.kernel_targets(), self.pd, self.seqs,
                                             self.batch_units_t.data_ptr(), self.nu, self.lb, self.le, self.row, self.cast, self.scales,
                                             stream=stream_ptr()), "batch scatter")
        _sync()
        return [p.buf.clone() for p in self.dsts]


def any_rig(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, seqs, src_kv=HND, dst_kvs=(NHD,), **kw):
    """The scatter plan of prefill rank `rank` (equal PP stages): one source pool with its stage's layers and heads, one pool per
    decode rank the plan names, in dst_kvs' formats in turn."""
    plan = tp_pp_scatter_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank)
    ranks = sorted({w.dst_rank for w in plan})
    dsts = [(L // dst_pp, max(1, H // dst_tp), dst_kvs[i % len(dst_kvs)]) for i in range(len(ranks))]
    targets = [(ranks.index(w.dst_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
               for w in plan]
    return AnyRig((L // src_pp, max(1, H // src_tp), src_kv), dsts, targets, seqs, **kw)


def edge_seqs(ps, pd):
    """Ranges that start and end inside blocks on both sides, one token, an empty range, one from 0, and one longer range."""
    big, small = max(ps, pd), min(ps, pd)
    return [(big // 2 + 1, 3 * big + small // 2 + 1), (5 * big - 1, 5 * big), (7, 7), (small + 1, 2 * big + 3), (0, big + small + 1),
            (6 * big + 2, 9 * big - 1)]


PLANS = {
    "tp2_to_tp4": (8, 2, 2, 1, 4, 1, 0),
    "tp1_to_tp8": (8, 2, 1, 1, 8, 1, 0),
    "tp2_to_tp16": (8, 2, 2, 1, 16, 1, 0),                 # every source head to two decode ranks
    "pp2tp2_rank3_to_pp3tp2": (4, 12, 2, 2, 2, 3, 3),      # a 6-layer source into 4-layer targets, with layer shifts
}
SMALL = [(5, 200), (40, 41), (3, 3), (17, 333)]


# ---------------------------------------------------------------------------------------------------------------------
# against the oracle
# ---------------------------------------------------------------------------------------------------------------------
PAIRS = [(3, 5), (5, 3), (24, 16), (16, 24), (48, 64), (64, 48), (544, 64), (64, 544)]


@pytest.mark.parametrize("ps,pd", PAIRS, ids=str)
def test_pages_that_do_not_divide(ps, pd):
    """TP2 -> TP16 (replicated heads) over ranges inside blocks on both sides, a one-token and an empty range."""
    r = any_rig(*PLANS["tp2_to_tp16"], edge_seqs(ps, pd), ps=ps, pd=pd, no=1, hd=32, seed=ps + 7 * pd)
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("ps,pd", [(24, 16), (64, 48), (16, 24), (48, 64)], ids=str)
def test_a_mixed_batch(ps, pd):
    """1 to 4000 tokens, empty sequences between others."""
    r = any_rig(*PLANS["tp1_to_tp8"], BATCHES["mixed"], ps=ps, pd=pd, no=1, hd=32, seed=ps * pd)
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("name", list(PLANS))
def test_plans_into_mixed_formats(name):
    r = any_rig(*PLANS[name], BATCHES["32x512"][:4] + SMALL, dst_kvs=(NHD, UTP, HND, UPP), ps=48, pd=64, hd=32, seed=len(name))
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("hd", [64, 80, 96])
@pytest.mark.parametrize("scaled", [False, True], ids=["unscaled", "scaled"])
@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16, CM.BF16_TO_FP8E4M3], ids=lambda c: c.name)
def test_casts_scales_and_head_dims(cast, scaled, hd):
    if scaled and cast == CM.NONE:
        pytest.skip("scales go with a cast")
    for layers, (ps, pd) in ((None, (24, 16)), (range(1, 3), (48, 64))):
        r = any_rig(8, 4, 1, 1, 4, 1, 0, SMALL + [(100, 170)], src_kv=NHD, dst_kvs=(UTP, UPP, HND, NHD), cast=cast, scaled=scaled,
                    layers=layers, hd=hd, ps=ps, pd=pd, seed=int(cast) + 3 * scaled + hd)
        r.run_and_check()
    _sync()


@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16], ids=lambda c: c.name)
def test_mla_latent_head(cast):
    """MLA's one 576-wide latent head to 8 decode ranks."""
    r = any_rig(1, 2, 1, 1, 8, 1, 0, edge_seqs(24, 16), ps=24, pd=16, no=1, hd=576, cast=cast, seed=57)
    assert len(r.targets) == 8
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("ps,pd", [(544, 64), (48, 64)], ids=str)
def test_shared_source_blocks(ps, pd):
    """Sequences that share source blocks; at 48 -> 64 the phased loads go through the source's table and several units read one
    source block."""
    r = any_rig(*PLANS["tp1_to_tp8"], BATCHES["mixed"], ps=ps, pd=pd, no=1, hd=32, share=True, seed=77 + ps)
    assert len(set(r.sids.tolist())) < len(r.sids)
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (16, 16)], ids=str)
def test_dividing_pages_write_the_batch_bytes(ps, pd):
    r = any_rig(*PLANS["tp2_to_tp16"], BATCHES["mixed"][:6] + SMALL, ps=ps, pd=pd, no=1, hd=32, cast=CM.FP8E4M3_TO_BF16, scaled=True,
                seed=ps * pd)
    r.run_and_check()
    got = [p.buf.clone() for p in r.dsts]
    for g, ref in zip(got, r.batch_scatter()):
        assert torch.equal(g, ref)
    _sync()


def test_empty_batches_signal():
    r = any_rig(*PLANS["tp1_to_tp8"], [(9, 9), (70, 70)], ps=24, pd=16, seed=4)
    for seqs in ([], [(9, 9), (70, 70)]):
        r.done.zero_()
        assert K.paged_repage_scatter_anypage(r.src.side(r.sids_t), r.src.nh, 24, r.kernel_targets(), 16, seqs, 0, 0, 0, r.le, r.row, 0, None,
                                              7, r.completion.data_ptr(), 8, stream_ptr()) == 0
        _sync()
        assert r.done.tolist() == [7] * 8 and r.completion.item() == 8
    assert all(torch.equal(a, p.buf) for a, p in zip(r.initial, r.dsts))
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# every instantiation of both families, reached under the profiler
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True))}
EXPECTED = {w + (pp,) for w in WALKS for pp in (True, False)}


class StreamAny(StreamRig):
    """StreamRig over an AnyRig: `unstreamed` is the unstreamed anypage scatter's result."""

    def launch(self, epoch, gate_mode, value):
        r = self.r
        K.check(K.paged_repage_scatter_anypage_streamed(r.src.side(r.sids_t), r.src.nh, r.ps, r.kernel_targets(), r.pd, r.seqs,
                                                        r.units_t.data_ptr(), r.nu, r.lb, r.le, r.row, r.cast, r.scales,
                                                        self.stream_desc(epoch, gate_mode, value), stream_ptr(self.side_stream)),
                "streamed anypage scatter")


def test_every_instantiation():
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c, p, sc in sorted(WALKS):
            for ppow2 in (True, False):
                ps, pd = (16, 24) if ppow2 else (40, 24)
                r = any_rig(8, 4, 2, 1, 4, 1, 0, SMALL, dst_kvs=(UTP, HND), cast=CM(c), scaled=sc, hd=64 if p else 80, ps=ps, pd=pd,
                            seed=c + 2 * p + 4 * sc + 8 * ppow2)
                r.run_and_check()
                s = StreamAny(r)
                s.r.src.buf.copy_(s.r.src.final)   # the flags released before the launch
                s.r.src.ready.fill_(3)
                _sync()
                s.launch(3, K.GATE_SPIN, 5)
                assert _finish(s.side_stream)
                _sync()
                s.check_end(3, 5)
    assert _found(prof, "kvbm_paged_repage_phased_push_kernel") == EXPECTED
    assert _found(prof, "kvbm_gated_repage_phased_push_kernel") == EXPECTED
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# streamed, behind a producer that writes the source after the launch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("ps,pd", [(544, 64), (16, 24)], ids=str)
def test_streamed_behind_a_late_producer(gate_mode, ps, pd):
    s = StreamAny(any_rig(*PLANS["pp2tp2_rank3_to_pp3tp2"], BATCHES["mixed"][:4] + SMALL, ps=ps, pd=pd, hd=32, no=1, seed=ps + pd,
                          cast=CM.FP8E4M3_TO_BF16, scaled=True))
    s.run(5, gate_mode, 77)
    s.check_end(5, 77)
    _sync()


@pytest.mark.parametrize("max_ctas", [1, 2, 3])
def test_spinning_batches_that_span_layers(max_ctas):
    """A handful of units per layer on 1-3 CTAs: claims of several units cross layer boundaries."""
    s = StreamAny(any_rig(8, 4, 2, 1, 4, 1, 0, [(3, 70), (5, 5), (100, 180), (1, 2)], ps=24, pd=16, no=1, seed=90 + max_ctas),
                  max_ctas=max_ctas)
    s.run(8, K.GATE_SPIN, 5)
    s.check_end(8, 5)
    _sync()


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_only_released_layers_move(gate_mode):
    """Release k source layers, observe once layer_done[k - 1] appears: only those layers landed, for every sequence, and no done
    flag is written."""
    from tests.test_gpu_transform_stream import CHECKER_SLEEP
    s = StreamAny(any_rig(8, 4, 2, 1, 16, 1, 0, SMALL + edge_seqs(48, 64), ps=48, pd=64, seed=41))
    r, k, epoch = s.r, 2, 7
    snaps = [p.buf.clone() for p in r.dsts]
    flags = [s.layer_done.clone(), r.done.clone(), s.st_done.clone()]
    _sync()
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
    _sync()


def test_a_gate_timeout_writes_no_done_flag():
    s = StreamAny(any_rig(8, 4, 2, 1, 4, 1, 0, SMALL, ps=24, pd=16, seed=71), timeout_ms=200)
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
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# TransferManager.execute_repage_scatter_anypage
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=59)
    yield m
    _sync()
    m.close()


@pytest.mark.parametrize("streamed", [False, True], ids=["unstreamed", "streamed"])
@pytest.mark.parametrize("ps,pd", [(24, 64), (64, 24)], ids=str)
def test_manager_anypage_scatter(mgr, streamed, ps, pd):
    """One call: the oracle's bytes, per-destination done flags, the done flag, bytes_moved over every window; streamed behind a
    producer that writes the source after the call."""
    rig = any_rig(*PLANS["tp2_to_tp16"], BATCHES["mixed"][:5] + SMALL, ps=ps, pd=pd, hd=32, no=1, seed=109 + ps)
    s = StreamAny(rig) if streamed else None
    r = rig
    sh, dhs, plan, reqs = _managed(mgr, r)
    flags = torch.zeros(len(dhs) + 1, dtype=torch.int32, device="cuda")
    kw = dict(done_flag=flags[len(dhs):].data_ptr(), epoch=4, per_dst_done_flags=[flags[d:].data_ptr() for d in range(len(dhs))])
    m0 = mgr.bytes_moved()
    if streamed:
        try:
            note = mgr.execute_repage_scatter_anypage(sh, dhs, reqs, plan, TransferOptions(gate_mode=K.GATE_SPIN, max_ctas=4, **kw),
                                                      ready_flags=r.src.ready.data_ptr(), layer_done_flags=s.layer_done.data_ptr())
            r.src.produce(range(s.nl), 4)
            note.wait(20.0)
        finally:
            s.rescue(4)
        assert s.layer_done.tolist() == [4] * s.nl
    else:
        mgr.execute_repage_scatter_anypage(sh, dhs, reqs, plan, TransferOptions(**kw)).wait(20.0)
    _sync()
    for p, want in zip(r.dsts, r.expected()):
        assert np.array_equal(p.buf.cpu().numpy(), want)
    assert flags.tolist() == [4] * (len(dhs) + 1)
    tokens = sum(te - tb for tb, te in r.seqs)
    assert mgr.bytes_moved() - m0 == sum(tokens * c * r.no * k * r.row for _p, _sl, _dl, c, _sb, _db, k in r.targets)
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# limits
# ---------------------------------------------------------------------------------------------------------------------
def test_the_exactness_bound_and_the_32_bit_token_bound():
    """The largest big page a 46337-token small page takes (46353) at phase small - 1, and a sequence ending on the last block of the
    larger page below 2^32; the first rejected pair next to it."""
    small = 46337
    big = (1 << 32) // small
    while (big + small - np.gcd(big, small)) * small >= (1 << 32) or big % small == 0:
        big -= 1
    assert big == 46353 and K.repage_anypage_units([], big, small) is not None and K.repage_anypage_units([], big + 1, small) is None
    g = int(np.gcd(big, small))
    j = next(j for j in range(1, small) if (j * big) % small == small - g)     # the largest phase: the last slot splits at big + small - g - 1
    last = ((1 << 32) - 1) // big * big                                        # the start of the last big block below 2^32
    seqs = [(j * big + 3, (j + 1) * big), (last - small - 5, last)]
    for ps, pd in ((small, big), (big, small)):
        r = any_rig(2, 1, 1, 1, 1, 1, 0, seqs, ps=ps, pd=pd, hd=8, no=1, seed=3)
        assert any(u[3] == small - g for u in r.units_np.tolist())
        r.run_and_check()
        launches = K.launch_count()
        assert K.paged_repage_scatter_anypage(r.src.side(r.sids_t), r.src.nh, ps if ps == small else big + 1, r.kernel_targets(),
                                              pd if pd == small else big + 1, seqs, r.units_t.data_ptr(), r.nu, r.lb, r.le,
                                              r.row) == K.CUDA_ERROR_INVALID_VALUE
        assert K.launch_count() == launches
    _sync()


TOKENS = range(5, 61)            # big-pool page 16: blocks 0 .. 3 of the sequence, whose table is BIG_IDS


def _small_side(nh, page, kv, seed, poison_free=True):
    n = table_len(TOKENS.start, TOKENS.stop, page)
    p = Pool(n + 2, BNL, BNO, page, nh, BHD * 2, kv, seed)
    ids = np.random.default_rng(seed).permutation(n + 2)[:n].astype(np.int32)
    return p, ids, torch.from_numpy(ids).cuda()


def _units(ps, pd):
    u, _, _ = K.repage_anypage_units([(TOKENS.start, TOKENS.stop)], ps, pd)
    return torch.from_numpy(u.view(np.int32).reshape(-1)).cuda(), len(u)


@pytest.mark.parametrize("ps", [6, 24], ids=["source_page_6", "source_page_24"])
def test_big_pool_as_target(big_pool, ps):
    """The 4.02 GiB pool as two targets (heads 0-3 and 4-7 from the same 4 source heads, so replicated heads land past 2^32) next
    to a small pool.  Source page 6: the big pool (page 16) is the larger page's side; 24: the smaller, its stores phased."""
    src, sids, sids_t = _small_side(4, ps, NHD, 90 + ps)
    small = Pool(6, BNL, BNO, BNT, 4, BHD * 2, UPP, 91)
    small0 = small.buf.clone()
    dids = np.array([4, 1, 5, 2], dtype=np.int32)
    bi, di = ids_dev(BIG_IDS), torch.from_numpy(dids).cuda()
    units_t, nu = _units(ps, BNT)
    bside = K.PermuteSide(big_pool.desc, bi.data_ptr(), int(UTP))
    targets = [K.ScatterTarget(bside, BNH, 0, 0, 4, 0, 0, BNL, 0), K.ScatterTarget(bside, BNH, 0, 4, 4, 0, 0, BNL, 0),
               K.ScatterTarget(small.side(di), 4, 0, 0, 4, 0, 0, BNL, 0)]
    want_small = {}

    def want(old):
        pools = [np.stack(old), small0.cpu().numpy()]
        ts = [(0, list(range(4)), int(UTP), BNH, BNL, (0, 0, BNL, 0, 0, 4)), (0, list(range(4)), int(UTP), BNH, BNL, (0, 0, BNL, 0, 4, 4)),
              (1, dids, int(UPP), 4, BNL, (0, 0, BNL, 0, 0, 4))]
        repage_scatter_batch((src.final_np, sids, src.kv, 4, BNL), ts, pools, BNO, ps, BNT, BHD * 2, [(TOKENS.start, TOKENS.stop)])
        want_small["pool"] = pools[1]
        return list(pools[0])

    _into_big(big_pool, lambda: K.paged_repage_scatter_anypage(src.side(sids_t), 4, ps, targets, BNT, [(TOKENS.start, TOKENS.stop)],
                                                              units_t.data_ptr(), nu, 0, BNL, BHD * 2, stream=stream_ptr()), want)
    assert np.array_equal(small.buf.cpu().numpy(), want_small["pool"])
    _sync()


@pytest.mark.parametrize("pd", [6, 24], ids=["target_page_6", "target_page_24"])
def test_big_pool_as_source(big_pool, pd):
    """Blocks past 2^32 read once and stored to two pools: target page 6 reads them as the larger page's side, 24 as the smaller
    side, its loads phased.  The big pool keeps every byte."""
    olds = [big_pool.block(b) for b in BIG_IDS]
    nd = table_len(TOKENS.start, TOKENS.stop, pd)
    dsts = [Pool(nd + 2, BNL, BNO, pd, BNH, BHD * 2, NHD, 93), Pool(nd + 2, BNL, BNO, pd, 4, BHD * 2, UTP, 94)]
    init = [p.buf.clone() for p in dsts]
    dids = [np.random.default_rng(95 + i).permutation(nd + 2)[:nd].astype(np.int32) for i in range(2)]
    dids_t = [torch.from_numpy(x).cuda() for x in dids]
    bi = ids_dev(BIG_IDS)
    units_t, nu = _units(BNT, pd)
    sside = K.PermuteSide(big_pool.desc, bi.data_ptr(), int(UPP))
    targets = [K.ScatterTarget(dsts[0].side(dids_t[0]), BNH, 0, 0, BNH, 0, 0, BNL, 0),
               K.ScatterTarget(dsts[1].side(dids_t[1]), 4, 4, 0, 4, 0, 0, BNL, 0)]
    pools = [x.cpu().numpy() for x in init]
    repage_scatter_batch((np.stack(olds), np.arange(4), int(UPP), BNH, BNL),
                         [(0, dids[0], int(NHD), BNH, BNL, (0, 0, BNL, 0, 0, BNH)), (1, dids[1], int(UTP), 4, BNL, (0, 0, BNL, 4, 0, 4))],
                         pools, BNO, BNT, pd, BHD * 2, [(TOKENS.start, TOKENS.stop)])
    try:
        assert K.paged_repage_scatter_anypage(sside, BNH, BNT, targets, pd, [(TOKENS.start, TOKENS.stop)], units_t.data_ptr(), nu, 0, BNL,
                                              BHD * 2, stream=stream_ptr()) == 0
        _sync()
        for p, w in zip(dsts, pools):
            assert np.array_equal(p.buf.cpu().numpy(), w)
        big_pool.assert_all_filled()
    except BaseException:
        big_pool.refill()
        raise
    _sync()

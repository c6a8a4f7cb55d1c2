"""GPU parity of re-paging between pages that need not divide: kvbm_kernels_paged_stage_repage_gather_anypage, its streamed form
and TransferManager.execute_repage_anypage.  Every case compares the whole destination pool, byte for byte, with
tests/repage_batch_oracle.py (tests/stage_repage_oracle.py per sequence), which states re-paging by sequence position and needs no
divisibility: the destination starts as random bytes, so every slot no sequence touches (guard blocks no table names, the slots of
a first or last block outside a range, heads no window covers, layers outside the layer range) is poison that must survive.  With
dividing pages the anypage entry is also compared with the batch entry on the same inputs.  Every test ends with a device
synchronize, so a profile window never loses a launch."""
import re

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import TransferOptions, tp_pp_reshard_plan
from tests.gpu_util import stream_ptr
from tests.repage_batch_oracle import repage_batch
from tests.test_gpu_layer_stream import _finish
from tests.test_gpu_repage_batch import PP2TP2, TP4_TP2, BatchRig, _requests, mixed_seqs
from tests.test_gpu_stage_gather import GATE_IDS, GATES, GUARD, _register
from tests.test_gpu_transform_stream import LAYER_SLEEP

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode


def _sync():
    torch.cuda.synchronize()


class AnyRig(BatchRig):
    """BatchRig over the anypage entries: the unit table is kvbm_kernels_repage_anypage_units', and the launches are the anypage
    gather's.  BatchRig builds the batch helper's table for dividing pages; for any other pair it is built here."""

    def __init__(self, *a, ps=16, pd=64, **kw):
        div = max(ps, pd) % min(ps, pd) == 0
        # BatchRig sizes its tables with the batch helper, which only takes dividing pages: build it at a dividing stand-in with
        # the same larger page, then re-cut the tables for the real pair.  The pools' blocks are sized by the pair's own counts.
        super().__init__(*a, ps=ps if div else _standin(ps, pd), pd=pd if div else _standin(pd, ps), **kw)
        if not div:
            self._recut(ps, pd, kw.get("seed", 0), kw.get("shared", ()), kw.get("poison", False))
        self.any_np, ns, nd = K.repage_anypage_units(self.seqs, ps, pd)
        assert (ns, nd) == (sum(len(x) for x in self.sids[0]), sum(len(x) for x in self.dids))
        self.any_units = torch.from_numpy(np.concatenate([self.any_np, np.zeros((1, 4), np.uint32)]).view(np.int32)).cuda()

    def _recut(self, ps, pd, seed, shared, poison):
        from tests.test_gpu_repage_batch import _blocks
        from tests.test_gpu_transform_stream import Pool
        self.ps, self.pd = ps, pd
        n_s = [_blocks(tb, te, ps) for tb, te in self.seqs]
        n_d = [_blocks(tb, te, pd) for tb, te in self.seqs]
        old = self.srcs
        self.srcs = [Pool(sum(n_s) + 2, p.nl, p.no, ps, p.nh, p.row, p.kv, seed + 10 + s, poison=poison) for s, p in enumerate(old)]
        for p in self.srcs:
            p.ready_all = torch.zeros(p.nl + GUARD, dtype=torch.int32, device="cuda")
            p.ready = p.ready_all[:p.nl]
        d = self.dst
        self.dst = Pool(sum(n_d) + 2, d.nl, d.no, pd, d.nh, d.row, d.kv, seed + 1)
        rng = np.random.default_rng(seed + 2)
        cut = lambda perm, counts: np.split(perm[:sum(counts)].astype(np.int32), np.cumsum(counts)[:-1])  # noqa: E731
        self.sids = [cut(rng.permutation(sum(n_s) + 2), n_s) for _ in old]
        self.dids = cut(rng.permutation(sum(n_d) + 2), n_d)
        for i, j in shared:
            first = self.seqs[i][0] // ps - self.seqs[j][0] // ps
            for s in range(len(old)):
                for k in range(len(self.sids[s][j])):
                    if 0 <= k - first < len(self.sids[s][i]):
                        self.sids[s][j][k] = self.sids[s][i][k - first]
        dev = lambda parts: torch.from_numpy(np.concatenate(list(parts) + [np.zeros(1, np.int32)])).cuda()  # noqa: E731
        self.sids_t = [dev(x) for x in self.sids]
        self.dids_t = dev(self.dids)
        self.units_np, self.units = None, None
        self.initial = self.dst.buf.clone()

    def args(self):
        return (self.sources(), self.ps, self.dst.side(self.dids_t), self.dst.nh, self.pd, self.seqs, self.any_units.data_ptr(),
                len(self.any_np), self.lb, self.le, self.row, self.cast, self.scales)

    def run(self):
        rc = K.paged_stage_repage_gather_anypage(*self.args(), self.done.data_ptr(), 5, self.completion.data_ptr(), 6, stream_ptr())
        _sync()
        return rc

    def expected(self, layers=None):
        d = self.dst
        seqs = [(tb, te, [self.sids[s][i] for s in range(len(self.srcs))], self.dids[i]) for i, (tb, te) in enumerate(self.seqs)]
        return repage_batch([(p.final_np, p.kv, p.nh, p.nl) for p in self.srcs], self.windows, self.initial.cpu().numpy(), d.kv, d.nh, d.nl,
                            self.no, self.ps, self.pd, self.row, seqs, self.cast, self.scales_np,
                            layers if layers is not None else range(self.lb, self.le))

    def check(self, singles=False):
        assert np.array_equal(self.dst.buf.cpu().numpy(), self.expected()), "the anypage gather differs from the oracle"

    def launch_streamed(self, epoch, gate_mode, timeout_ms=3000):
        K.check(K.paged_stage_repage_gather_anypage_streamed(*self.args(), self.stream_desc(epoch, gate_mode, timeout_ms),
                                                             stream_ptr(self.side_stream)), "launch")

    def produce(self, layers, epoch, stream):
        with torch.cuda.stream(stream):
            for p in self.srcs:
                for l in layers:
                    if l < p.nl:
                        torch.cuda._sleep(LAYER_SLEEP)
                        p.layer(p.buf, l).copy_(p.layer(p.final, l))
                        K.check(K.set_flags(p.ready.data_ptr(), l, 1, epoch, stream_ptr(stream)), "set_flags")

    def release_all(self, epoch):
        s = torch.cuda.Stream()
        for p in self.srcs:
            K.set_flags(p.ready.data_ptr(), 0, p.nl, epoch, stream_ptr(s))
        K.set_flags(self.layer_done.data_ptr(), self.lb, self.le - self.lb, epoch, stream_ptr(s))
        assert _finish(s) and _finish(self.side_stream)
        _sync()

    def run_streamed(self, epoch, gate_mode, timeout_ms=3000):
        """A late producer: the sources start as poison, the launch comes first, then one producer stream writes every source layer
        by layer and releases its flags."""
        prod = torch.cuda.Stream()
        with torch.cuda.stream(prod):      # every torch kernel of the producer once, then the poison back
            torch.cuda._sleep(100)
            for p in self.srcs:
                p.layer(p.buf, 0).copy_(p.layer(p.final, 0))
        _sync()
        for p in self.srcs:
            p.buf.copy_(p.poison)
            if gate_mode == K.GATE_STREAM_WAIT:
                p.ready_all[p.nl:].fill_(epoch)
        _sync()
        try:
            self.launch_streamed(epoch, gate_mode, timeout_ms)
            self.produce(range(max(p.nl for p in self.srcs)), epoch, prod)
            assert _finish(self.side_stream) and _finish(prod), "the streamed anypage gather did not finish"
        finally:
            self.release_all(epoch)
        self.check()
        assert self.done.item() == epoch and self.completion.item() == epoch
        assert not self.ws.any().item(), "the workspace must be left zeroed"


def _standin(p, other):
    """A page that divides or is divided by `other`'s stand-in: the larger of the pair keeps its page, the smaller becomes 1."""
    return p if p > other else 1


def any_rig(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, seqs, src_kv=KV.OperationalNHD, dst_kv=KV.OperationalNHD, **kw):
    plan = tp_pp_reshard_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank)
    ranks = sorted({w.src_rank for w in plan})
    srcs = [(L // src_pp, max(1, H // src_tp), src_kv) for _ in ranks]
    windows = [(ranks.index(w.src_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
               for w in plan]
    return AnyRig(srcs, windows, L // dst_pp, max(1, H // dst_tp), dst_kv, seqs, **kw)


def edge_seqs(ps, pd):
    """Ranges that start and end inside blocks on both sides, one token, an empty range, and one from 0."""
    big, small = max(ps, pd), min(ps, pd)
    return [(big // 2 + 1, 3 * big + small // 2 + 1), (5 * big - 1, 5 * big), (7, 7), (small + 1, 2 * big + 3), (0, big + small + 1),
            (6 * big + 2, 9 * big - 1)]


# ---------------------------------------------------------------------------------------------------------------------
# against the oracle
# ---------------------------------------------------------------------------------------------------------------------
PAIRS = [(3, 5), (5, 3), (24, 16), (16, 24), (48, 64), (64, 48), (544, 64), (64, 544), (7, 1)]


@pytest.mark.parametrize("ps,pd", PAIRS, ids=lambda p: str(p))
def test_pages_that_do_not_divide(ps, pd):
    r = any_rig(*TP4_TP2, edge_seqs(ps, pd), src_kv=KV.OperationalHND, seed=ps + 7 * pd, no=1 if max(ps, pd) > 100 else 2)
    assert r.run() == 0
    r.check()
    assert r.done.item() == 5 and r.completion.item() == 6
    _sync()


@pytest.mark.parametrize("ps,pd", [(24, 16), (64, 544)], ids=lambda p: str(p))
def test_pp_tp_stage_plan_and_shared_source_blocks(ps, pd):
    r = any_rig(*PP2TP2, [(0, 300), (70, 400), (130, 140), (5, 6)], ps=ps, pd=pd, seed=ps, shared=[(0, 1), (0, 2)], dst_kv=KV.UniversalPP,
                no=1)
    assert any(set(r.sids[0][0]) & set(r.sids[0][j]) for j in (1, 2))
    assert r.run() == 0
    r.check()
    _sync()


@pytest.mark.parametrize("hd", [64, 80, 96])
@pytest.mark.parametrize("scaled", [False, True], ids=["unscaled", "scaled"])
@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16, CM.BF16_TO_FP8E4M3], ids=lambda c: c.name)
def test_casts_scales_and_head_dims(cast, scaled, hd):
    if scaled and cast == CM.NONE:
        pytest.skip("scales go with a cast")
    for layers, (ps, pd) in ((None, (24, 16)), (range(1, 3), (48, 64))):
        r = any_rig(*PP2TP2, mixed_seqs(6, hd, longest=400), dst_kv=KV.UniversalTP, cast=cast, scaled=scaled, layers=layers, hd=hd, ps=ps,
                    pd=pd, seed=int(cast) + 3 * scaled + hd)
        assert r.run() == 0
        r.check()
    _sync()


@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16], ids=lambda c: c.name)
def test_mla_one_head(cast):
    r = any_rig(1, 4, 1, 2, 1, 1, 0, edge_seqs(24, 16), ps=24, pd=16, hd=576, no=1, cast=cast, seed=5)
    assert r.run() == 0
    r.check()
    _sync()


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (16, 16), (1, 48), (48, 12)], ids=lambda p: str(p))
def test_dividing_pages_write_the_batch_bytes(ps, pd):
    r = any_rig(*PP2TP2, mixed_seqs(9, ps + pd), ps=ps, pd=pd, seed=ps * pd, cast=CM.FP8E4M3_TO_BF16, scaled=True)
    assert r.run() == 0
    got = r.dst.buf.clone()
    r.dst.buf.copy_(r.initial)
    assert K.paged_stage_repage_gather_batch(r.sources(), ps, r.dst.side(r.dids_t), r.dst.nh, pd, r.seqs, r.units.data_ptr(), len(r.units_np),
                                             r.lb, r.le, r.row, r.cast, r.scales, stream=stream_ptr()) == 0
    _sync()
    assert torch.equal(got, r.dst.buf)
    r.check()
    _sync()


def test_the_exactness_bound_and_the_32_bit_token_bound():
    """The largest big page a 46337-token small page accepts, and a range that ends on the last block of the larger page below 2^32,
    in a block whose phase + q reaches big + small - gcd - 1."""
    small = 46337
    big = (1 << 32) // small
    while (big + small - np.gcd(big, small)) * small >= (1 << 32):
        big -= 1
    assert K.repage_anypage_units([], big, small) is not None and K.repage_anypage_units([], big + 1, small) is None
    g = int(np.gcd(big, small))
    # a big block j whose phase (j * big) % small is small - g, the largest: its last slot splits at big + small - g - 1
    j = next(j for j in range(1, small) if (j * big) % small == small - g)
    seqs = [(j * big + 3, (j + 1) * big)]
    last = ((1 << 32) - 1) // big * big                              # the start of the last big block below 2^32
    seqs.append((last - small - 5, last))
    for ps, pd in ((small, big), (big, small)):
        r = any_rig(2, 1, 1, 1, 1, 1, 0, seqs, ps=ps, pd=pd, hd=8, no=1, seed=3)
        assert r.run() == 0
        r.check()
    _sync()


def test_empty_batches_signal():
    for seqs, layers in (([], None), ([(9, 9), (24, 24)], None), ([(0, 100)], range(1, 1))):
        z = any_rig(*TP4_TP2, seqs, layers=layers, ps=24, pd=16, seed=4)
        assert z.run() == 0
        assert torch.equal(z.dst.buf, z.initial) and z.done.item() == 5 and z.completion.item() == 6
        K.check(K.paged_stage_repage_gather_anypage_streamed(*z.args(), z.stream_desc(7, K.GATE_SPIN, 1000), stream_ptr()), "streamed")
        _sync()
        assert torch.equal(z.dst.buf, z.initial) and z.done.item() == 7 and z.completion.item() == 7
        assert not z.layer_done.any().item() and not z.ws.any().item()
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# every instantiation of the two families, reached under the profiler
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True))}
EXPECTED = {(f, w + (pp,)) for f in ("paged", "gated") for w in WALKS for pp in (True, False)}


def test_every_instantiation():
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c, p, s in sorted(WALKS):
            for ppow2 in (True, False):
                for gated in (False, True):
                    ps, pd = (16, 24) if ppow2 else (24, 40)
                    r = any_rig(*PP2TP2, [(5, 150), (40, 41), (96, 200)], dst_kv=KV.UniversalTP, cast=CM(c), scaled=s, hd=64 if p else 80,
                                ps=ps, pd=pd, seed=c + 2 * p + 4 * s + 8 * ppow2)
                    if gated:
                        for q in r.srcs:
                            q.ready.fill_(9)
                        _sync()
                        K.check(K.paged_stage_repage_gather_anypage_streamed(*r.args(), r.stream_desc(9, K.GATE_SPIN, 10000), stream_ptr()),
                                "gated")
                        _sync()
                    else:
                        assert r.run() == 0
                    r.check()
        _sync()
    found = set()
    for e in prof.events():
        for m in re.finditer(r"kvbm_(paged|gated)_repage_anypage_kernel<([^<>]*)>", e.name):
            c, p, s, pp = (a.strip().replace("(int)", "") for a in m.group(2).split(","))
            found.add((m.group(1), (int(c), p == "true", s == "true", pp == "true")))
    assert found == EXPECTED
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# streamed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("ps,pd", [(24, 16), (64, 544)], ids=lambda p: str(p))
def test_streamed_behind_a_late_producer(gate_mode, ps, pd):
    r = any_rig(*PP2TP2, mixed_seqs(7, 3, longest=700), src_kv=KV.OperationalHND, dst_kv=KV.UniversalTP, ps=ps, pd=pd, seed=7, poison=True,
                cast=CM.FP8E4M3_TO_BF16, scaled=True, no=1)
    r.run_streamed(3, gate_mode)
    assert r.layer_done.tolist() == [3] * r.dst.nl
    _sync()


@pytest.mark.parametrize("max_ctas", [1, 2, 3])
def test_spinning_batches_that_span_layers(max_ctas):
    """A handful of units per layer on 1-3 CTAs: claims of several units cross layer boundaries."""
    r = any_rig(*PP2TP2, [(3, 70), (5, 5), (100, 180), (1, 2)], ps=24, pd=16, no=1, seed=90 + max_ctas, poison=True, max_ctas=max_ctas)
    r.run_streamed(8, K.GATE_SPIN)
    _sync()


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_only_released_layers_move(gate_mode):
    """Release k layers of every source, wait for layer_done[k - 1]: only those layers landed, and no done flag is written."""
    r = any_rig(*TP4_TP2, edge_seqs(24, 16), ps=24, pd=16, seed=41, poison=True)
    r.lb, r.le = 0, r.dst.nl
    nl, k, epoch = r.dst.nl, 1, 7
    prod, checker = torch.cuda.Stream(), torch.cuda.Stream()
    for p in r.srcs:
        p.buf.copy_(p.poison)
        if gate_mode == K.GATE_STREAM_WAIT:
            p.ready_all[p.nl:].fill_(epoch)
    _sync()
    snap, flags = r.dst.buf.clone(), [r.layer_done.clone(), r.done.clone()]
    try:
        r.launch_streamed(epoch, gate_mode, 3000)
        r.produce(range(k), epoch, prod)
        with torch.cuda.stream(checker):
            K.check(K.wait_flag(r.layer_done.data_ptr() + 4 * (k - 1), epoch, stream_ptr(checker)), "wait_flag")
            torch.cuda._sleep(2_000_000)
            for t, f in zip(flags, (r.layer_done, r.done)):
                t.copy_(f)
            snap.copy_(r.dst.buf)
        assert _finish(checker), "layer_done of the released layers did not appear"
        r.produce(range(k, nl), epoch, prod)
        assert _finish(r.side_stream) and _finish(prod)
    finally:
        r.release_all(epoch)
        assert _finish(checker)
    r.check()
    assert np.array_equal(snap.cpu().numpy(), r.expected(range(0, k)))
    assert flags[0].tolist() == [epoch if l < k else 0 for l in range(nl)] and flags[1].item() == 0
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# through the TransferManager
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    from dynamo_b200.physical import TransferManager
    m = TransferManager(device=0, worker_id=17)
    yield m
    _sync()
    m.close()


@pytest.mark.parametrize("streamed", [False, True], ids=["unstreamed", "streamed"])
@pytest.mark.parametrize("ps,pd", [(24, 64), (64, 24)], ids=lambda p: str(p))
def test_manager_anypage(mgr, streamed, ps, pd):
    H, L = 8, 4
    plan = tp_pp_reshard_plan(H, L, 2, 2, 1, 1, 0)
    r = any_rig(H, L, 2, 2, 1, 1, 0, mixed_seqs(12, 5), src_kv=KV.UniversalTP, dst_kv=KV.OperationalNHD, ps=ps, pd=pd, seed=ps,
                layers=range(1, 4))
    ranks = sorted({w.src_rank for w in plan})
    hs = {rk: _register(mgr, r.srcs[i], KV.UniversalTP) for i, rk in enumerate(ranks)}
    dh = _register(mgr, r.dst, KV.OperationalNHD)
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    kw = dict(done_flag=flag.data_ptr(), epoch=4, layer_range=range(1, 4))
    moved0, launches = mgr.bytes_moved(), K.launch_count()
    if streamed:
        for p in r.srcs:
            p.ready.fill_(4)
        _sync()
        note = mgr.execute_repage_anypage(hs, dh, _requests(r, ranks), plan, TransferOptions(gate_mode=K.GATE_STREAM_WAIT, **kw),
                                          ready_flags={rk: r.srcs[i].ready.data_ptr() for i, rk in enumerate(ranks)},
                                          layer_done_flags=r.layer_done.data_ptr())
    else:
        note = mgr.execute_repage_anypage(hs, dh, _requests(r, ranks), plan, TransferOptions(**kw))
    note.wait(30.0)
    _sync()
    r.check()
    assert flag.item() == 4
    inside = lambda w: max(0, min(4, w.dst_layer_begin + w.layer_count) - max(1, w.dst_layer_begin))  # noqa: E731
    tokens = sum(te - tb for tb, te in r.seqs)
    assert mgr.bytes_moved() - moved0 == sum(tokens * inside(w) * r.no * w.head_count * r.row for w in plan)
    if streamed:
        assert r.layer_done.tolist() == [4 if 1 <= l < 4 else 0 for l in range(4)]
    else:
        assert 1 <= K.launch_count() - launches <= 2
    _sync()

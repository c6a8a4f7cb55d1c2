"""GPU parity of a batch of sequences in one re-paging launch: kvbm_kernels_paged_stage_repage_gather_batch, its streamed form and
TransferManager.execute_repage_batch.  Every case compares the whole destination pool, byte for byte, with
tests/repage_batch_oracle.py and with the pool that n launches of kvbm_kernels_paged_stage_repage_gather leave, one per
sequence: the destination starts as random bytes, so every slot no sequence touches (guard blocks no table names, the slots of a
first or last block outside a range, heads no window covers, layers outside the layer range) is poison that must survive.

The streamed cases keep tests/test_gpu_stage_gather.py's discipline: poisoned sources, the launch first, one producer stream that
releases layer by layer, guard words after every source's flags, every flag released in a `finally`; tests/conftest.py sets
CUDA_MODULE_LOADING=EAGER for them, as for every stream test."""
import re

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import ErrorCode, KvbmError, TransferManager, TransferOptions, tp_pp_reshard_plan
from tests.gpu_util import stream_ptr
from tests.repage_batch_oracle import repage_batch
from tests.test_gpu_layer_stream import _finish
from tests.test_gpu_stage_gather import ELEMS, GATE_IDS, GATES, GUARD, _register
from tests.test_gpu_transform_stream import LAYER_SLEEP, Pool, _i32

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
ALL = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]


def _blocks(tb, te, page):
    return 0 if tb == te else -(-te // page) - tb // page


def mixed_seqs(n, seed, longest=3000, page=64):
    """n ranges of mixed lengths, 1 token to `longest`, most short; starts mostly inside a block (a prefix-cache hit), some on a
    block boundary, some at 0; one empty sequence in every batch of more than 2."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        tb = int(rng.integers(0, 5 * page)) if i % 4 else int(rng.integers(0, 4)) * page
        length = 1 if i % 7 == 3 else int(rng.integers(1, longest)) if i % 16 == 0 else int(rng.integers(1, 3 * page))
        out.append((tb, tb + (0 if (n > 2 and i == 2) else length)))
    return out


class BatchRig:
    """srcs: (num_layers, num_heads, kv) per source pool; windows: (source, src_layer_begin, dst_layer_begin, layer_count,
    src_head_begin, dst_head_begin, head_count); seqs: (token_begin, token_end) per sequence.  Every sequence gets its own blocks
    on both sides; `shared` names pairs (i, j) whose sequence j reads sequence i's source blocks for the blocks both have."""

    def __init__(self, srcs, windows, dst_nl, dst_nh, dst_kv, seqs, ps=16, pd=64, no=2, hd=64, cast=CM.NONE, scaled=False, layers=None, seed=0,
                 poison=False, max_ctas=4, shared=()):
        se, de = ELEMS[cast]
        self.row, self.cast, self.windows, self.no, self.ps, self.pd, self.max_ctas = hd * se, int(cast), windows, no, ps, pd, max_ctas
        self.seqs = list(seqs)
        self.lb, self.le = (layers.start, layers.stop) if layers is not None else (0, dst_nl)
        n_s = [_blocks(tb, te, ps) for tb, te in self.seqs]
        n_d = [_blocks(tb, te, pd) for tb, te in self.seqs]
        self.srcs = [Pool(sum(n_s) + 2, nl, no, ps, nh, hd * se, kv, seed + 10 + s, poison=poison) for s, (nl, nh, kv) in enumerate(srcs)]
        for p in self.srcs:
            p.ready_all = torch.zeros(p.nl + GUARD, dtype=torch.int32, device="cuda")
            p.ready = p.ready_all[:p.nl]
        self.dst = Pool(sum(n_d) + 2, dst_nl, no, pd, dst_nh, hd * de, dst_kv, seed + 1)
        rng = np.random.default_rng(seed + 2)
        cut = lambda perm, counts: np.split(perm[:sum(counts)].astype(np.int32), np.cumsum(counts)[:-1])  # noqa: E731
        self.sids = [cut(rng.permutation(sum(n_s) + 2), n_s) for _ in srcs]      # [source][sequence]
        self.dids = cut(rng.permutation(sum(n_d) + 2), n_d)                      # [sequence]
        for i, j in shared:
            first = self.seqs[i][0] // ps - self.seqs[j][0] // ps                # sequence i's block 0 is sequence j's block `first`
            for s in range(len(srcs)):
                for k in range(len(self.sids[s][j])):
                    if 0 <= k - first < len(self.sids[s][i]):
                        self.sids[s][j][k] = self.sids[s][i][k - first]
        dev = lambda parts: torch.from_numpy(np.concatenate(list(parts) + [np.zeros(1, np.int32)])).cuda()  # noqa: E731
        self.sids_t = [dev(x) for x in self.sids]
        self.dids_t = dev(self.dids)
        self.units_np, ns, nd = K.repage_batch_units(self.seqs, ps, pd)
        assert (ns, nd) == (sum(n_s), sum(n_d))
        self.units = torch.from_numpy(np.concatenate([self.units_np, np.zeros((1, 4), np.uint32)]).view(np.int32)).cuda()
        self.initial = self.dst.buf.clone()
        self.scales_np = (rng.uniform(0.1, 4.0, dst_nl * no) * (1 + np.arange(dst_nl * no) * 1e-2)).astype(np.float32) if scaled else None
        self.scales = torch.from_numpy(self.scales_np).cuda() if scaled else None
        self.layer_done = torch.zeros(dst_nl, dtype=torch.int32, device="cuda")
        self.done = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.completion = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.ws = torch.zeros(K.sync_workspace_words(dst_nl), dtype=torch.int32, device="cuda")
        self.side_stream = torch.cuda.Stream()

    def sources(self, ids=None):
        ids = ids or self.sids_t
        return [K.StageSource(K.PermuteSource(self.srcs[s].side(ids[s]), self.srcs[s].nh, sb, db, k), sl, dl, c)
                for s, sl, dl, c, sb, db, k in self.windows]

    def expected(self):
        d = self.dst
        seqs = [(tb, te, [self.sids[s][i] for s in range(len(self.srcs))], self.dids[i]) for i, (tb, te) in enumerate(self.seqs)]
        return repage_batch([(p.final_np, p.kv, p.nh, p.nl) for p in self.srcs], self.windows, self.initial.cpu().numpy(), d.kv, d.nh, d.nl,
                            self.no, self.ps, self.pd, self.row, seqs, self.cast, self.scales_np, range(self.lb, self.le))

    def args(self):
        return (self.sources(), self.ps, self.dst.side(self.dids_t), self.dst.nh, self.pd, self.seqs, self.units.data_ptr(),
                len(self.units_np), self.lb, self.le, self.row, self.cast, self.scales)

    def run(self):
        rc = K.paged_stage_repage_gather_batch(*self.args(), self.done.data_ptr(), 5, self.completion.data_ptr(), 6, stream_ptr())
        torch.cuda.synchronize()
        return rc

    def singles(self, order=None):
        """The pool n single launches leave, from the same initial bytes (the rig's destination is restored afterwards)."""
        kept = self.dst.buf.clone()
        self.dst.buf.copy_(self.initial)
        for i in (order if order is not None else range(len(self.seqs))):
            tb, te = self.seqs[i]
            ids = [torch.from_numpy(np.concatenate([x[i], np.zeros(1, np.int32)])).cuda() for x in self.sids]
            did = torch.from_numpy(np.concatenate([self.dids[i], np.zeros(1, np.int32)])).cuda()
            K.check(K.paged_stage_repage_gather(self.sources(ids), self.ps, self.dst.side(did), self.dst.nh, self.pd, tb, te, self.lb, self.le,
                                                self.row, self.cast, self.scales, stream=stream_ptr()), "single")
            torch.cuda.synchronize()
        out = self.dst.buf.clone()
        self.dst.buf.copy_(kept)
        return out

    def check(self, singles=True):
        got = self.dst.buf.cpu().numpy()
        assert np.array_equal(got, self.expected()), "the batch differs from the oracle"
        if singles:
            assert torch.equal(self.dst.buf, self.singles()), "the batch differs from n single launches"

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
        st.completion_value = epoch           # the epoch word as completion
        st.gate_mode = gate_mode
        st.gate_timeout_ms = timeout_ms
        st.max_ctas = self.max_ctas
        return st

    def run_streamed(self, epoch, gate_mode, timeout_ms=3000):
        """A late producer on its own stream (one for all sources) writes each source layer by layer and releases its flag; a
        checker stream waits for each layer_done flag in turn, so every one of them was observed at its epoch."""
        p0 = self.srcs[0].stream
        checker = torch.cuda.Stream()
        for p in self.srcs:        # every torch kernel of the producer once, then the poison back
            with torch.cuda.stream(p0):
                torch.cuda._sleep(100)
                p.layer(p.buf, 0).copy_(p.layer(p.final, 0))
        torch.cuda.synchronize()
        first = {}
        for s, _sl, dl, *_r in self.windows:
            first[s] = min(first.get(s, 1 << 30), dl)
        for p in self.srcs:
            p.buf.copy_(p.poison)
            if gate_mode == K.GATE_STREAM_WAIT:     # the stream-wait form has no timeout: its guards stay released
                p.ready_all[p.nl:].fill_(epoch)
        torch.cuda.synchronize()
        try:
            K.check(K.paged_stage_repage_gather_batch_streamed(*self.args(), self.stream_desc(epoch, gate_mode, timeout_ms),
                                                               stream_ptr(self.side_stream)), "launch")
            for l in range(self.lb, self.le):
                K.check(K.wait_flag(self.layer_done[l:].data_ptr(), epoch, stream_ptr(checker)), "wait_flag")
            with torch.cuda.stream(p0):
                for s in sorted(first, key=lambda x: first[x]):
                    p = self.srcs[s]
                    for l in range(p.nl):
                        torch.cuda._sleep(LAYER_SLEEP)
                        p.layer(p.buf, l).copy_(p.layer(p.final, l))
                        K.check(K.set_flags(p.ready.data_ptr(), l, 1, epoch, stream_ptr(p0)), "set_flags")
            assert _finish(self.side_stream) and _finish(p0) and _finish(checker), "the streamed batch did not finish"
        finally:
            s = torch.cuda.Stream()
            for p in self.srcs:
                K.set_flags(p.ready.data_ptr(), 0, p.nl, epoch, stream_ptr(s))
            K.set_flags(self.layer_done.data_ptr(), self.lb, self.le - self.lb, epoch, stream_ptr(s))   # frees the checker on failure
            assert _finish(s) and _finish(self.side_stream) and _finish(checker)
            torch.cuda.synchronize()
        self.check()
        assert [_i32(v) for v in self.layer_done.tolist()] == [epoch if self.lb <= l < self.le else 0 for l in range(self.dst.nl)]
        assert self.done.item() == epoch and self.completion.item() == epoch
        assert not self.ws.any().item(), "the workspace must be left zeroed"


def plan_rig(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, seqs, src_kv=KV.OperationalNHD, dst_kv=KV.OperationalNHD, **kw):
    """A rig of tp_pp_reshard_plan's windows: one pool per source rank the plan names, with its stage's layers and its heads."""
    plan = tp_pp_reshard_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank)
    ranks = sorted({w.src_rank for w in plan})
    srcs = [(L // src_pp, max(1, H // src_tp), src_kv) for _ in ranks]
    windows = [(ranks.index(w.src_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
               for w in plan]
    return BatchRig(srcs, windows, L // dst_pp, max(1, H // dst_tp), dst_kv, seqs, **kw)


TP4_TP2 = (8, 2, 4, 1, 2, 1, 0)       # H, L, src_tp, src_pp, dst_tp, dst_pp, rank
TP8_TP1 = (8, 2, 8, 1, 1, 1, 0)
PP2TP2 = (4, 4, 2, 2, 1, 1, 0)
ONE = (2, 2, 1, 1, 1, 1, 0)           # one source over every head and layer: still the batch gather kernels


# ---------------------------------------------------------------------------------------------------------------------
# against the oracle and n single launches
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 33, 257])
def test_batch_sizes(n):
    r = plan_rig(*TP4_TP2, mixed_seqs(n, n), src_kv=KV.OperationalHND, seed=n, no=1 if n > 100 else 2)
    assert r.run() == 0
    r.check()
    assert r.done.item() == 5 and r.completion.item() == 6


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (1, 16), (16, 1), (16, 16), (48, 12), (12, 48)], ids=lambda p: str(p))
@pytest.mark.parametrize("name,plan", [("tp4_to_tp2", TP4_TP2), ("tp8_to_tp1", TP8_TP1), ("pp2tp2_to_tp1", PP2TP2), ("one_source", ONE)])
def test_plans_and_pages(name, plan, ps, pd):
    """Prefix-hit starts inside a block, a 1-token sequence, an empty one, and a range whose first small blocks precede it."""
    big = max(ps, pd)
    seqs = [(big // 2 + 1, 3 * big + 3), (5 * big - 1, 5 * big), (7, 7), (2 * big, 4 * big), (big - 1, big + 1), (0, 2 * big + 5)]
    r = plan_rig(*plan, seqs, src_kv=KV.OperationalHND, dst_kv=KV.OperationalNHD, ps=ps, pd=pd, seed=ps + pd + len(name))
    assert r.run() == 0
    r.check()
    if name == "tp4_to_tp2":          # any order of the single launches: no two sequences share a destination block
        assert torch.equal(r.dst.buf, r.singles(order=list(reversed(range(len(seqs))))))


def test_two_sequences_sharing_source_blocks():
    """A shared prefix: sequence 1 reads sequence 0's source blocks (from its own prefix hit on) and its own past them."""
    for ps, pd in ((16, 64), (64, 16), (16, 16)):
        r = plan_rig(*TP4_TP2, [(0, 200), (70, 300), (130, 140)], ps=ps, pd=pd, seed=ps, shared=[(0, 1), (0, 2)])
        assert any(set(r.sids[0][0]) & set(r.sids[0][j]) for j in (1, 2))
        assert r.run() == 0
        r.check()


@pytest.mark.parametrize("dst_kv", ALL, ids=lambda k: k.name)
@pytest.mark.parametrize("src_kv", ALL, ids=lambda k: k.name)
def test_every_format_pair(src_kv, dst_kv):
    ps, pd = (16, 64) if (int(src_kv) + int(dst_kv)) % 2 else (64, 16)
    r = plan_rig(*PP2TP2, mixed_seqs(5, int(src_kv)), src_kv=src_kv, dst_kv=dst_kv, ps=ps, pd=pd, seed=10 * int(src_kv) + int(dst_kv))
    assert r.run() == 0
    r.check()


@pytest.mark.parametrize("hd", [128, 80])
@pytest.mark.parametrize("scaled", [False, True], ids=["unscaled", "scaled"])
@pytest.mark.parametrize("cast", [CM.FP8E4M3_TO_BF16, CM.BF16_TO_FP8E4M3], ids=lambda c: c.name)
def test_casts_scales_head_dims_and_layer_sub_ranges(cast, scaled, hd):
    for layers, (ps, pd) in ((None, (16, 64)), (range(1, 3), (48, 12))):
        r = plan_rig(*PP2TP2, mixed_seqs(6, hd), dst_kv=KV.UniversalPP, cast=cast, scaled=scaled, layers=layers, hd=hd, ps=ps, pd=pd,
                     seed=int(cast) + 3 * scaled + hd)
        assert r.run() == 0
        r.check()


@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16], ids=lambda c: c.name)
def test_mla_one_head(cast):
    r = plan_rig(1, 4, 1, 2, 1, 1, 0, mixed_seqs(4, 9), ps=64, pd=16, hd=576, no=1, cast=cast, seed=5)
    assert r.run() == 0
    r.check()


def test_a_batch_of_one_is_the_single_entry_and_zero_work_signals():
    r = plan_rig(*TP4_TP2, [(37, 411)], seed=3)
    assert r.run() == 0
    assert torch.equal(r.dst.buf, r.singles()) and not torch.equal(r.dst.buf, r.initial)
    # nothing to move: the destination keeps every byte and both words are still written
    for seqs, layers in (([], None), ([(9, 9), (64, 64)], None), ([(0, 100)], range(1, 1))):
        z = plan_rig(*TP4_TP2, seqs, layers=layers, seed=4)
        assert z.run() == 0
        assert torch.equal(z.dst.buf, z.initial) and z.done.item() == 5 and z.completion.item() == 6
        st = z.stream_desc(7, K.GATE_SPIN, 1000)
        K.check(K.paged_stage_repage_gather_batch_streamed(*z.args(), st, stream_ptr()), "streamed")
        torch.cuda.synchronize()
        assert torch.equal(z.dst.buf, z.initial) and z.done.item() == 7 and z.completion.item() == 7
        assert not z.layer_done.any().item() and not z.ws.any().item()


# ---------------------------------------------------------------------------------------------------------------------
# every instantiation of the two batch families, reached under the profiler
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True))}
EXPECTED = {(f, w + (pp,)) for f in ("paged", "gated") for w in WALKS for pp in (True, False)}


def test_batches_reach_every_batch_instantiation():
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c, p, s in sorted(WALKS):
            for ppow2 in (True, False):
                for gated in (False, True):
                    ps, pd = (16, 64) if ppow2 else (48, 12)
                    r = plan_rig(*PP2TP2, [(5, 150), (40, 41), (96, 200)], dst_kv=KV.UniversalTP, cast=CM(c), scaled=s, hd=64 if p else 80,
                                 ps=ps, pd=pd, seed=c + 2 * p + 4 * s + 8 * ppow2)
                    if gated:
                        for q in r.srcs:
                            q.ready.fill_(9)
                        torch.cuda.synchronize()
                        K.check(K.paged_stage_repage_gather_batch_streamed(*r.args(), r.stream_desc(9, K.GATE_SPIN, 10000), stream_ptr()),
                                "gated")
                        torch.cuda.synchronize()
                    else:
                        assert r.run() == 0
                    r.check(singles=False)
    found = set()
    for e in prof.events():
        for m in re.finditer(r"kvbm_(paged|gated)_batch_repage_gather_kernel<([^<>]*)>", e.name):
            c, p, s, pp = (a.strip().replace("(int)", "") for a in m.group(2).split(","))
            found.add((m.group(1), (int(c), p == "true", s == "true", pp == "true")))
    assert found == EXPECTED


# ---------------------------------------------------------------------------------------------------------------------
# streamed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("name,plan,ps,pd", [("tp4_to_tp2", TP4_TP2, 16, 64), ("pp2tp2_to_tp1", PP2TP2, 64, 16), ("pp2tp2_48", PP2TP2, 12, 48)])
def test_streamed_behind_a_late_producer(gate_mode, name, plan, ps, pd):
    r = plan_rig(*plan, mixed_seqs(9, 3, longest=700), src_kv=KV.OperationalHND, dst_kv=KV.UniversalTP, ps=ps, pd=pd, seed=7, poison=True,
                 cast=CM.FP8E4M3_TO_BF16, scaled=True)
    r.run_streamed(3, gate_mode)


def test_streamed_layer_sub_range_spinning():
    r = plan_rig(*PP2TP2, mixed_seqs(5, 11), ps=16, pd=64, seed=8, poison=True, layers=range(1, 4), max_ctas=2)
    r.run_streamed(6, K.GATE_SPIN)


# ---------------------------------------------------------------------------------------------------------------------
# through the TransferManager
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=11)
    yield m
    torch.cuda.synchronize()
    m.close()


def _requests(r, ranks):
    """The rig's sequences as execute_repage_batch takes them."""
    return [(range(tb, te), {rk: [int(x) for x in r.sids[i][q]] for i, rk in enumerate(ranks)}, [int(x) for x in r.dids[q]])
            for q, (tb, te) in enumerate(r.seqs)]


def _manager_rig(mgr, ranges, seed, **kw):
    H, L = 8, 4
    plan = tp_pp_reshard_plan(H, L, 2, 2, 1, 1, 0)
    r = plan_rig(H, L, 2, 2, 1, 1, 0, ranges, src_kv=KV.UniversalTP, dst_kv=KV.OperationalNHD, seed=seed, **kw)
    ranks = sorted({w.src_rank for w in plan})
    hs = {rk: _register(mgr, r.srcs[i], KV.UniversalTP) for i, rk in enumerate(ranks)}
    dh = _register(mgr, r.dst, KV.OperationalNHD)
    return r, plan, ranks, hs, dh


@pytest.mark.parametrize("n", [3, 40, 300])
@pytest.mark.parametrize("streamed", [False, True], ids=["unstreamed", "streamed"])
def test_manager_batch(mgr, streamed, n):
    """One launch, one notification, one done flag, the oracle's and the single launches' bytes, bytes_moved the single calls' sum.
    300 sequences outgrow a slot's arena and take its owned allocation."""
    r, plan, ranks, hs, dh = _manager_rig(mgr, mixed_seqs(n, 20 + n), 20 + n, layers=range(1, 4))
    seqs = _requests(r, ranks)
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    kw = dict(done_flag=flag.data_ptr(), epoch=4, layer_range=range(1, 4))
    launches, moved0, h2d0 = K.launch_count(), mgr.bytes_moved(), mgr.h2d_bytes()
    if streamed:
        for p in r.srcs:
            p.ready.fill_(4)
        torch.cuda.synchronize()
        note = mgr.execute_repage_batch(hs, dh, seqs, plan, TransferOptions(gate_mode=K.GATE_STREAM_WAIT, **kw),
                                        ready_flags={rk: r.srcs[i].ready.data_ptr() for i, rk in enumerate(ranks)},
                                        layer_done_flags=r.layer_done.data_ptr())
    else:
        note = mgr.execute_repage_batch(hs, dh, seqs, plan, TransferOptions(**kw))
    note.wait(30.0)
    torch.cuda.synchronize()
    launched = K.launch_count() - launches
    r.check()
    assert flag.item() == 4
    inside = lambda w: max(0, min(4, w.dst_layer_begin + w.layer_count) - max(1, w.dst_layer_begin))  # noqa: E731
    tokens = sum(te - tb for tb, te in r.seqs)
    assert mgr.bytes_moved() - moved0 == sum(tokens * inside(w) * r.no * w.head_count * r.row for w in plan)
    if not streamed:
        assert 1 <= launched <= 2                        # the batch kernel and the signal, however many sequences
    else:
        assert r.layer_done.tolist() == [4 if 1 <= l < 4 else 0 for l in range(4)]
    ids = len(ranks) * sum(len(x) for x in r.sids[0]) + sum(len(x) for x in r.dids)
    assert mgr.h2d_bytes() - h2d0 == 4 * ((ids + 3) // 4 * 4) + 16 * len(r.units_np)   # one staged copy: the ids, padded to 16 B, and the units


def test_manager_destination_blocks_are_unique_and_source_blocks_may_be_shared(mgr):
    r, plan, ranks, hs, dh = _manager_rig(mgr, [(10, 200), (10, 200), (64, 65)], 31)
    for s in range(len(r.srcs)):            # sequence 1 reads sequence 0's source blocks: a shared prefix
        r.sids[s][1] = r.sids[s][0]
    seqs = _requests(r, ranks)
    tokens, src, dst = seqs[1]
    with pytest.raises(KvbmError) as e:      # ... but may not write one of its destination blocks
        mgr.execute_repage_batch(hs, dh, [seqs[0], (tokens, src, [seqs[0][2][1]] + dst[1:]), seqs[2]], plan)
    assert e.value.code == ErrorCode.DUPLICATE_DST and f"duplicates = [{seqs[0][2][1]}]" in e.value.msg
    torch.cuda.synchronize()
    assert torch.equal(r.dst.buf, r.initial)
    mgr.execute_repage_batch(hs, dh, seqs, plan).wait(30.0)
    torch.cuda.synchronize()
    r.check()


def test_manager_head_window_plan_is_pp1(mgr):
    """A HeadWindow plan with num_layers is the identity layer window over every layer."""
    from dynamo_b200.physical import tp_reshard_plan
    H, L = 8, 2
    plan = tp_reshard_plan(H, 4, 2, 0)
    r = plan_rig(H, L, 4, 1, 2, 1, 0, mixed_seqs(5, 2), seed=12)
    ranks = sorted({w.src_rank for w in plan})
    hs = {rk: _register(mgr, r.srcs[i], KV.OperationalNHD) for i, rk in enumerate(ranks)}
    dh = _register(mgr, r.dst, KV.OperationalNHD)
    mgr.execute_repage_batch(hs, dh, _requests(r, ranks), plan, num_layers=L).wait(30.0)
    torch.cuda.synchronize()
    r.check()

"""GPU parity of the routed re-paging gather (each sequence of a decode step pulled from the prefill workers that served it, in one
launch): kvbm_kernels_paged_stage_repage_gather_routed, its streamed form and TransferManager.execute_repage_batch_routed.  The
destination pool starts as poison and is compared whole with a per-sequence oracle: tests/stage_repage_oracle.stage_repage_gather
over each sequence's range with its routed windows only.  At the kernel entry every source-table position of a sequence not routed
to that source names one of the source's sentinel blocks, whose bytes are all SENTINEL, so a kernel that reads an unrouted window
writes that pattern and fails the comparison.  One streamed launch runs at a time; every test ends with a device synchronize."""
import re
import time

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import (ErrorCode, KvbmError, LayoutConfig, ShardWindow, StorageKind, TransferManager, TransferOptions,
                                  tile_reshard_plan, tp_pp_reshard_plan)
from tests.gpu_util import stream_ptr
from tests.stage_repage_oracle import stage_repage_gather

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
ELEMS = {CM.NONE: (2, 2), CM.FP8E4M3_TO_BF16: (1, 2), CM.BF16_TO_FP8E4M3: (2, 1)}
GATES = [K.GATE_SPIN, K.GATE_STREAM_WAIT]
GATE_IDS = ["spin", "stream_wait"]
MASK = 0xFFFFFFFF
LAYER_SLEEP = 300_000      # cycles a producer sleeps before each layer (~0.15 ms)
HOST_TIMEOUT_S = 15.0      # longer than any gate timeout here
MAX_CTAS = 4
SENTINELS = 2              # blocks per source pool that only unrouted table positions name
SENTINEL = 0x7B            # their bytes


def _i32(v):
    v &= MASK
    return v - (1 << 32) if v >= 1 << 31 else v


def _sync():
    torch.cuda.synchronize()


def _finish(stream, timeout_s=HOST_TIMEOUT_S):
    """Wait on the host, with a deadline, for the work enqueued on `stream` so far; False when the deadline passed."""
    ev = torch.cuda.Event()
    ev.record(stream)
    t0 = time.monotonic()
    while not ev.query():
        if time.monotonic() - t0 > timeout_s:
            return False
        time.sleep(0.0005)
    return True


def table_len(tb, te, page):
    return 0 if tb == te else -(-te // page) - tb // page


class Pool:
    """A fully contiguous device pool of nb blocks [nl, no, region]: its final bytes, their poison (final ^ 0xA5) and its ready
    flags.  The last `sentinels` blocks hold SENTINEL bytes in both."""

    def __init__(self, nb, nl, no, page, nh, row, kv, seed, poison=False, sentinels=0):
        self.nb, self.nl, self.no, self.page, self.nh, self.row, self.kv = nb, nl, no, page, nh, row, int(kv)
        self.region = page * nh * row
        self.block = nl * no * self.region
        rng = np.random.default_rng(seed)
        self.final_np = rng.integers(0, 256, (nb, self.block), dtype=np.uint8)
        self.sentinel = list(range(nb - sentinels, nb))
        self.final_np[self.sentinel] = SENTINEL
        bad = self.final_np ^ 0xA5
        bad[self.sentinel] = SENTINEL
        self.final, self.poison = torch.from_numpy(self.final_np).cuda(), torch.from_numpy(bad).cuda()
        self.buf = (self.poison if poison else self.final).clone()
        self.layer_base = torch.tensor([self.buf.data_ptr() + l * no * self.region for l in range(nl)], dtype=torch.int64, device="cuda")
        self.ready = torch.zeros(nl, dtype=torch.int32, device="cuda")

    def side(self, ids):
        return K.PermuteSide(K.PagedLayout(self.layer_base.data_ptr(), self.block, self.region, self.region, self.nl, self.no, self.nb),
                             ids.data_ptr(), self.kv)

    def layer(self, t, l):
        return t.view(self.nb, self.nl, -1)[:, l]


def _dev(x):
    x = np.asarray(x, dtype=np.int32)
    return torch.from_numpy(x if len(x) else np.zeros(1, np.int32)).cuda()


class GatherRig:
    """pools: (num_layers, num_heads, kv) per source pool at page ps; windows: (pool, src_layer_begin, dst_layer_begin, layer_count,
    src_head_begin, dst_head_begin, head_count), one kernel source each; dst: (num_layers, num_heads, kv) at pd; seqs: (token_begin,
    token_end, pool mask).  A sequence is routed to every window of the pools in its mask.  share: the source tables draw their
    blocks with repeats (shared prefixes)."""

    def __init__(self, pools, windows, dst, seqs, ps=16, pd=64, no=2, hd=64, cast=CM.NONE, scaled=False, layers=None, seed=0, share=False):
        se, de = ELEMS[cast]
        self.row, self.cast, self.windows, self.no, self.ps, self.pd = hd * se, int(cast), list(windows), no, ps, pd
        self.seqs = [tuple(int(x) for x in s) for s in seqs]
        dnl, dnh, dkv = dst
        self.lb, self.le = (layers.start, layers.stop) if layers else (0, dnl)
        ns = sum(table_len(tb, te, ps) for tb, te, _ in self.seqs)
        nd = sum(table_len(tb, te, pd) for tb, te, _ in self.seqs)
        nsb = ns // 2 + 2 if share else ns + 2
        self.srcs = [Pool(nsb + SENTINELS, nl, no, ps, nh, self.row, kv, seed + 10 + i, sentinels=SENTINELS) for i, (nl, nh, kv) in enumerate(pools)]
        self.dst = Pool(nd + 2, dnl, no, pd, dnh, hd * de, dkv, seed + 1, poison=True)
        rng = np.random.default_rng(seed + 2)
        self.sids = []
        for p, pool in enumerate(self.srcs):
            ids, so = (rng.integers(0, nsb, ns) if share else rng.permutation(nsb)[:ns]).astype(np.int32), 0
            for tb, te, m in self.seqs:
                a = table_len(tb, te, ps)
                if not (m >> p) & 1:
                    ids[so:so + a] = [pool.sentinel[k % SENTINELS] for k in range(a)]
                so += a
            self.sids.append(ids)
        self.dids = rng.permutation(nd + 2)[:nd].astype(np.int32)
        self.kseqs = [(tb, te, self.window_mask(m)) for tb, te, m in self.seqs]
        u = K.repage_route_units(self.kseqs, ps, pd)
        assert u is not None and (u[1], u[2]) == (ns, nd)
        self.units_np, self.nu = u[0], len(u[0])
        self.sids_t, self.dids_t = [_dev(x) for x in self.sids], _dev(self.dids)
        self.units_t = _dev(np.ascontiguousarray(self.units_np).view(np.int32).reshape(-1))
        self.initial = self.dst.buf.clone()
        self.scales_np = (rng.uniform(0.1, 4.0, dnl * no) * (1 + np.arange(dnl * no) * 1e-2)).astype(np.float32) if scaled else None
        self.scales = torch.from_numpy(self.scales_np).cuda() if scaled else None
        self.done = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.completion = torch.zeros(1, dtype=torch.int32, device="cuda")

    def window_mask(self, m):
        return sum(1 << j for j, w in enumerate(self.windows) if (m >> w[0]) & 1)

    def sources(self, ids=None, windows=None):
        ids = ids or self.sids_t
        return [K.StageSource(K.PermuteSource(self.srcs[p].side(ids[p]), self.srcs[p].nh, sb, db, k), sl, dl, c)
                for p, sl, dl, c, sb, db, k in (windows or self.windows)]

    def args(self):
        return (self.sources(), self.ps, self.dst.side(self.dids_t), self.dst.nh, self.pd, self.kseqs, self.units_t.data_ptr(), self.nu,
                self.lb, self.le, self.row, self.cast, self.scales)

    def launch(self, epoch=5, value=6):
        return K.paged_stage_repage_gather_routed(*self.args(), self.done.data_ptr(), epoch, self.completion.data_ptr(), value, stream_ptr())

    def expected(self, layers=None):
        pool = self.initial.cpu().numpy().copy()
        layers = layers if layers is not None else range(self.lb, self.le)
        so = do = 0
        for tb, te, m in self.seqs:
            a, b = table_len(tb, te, self.ps), table_len(tb, te, self.pd)
            if a:
                routed = [p for p in range(len(self.srcs)) if (m >> p) & 1]
                srcs = [([self.srcs[p].final_np[x] for x in self.sids[p][so:so + a]], self.srcs[p].kv, self.srcs[p].nh, self.srcs[p].nl)
                        for p in routed]
                wins = [(routed.index(p),) + tuple(w) for p, *w in self.windows if (m >> p) & 1]
                d = self.dst
                out = stage_repage_gather(srcs, wins, [pool[x] for x in self.dids[do:do + b]], d.kv, d.nh, d.nl, self.no, self.ps, self.pd,
                                          self.row, tb, te, self.cast, self.scales_np, layers)
                for x, blk in zip(self.dids[do:do + b], out):
                    pool[x] = blk
            so, do = so + a, do + b
        return pool

    def check_pool(self, want=None):
        got = self.dst.buf.cpu().numpy()
        if self.cast == CM.NONE:
            assert not (got.reshape(-1, 16) == SENTINEL).all(1).any(), "a sentinel source block was read"
        assert np.array_equal(got, self.expected() if want is None else want)

    def run_and_check(self, epoch=5, value=6):
        assert self.launch(epoch, value) == 0
        _sync()
        self.check_pool()
        assert self.done.item() == epoch and self.completion.item() == value

    def reset(self):
        self.dst.buf.copy_(self.initial)
        _sync()


def _plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers):
    """Decode rank `rank`'s plan from one prefill group, its ranks renumbered 0..R-1, tiled over `workers` identical workers."""
    one = tp_pp_reshard_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank)
    ranks = sorted({w.src_rank for w in one})
    one = [ShardWindow(ranks.index(w.src_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin,
                       w.head_count) for w in one]
    return tile_reshard_plan(one, workers, len(ranks)), len(ranks)


def _masks(how, n, npools, per_worker, rng):
    """Pool masks: each sequence from one random worker, a random non-empty subset of pools, or every pool."""
    workers = npools // per_worker
    out = []
    for _ in range(n):
        if how == "worker":
            k = int(rng.integers(0, workers))
            out.append(((1 << per_worker) - 1) << (k * per_worker))
        elif how == "random":
            out.append(int(rng.integers(1, 1 << npools)))
        else:
            out.append((1 << npools) - 1)
    return out


def _rig(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers, ranges, how="worker", src_kv=KV.OperationalHND, dst_kv=KV.OperationalNHD,
         seed=0, **kw):
    plan, per = _plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers)
    npools = workers * per
    masks = _masks(how, len(ranges), npools, per, np.random.default_rng(seed + 1000))
    pools = [(L // src_pp, max(1, H // src_tp), src_kv)] * npools
    windows = [(w.src_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan]
    r = GatherRig(pools, windows, (L // dst_pp, max(1, H // dst_tp), dst_kv), [(tb, te, m) for (tb, te), m in zip(ranges, masks)], seed=seed,
                  **kw)
    r.plan, r.per_worker = plan, per
    return r


def _batch(n, length, first=3, step=11):
    return [(first + step * i, first + step * i + length) for i in range(n)]


def _mixed(seed=7):
    """1 to 4000 tokens, empty sequences between others."""
    rng = np.random.default_rng(seed)
    out = []
    for i, n in enumerate([1, 4000] + [int(x) for x in rng.integers(1, 4001, 8)]):
        tb = int(rng.integers(1, 300)) | 1
        out.append((tb, tb + n))
        if i % 3 == 1:
            out.append((tb + 5, tb + 5))
    return out


SMALL = [(5, 200), (40, 41), (3, 3), (17, 333)]
# (H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers): windows = workers x windows per worker
SHAPES = {
    "4x_tp4_to_tp2": (8, 2, 4, 1, 2, 1, 0, 4),          # 2 windows per worker, overlapping across workers
    "2x_tp8_to_tp1": (8, 2, 8, 1, 1, 1, 0, 2),          # 8 windows per worker, 16 sources
    "tp4_to_tp1": (8, 2, 4, 1, 1, 1, 0, 1),             # 4 disjoint windows: any subset of sources
}


# ---------------------------------------------------------------------------------------------------------------------
# unstreamed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (1, 16), (16, 16), (48, 96), (96, 48)], ids=str)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_routed_plans_and_pages(shape, ps, pd):
    how = "random" if shape == "tp4_to_tp1" else "worker"
    r = _rig(*SHAPES[shape], _mixed()[:7] + SMALL, how=how, ps=ps, pd=pd, no=1, hd=32, seed=ps + pd + len(shape))
    assert any(m != (1 << len(r.srcs)) - 1 for _, _, m in r.seqs)
    r.run_and_check()
    _sync()


def test_mla_from_8_dp_workers():
    """MLA's one 576-wide latent head, every worker's window writing it: each sequence from one worker."""
    r = _rig(1, 3, 1, 1, 1, 1, 0, 8, SMALL + _batch(12, 300), no=1, hd=576, ps=64, pd=64, seed=57)
    assert len(r.windows) == 8 and all(w[5] == 0 for w in r.windows)
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("rank", [2, 4], ids=["two_stages", "one_stage"])
def test_pp2_workers_tiled(rank):
    """Decode rank `rank` of PP3 x TP2 from 2 PP2 x TP2 prefill workers: decode stage 1 reads both prefill stages (layer shifts of
    either sign), stage 2 the second only."""
    r = _rig(4, 12, 2, 2, 2, 3, rank, 2, _batch(6, 300) + SMALL, seed=rank + 5)
    shifts = {w[1] - w[2] for w in r.windows}
    assert shifts == ({4, -2} if rank == 2 else {2})
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("cast,scaled", [(CM.FP8E4M3_TO_BF16, False), (CM.FP8E4M3_TO_BF16, True), (CM.BF16_TO_FP8E4M3, False),
                                         (CM.BF16_TO_FP8E4M3, True)], ids=["up", "up_scaled", "down", "down_scaled"])
def test_casts_and_scales(cast, scaled):
    r = _rig(*SHAPES["4x_tp4_to_tp2"][:1], 4, *SHAPES["4x_tp4_to_tp2"][2:], SMALL + _batch(6, 100), src_kv=KV.OperationalNHD,
             dst_kv=KV.UniversalTP, cast=cast, scaled=scaled, layers=range(1, 3), seed=int(cast) + 3 * scaled)
    r.run_and_check()
    _sync()


def test_shared_source_blocks_and_300_sequences():
    r = _rig(*SHAPES["4x_tp4_to_tp2"], _batch(300, 70, step=3), no=1, hd=32, share=True, seed=77)
    assert len({m for _, _, m in r.seqs}) > 1
    r.run_and_check()
    _sync()


def test_all_ones_equals_the_batch_gather():
    r = _rig(*SHAPES["tp4_to_tp1"], _mixed() + SMALL, how="all", no=1, hd=32, seed=88)
    r.run_and_check()
    routed = r.dst.buf.clone()
    r.reset()
    u = K.repage_batch_units([(tb, te) for tb, te, _ in r.seqs], r.ps, r.pd)
    ut = _dev(np.ascontiguousarray(u[0]).view(np.int32).reshape(-1))
    assert K.paged_stage_repage_gather_batch(r.sources(), r.ps, r.dst.side(r.dids_t), r.dst.nh, r.pd, [(tb, te) for tb, te, _ in r.seqs],
                                             ut.data_ptr(), len(u[0]), r.lb, r.le, r.row, r.cast, r.scales, stream=stream_ptr()) == 0
    _sync()
    assert torch.equal(routed, r.dst.buf)
    _sync()


def test_one_worker_per_sequence_equals_one_batch_gather_per_worker():
    r = _rig(*SHAPES["2x_tp8_to_tp1"], _batch(10, 130, step=13) + SMALL, no=1, hd=32, seed=89)
    r.run_and_check()
    routed = r.dst.buf.clone()
    r.reset()
    per, spans, so, do = r.per_worker, [], 0, 0
    for tb, te, m in r.seqs:
        a, b = table_len(tb, te, r.ps), table_len(tb, te, r.pd)
        spans.append((so, a, do, b))
        so, do = so + a, do + b
    for k in range(len(r.srcs) // per):
        idx = [i for i, (_, _, m) in enumerate(r.seqs) if (m >> (k * per)) & 1]
        seqs = [r.seqs[i][:2] for i in idx]
        ids = [_dev(np.concatenate([r.sids[p][spans[i][0]:spans[i][0] + spans[i][1]] for i in idx])) for p in range(len(r.srcs))]
        did = _dev(np.concatenate([r.dids[spans[i][2]:spans[i][2] + spans[i][3]] for i in idx]))
        u = K.repage_batch_units(seqs, r.ps, r.pd)
        ut = _dev(np.ascontiguousarray(u[0]).view(np.int32).reshape(-1))
        wins = [w for w in r.windows if w[0] // per == k]
        K.check(K.paged_stage_repage_gather_batch(r.sources(ids, wins), r.ps, r.dst.side(did), r.dst.nh, r.pd, seqs, ut.data_ptr(), len(u[0]),
                                                  r.lb, r.le, r.row, r.cast, r.scales, stream=stream_ptr()), "per-worker batch")
        _sync()
    assert torch.equal(routed, r.dst.buf)
    _sync()


def test_empty_batches_signal():
    r = _rig(*SHAPES["4x_tp4_to_tp2"], [(9, 9), (70, 70)], seed=4)
    for seqs in ([], [(9, 9, 1), (70, 70, 2)]):
        r.done.zero_()
        assert K.paged_stage_repage_gather_routed(r.sources(), 16, r.dst.side(r.dids_t), r.dst.nh, 64, seqs, 0, 0, 0, r.le, r.row, 0, None,
                                                  r.done.data_ptr(), 7, r.completion.data_ptr(), 8, stream_ptr()) == 0
        _sync()
        assert r.done.item() == 7 and r.completion.item() == 8
    assert torch.equal(r.initial, r.dst.buf)
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# the streamed routed gather, behind a producer that writes the sources after the launch
# ---------------------------------------------------------------------------------------------------------------------
class StreamGather:
    """A GatherRig whose sources are written after the launch; `unstreamed` holds the pool the unstreamed routed gather leaves.
    flags[p]: pool p's ready flags (its device `ready`, or a caller's)."""

    def __init__(self, rig, max_ctas=MAX_CTAS, timeout_ms=10000, flags=None):
        self.r, self.max_ctas, self.timeout_ms = rig, max_ctas, timeout_ms
        self.flags = flags or {}
        self.nl = rig.dst.nl
        self.want = rig.expected()
        assert rig.launch(1, 1) == 0
        _sync()
        self.unstreamed = rig.dst.buf.clone()
        self.layer_done = torch.zeros(self.nl, dtype=torch.int32, device="cuda")
        self.ws = torch.zeros(K.sync_workspace_words(self.nl), dtype=torch.int32, device="cuda")
        self.side_stream, self.producer = torch.cuda.Stream(), torch.cuda.Stream()
        with torch.cuda.stream(self.producer):   # every torch kernel of the producer once
            torch.cuda._sleep(100)
            for p in rig.srcs:
                p.layer(p.buf, 0).copy_(p.layer(p.final, 0))
        _sync()
        self.reset()

    def reset(self):
        r = self.r
        for p in r.srcs:
            p.buf.copy_(p.poison)
            p.ready.zero_()
        r.dst.buf.copy_(r.initial)
        for t in (self.layer_done, r.done, r.completion):
            t.zero_()
        _sync()

    def flag(self, p):
        return self.flags.get(p, self.r.srcs[p].ready.data_ptr())

    def stream_desc(self, epoch, gate_mode, value):
        st = K.PermuteStream()
        for j, w in enumerate(self.r.windows):
            st.layer_ready_flags[j] = self.flag(w[0])
        st.layer_done_flags = self.layer_done.data_ptr()
        st.done_flag = self.r.done.data_ptr()
        st.epoch = epoch & MASK
        st.sync_workspace = self.ws.data_ptr()
        st.completion_flag = self.r.completion.data_ptr()
        st.completion_value = value & MASK
        st.gate_mode = gate_mode
        st.gate_timeout_ms = self.timeout_ms
        st.max_ctas = self.max_ctas
        return st

    def launch(self, epoch, gate_mode, value):
        K.check(K.paged_stage_repage_gather_routed_streamed(*self.r.args(), self.stream_desc(epoch, gate_mode, value),
                                                            stream_ptr(self.side_stream)), "streamed routed gather")

    def produce(self, layers, epoch, pools=None):
        """On the producer stream: per source layer, sleep, write every pool's layer and release its flag."""
        with torch.cuda.stream(self.producer):
            for l in layers:
                torch.cuda._sleep(LAYER_SLEEP)
                for i in (pools if pools is not None else range(len(self.r.srcs))):
                    p = self.r.srcs[i]
                    if l < p.nl:
                        p.layer(p.buf, l).copy_(p.layer(p.final, l))
                        K.check(K.set_flags(p.ready.data_ptr(), l, 1, epoch & MASK, stream_ptr(self.producer)), "set_flags")

    def rescue(self, epoch):
        """Release every device flag from a fresh stream and let the launch and the producer drain."""
        s = torch.cuda.Stream()
        for p in self.r.srcs:
            K.set_flags(p.ready.data_ptr(), 0, p.nl, epoch & MASK, stream_ptr(s))
        assert _finish(s) and _finish(self.side_stream) and _finish(self.producer), "a streamed launch is still waiting"
        _sync()

    def run(self, epoch, gate_mode, value):
        try:
            self.launch(epoch, gate_mode, value)
            self.produce(range(max(p.nl for p in self.r.srcs)), epoch)
            assert _finish(self.side_stream) and _finish(self.producer), "the streamed routed gather did not finish"
        finally:
            self.rescue(epoch)

    def check_end(self, epoch, value):
        r = self.r
        r.check_pool(self.want)
        assert torch.equal(r.dst.buf, self.unstreamed)
        assert [_i32(v) for v in self.layer_done.tolist()] == [_i32(epoch) if r.lb <= l < r.le else 0 for l in range(self.nl)]
        assert r.done.item() == _i32(epoch) and r.completion.item() == _i32(value)
        assert not self.ws.any().item(), "the workspace must be left zeroed"


SRC_KV = dict(src_kv=KV.OperationalHND)   # one layer of a source block is one contiguous run the producer writes


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("shape", ["4x_tp4_to_tp2", "pp2tp2_x2_to_pp3tp2_rank3"])
def test_streamed_layers_written_after_the_launch(gate_mode, shape):
    args = SHAPES.get(shape, (4, 12, 2, 2, 2, 3, 3, 2))
    s = StreamGather(_rig(*args, _mixed()[:6] + SMALL, hd=32, seed=len(shape), **SRC_KV))
    s.run(5, gate_mode, 77)
    s.check_end(5, 77)
    _sync()


@pytest.mark.parametrize("max_ctas", [1, 2, 3])
def test_spinning_batches_that_span_layers(max_ctas):
    """A handful of units per layer on 1-3 CTAs: claims of several units cross layer boundaries."""
    s = StreamGather(_rig(8, 4, 4, 1, 2, 1, 0, 2, [(3, 70), (5, 5), (100, 180), (1, 2)], no=1, seed=90 + max_ctas, **SRC_KV),
                     max_ctas=max_ctas)
    s.run(8, K.GATE_SPIN, 5)
    s.check_end(8, 5)
    _sync()


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_only_released_layers_move(gate_mode):
    """Release k layers of every source, wait for layer_done[k - 1]: only those layers landed, and no done flag is written."""
    s = StreamGather(_rig(8, 4, 4, 1, 2, 1, 0, 2, SMALL + _batch(5, 200), seed=41, **SRC_KV))
    r, k, epoch = s.r, 2, 7
    checker = torch.cuda.Stream()
    snap, flags = r.dst.buf.clone(), [s.layer_done.clone(), r.done.clone()]
    try:
        s.launch(epoch, gate_mode, 1)
        s.produce(range(k), epoch)
        with torch.cuda.stream(checker):
            K.check(K.wait_flag(s.layer_done.data_ptr() + 4 * (k - 1), epoch, stream_ptr(checker)), "wait_flag")
            torch.cuda._sleep(2_000_000)
            for t, f in zip(flags, (s.layer_done, r.done)):
                t.copy_(f)
            snap.copy_(r.dst.buf)
        assert _finish(checker), "layer_done of the released layers did not appear"
        s.produce(range(k, s.nl), epoch)
        assert _finish(s.side_stream) and _finish(s.producer)
    finally:
        if not _finish(checker, 2.0):
            K.set_flags(s.layer_done.data_ptr(), 0, s.nl, epoch, stream_ptr(torch.cuda.Stream()))
        s.rescue(epoch)
        assert _finish(checker)
    s.check_end(epoch, 1)
    assert np.array_equal(snap.cpu().numpy(), r.expected(range(0, k)))
    assert flags[0].tolist() == [epoch if l < k else 0 for l in range(s.nl)] and flags[1].item() == 0
    _sync()


def test_a_lockstep_producer():
    """The producer waits for layer_done[l] before it writes layer l + 1 (spinning form)."""
    s = StreamGather(_rig(*SHAPES["4x_tp4_to_tp2"], _batch(20, 64 * 3, step=17), seed=55, **SRC_KV), max_ctas=8, timeout_ms=3000)
    r, epoch = s.r, 11
    try:
        s.launch(epoch, K.GATE_SPIN, 12)
        with torch.cuda.stream(s.producer):
            for l in range(s.nl):
                for p in r.srcs:
                    p.layer(p.buf, l).copy_(p.layer(p.final, l))
                    K.check(K.set_flags(p.ready.data_ptr(), l, 1, epoch, stream_ptr(s.producer)), "set_flags")
                K.check(K.wait_flag(s.layer_done.data_ptr() + 4 * l, epoch, stream_ptr(s.producer)), "wait_flag")
        assert _finish(s.producer) and _finish(s.side_stream), "the lockstep producer did not finish"
    finally:
        s.rescue(epoch)
    assert r.completion.item() == 12, "the gate timed out"
    s.check_end(epoch, 12)
    _sync()


def test_default_grid_leaves_the_producer_room():
    s = StreamGather(_rig(*SHAPES["4x_tp4_to_tp2"], _batch(40, 64 * 2, step=29), seed=61, **SRC_KV), max_ctas=0)
    assert s.r.nu * s.r.no >= torch.cuda.get_device_properties(0).multi_processor_count // 2
    s.run(6, K.GATE_SPIN, 61)
    s.check_end(6, 61)
    _sync()


def test_a_gate_timeout_writes_no_done_flag():
    s = StreamGather(_rig(*SHAPES["4x_tp4_to_tp2"], SMALL + _batch(3, 100), seed=71, **SRC_KV), timeout_ms=200)
    r, epoch = s.r, 4
    try:
        s.launch(epoch, K.GATE_SPIN, 9)
        s.produce(range(1), epoch)
        assert _finish(s.side_stream), "the gate did not time out"
    finally:
        s.rescue(epoch)
    assert _i32(r.completion.item()) == _i32(MASK) and r.done.item() == 0
    assert not s.ws.any().item()
    _sync()


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_an_unrouted_source_is_never_waited_on(gate_mode):
    """Worker 1's sources are named by no sequence and their ready flags, in mapped pinned host memory, are never released by the
    producer.  The host waits for the transfer with a deadline and only then releases them itself, so a build that waits on them
    finishes late and fails instead of hanging."""
    ranges = SMALL + _batch(6, 150)
    r = _rig(*SHAPES["4x_tp4_to_tp2"], ranges, seed=31, **SRC_KV)
    per = r.per_worker
    r2 = GatherRig([(p.nl, p.nh, p.kv) for p in r.srcs], r.windows, (r.dst.nl, r.dst.nh, r.dst.kv),
                   [(tb, te, ((1 << per) - 1) << (per * (0 if i % 2 else 2))) for i, (tb, te) in enumerate(ranges)], hd=64, seed=31)
    idle = [p for p in range(len(r2.srcs)) if not any((m >> p) & 1 for _, _, m in r2.seqs)]
    assert idle
    host = torch.zeros((len(idle), r2.dst.nl + 1), dtype=torch.int32).pin_memory()
    s = StreamGather(r2, flags={p: host[i].data_ptr() for i, p in enumerate(idle)})
    epoch = 3
    try:
        s.launch(epoch, gate_mode, 21)
        s.produce(range(r2.dst.nl), epoch, pools=[p for p in range(len(r2.srcs)) if p not in idle])
        finished = _finish(s.side_stream, 5.0)
    finally:
        host.numpy()[:] = epoch
        s.rescue(epoch)
    assert finished, "the transfer waited on a source no sequence is routed to"
    s.check_end(epoch, 21)
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# every instantiation of both families, reached under the profiler
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True))}
EXPECTED = {w + (pp,) for w in WALKS for pp in (True, False)}


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
                r = _rig(8, 4, 4, 1, 2, 1, 0, 2, SMALL, dst_kv=KV.UniversalTP, cast=CM(c), scaled=sc, hd=64 if p else 80, ps=ps, pd=pd,
                         seed=c + 2 * p + 4 * sc + 8 * ppow2, **SRC_KV)
                r.run_and_check()     # synchronizes before the oracle check
                s = StreamGather(r)
                for x in r.srcs:      # the flags released before the launch
                    x.buf.copy_(x.final)
                    x.ready.fill_(3)
                _sync()
                s.launch(3, K.GATE_SPIN, 5)
                assert _finish(s.side_stream)
                _sync()
                s.check_end(3, 5)
    assert _found(prof, "kvbm_paged_repage_fanin_kernel") == EXPECTED
    assert _found(prof, "kvbm_gated_repage_fanin_kernel") == EXPECTED
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# TransferManager.execute_repage_batch_routed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=61)
    yield m
    _sync()
    m.close()


def _register(mgr, p):
    cfg = LayoutConfig(p.nb, p.nl, p.no, p.page, p.nh * (p.row // 2), dtype_width_bytes=2, num_heads=p.nh)
    h = mgr.register_fully_contiguous(cfg, p.buf.data_ptr(), p.buf.numel(), StorageKind.Device, 0)
    mgr.set_kv_block_layout(h, KV(p.kv))
    return h


def _managed(mgr, r):
    """Register the rig's pools; the plan (source rank = pool) and the routed requests, each with its routed sources' ids."""
    sources = {p: _register(mgr, x) for p, x in enumerate(r.srcs)}
    dh = _register(mgr, r.dst)
    plan = [ShardWindow(*w) for w in r.windows]
    reqs, so, do = [], 0, 0
    for tb, te, m in r.seqs:
        a, b = table_len(tb, te, r.ps), table_len(tb, te, r.pd)
        ids = {p: [int(x) for x in r.sids[p][so:so + a]] for p in range(len(r.srcs)) if (m >> p) & 1}
        reqs.append((range(tb, te), ids, [int(x) for x in r.dids[do:do + b]]))
        so, do = so + a, do + b
    return sources, dh, plan, reqs


def _routed_bytes(r):
    total = 0
    for tb, te, m in r.seqs:
        for p, sl, dl, c, sb, db, k in r.windows:
            if (m >> p) & 1:
                total += (te - tb) * max(0, min(r.le, dl + c) - max(r.lb, dl)) * r.no * k * r.dst.row
    return total


def test_manager_routed(mgr):
    r = _rig(*SHAPES["4x_tp4_to_tp2"], _mixed() + SMALL, no=1, hd=32, seed=101)
    sources, dh, plan, reqs = _managed(mgr, r)
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    m0 = mgr.bytes_moved()
    mgr.execute_repage_batch_routed(sources, dh, reqs, plan, TransferOptions(done_flag=flag.data_ptr(), epoch=4)).wait(20.0)
    _sync()
    assert mgr.bytes_moved() - m0 == _routed_bytes(r) > 0
    r.check_pool()
    assert flag.item() == 4
    _sync()


def test_manager_300_sequences(mgr):
    r = _rig(*SHAPES["2x_tp8_to_tp1"], _batch(300, 70, step=3), no=1, hd=32, seed=107)
    sources, dh, plan, reqs = _managed(mgr, r)
    mgr.execute_repage_batch_routed(sources, dh, reqs, plan).wait(20.0)
    _sync()
    r.check_pool()
    _sync()


def test_manager_duplicate_and_overlap_rejections(mgr):
    """A destination block named twice in the batch is KVBM_ERR_DUPLICATE_DST; a sequence routed to two workers whose windows
    share destination heads is KVBM_ERR_OVERLAP; nothing moves."""
    r = _rig(*SHAPES["4x_tp4_to_tp2"], [(3, 70), (100, 180)], seed=103)
    sources, dh, plan, reqs = _managed(mgr, r)
    before = r.dst.buf.clone()
    dup = [reqs[0], (reqs[1][0], reqs[1][1], [reqs[0][2][0]] + reqs[1][2][1:])]
    with pytest.raises(KvbmError) as e:
        mgr.execute_repage_batch_routed(sources, dh, dup, plan)
    assert e.value.code == ErrorCode.DUPLICATE_DST
    both = [reqs[0], (reqs[1][0], {p: list(range(len(reqs[1][1][next(iter(reqs[1][1]))]))) for p in range(len(r.srcs))}, reqs[1][2])]
    with pytest.raises(KvbmError) as e:
        mgr.execute_repage_batch_routed(sources, dh, both, plan)
    assert e.value.code == ErrorCode.OVERLAP and "overlap in the destination" in e.value.msg
    _sync()
    assert torch.equal(before, r.dst.buf)


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_manager_streamed_routed(mgr, gate_mode):
    s = StreamGather(_rig(*SHAPES["4x_tp4_to_tp2"], _mixed()[:5] + SMALL, hd=32, seed=109, **SRC_KV))
    r = s.r
    sources, dh, plan, reqs = _managed(mgr, r)
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    opts = TransferOptions(done_flag=flag.data_ptr(), epoch=4, gate_mode=gate_mode, max_ctas=MAX_CTAS)
    try:
        note = mgr.execute_repage_batch_routed(sources, dh, reqs, plan, opts, ready_flags={p: x.ready.data_ptr() for p, x in enumerate(r.srcs)},
                                               layer_done_flags=s.layer_done.data_ptr())
        s.produce(range(r.dst.nl), 4)
        note.wait(20.0)
    finally:
        s.rescue(4)
    r.check_pool(s.want)
    assert flag.item() == 4 and s.layer_done.tolist() == [4] * s.nl
    _sync()

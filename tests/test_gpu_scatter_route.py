"""GPU parity of the routed re-paging scatter (each sequence of a prefill batch pushed to its own decode workers in one launch):
kvbm_kernels_paged_repage_scatter_routed, its streamed form and TransferManager.execute_repage_scatter_routed.  Every destination
pool starts as poison and is compared whole with the routed oracle: tests/scatter_oracle.repage_scatter applied per sequence to its
routed targets over its slices of the concatenated tables.  At the kernel entry every table position of a sequence not routed to
that pool names one of the pool's sentinel blocks (real, poisoned, named by no routed position), which must still hold their poison
afterwards.  Every sequence starts inside a block of the larger page.  One streamed launch runs at a time; every test ends with a
device synchronize."""
import re
import time

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import (ErrorCode, KvbmError, LayoutConfig, ScatterWindow, StorageKind, TransferManager, TransferOptions,
                                  tile_scatter_plan, tp_pp_scatter_plan)
from tests.gpu_util import stream_ptr
from tests.scatter_batch_oracle import table_len
from tests.scatter_oracle import repage_scatter

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
ELEMS = {CM.NONE: (2, 2), CM.FP8E4M3_TO_BF16: (1, 2), CM.BF16_TO_FP8E4M3: (2, 1)}
GATES = [K.GATE_SPIN, K.GATE_STREAM_WAIT]
GATE_IDS = ["spin", "stream_wait"]
MASK = 0xFFFFFFFF
LAYER_SLEEP = 300_000      # cycles a producer sleeps before each layer (~0.15 ms)
CHECKER_SLEEP = 2_000_000  # ~1 ms
HOST_TIMEOUT_S = 15.0      # longer than any gate timeout here
MAX_CTAS = 4
SENTINELS = 2              # blocks per destination pool that only unrouted table positions name


def _i32(v):
    v &= MASK
    return v - (1 << 32) if v >= 1 << 31 else v


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


class Pool:
    """A fully contiguous device pool of nb blocks [nl, no, region], with its final bytes and their poison (final ^ 0xA5)."""

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
        """On this pool's producer stream: per layer sleep, write its final bytes, release its flag."""
        with torch.cuda.stream(self.stream):
            for l in layers:
                torch.cuda._sleep(LAYER_SLEEP)
                self.layer(self.buf, l).copy_(self.layer(self.final, l))
                K.check(K.set_flags(self.ready.data_ptr(), l, 1, epoch, stream_ptr(self.stream)), "set_flags")


def routed_oracle(src, sids, targets, pools, no, ps, pd, row, seqs, cast=CM.NONE, scales=None, layers=None):
    """The routed scatter from the semantics: for each sequence (tb, te, mask), tests/scatter_oracle.repage_scatter over its range
    and its slices of the concatenated tables, with the targets whose bit is set only.  targets: (pool index, concatenated ids, kv,
    num_heads, num_layers, window).  Updates pools in place."""
    so = do = 0
    for tb, te, m in seqs:
        a, b = table_len(tb, te, ps), table_len(tb, te, pd)
        if a:
            tg = [(p, ids[do:do + b], kv, nh, nl, w) for t, (p, ids, kv, nh, nl, w) in enumerate(targets) if (m >> t) & 1]
            repage_scatter(([src.final_np[x] for x in sids[so:so + a]], src.kv, src.nh, src.nl), tg, pools, no, ps, pd, row, tb, te, int(cast),
                           scales, layers)
        so, do = so + a, do + b


class RouteRig:
    """src: (num_layers, num_heads, kv) of the source pool at page ps; dsts: (num_layers, num_heads, kv) per destination pool at pd;
    targets: (pool, src_layer_begin, dst_layer_begin, layer_count, src_head_begin, dst_head_begin, head_count); seqs: (token_begin,
    token_end, target mask).  Every destination pool is poisoned and has SENTINELS blocks that each table position of a sequence
    not routed to that pool names; every target of a pool takes that pool's one concatenated table.  share: the source table
    draws its blocks with repeats."""

    def __init__(self, src, dsts, targets, seqs, ps=16, pd=64, no=2, hd=64, cast=CM.NONE, scaled=False, layers=None, seed=0, share=False):
        se, de = ELEMS[cast]
        self.row, self.cast, self.targets, self.no, self.ps, self.pd = hd * se, int(cast), targets, no, ps, pd
        self.seqs = [tuple(int(x) for x in s) for s in seqs]
        nl, nh, kv = src
        self.lb, self.le = (layers.start, layers.stop) if layers else (0, nl)
        ns = sum(table_len(tb, te, ps) for tb, te, _ in self.seqs)
        nd = sum(table_len(tb, te, pd) for tb, te, _ in self.seqs)
        nsb = ns // 2 + 2 if share else ns + 2
        self.src = Pool(nsb, nl, no, ps, nh, hd * se, kv, seed + 10)
        self.dsts = [Pool(nd + 2 + SENTINELS, dnl, no, pd, dnh, hd * de, dkv, seed + 20 + i, poison=True)
                     for i, (dnl, dnh, dkv) in enumerate(dsts)]
        rng = np.random.default_rng(seed + 2)
        self.sids = (rng.integers(0, nsb, ns) if share else rng.permutation(nsb)[:ns]).astype(np.int32)
        self.sentinel = [list(range(nd + 2, nd + 2 + SENTINELS)) for _ in dsts]
        self.dids = []
        for p in range(len(dsts)):
            ids, do = rng.permutation(nd + 2)[:nd].astype(np.int32), 0
            for tb, te, m in self.seqs:
                b = table_len(tb, te, pd)
                if not self.routed_to_pool(m, p):
                    ids[do:do + b] = [self.sentinel[p][k % SENTINELS] for k in range(b)]
                do += b
            self.dids.append(ids)
        u = K.repage_route_units(self.seqs, ps, pd)
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

    def routed_to_pool(self, m, p):
        return any((m >> t) & 1 and tg[0] == p for t, tg in enumerate(self.targets))

    def kernel_targets(self, dids_t=None):
        dids_t = dids_t or self.dids_t
        return [K.ScatterTarget(self.dsts[p].side(dids_t[p]), self.dsts[p].nh, sb, db, k, sl, dl, c, self.done[t:].data_ptr())
                for t, (p, sl, dl, c, sb, db, k) in enumerate(self.targets)]

    def launch(self, epoch=5, value=6):
        return K.paged_repage_scatter_routed(self.src.side(self.sids_t), self.src.nh, self.ps, self.kernel_targets(), self.pd, self.seqs,
                                             self.units_t.data_ptr(), self.nu, self.lb, self.le, self.row, self.cast, self.scales, epoch,
                                             self.completion.data_ptr(), value, stream_ptr())

    def oracle_targets(self):
        return [(p, self.dids[p], self.dsts[p].kv, self.dsts[p].nh, self.dsts[p].nl, (sl, dl, c, sb, db, k))
                for p, sl, dl, c, sb, db, k in self.targets]

    def expected(self, layers=None):
        pools = [x.cpu().numpy() for x in self.initial]
        routed_oracle(self.src, self.sids, self.oracle_targets(), pools, self.no, self.ps, self.pd, self.row, self.seqs, self.cast,
                      self.scales_np, layers if layers is not None else range(self.lb, self.le))
        return pools

    def check_pools(self, want=None):
        for p, w, sent in zip(self.dsts, want or self.expected(), self.sentinel):
            got = p.buf.cpu().numpy()
            assert np.array_equal(got[sent], p.final_np[sent] ^ 0xA5), "a sentinel block was written"
            assert np.array_equal(got, w)

    def run_and_check(self, epoch=5, value=6):
        assert self.launch(epoch, value) == 0
        torch.cuda.synchronize()
        self.check_pools()
        assert self.done.tolist() == [epoch] * len(self.targets) and self.completion.item() == value

    def reset_pools(self):
        for p, x in zip(self.dsts, self.initial):
            p.buf.copy_(x)
        torch.cuda.synchronize()


def _worker_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers):
    """Prefill rank `rank`'s plan into one decode group, its ranks renumbered 0..R-1, tiled over `workers` identical workers."""
    one = tp_pp_scatter_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank)
    ranks = sorted({w.dst_rank for w in one})
    one = [ScatterWindow(ranks.index(w.dst_rank), w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin,
                         w.dst_head_begin, w.head_count) for w in one]
    return tile_scatter_plan(one, workers, len(ranks)), len(ranks)


def _masks(how, n, plan, per_worker, rng):
    """Target masks over the plan's windows: each sequence to one random worker, a random non-empty subset of windows, every
    window, or one random window."""
    nt = len(plan)
    workers = max(w.dst_rank for w in plan) // per_worker + 1
    out = []
    for _ in range(n):
        if how == "worker":
            k = int(rng.integers(0, workers))
            out.append(sum(1 << j for j, w in enumerate(plan) if w.dst_rank // per_worker == k))
        elif how == "random":
            out.append(int(rng.integers(1, 1 << nt)))
        elif how == "all":
            out.append((1 << nt) - 1)
        else:
            out.append(1 << int(rng.integers(0, nt)))
    return out


def _rig(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers, ranges, how="worker", src_kv=KV.OperationalHND,
         dst_kvs=(KV.OperationalNHD,), seed=0, **kw):
    plan, per = _worker_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers)
    rng = np.random.default_rng(seed + 1000)
    masks = _masks(how, len(ranges), plan, per, rng)
    ndst = workers * per
    dsts = [(L // dst_pp, max(1, H // dst_tp), dst_kvs[i % len(dst_kvs)]) for i in range(ndst)]
    targets = [(w.dst_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
               for w in plan]
    seqs = [(tb, te, m) for (tb, te), m in zip(ranges, masks)]
    r = RouteRig((L // src_pp, max(1, H // src_tp), src_kv), dsts, targets, seqs, seed=seed, **kw)
    r.plan, r.per_worker = plan, per
    return r


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


SMALL = [(5, 200), (40, 41), (3, 3), (17, 333)]
# (H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers): targets = workers x windows per worker
SHAPES = {
    "tp2_to_2x_tp4": (8, 2, 2, 1, 4, 1, 0, 2),          # 2 windows per worker, 4 targets
    "tp1_to_4x_tp4": (8, 2, 1, 1, 4, 1, 0, 4),          # 4 windows per worker, 16 targets
    "tp2_to_8x_tp4": (8, 2, 2, 1, 4, 1, 0, 8),          # 2 windows per worker, 16 targets
    "tp1_to_2x_tp1": (4, 2, 1, 1, 1, 1, 0, 2),          # 1 window per worker, 2 targets
}


def _sync():
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# unstreamed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("how", ["worker", "random", "onehot"])
def test_sentinel_padding_is_never_touched(how):
    """Every unrouted table position names a poisoned sentinel block; a kernel that ignores the mask writes them."""
    r = _rig(*SHAPES["tp2_to_8x_tp4"], _batch(24, 150, step=7) + SMALL, how=how, no=1, hd=32, seed=len(how))
    assert any(not r.routed_to_pool(m, p) for _, _, m in r.seqs for p in range(len(r.dsts)))
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (16, 16), (1, 16), (48, 96), (96, 48)], ids=str)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_random_masks_and_pages(shape, ps, pd):
    r = _rig(*SHAPES[shape], _mixed()[:7] + SMALL, how="random", ps=ps, pd=pd, no=1, hd=32, seed=ps + pd + len(shape))
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("cast,scaled", [(CM.FP8E4M3_TO_BF16, False), (CM.FP8E4M3_TO_BF16, True), (CM.BF16_TO_FP8E4M3, False),
                                         (CM.BF16_TO_FP8E4M3, True)], ids=["up", "up_scaled", "down", "down_scaled"])
def test_casts_and_scales(cast, scaled):
    """TP1 -> 2 workers at TP4 in four destination formats, source layers 1..3 of 4."""
    r = _rig(8, 4, 1, 1, 4, 1, 0, 2, SMALL + _batch(6, 100), how="random", src_kv=KV.OperationalNHD,
             dst_kvs=(KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD), cast=cast, scaled=scaled,
             layers=range(1, 3), seed=int(cast) + 3 * scaled)
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("rank", [0, 3], ids=["shift_ge_0", "shift_lt_0"])
def test_pp_plans(rank):
    """PP2 x TP2 prefill rank `rank` into 2 workers at PP3 x TP2: layer shifts of either sign."""
    r = _rig(4, 12, 2, 2, 2, 3, rank, 2, _batch(6, 300) + SMALL, how="worker", seed=rank + 5)
    assert len({t[2] - t[1] for t in r.targets}) > 1
    r.run_and_check()
    _sync()


def test_mla_to_8_dp_ranks_one_rank_per_sequence():
    """MLA's one 576-wide latent head; each decode DP rank owns whole sequences."""
    r = _rig(1, 3, 1, 1, 1, 1, 0, 8, SMALL + _batch(12, 300), how="worker", no=1, hd=576, ps=64, pd=64, seed=57)
    assert len(r.targets) == 8 and all(bin(m).count("1") == 1 for _, _, m in r.seqs)
    r.run_and_check()
    _sync()


def test_shared_source_blocks_across_workers():
    r = _rig(*SHAPES["tp2_to_2x_tp4"], _mixed(), how="worker", no=1, hd=32, share=True, seed=77)
    assert len(set(r.sids.tolist())) < len(r.sids)
    assert len({m for _, _, m in r.seqs}) > 1
    r.run_and_check()
    _sync()


def test_all_ones_equals_the_batch_scatter():
    r = _rig(*SHAPES["tp2_to_8x_tp4"], _mixed() + SMALL, how="all", no=1, hd=32, seed=88)
    r.run_and_check()
    routed = [p.buf.clone() for p in r.dsts]
    r.reset_pools()
    u = K.repage_batch_units([(tb, te) for tb, te, _ in r.seqs], r.ps, r.pd)
    ut = torch.from_numpy(np.ascontiguousarray(u[0]).view(np.int32).reshape(-1)).cuda()
    assert K.paged_repage_scatter_batch(r.src.side(r.sids_t), r.src.nh, r.ps, r.kernel_targets(), r.pd, [(tb, te) for tb, te, _ in r.seqs],
                                        ut.data_ptr(), len(u[0]), r.lb, r.le, r.row, r.cast, r.scales, stream=stream_ptr()) == 0
    _sync()
    assert all(torch.equal(a, p.buf) for a, p in zip(routed, r.dsts))
    _sync()


def test_one_hot_equals_one_single_target_scatter_per_sequence():
    r = _rig(*SHAPES["tp1_to_4x_tp4"], _batch(10, 130, step=13) + SMALL, how="onehot", no=1, hd=32, seed=89)
    r.run_and_check()
    routed = [p.buf.clone() for p in r.dsts]
    r.reset_pools()
    so = do = 0
    for tb, te, m in r.seqs:
        a, b = table_len(tb, te, r.ps), table_len(tb, te, r.pd)
        if a:
            t = m.bit_length() - 1
            p, sl, dl, c, sb, db, k = r.targets[t]
            s_t, d_t = r.sids_t[so:so + a], r.dids_t[p][do:do + b]
            tg = [K.ScatterTarget(r.dsts[p].side(d_t), r.dsts[p].nh, sb, db, k, sl, dl, c, None)]
            K.check(K.paged_repage_scatter(r.src.side(s_t), r.src.nh, r.ps, tg, r.pd, tb, te, r.lb, r.le, r.row, r.cast, r.scales,
                                           stream=stream_ptr()), "single scatter")
            _sync()
        so, do = so + a, do + b
    assert all(torch.equal(a, p.buf) for a, p in zip(routed, r.dsts))
    _sync()


def test_empty_batches_signal():
    r = _rig(*SHAPES["tp2_to_2x_tp4"], [(9, 9), (70, 70)], seed=4)
    for seqs in ([], [(9, 9, 1), (70, 70, 2)]):
        r.done.zero_()
        assert K.paged_repage_scatter_routed(r.src.side(r.sids_t), r.src.nh, 16, r.kernel_targets(), 64, seqs, 0, 0, 0, r.le, r.row, 0, None,
                                             7, r.completion.data_ptr(), 8, stream_ptr()) == 0
        _sync()
        assert r.done.tolist() == [7] * len(r.targets) and r.completion.item() == 8
    assert all(torch.equal(a, p.buf) for a, p in zip(r.initial, r.dsts))
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# limits
# ---------------------------------------------------------------------------------------------------------------------
def test_sixteen_targets_with_sequences_for_target_15_alone_and_256_pairs():
    dsts = [(2, 16, KV.OperationalHND if i % 2 else KV.UniversalTP) for i in range(16)]
    targets = [(i, 0, 0, 2, 0, 0, 16) for i in range(16)]
    rng = np.random.default_rng(16)
    seqs = [(tb, te, 1 << 15) for tb, te in _batch(4, 90)] + [(tb, te, int(rng.integers(1, 1 << 16))) for tb, te in _batch(4, 70, first=500)]
    r = RouteRig((2, 16, KV.OperationalNHD), dsts, targets, seqs, no=1, seed=16)
    assert sum(t[6] for t in r.targets) == 256
    r.run_and_check()
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# the streamed routed scatter, behind a producer that writes the source after the launch
# ---------------------------------------------------------------------------------------------------------------------
class StreamRoute:
    """A RouteRig whose source is written after the launch; `unstreamed` holds the pools the unstreamed routed scatter leaves."""

    def __init__(self, rig, max_ctas=MAX_CTAS, timeout_ms=10000):
        self.r, self.max_ctas, self.timeout_ms = rig, max_ctas, timeout_ms
        src = rig.src
        self.nl = src.nl
        self.want = rig.expected()
        assert rig.launch(1, 1) == 0
        _sync()
        self.unstreamed = [p.buf.clone() for p in rig.dsts]
        self.layer_done = torch.zeros(self.nl, dtype=torch.int32, device="cuda")
        self.st_done = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.ws = torch.zeros(K.sync_workspace_words(self.nl), dtype=torch.int32, device="cuda")
        self.side_stream, self.checker = torch.cuda.Stream(), torch.cuda.Stream()
        for s in (src.stream, self.checker):   # every torch kernel of the producer and the checker once
            with torch.cuda.stream(s):
                torch.cuda._sleep(100)
                for l in range(self.nl):
                    src.layer(src.buf, l).copy_(src.layer(src.final, l))
                for p in rig.dsts:
                    p.buf.copy_(p.buf)
        _sync()
        self.reset()

    def reset(self):
        r = self.r
        r.src.buf.copy_(r.src.poison)
        for p, x in zip(r.dsts, r.initial):
            p.buf.copy_(x)
        for t in (r.src.ready, self.layer_done, self.st_done, r.done, r.completion):
            t.zero_()
        _sync()

    def stream_desc(self, epoch, gate_mode, value):
        st = K.PermuteStream()
        st.layer_ready_flags[0] = self.r.src.ready.data_ptr()
        st.layer_done_flags = self.layer_done.data_ptr()
        st.done_flag = self.st_done.data_ptr()
        st.epoch = epoch & MASK
        st.sync_workspace = self.ws.data_ptr()
        st.completion_flag = self.r.completion.data_ptr()
        st.completion_value = value & MASK
        st.gate_mode = gate_mode
        st.gate_timeout_ms = self.timeout_ms
        st.max_ctas = self.max_ctas
        return st

    def launch(self, epoch, gate_mode, value):
        r = self.r
        K.check(K.paged_repage_scatter_routed_streamed(r.src.side(r.sids_t), r.src.nh, r.ps, r.kernel_targets(), r.pd, r.seqs,
                                                       r.units_t.data_ptr(), r.nu, r.lb, r.le, r.row, r.cast, r.scales,
                                                       self.stream_desc(epoch, gate_mode, value), stream_ptr(self.side_stream)),
                "streamed routed scatter")

    def rescue(self, epoch):
        """Release every flag from a fresh stream and let the launch, the producer and the checker drain."""
        s = torch.cuda.Stream()
        K.set_flags(self.r.src.ready.data_ptr(), 0, self.nl, epoch & MASK, stream_ptr(s))
        assert _finish(s) and _finish(self.side_stream), "a streamed launch is still waiting"
        for w in (self.r.src.stream, self.checker):
            if not _finish(w, 2.0):
                K.set_flags(self.layer_done.data_ptr(), 0, self.nl, epoch & MASK, stream_ptr(s))
                assert _finish(w), "a producer or checker is still waiting"
        _sync()

    def run(self, epoch, gate_mode, value):
        try:
            self.launch(epoch, gate_mode, value)
            self.r.src.produce(range(self.nl), epoch & MASK)
            assert _finish(self.side_stream) and _finish(self.r.src.stream), "the streamed routed scatter did not finish"
        finally:
            self.rescue(epoch)

    def check_end(self, epoch, value):
        r = self.r
        r.check_pools(self.want)
        for p, ref in zip(r.dsts, self.unstreamed):
            assert torch.equal(p.buf, ref)
        assert [_i32(v) for v in self.layer_done.tolist()] == [_i32(epoch) if r.lb <= l < r.le else 0 for l in range(self.nl)]
        assert r.done.tolist() == [_i32(epoch)] * len(r.targets)
        assert self.st_done.item() == _i32(epoch) and r.completion.item() == _i32(value)
        assert not self.ws.any().item(), "the workspace must be left zeroed"


SRC_KV = dict(src_kv=KV.OperationalHND)   # one layer of a source block is one contiguous run the producer writes


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("shape", ["tp2_to_8x_tp4", "pp2tp2_rank3_to_2x_pp3tp2"])
def test_streamed_layers_written_after_the_launch(gate_mode, shape):
    args = SHAPES.get(shape, (4, 12, 2, 2, 2, 3, 3, 2))
    s = StreamRoute(_rig(*args, _mixed()[:6] + SMALL, how="worker", hd=32, seed=len(shape), **SRC_KV))
    s.run(5, gate_mode, 77)
    s.check_end(5, 77)
    _sync()


@pytest.mark.parametrize("max_ctas", [1, 2, 3])
def test_spinning_batches_that_span_layers(max_ctas):
    """A handful of units per layer on 1-3 CTAs: claims of several units cross layer boundaries."""
    s = StreamRoute(_rig(8, 4, 2, 1, 4, 1, 0, 2, [(3, 70), (5, 5), (100, 180), (1, 2)], how="random", no=1, seed=90 + max_ctas, **SRC_KV),
                    max_ctas=max_ctas)
    s.run(8, K.GATE_SPIN, 5)
    s.check_end(8, 5)
    _sync()


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_only_released_layers_move(gate_mode):
    """Release k source layers, observe once layer_done[k - 1] appears: only those layers landed, for every sequence in its own
    targets, and no done flag is written."""
    s = StreamRoute(_rig(8, 4, 2, 1, 4, 1, 0, 4, SMALL + _batch(5, 200), how="worker", seed=41, **SRC_KV))
    r, k, epoch = s.r, 2, 7
    snaps = [p.buf.clone() for p in r.dsts]
    flags = [s.layer_done.clone(), r.done.clone(), s.st_done.clone()]
    with torch.cuda.stream(s.checker):
        for t, p in zip(snaps, r.dsts):
            t.copy_(p.buf)
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
    partial = r.expected(range(0, k))
    for t, want in zip(snaps, partial):
        assert np.array_equal(t.cpu().numpy(), want)
    assert flags[0].tolist() == [epoch if l < k else 0 for l in range(s.nl)]
    assert not flags[1].any().item() and flags[2].item() == 0
    _sync()


def test_a_lockstep_producer():
    """The producer waits for layer_done[l] before it writes layer l + 1 (spinning form)."""
    s = StreamRoute(_rig(*SHAPES["tp2_to_8x_tp4"], _batch(20, 64 * 3, step=17), how="worker", seed=55, **SRC_KV), max_ctas=8,
                    timeout_ms=3000)
    r, epoch = s.r, 11
    try:
        s.launch(epoch, K.GATE_SPIN, 12)
        with torch.cuda.stream(r.src.stream):
            for l in range(s.nl):
                r.src.layer(r.src.buf, l).copy_(r.src.layer(r.src.final, l))
                K.check(K.set_flags(r.src.ready.data_ptr(), l, 1, epoch, stream_ptr(r.src.stream)), "set_flags")
                K.check(K.wait_flag(s.layer_done.data_ptr() + 4 * l, epoch, stream_ptr(r.src.stream)), "wait_flag")
        assert _finish(r.src.stream) and _finish(s.side_stream), "the lockstep producer did not finish"
    finally:
        s.rescue(epoch)
    assert r.completion.item() == 12, "the gate timed out"
    s.check_end(epoch, 12)
    _sync()


def test_default_grid_leaves_the_producer_room():
    """max_ctas 0 (half the SMs) with enough units per layer for the whole default grid, next to a same-GPU producer."""
    s = StreamRoute(_rig(*SHAPES["tp2_to_8x_tp4"], _batch(40, 64 * 2, step=29), how="worker", seed=61, **SRC_KV), max_ctas=0)
    assert s.r.nu * s.r.no >= torch.cuda.get_device_properties(0).multi_processor_count // 2
    s.run(6, K.GATE_SPIN, 61)
    s.check_end(6, 61)
    _sync()


def test_a_gate_timeout_writes_no_done_flag():
    s = StreamRoute(_rig(*SHAPES["tp2_to_2x_tp4"], SMALL + _batch(3, 100), how="worker", seed=71, **SRC_KV), timeout_ms=200)
    r, epoch = s.r, 4
    try:
        s.launch(epoch, K.GATE_SPIN, 9)
        r.src.produce(range(1), epoch)
        assert _finish(s.side_stream), "the gate did not time out"
    finally:
        s.rescue(epoch)
    assert _i32(r.completion.item()) == _i32(MASK)
    assert not r.done.any().item() and s.st_done.item() == 0
    assert not s.ws.any().item()
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
                r = _rig(8, 4, 2, 1, 4, 1, 0, 2, SMALL, how="random", dst_kvs=(KV.UniversalTP, KV.OperationalHND), cast=CM(c), scaled=sc,
                         hd=64 if p else 80, ps=ps, pd=pd, seed=c + 2 * p + 4 * sc + 8 * ppow2, **SRC_KV)
                r.run_and_check()     # synchronizes before the oracle check
                s = StreamRoute(r)
                s.r.src.buf.copy_(s.r.src.final)   # the flags released before the launch
                s.r.src.ready.fill_(3)
                _sync()
                s.launch(3, K.GATE_SPIN, 5)
                assert _finish(s.side_stream)
                _sync()
                s.check_end(3, 5)
    assert _found(prof, "kvbm_paged_repage_route_kernel") == EXPECTED
    assert _found(prof, "kvbm_gated_repage_route_kernel") == EXPECTED
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# TransferManager.execute_repage_scatter_routed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=59)
    yield m
    _sync()
    m.close()


def _register(mgr, p, kv):
    cfg = LayoutConfig(p.nb, p.nl, p.no, p.page, p.nh * (p.row // 2), dtype_width_bytes=2, num_heads=p.nh)
    h = mgr.register_fully_contiguous(cfg, p.buf.data_ptr(), p.buf.numel(), StorageKind.Device, 0)
    mgr.set_kv_block_layout(h, kv)
    return h


def _managed(mgr, r):
    """Register the rig's pools; the plan (destination = pool) and the routed requests, each with its routed destinations' ids."""
    sh = _register(mgr, r.src, KV(r.src.kv))
    dhs = [_register(mgr, p, KV(p.kv)) for p in r.dsts]
    plan = [ScatterWindow(p, sl, dl, c, sb, db, k) for p, sl, dl, c, sb, db, k in r.targets]
    reqs, so, do = [], 0, 0
    for tb, te, m in r.seqs:
        a, b = table_len(tb, te, r.ps), table_len(tb, te, r.pd)
        pools = [p for p in range(len(r.dsts)) if r.routed_to_pool(m, p)]
        reqs.append((range(tb, te), [int(x) for x in r.sids[so:so + a]], {p: [int(x) for x in r.dids[p][do:do + b]] for p in pools}))
        so, do = so + a, do + b
    return sh, dhs, plan, reqs


def _routed_bytes(r):
    """What lands: each routed window's destination bytes over its layers inside the range."""
    total = 0
    for tb, te, m in r.seqs:
        for t, (p, sl, dl, c, sb, db, k) in enumerate(r.targets):
            if (m >> t) & 1:
                lo, hi = max(r.lb, sl), min(r.le, sl + c)
                total += (te - tb) * max(0, hi - lo) * r.no * k * r.dsts[p].row
    return total


def test_manager_routed(mgr):
    r = _rig(*SHAPES["tp2_to_8x_tp4"], _mixed() + SMALL, how="worker", no=1, hd=32, seed=101)
    sh, dhs, plan, reqs = _managed(mgr, r)
    flags = torch.zeros(len(dhs) + 1, dtype=torch.int32, device="cuda")
    opts = TransferOptions(done_flag=flags[len(dhs):].data_ptr(), epoch=4, per_dst_done_flags=[flags[d:].data_ptr() for d in range(len(dhs))])
    m0 = mgr.bytes_moved()
    mgr.execute_repage_scatter_routed(sh, dhs, reqs, plan, opts).wait(20.0)
    _sync()
    assert mgr.bytes_moved() - m0 == _routed_bytes(r) > 0
    r.check_pools()
    assert flags.tolist() == [4] * (len(dhs) + 1)
    _sync()


def test_manager_300_sequences_outgrow_a_staging_slot(mgr):
    r = _rig(*SHAPES["tp2_to_8x_tp4"], _batch(300, 70, step=3), how="worker", no=1, hd=32, seed=107)
    sh, dhs, plan, reqs = _managed(mgr, r)
    mgr.execute_repage_scatter_routed(sh, dhs, reqs, plan).wait(20.0)
    _sync()
    r.check_pools()
    _sync()


def test_manager_duplicates_among_routed_sequences_only(mgr):
    """A destination block named by two sequences routed to different workers is accepted (the other sequence never sends that
    destination's list); named twice among one destination's routed sequences it is KVBM_ERR_DUPLICATE_DST and nothing moves."""
    r = _rig(*SHAPES["tp1_to_2x_tp1"], [(3, 70), (100, 180), (200, 260)], how="worker", seed=103)
    r.seqs = [(3, 70, 1), (100, 180, 2), (200, 260, 1)]
    sh, dhs, plan, _ = _managed(mgr, r)
    a, b, c = (range(3, 70), [0, 1, 2, 3, 4]), (range(100, 180), [5, 6, 7, 8, 9, 10]), (range(200, 260), [11, 12, 13, 14, 15])
    ok = [a + ({0: [0, 1]},), b + ({1: [0, 1]},), c + ({0: [2, 3]},)]
    mgr.execute_repage_scatter_routed(sh, dhs, ok, plan).wait(20.0)
    _sync()
    before = [p.buf.clone() for p in r.dsts]
    dup = [a + ({0: [4, 5]},), b + ({1: [4, 5]},), c + ({0: [5, 6]},)]
    with pytest.raises(KvbmError) as e:
        mgr.execute_repage_scatter_routed(sh, dhs, dup, plan)
    assert e.value.code == ErrorCode.DUPLICATE_DST
    _sync()
    assert all(torch.equal(x, p.buf) for x, p in zip(before, r.dsts))


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_manager_streamed_routed(mgr, gate_mode):
    s = StreamRoute(_rig(*SHAPES["tp2_to_8x_tp4"], _mixed()[:5] + SMALL, how="worker", hd=32, seed=109, **SRC_KV))
    r = s.r
    sh, dhs, plan, reqs = _managed(mgr, r)
    flags = torch.zeros(len(dhs) + 1, dtype=torch.int32, device="cuda")
    opts = TransferOptions(done_flag=flags[len(dhs):].data_ptr(), epoch=4, gate_mode=gate_mode, max_ctas=MAX_CTAS,
                           per_dst_done_flags=[flags[d:].data_ptr() for d in range(len(dhs))])
    try:
        note = mgr.execute_repage_scatter_routed(sh, dhs, reqs, plan, opts, ready_flags=r.src.ready.data_ptr(),
                                                 layer_done_flags=s.layer_done.data_ptr())
        r.src.produce(range(s.nl), 4)
        note.wait(20.0)
    finally:
        s.rescue(4)
    r.check_pools(s.want)
    assert flags.tolist() == [4] * (len(dhs) + 1)
    assert s.layer_done.tolist() == [4] * s.nl
    _sync()


def test_manager_gate_timeout(mgr):
    s = StreamRoute(_rig(*SHAPES["tp2_to_2x_tp4"], SMALL, how="worker", seed=113, **SRC_KV))
    r = s.r
    sh, dhs, plan, reqs = _managed(mgr, r)
    flags = torch.zeros(len(dhs) + 1, dtype=torch.int32, device="cuda")
    opts = TransferOptions(done_flag=flags[len(dhs):].data_ptr(), epoch=6, gate_mode=K.GATE_SPIN, max_ctas=MAX_CTAS, gate_timeout_ms=200,
                           per_dst_done_flags=[flags[d:].data_ptr() for d in range(len(dhs))])
    try:
        note = mgr.execute_repage_scatter_routed(sh, dhs, reqs, plan, opts, ready_flags=r.src.ready.data_ptr())
        r.src.produce(range(1), 6)
        with pytest.raises(KvbmError) as e:
            note.wait(20.0)
        assert e.value.code == ErrorCode.TIMEOUT
    finally:
        s.rescue(6)
    assert not flags.any().item()
    _sync()

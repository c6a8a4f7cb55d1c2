"""GPU parity of routed re-paging between pages that need not divide (each sequence of a batch pushed to, or pulled from, its own
workers in one launch, for any two page sizes): kvbm_kernels_paged_repage_scatter_routed_anypage,
kvbm_kernels_paged_stage_repage_gather_routed_anypage, their streamed forms and TransferManager.execute_repage_scatter_routed_anypage /
execute_repage_batch_routed_anypage.  The rigs are the routed scatter's and the routed gather's (tests/test_gpu_scatter_route.py,
tests/test_gpu_gather_route.py) with the unit table of kvbm_kernels_repage_route_anypage_units, which has the routed helper's counts:
poisoned destination pools compared whole with the per-sequence routed oracles (tests/scatter_oracle.py and
tests/stage_repage_oracle.py, which place token p at slot p % P of block table[p // P] for any page P), and at every unrouted table
position a sentinel block that must never be written (push) or read (pull).  One streamed launch runs at a time; every test ends
with a device synchronize."""
from unittest import mock

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import ScatterWindow, ShardWindow, TransferManager, TransferOptions
from tests.gpu_util import stream_ptr
from tests.scatter_batch_oracle import table_len
from tests.test_gpu_gather_route import GatherRig, StreamGather, _plan
from tests.test_gpu_gather_route import _managed as _managed_gather
from tests.test_gpu_gather_route import _masks as _gather_masks
from tests.test_gpu_gather_route import _register as _register_gather_pool
from tests.test_gpu_gather_route import _routed_bytes as _gather_bytes
from tests.test_gpu_reroute_limits import _as_destination, _as_source, _check_filled, _into_big_rows
from tests.test_gpu_scatter_route import (GATE_IDS, GATES, MASK, MAX_CTAS, SMALL, RouteRig, StreamRoute, _batch, _finish, _found, _i32,
                                          _mixed, _worker_plan)
from tests.test_gpu_scatter_route import _managed as _managed_route
from tests.test_gpu_scatter_route import _masks as _scatter_masks
from tests.test_gpu_scatter_route import _register as _register_pool
from tests.test_gpu_scatter_route import _routed_bytes as _scatter_bytes
from tests.test_gpu_transform_limits import BHD, BNH, BNL, BNO, BNT, big_pool  # noqa: F401  (big_pool: the fixture)

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
NHD, HND, UTP, UPP = KV.OperationalNHD, KV.OperationalHND, KV.UniversalTP, KV.UniversalPP
SRC_KV = dict(src_kv=HND)   # one layer of a source block is one contiguous run the producer writes


def _sync():
    torch.cuda.synchronize()


def _dev(x):
    x = np.ascontiguousarray(x)
    return torch.from_numpy(x.view(np.int32).reshape(-1) if len(x) else np.zeros(1, np.int32)).cuda()


def _anypage_helper():
    """The rigs build their unit table with K.repage_route_units; here it is the routed anypage helper's (same counts)."""
    return mock.patch.object(K, "repage_route_units", K.repage_route_anypage_units)


class DealRig(RouteRig):
    """RouteRig over the routed anypage scatter."""

    def __init__(self, *a, **kw):
        with _anypage_helper():
            super().__init__(*a, **kw)

    def launch(self, epoch=5, value=6):
        return K.paged_repage_scatter_routed_anypage(self.src.side(self.sids_t), self.src.nh, self.ps, self.kernel_targets(), self.pd,
                                                     self.seqs, self.units_t.data_ptr(), self.nu, self.lb, self.le, self.row, self.cast,
                                                     self.scales, epoch, self.completion.data_ptr(), value, stream_ptr())


class CollectRig(GatherRig):
    """GatherRig over the routed anypage gather."""

    def __init__(self, *a, **kw):
        with _anypage_helper():
            super().__init__(*a, **kw)

    def launch(self, epoch=5, value=6):
        return K.paged_stage_repage_gather_routed_anypage(*self.args(), self.done.data_ptr(), epoch, self.completion.data_ptr(), value,
                                                          stream_ptr())


class StreamDeal(StreamRoute):
    def launch(self, epoch, gate_mode, value):
        r = self.r
        K.check(K.paged_repage_scatter_routed_anypage_streamed(r.src.side(r.sids_t), r.src.nh, r.ps, r.kernel_targets(), r.pd, r.seqs,
                                                               r.units_t.data_ptr(), r.nu, r.lb, r.le, r.row, r.cast, r.scales,
                                                               self.stream_desc(epoch, gate_mode, value), stream_ptr(self.side_stream)),
                "streamed routed anypage scatter")


class StreamCollect(StreamGather):
    def launch(self, epoch, gate_mode, value):
        K.check(K.paged_stage_repage_gather_routed_anypage_streamed(*self.r.args(), self.stream_desc(epoch, gate_mode, value),
                                                                    stream_ptr(self.side_stream)), "streamed routed anypage gather")


def deal_rig(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers, ranges, how="worker", src_kv=HND, dst_kvs=(NHD,), seed=0, **kw):
    """tests/test_gpu_scatter_route._rig over DealRig: prefill rank `rank`'s plan tiled over `workers` decode workers."""
    plan, per = _worker_plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers)
    masks = _scatter_masks(how, len(ranges), plan, per, np.random.default_rng(seed + 1000))
    dsts = [(L // dst_pp, max(1, H // dst_tp), dst_kvs[i % len(dst_kvs)]) for i in range(workers * per)]
    targets = [(w.dst_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
               for w in plan]
    r = DealRig((L // src_pp, max(1, H // src_tp), src_kv), dsts, targets, [(tb, te, m) for (tb, te), m in zip(ranges, masks)], seed=seed,
                **kw)
    r.plan, r.per_worker = plan, per
    return r


def collect_rig(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers, ranges, how="worker", src_kv=HND, dst_kv=NHD, seed=0, **kw):
    """tests/test_gpu_gather_route._rig over CollectRig: decode rank `rank`'s plan from `workers` prefill workers."""
    plan, per = _plan(H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers)
    masks = _gather_masks(how, len(ranges), workers * per, per, np.random.default_rng(seed + 1000))
    pools = [(L // src_pp, max(1, H // src_tp), src_kv)] * (workers * per)
    windows = [(w.src_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan]
    r = CollectRig(pools, windows, (L // dst_pp, max(1, H // dst_tp), dst_kv), [(tb, te, m) for (tb, te), m in zip(ranges, masks)],
                   seed=seed, **kw)
    r.plan, r.per_worker = plan, per
    return r


def edge_ranges(ps, pd):
    """Ranges that start and end inside blocks on both sides, one token, an empty range, one from 0, and longer ones."""
    big, small = max(ps, pd), min(ps, pd)
    return [(big // 2 + 1, 3 * big + small // 2 + 1), (5 * big - 1, 5 * big), (7, 7), (small + 1, 2 * big + 3), (0, big + small + 1),
            (6 * big + 2, 9 * big - 1), (2 * big + 5, 4 * big + small - 2)]


# (H, L, src_tp, src_pp, dst_tp, dst_pp, rank, workers) -- push: prefill rank into decode workers; pull: decode rank from prefill workers
PUSH = {"tp2_to_2x_tp16": (8, 2, 2, 1, 16, 1, 0, 2), "tp1_to_2x_tp8": (8, 2, 1, 1, 8, 1, 0, 2), "tp2_to_8x_tp4": (8, 2, 2, 1, 4, 1, 0, 8)}
PULL = {"4x_tp4_to_tp2": (8, 2, 4, 1, 2, 1, 0, 4), "2x_tp8_to_tp1": (8, 2, 8, 1, 1, 1, 0, 2), "tp4_to_tp1": (8, 2, 4, 1, 1, 1, 0, 1)}
PAIRS = [(3, 5), (5, 3), (24, 16), (16, 24), (48, 64), (64, 48), (544, 64), (64, 544)]
HOWS = ["worker", "random", "onehot"]


def _has_phase(r):
    return bool((r.units_np[:, 3] >> 16).any())


# ---------------------------------------------------------------------------------------------------------------------
# the push against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ps,pd", PAIRS, ids=str)
@pytest.mark.parametrize("shape", list(PUSH))
def test_push_pages_plans_and_masks(shape, ps, pd):
    """Every pair under the TP plans, masks cycling worker / random / one-hot; unrouted positions name poisoned sentinels."""
    how = HOWS[(ps + pd + len(shape)) % 3]
    r = deal_rig(*PUSH[shape], edge_ranges(ps, pd), how=how, ps=ps, pd=pd, no=1, hd=32, seed=ps + 3 * pd + len(shape))
    assert _has_phase(r) and any(not r.routed_to_pool(m, p) for _, _, m in r.seqs for p in range(len(r.dsts)))
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("rank", [0, 3], ids=["shift_ge_0", "shift_lt_0"])
def test_push_pp_plans(rank):
    """PP2 x TP2 prefill rank `rank` into 2 workers at PP3 x TP2, 48 -> 64."""
    r = deal_rig(4, 12, 2, 2, 2, 3, rank, 2, _batch(6, 300) + SMALL, ps=48, pd=64, seed=rank + 5)
    assert len({t[2] - t[1] for t in r.targets}) > 1
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("hd", [64, 80, 96])
@pytest.mark.parametrize("cast,scaled", [(CM.NONE, False), (CM.FP8E4M3_TO_BF16, False), (CM.FP8E4M3_TO_BF16, True), (CM.BF16_TO_FP8E4M3, False),
                                         (CM.BF16_TO_FP8E4M3, True)], ids=["none", "up", "up_scaled", "down", "down_scaled"])
def test_push_casts_scales_and_head_dims(cast, scaled, hd):
    for layers, (ps, pd) in ((None, (24, 16)), (range(1, 3), (48, 64))):
        r = deal_rig(8, 4, 1, 1, 4, 1, 0, 2, SMALL + _batch(4, 100), how="random", src_kv=NHD, dst_kvs=(UTP, UPP, HND, NHD), cast=cast,
                     scaled=scaled, layers=layers, hd=hd, ps=ps, pd=pd, seed=int(cast) + 3 * scaled + hd)
        r.run_and_check()
    _sync()


@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16], ids=lambda c: c.name)
def test_push_mla_to_8_dp_ranks(cast):
    """MLA's one 576-wide latent head from 544-token blocks to 8 DP ranks of 64-token pages, each rank owning whole sequences."""
    r = deal_rig(1, 2, 1, 1, 1, 1, 0, 8, SMALL + _batch(8, 700, step=97), ps=544, pd=64, no=1, hd=576, cast=cast, seed=57)
    assert len(r.targets) == 8 and all(bin(m).count("1") == 1 for _, _, m in r.seqs)
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("ps,pd", [(544, 64), (48, 64)], ids=str)
def test_push_shared_source_blocks(ps, pd):
    r = deal_rig(*PUSH["tp2_to_8x_tp4"], _mixed(), ps=ps, pd=pd, no=1, hd=32, share=True, seed=77 + ps)
    assert len(set(r.sids.tolist())) < len(r.sids)
    r.run_and_check()
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# the pull against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ps,pd", PAIRS, ids=str)
@pytest.mark.parametrize("shape", list(PULL))
def test_pull_pages_plans_and_masks(shape, ps, pd):
    how = "random" if shape == "tp4_to_tp1" else "worker"
    r = collect_rig(*PULL[shape], edge_ranges(ps, pd), how=how, ps=ps, pd=pd, no=1, hd=32, seed=ps + 3 * pd + len(shape))
    assert _has_phase(r) and any(m != (1 << len(r.srcs)) - 1 for _, _, m in r.seqs)
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("rank", [2, 4], ids=["two_stages", "one_stage"])
def test_pull_pp_workers_tiled(rank):
    r = collect_rig(4, 12, 2, 2, 2, 3, rank, 2, _batch(6, 300) + SMALL, ps=64, pd=48, seed=rank + 5)
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("hd", [64, 80, 96])
@pytest.mark.parametrize("cast,scaled", [(CM.NONE, False), (CM.FP8E4M3_TO_BF16, False), (CM.FP8E4M3_TO_BF16, True), (CM.BF16_TO_FP8E4M3, False),
                                         (CM.BF16_TO_FP8E4M3, True)], ids=["none", "up", "up_scaled", "down", "down_scaled"])
def test_pull_casts_scales_and_head_dims(cast, scaled, hd):
    for layers, (ps, pd) in ((None, (16, 24)), (range(1, 3), (64, 48))):
        r = collect_rig(8, 4, 4, 1, 2, 1, 0, 2, SMALL + _batch(4, 100), src_kv=NHD, dst_kv=UTP, cast=cast, scaled=scaled, layers=layers,
                        hd=hd, ps=ps, pd=pd, seed=int(cast) + 3 * scaled + hd)
        r.run_and_check()
    _sync()


@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16], ids=lambda c: c.name)
def test_pull_mla_from_8_dp_workers(cast):
    """MLA's latent head from 8 DP prefill workers of 544-token blocks into 64-token pages, each sequence from one worker."""
    r = collect_rig(1, 2, 1, 1, 1, 1, 0, 8, SMALL + _batch(8, 700, step=97), ps=544, pd=64, no=1, hd=576, cast=cast, seed=58)
    assert len(r.windows) == 8
    r.run_and_check()
    _sync()


@pytest.mark.parametrize("ps,pd", [(544, 64), (48, 64)], ids=str)
def test_pull_shared_source_blocks(ps, pd):
    r = collect_rig(*PULL["4x_tp4_to_tp2"], _batch(60, 170, step=7), ps=ps, pd=pd, no=1, hd=32, share=True, seed=78 + ps)
    r.run_and_check()
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# the three equivalences, byte for byte
# ---------------------------------------------------------------------------------------------------------------------
def test_push_all_ones_is_the_anypage_scatter():
    r = deal_rig(*PUSH["tp2_to_8x_tp4"], _mixed() + SMALL, how="all", ps=544, pd=64, no=1, hd=32, seed=88)
    r.run_and_check()
    routed = [p.buf.clone() for p in r.dsts]
    r.reset_pools()
    seqs = [(tb, te) for tb, te, _ in r.seqs]
    u = K.repage_anypage_units(seqs, r.ps, r.pd)
    ut = _dev(u[0])
    assert K.paged_repage_scatter_anypage(r.src.side(r.sids_t), r.src.nh, r.ps, r.kernel_targets(), r.pd, seqs, ut.data_ptr(), len(u[0]),
                                          r.lb, r.le, r.row, r.cast, r.scales, stream=stream_ptr()) == 0
    _sync()
    assert all(torch.equal(a, p.buf) for a, p in zip(routed, r.dsts))
    _sync()


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (16, 16)], ids=str)
def test_push_dividing_pages_are_the_routed_scatter(ps, pd):
    r = deal_rig(*PUSH["tp2_to_2x_tp16"], _mixed()[:6] + SMALL, how="random", ps=ps, pd=pd, no=1, hd=32, cast=CM.FP8E4M3_TO_BF16,
                 scaled=True, seed=ps * pd)
    r.run_and_check()
    routed = [p.buf.clone() for p in r.dsts]
    r.reset_pools()
    u = K.repage_route_units(r.seqs, ps, pd)
    assert u[0].tobytes() == r.units_np.tobytes()
    ut = _dev(u[0])
    assert K.paged_repage_scatter_routed(r.src.side(r.sids_t), r.src.nh, ps, r.kernel_targets(), pd, r.seqs, ut.data_ptr(), len(u[0]),
                                         r.lb, r.le, r.row, r.cast, r.scales, stream=stream_ptr()) == 0
    _sync()
    assert all(torch.equal(a, p.buf) for a, p in zip(routed, r.dsts))
    _sync()


def _spans(r):
    out, so, do = [], 0, 0
    for tb, te, _ in r.seqs:
        a, b = table_len(tb, te, r.ps), table_len(tb, te, r.pd)
        out.append((so, a, do, b))
        so, do = so + a, do + b
    return out


@pytest.mark.parametrize("ps,pd", [(24, 16), (544, 64)], ids=str)
def test_push_one_worker_per_sequence_is_one_anypage_scatter_per_worker(ps, pd):
    r = deal_rig(*PUSH["tp1_to_2x_tp8"], _batch(10, 130, step=13) + SMALL, how="worker", ps=ps, pd=pd, no=1, hd=32, seed=89)
    r.run_and_check()
    routed = [p.buf.clone() for p in r.dsts]
    r.reset_pools()
    spans, per = _spans(r), r.per_worker
    for k in range(len(r.dsts) // per):
        idx = [i for i, (_, _, m) in enumerate(r.seqs) if r.routed_to_pool(m, k * per)]
        if not idx:
            continue
        seqs = [r.seqs[i][:2] for i in idx]
        sid = _dev(np.concatenate([r.sids[spans[i][0]:spans[i][0] + spans[i][1]] for i in idx]).astype(np.int32))
        dids = [_dev(np.concatenate([r.dids[p][spans[i][2]:spans[i][2] + spans[i][3]] for i in idx]).astype(np.int32))
                for p in range(len(r.dsts))]
        tg = [t for t, x in zip(r.kernel_targets(dids), r.targets) if x[0] // per == k]
        u = K.repage_anypage_units(seqs, ps, pd)
        ut = _dev(u[0])
        K.check(K.paged_repage_scatter_anypage(r.src.side(sid), r.src.nh, ps, tg, pd, seqs, ut.data_ptr(), len(u[0]), r.lb, r.le, r.row,
                                               r.cast, r.scales, stream=stream_ptr()), "per-worker anypage scatter")
        _sync()
    assert all(torch.equal(a, p.buf) for a, p in zip(routed, r.dsts))
    _sync()


def test_pull_all_ones_is_the_anypage_gather():
    r = collect_rig(*PULL["tp4_to_tp1"], _mixed() + SMALL, how="all", ps=544, pd=64, no=1, hd=32, seed=88)
    r.run_and_check()
    routed = r.dst.buf.clone()
    r.reset()
    seqs = [(tb, te) for tb, te, _ in r.seqs]
    u = K.repage_anypage_units(seqs, r.ps, r.pd)
    ut = _dev(u[0])
    assert K.paged_stage_repage_gather_anypage(r.sources(), r.ps, r.dst.side(r.dids_t), r.dst.nh, r.pd, seqs, ut.data_ptr(), len(u[0]),
                                               r.lb, r.le, r.row, r.cast, r.scales, stream=stream_ptr()) == 0
    _sync()
    assert torch.equal(routed, r.dst.buf)
    _sync()


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (16, 16)], ids=str)
def test_pull_dividing_pages_are_the_routed_gather(ps, pd):
    r = collect_rig(*PULL["4x_tp4_to_tp2"], _mixed()[:6] + SMALL, ps=ps, pd=pd, no=1, hd=32, cast=CM.FP8E4M3_TO_BF16, scaled=True,
                    seed=ps * pd)
    r.run_and_check()
    routed = r.dst.buf.clone()
    r.reset()
    u = K.repage_route_units(r.kseqs, ps, pd)
    assert u[0].tobytes() == r.units_np.tobytes()
    ut = _dev(u[0])
    args = list(r.args())
    args[6] = ut.data_ptr()
    assert K.paged_stage_repage_gather_routed(*args, stream=stream_ptr()) == 0
    _sync()
    assert torch.equal(routed, r.dst.buf)
    _sync()


@pytest.mark.parametrize("ps,pd", [(16, 24), (544, 64)], ids=str)
def test_pull_one_worker_per_sequence_is_one_anypage_gather_per_worker(ps, pd):
    r = collect_rig(*PULL["2x_tp8_to_tp1"], _batch(10, 130, step=13) + SMALL, ps=ps, pd=pd, no=1, hd=32, seed=89)
    r.run_and_check()
    routed = r.dst.buf.clone()
    r.reset()
    spans, per = _spans(r), r.per_worker
    for k in range(len(r.srcs) // per):
        idx = [i for i, (_, _, m) in enumerate(r.seqs) if (m >> (k * per)) & 1]
        if not idx:
            continue
        seqs = [r.seqs[i][:2] for i in idx]
        ids = [_dev(np.concatenate([r.sids[p][spans[i][0]:spans[i][0] + spans[i][1]] for i in idx]).astype(np.int32))
               for p in range(len(r.srcs))]
        did = _dev(np.concatenate([r.dids[spans[i][2]:spans[i][2] + spans[i][3]] for i in idx]).astype(np.int32))
        u = K.repage_anypage_units(seqs, ps, pd)
        ut = _dev(u[0])
        wins = [w for w in r.windows if w[0] // per == k]
        K.check(K.paged_stage_repage_gather_anypage(r.sources(ids, wins), ps, r.dst.side(did), r.dst.nh, pd, seqs, ut.data_ptr(), len(u[0]),
                                                    r.lb, r.le, r.row, r.cast, r.scales, stream=stream_ptr()), "per-worker anypage gather")
        _sync()
    assert torch.equal(routed, r.dst.buf)
    _sync()


def test_empty_batches_signal():
    r = deal_rig(*PUSH["tp1_to_2x_tp8"], [(9, 9), (70, 70)], ps=24, pd=16, seed=4)
    g = collect_rig(*PULL["4x_tp4_to_tp2"], [(9, 9), (70, 70)], ps=24, pd=16, seed=4)
    for seqs in ([], [(9, 9, 1), (70, 70, 2)]):
        r.done.zero_()
        g.done.zero_()
        assert K.paged_repage_scatter_routed_anypage(r.src.side(r.sids_t), r.src.nh, 24, r.kernel_targets(), 16, seqs, 0, 0, 0, r.le, r.row,
                                                     0, None, 7, r.completion.data_ptr(), 8, stream_ptr()) == 0
        assert K.paged_stage_repage_gather_routed_anypage(g.sources(), 24, g.dst.side(g.dids_t), g.dst.nh, 16, seqs, 0, 0, 0, g.le, g.row, 0,
                                                          None, g.done.data_ptr(), 7, g.completion.data_ptr(), 8, stream_ptr()) == 0
        _sync()
        assert r.done.tolist() == [7] * len(r.targets) and r.completion.item() == 8
        assert g.done.item() == 7 and g.completion.item() == 8
    assert all(torch.equal(a, p.buf) for a, p in zip(r.initial, r.dsts)) and torch.equal(g.initial, g.dst.buf)
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# every instantiation of the four families, reached under the profiler
# ---------------------------------------------------------------------------------------------------------------------
WALKS = {(c, p, s) for c in (0, 1, 2) for p in (True, False) for s in ((False,) if c == 0 else (False, True))}
EXPECTED = {w + (pp,) for w in WALKS for pp in (True, False)}


def test_every_instantiation():
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c, p, sc in sorted(WALKS):
            for ppow2 in (True, False):
                ps, pd = (16, 24) if ppow2 else (40, 24)
                kw = dict(cast=CM(c), scaled=sc, hd=64 if p else 80, seed=c + 2 * p + 4 * sc + 8 * ppow2)
                r = deal_rig(8, 4, 2, 1, 4, 1, 0, 2, SMALL, how="random", dst_kvs=(UTP, HND), ps=ps, pd=pd, **kw, **SRC_KV)
                r.run_and_check()
                s = StreamDeal(r)
                s.r.src.buf.copy_(s.r.src.final)   # the flags released before the launch
                s.r.src.ready.fill_(3)
                _sync()
                s.launch(3, K.GATE_SPIN, 5)
                assert _finish(s.side_stream)
                _sync()
                s.check_end(3, 5)
                g = collect_rig(8, 4, 4, 1, 2, 1, 0, 2, SMALL, dst_kv=UTP, ps=pd, pd=ps, **kw, **SRC_KV)
                g.run_and_check()
                t = StreamCollect(g)
                for x in g.srcs:
                    x.buf.copy_(x.final)
                    x.ready.fill_(3)
                _sync()
                t.launch(3, K.GATE_SPIN, 5)
                assert _finish(t.side_stream)
                _sync()
                t.check_end(3, 5)
    for family in ("kvbm_paged_repage_deal_kernel", "kvbm_gated_repage_deal_kernel", "kvbm_paged_repage_collect_kernel",
                   "kvbm_gated_repage_collect_kernel"):
        assert _found(prof, family) == EXPECTED, family
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# streamed, behind a producer that writes the sources after the launch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("ps,pd", [(544, 64), (16, 24)], ids=str)
def test_push_streamed_behind_a_late_producer(gate_mode, ps, pd):
    s = StreamDeal(deal_rig(4, 12, 2, 2, 2, 3, 3, 2, _mixed()[:5] + SMALL, ps=ps, pd=pd, hd=32, no=1, cast=CM.FP8E4M3_TO_BF16, scaled=True,
                            seed=ps + pd, **SRC_KV))
    s.run(5, gate_mode, 77)
    s.check_end(5, 77)
    _sync()


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("ps,pd", [(544, 64), (24, 16)], ids=str)
def test_pull_streamed_behind_a_late_producer(gate_mode, ps, pd):
    s = StreamCollect(collect_rig(4, 12, 2, 2, 2, 3, 3, 2, _mixed()[:5] + SMALL, ps=ps, pd=pd, hd=32, no=1, cast=CM.FP8E4M3_TO_BF16,
                                  scaled=True, seed=ps + pd, **SRC_KV))
    s.run(5, gate_mode, 77)
    s.check_end(5, 77)
    _sync()


@pytest.mark.parametrize("max_ctas", [1, 2, 3])
def test_spinning_batches_that_span_layers(max_ctas):
    """A handful of units per layer on 1-3 CTAs: claims of several units cross layer boundaries, push and pull."""
    ranges = [(3, 70), (5, 5), (100, 180), (1, 2)]
    s = StreamDeal(deal_rig(8, 4, 2, 1, 4, 1, 0, 2, ranges, ps=24, pd=16, no=1, seed=90 + max_ctas, **SRC_KV), max_ctas=max_ctas)
    s.run(8, K.GATE_SPIN, 5)
    s.check_end(8, 5)
    t = StreamCollect(collect_rig(8, 4, 4, 1, 2, 1, 0, 2, ranges, ps=16, pd=24, no=1, seed=90 + max_ctas, **SRC_KV), max_ctas=max_ctas)
    t.run(8, K.GATE_SPIN, 5)
    t.check_end(8, 5)
    _sync()


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_push_only_released_layers_move(gate_mode):
    """Release k source layers, observe once layer_done[k - 1] appears: only those layers landed, for every routed sequence, and no
    done flag is written."""
    from tests.test_gpu_scatter_route import CHECKER_SLEEP
    s = StreamDeal(deal_rig(8, 4, 2, 1, 4, 1, 0, 2, SMALL + edge_ranges(48, 64), ps=48, pd=64, seed=41, **SRC_KV))
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
    for t, want in zip(snaps, r.expected(range(0, k))):
        assert np.array_equal(t.cpu().numpy(), want)
    assert flags[0].tolist() == [epoch if l < k else 0 for l in range(s.nl)]
    assert not flags[1].any().item() and flags[2].item() == 0
    _sync()


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_pull_only_released_layers_move(gate_mode):
    s = StreamCollect(collect_rig(8, 4, 4, 1, 2, 1, 0, 2, SMALL + edge_ranges(64, 48), ps=64, pd=48, seed=41, **SRC_KV))
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


def test_a_gate_timeout_writes_no_done_flag():
    s = StreamDeal(deal_rig(8, 4, 2, 1, 4, 1, 0, 2, SMALL + _batch(3, 100), ps=24, pd=16, seed=71, **SRC_KV), timeout_ms=200)
    r, epoch = s.r, 4
    try:
        s.launch(epoch, K.GATE_SPIN, 9)
        r.src.produce(range(1), epoch)
        assert _finish(s.side_stream), "the gate did not time out"
    finally:
        s.rescue(epoch)
    assert _i32(r.completion.item()) == _i32(MASK) and not r.done.any().item() and s.st_done.item() == 0
    assert not s.ws.any().item()
    t = StreamCollect(collect_rig(*PULL["4x_tp4_to_tp2"], SMALL + _batch(3, 100), ps=16, pd=24, seed=71, **SRC_KV), timeout_ms=200)
    g = t.r
    try:
        t.launch(epoch, K.GATE_SPIN, 9)
        t.produce(range(1), epoch)
        assert _finish(t.side_stream), "the gate did not time out"
    finally:
        t.rescue(epoch)
    assert _i32(g.completion.item()) == _i32(MASK) and g.done.item() == 0
    assert not t.ws.any().item()
    _sync()


@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_an_unrouted_source_is_never_waited_on(gate_mode):
    """Worker 1's sources are named by no sequence and their ready flags, in mapped pinned host memory, are never released by the
    producer; the host waits with a deadline and only then releases them, so a build that waits on them fails instead of hanging."""
    ranges = SMALL + _batch(6, 150)
    r = collect_rig(*PULL["4x_tp4_to_tp2"], ranges, ps=48, pd=64, seed=31, **SRC_KV)
    per = r.per_worker
    r2 = CollectRig([(p.nl, p.nh, p.kv) for p in r.srcs], r.windows, (r.dst.nl, r.dst.nh, r.dst.kv),
                    [(tb, te, ((1 << per) - 1) << (per * (0 if i % 2 else 2))) for i, (tb, te) in enumerate(ranges)], ps=48, pd=64, hd=64,
                    seed=31)
    idle = [p for p in range(len(r2.srcs)) if not any((m >> p) & 1 for _, _, m in r2.seqs)]
    assert idle
    host = torch.zeros((len(idle), r2.dst.nl + 1), dtype=torch.int32).pin_memory()
    s = StreamCollect(r2, flags={p: host[i].data_ptr() for i, p in enumerate(idle)})
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


def test_producers_enqueued_first_and_from_their_own_thread():
    """The producer's work is enqueued before the streamed launch, and from a thread of its own while the launch is enqueued
    (stream-wait form), so no enqueue order of many stream-wait launches can hold the producer back."""
    import threading
    for order in ("producer_first", "producer_thread"):
        s = StreamDeal(deal_rig(8, 4, 2, 1, 4, 1, 0, 2, _mixed()[:4] + SMALL, ps=544, pd=64, no=1, hd=32, seed=97, **SRC_KV))
        epoch = 6
        try:
            if order == "producer_first":
                s.r.src.produce(range(s.nl), epoch)
                s.launch(epoch, K.GATE_STREAM_WAIT, 12)
            else:
                th = threading.Thread(target=lambda: s.r.src.produce(range(s.nl), epoch))
                th.start()
                s.launch(epoch, K.GATE_STREAM_WAIT, 12)
                th.join()
            assert _finish(s.side_stream) and _finish(s.r.src.stream)
        finally:
            s.rescue(epoch)
        s.check_end(epoch, 12)
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# the manager
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=71)
    yield m
    _sync()
    m.close()


@pytest.mark.parametrize("streamed", [False, True], ids=["unstreamed", "streamed"])
@pytest.mark.parametrize("ps,pd", [(544, 64), (24, 64)], ids=str)
def test_manager_push(mgr, streamed, ps, pd):
    r = deal_rig(*PUSH["tp2_to_8x_tp4"], _mixed()[:5] + SMALL, ps=ps, pd=pd, no=1, hd=32, seed=101 + ps, **SRC_KV)
    s = StreamDeal(r) if streamed else None
    sh, dhs, plan, reqs = _managed_route(mgr, r)
    flags = torch.zeros(len(dhs) + 1, dtype=torch.int32, device="cuda")
    kw = dict(done_flag=flags[len(dhs):].data_ptr(), epoch=4, per_dst_done_flags=[flags[d:].data_ptr() for d in range(len(dhs))])
    m0 = mgr.bytes_moved()
    if streamed:
        try:
            note = mgr.execute_repage_scatter_routed_anypage(sh, dhs, reqs, plan, TransferOptions(gate_mode=K.GATE_SPIN, max_ctas=MAX_CTAS, **kw),
                                                             ready_flags=r.src.ready.data_ptr(), layer_done_flags=s.layer_done.data_ptr())
            r.src.produce(range(s.nl), 4)
            note.wait(20.0)
        finally:
            s.rescue(4)
        assert s.layer_done.tolist() == [4] * s.nl
    else:
        mgr.execute_repage_scatter_routed_anypage(sh, dhs, reqs, plan, TransferOptions(**kw)).wait(20.0)
    _sync()
    assert mgr.bytes_moved() - m0 == _scatter_bytes(r) > 0
    r.check_pools(s.want if streamed else None)
    assert flags.tolist() == [4] * (len(dhs) + 1)
    _sync()


@pytest.mark.parametrize("streamed", [False, True], ids=["unstreamed", "streamed"])
@pytest.mark.parametrize("ps,pd", [(544, 64), (64, 24)], ids=str)
def test_manager_pull(mgr, streamed, ps, pd):
    r = collect_rig(*PULL["4x_tp4_to_tp2"], _mixed()[:5] + SMALL, ps=ps, pd=pd, no=1, hd=32, seed=102 + ps, **SRC_KV)
    s = StreamCollect(r) if streamed else None
    sources, dh, plan, reqs = _managed_gather(mgr, r)
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    m0 = mgr.bytes_moved()
    if streamed:
        opts = TransferOptions(done_flag=flag.data_ptr(), epoch=4, gate_mode=K.GATE_STREAM_WAIT, max_ctas=MAX_CTAS)
        try:
            note = mgr.execute_repage_batch_routed_anypage(sources, dh, reqs, plan, opts,
                                                           ready_flags={p: x.ready.data_ptr() for p, x in enumerate(r.srcs)},
                                                           layer_done_flags=s.layer_done.data_ptr())
            s.produce(range(r.dst.nl), 4)
            note.wait(20.0)
        finally:
            s.rescue(4)
        assert s.layer_done.tolist() == [4] * s.nl
    else:
        mgr.execute_repage_batch_routed_anypage(sources, dh, reqs, plan, TransferOptions(done_flag=flag.data_ptr(), epoch=4)).wait(20.0)
    _sync()
    assert mgr.bytes_moved() - m0 == _gather_bytes(r) > 0
    r.check_pool(s.want if streamed else None)
    assert flag.item() == 4
    _sync()


HIGH_MASKS = [1 << 15, 1 << 15, 1, 0xFFFF, 0x8001, 0x00F0, 1 << 15, 0x7FFF]


def _phase_ranges(big, small, n):
    """n ranges, each starting on a big block whose phase is nonzero."""
    out, j = [], 1
    while len(out) < n:
        if (j * big) % small:
            out.append((j * big + 1, j * big + big + small // 2))
        j += 3
    return out


@pytest.mark.parametrize("streamed", [False, True], ids=["unstreamed", "streamed"])
def test_manager_push_to_ranks_16_to_31_with_a_phase(mgr, streamed):
    """32 destinations, windows writing 16-31 only, several sequences to rank 31 alone, 24 -> 16: the window mask (bits 0-15) and
    the phase share each record's fourth word.  Destinations 0-15 keep their bytes."""
    dsts = [(2, 1, (NHD, UTP)[p % 2]) for p in range(16)]
    targets = [(p, 0, 0, 2, p, 0, 1) for p in range(16)]
    seqs = [(tb, te, m) for (tb, te), m in zip(_phase_ranges(24, 16, len(HIGH_MASKS)), HIGH_MASKS)]
    r = DealRig((2, 16, HND), dsts, targets, seqs, ps=24, pd=16, no=1, hd=32, seed=32)
    assert _has_phase(r) and (r.units_np[:, 3] & 0xFFFF).max() == 0xFFFF
    s = StreamDeal(r) if streamed else None
    idle = [DealRig((2, 1, HND), [(2, 1, NHD)], [(0, 0, 0, 2, 0, 0, 1)], [(0, 1, 1)], ps=24, pd=16, no=1, hd=32, seed=40 + k).dsts[0]
            for k in range(16)]
    idle0 = [p.buf.clone() for p in idle]
    sh = _register_pool(mgr, r.src, KV(r.src.kv))
    dhs = [_register_pool(mgr, p, KV(p.kv)) for p in idle] + [_register_pool(mgr, p, KV(p.kv)) for p in r.dsts]
    plan = [ScatterWindow(16 + p, sl, dl, c, sb, db, k) for p, sl, dl, c, sb, db, k in r.targets]
    reqs, spans = [], _spans(r)
    for (tb, te, m), (so, a, do, b) in zip(r.seqs, spans):
        reqs.append((range(tb, te), [int(x) for x in r.sids[so:so + a]],
                     {16 + p: [int(x) for x in r.dids[p][do:do + b]] for p in range(16) if (m >> p) & 1}))
    assert sum(set(q[2]) == {31} for q in reqs) >= 3
    if streamed:
        try:
            note = mgr.execute_repage_scatter_routed_anypage(sh, dhs, reqs, plan, TransferOptions(epoch=4, gate_mode=K.GATE_SPIN,
                                                                                                  max_ctas=MAX_CTAS),
                                                             ready_flags=r.src.ready.data_ptr())
            r.src.produce(range(s.nl), 4)
            note.wait(20.0)
        finally:
            s.rescue(4)
    else:
        mgr.execute_repage_scatter_routed_anypage(sh, dhs, reqs, plan).wait(20.0)
    _sync()
    r.check_pools(s.want if streamed else None)
    assert all(torch.equal(p.buf, x) for p, x in zip(idle, idle0))
    _sync()


def _c_pull(mgr, handles, dh, reqs, plan):
    """kvbm_manager_execute_repage_batch_routed_anypage with the source list as given (TransferManager passes only the ranks its
    plan reads): reqs are (tokens, {source rank: ids}, dst ids); the mask is the dict's keys."""
    import ctypes as C
    from dynamo_b200 import physical as P
    keep, n = [], len(handles)
    cs = (P._CRepageRouteSeq * max(1, len(reqs)))()
    for c, (tokens, ids, dids) in zip(cs, reqs):
        arrs = {r: (C.c_size_t * max(1, len(x)))(*x) for r, x in ids.items()}
        sp = (C.c_void_p * n)(*[C.addressof(arrs[r]) if r in arrs else None for r in range(n)])
        d = (C.c_size_t * max(1, len(dids)))(*dids)
        keep += [arrs, sp, d]
        c.token_begin, c.token_end, c.src_ids, c.n_src = tokens.start, tokens.stop, C.addressof(sp), len(next(iter(ids.values())))
        c.dst_ids, c.n_dst, c.src_mask = C.addressof(d), len(dids), sum(1 << r for r in ids)
    ws = (P._CShardWindow * len(plan))(*[P._CShardWindow(w.src_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin,
                                                          w.dst_head_begin, w.head_count) for w in plan])
    srcs = (C.c_uint64 * n)(*handles)
    o, tok = P.TransferOptions()._c(), C.c_uint64()
    P._check(P.lib().kvbm_manager_execute_repage_batch_routed_anypage(mgr._h, n, srcs, dh, cs, len(reqs), ws, len(plan), None, C.byref(o),
                                                                     C.byref(tok)))
    return P.TransferCompleteNotification(mgr, tok.value)


def test_manager_pull_from_ranks_16_to_31_with_a_phase(mgr):
    """The C entry with 32 sources, windows reading 16-31 only, several sequences from source 31 alone, 16 -> 24."""
    pools = [(2, 1, (HND, UTP)[p % 2]) for p in range(16)]
    windows = [(p, 0, 0, 2, 0, p, 1) for p in range(16)]
    seqs = [(tb, te, m) for (tb, te), m in zip(_phase_ranges(24, 16, len(HIGH_MASKS)), HIGH_MASKS)]
    r = CollectRig(pools, windows, (2, 16, NHD), seqs, ps=16, pd=24, no=1, hd=32, seed=33)
    assert _has_phase(r)
    idle = CollectRig([(2, 1, HND)], [(0, 0, 0, 2, 0, 0, 1)], (2, 1, NHD), [(0, 1, 1)], ps=16, pd=24, no=1, hd=32, seed=34).srcs[0]
    handles = [_register_gather_pool(mgr, idle)] * 16 + [_register_gather_pool(mgr, x) for x in r.srcs]
    dh = _register_gather_pool(mgr, r.dst)
    plan = [ShardWindow(16 + p, sl, dl, c, sb, db, k) for p, sl, dl, c, sb, db, k in r.windows]
    reqs = []
    for (tb, te, m), (so, a, do, b) in zip(r.seqs, _spans(r)):
        reqs.append((range(tb, te), {16 + p: [int(x) for x in r.sids[p][so:so + a]] for p in range(16) if (m >> p) & 1},
                     [int(x) for x in r.dids[do:do + b]]))
    _c_pull(mgr, handles, dh, reqs, plan).wait(20.0)
    _sync()
    r.check_pool()
    _sync()


def test_sixteen_targets_with_a_sequence_for_target_15_alone_at_the_largest_phase():
    """46337 / 46353 (the largest non-dividing pair the bound takes) with sixteen targets: a sequence routed to target 15 alone in a
    big block of phase small - 1, so bit 15 of the mask sits next to a phase of 2^15 or more."""
    small, big = 46337, 46353
    j = next(j for j in range(1, small) if (j * big) % small == small - 1)
    seqs = [(j * big + 3, j * big + 40, 1 << 15), (j * big + 100, j * big + 150, 0xFFFF), (5, 60, 1)]
    dsts = [(1, 1, (NHD, UTP)[t % 2]) for t in range(16)]
    targets = [(t, 0, 0, 1, 0, 0, 1) for t in range(16)]
    for ps, pd in ((big, small), (small, big)):
        r = DealRig((1, 1, HND), dsts, targets, seqs, ps=ps, pd=pd, no=1, hd=8, seed=15)
        assert any(u[3] == (1 << 15) | ((small - 1) << 16) for u in r.units_np.tolist())
        r.run_and_check()
        g = CollectRig([(1, 1, HND)] * 16, [(p, 0, 0, 1, 0, p, 1) for p in range(16)], (1, 16, NHD), seqs, ps=ps, pd=pd, no=1, hd=8, seed=16)
        assert any((u[3] & 0xFFFF) == 1 << 15 and (u[3] >> 16) >= 1 << 15 for u in g.units_np.tolist())
        g.run_and_check()
    _sync()


# ---------------------------------------------------------------------------------------------------------------------
# the 4.02 GiB pool of tests/test_gpu_transform_limits.py, as destination and as source, on both page sides
# ---------------------------------------------------------------------------------------------------------------------
def _deal_dst(ps):
    """A 4-head source into the big pool's heads 0-3 and 4-7 and a small pool: sequence 0 to every target, 1 to the small pool
    only (its big-pool positions unrouted), 2 to the big pool's heads 4-7 only."""
    return DealRig((BNL, 4, NHD), [(BNL, BNH, UTP), (BNL, 4, HND)], [(0, 0, 0, BNL, 0, 0, 4), (0, 0, 0, BNL, 0, 4, 4), (1, 0, 0, BNL, 0, 0, 4)],
                   [(5, 29, 0b111), (40, 60, 0b100), (115, 141, 0b010)], ps=ps, pd=BNT, seed=ps + 1, no=BNO, hd=BHD)


def _collect_dst(ps):
    return CollectRig([(BNL, 4, HND), (BNL, 4, NHD)], [(0, 0, 0, BNL, 0, 0, 4), (1, 0, 0, BNL, 0, 4, 4)], (BNL, BNH, UTP),
                      [(5, 29, 0b11), (40, 47, 0b01), (115, 120, 0b10)], ps=ps, pd=BNT, seed=ps + 2, no=BNO, hd=BHD)


@pytest.mark.parametrize("ps", [6, 24], ids=["larger_page_side", "smaller_page_side"])
@pytest.mark.parametrize("family", ["push", "pull"])
def test_big_pool_as_destination(big_pool, family, ps):
    if family == "push":
        r = _deal_dst(ps)
        pool, table, unrouted, initial = r.dsts[0], r.dids[0], tuple(r.sentinel[0]), r.initial[0]
        expected = lambda: (lambda p: (p, p[0]))(r.expected())  # noqa: E731
    else:
        r = _collect_dst(ps)
        pool, table, unrouted, initial = r.dst, r.dids, (), r.initial
        expected = lambda: (lambda p: (p, p))(r.expected())  # noqa: E731
    assert _has_phase(r)
    remap = _as_destination(big_pool, pool, table, unrouted)
    pools = _into_big_rows(big_pool, r.launch, initial, remap, expected)
    if family == "push":
        assert np.array_equal(r.dsts[1].buf.cpu().numpy(), pools[1])
    _sync()


@pytest.mark.parametrize("pd", [6, 24], ids=["larger_page_side", "smaller_page_side"])
@pytest.mark.parametrize("family", ["push", "pull"])
def test_big_pool_as_source(big_pool, family, pd):
    if family == "push":
        r = DealRig((BNL, BNH, UTP), [(BNL, BNH, NHD), (BNL, 4, UTP)], [(0, 0, 0, BNL, 0, 0, BNH), (1, 0, 0, BNL, 4, 0, 4)],
                    [(5, 29, 0b11), (40, 60, 0b10), (115, 141, 0b01)], ps=BNT, pd=pd, seed=pd + 5, no=BNO, hd=BHD)
        _as_source(big_pool, r.src, r.sids)
    else:
        r = CollectRig([(BNL, BNH, UTP), (BNL, BNH, HND)], [(0, 0, 0, BNL, 0, 0, BNH), (1, 0, 0, BNL, 0, 0, BNH)], (BNL, BNH, NHD),
                       [(5, 29, 0b01), (40, 60, 0b10), (115, 141, 0b01)], ps=BNT, pd=pd, seed=pd + 6, no=BNO, hd=BHD)
        _as_source(big_pool, r.srcs[0], r.sids[0])
    assert _has_phase(r)
    assert r.launch() == 0
    _sync()
    if family == "push":
        r.check_pools()
    else:
        assert np.array_equal(r.dst.buf.cpu().numpy(), r.expected())
    _check_filled(big_pool)
    _sync()


def test_rejections_launch_nothing():
    """A mask bit 16 on a 16-target launch is rejected before any launch, as is the first pair past the exactness bound."""
    r = deal_rig(*PUSH["tp1_to_2x_tp8"], SMALL, ps=24, pd=16, seed=3)
    before = K.launch_count()
    bad = [(tb, te, m | (1 << 16)) for tb, te, m in r.seqs]
    assert K.paged_repage_scatter_routed_anypage(r.src.side(r.sids_t), r.src.nh, 24, r.kernel_targets(), 16, bad, r.units_t.data_ptr(), r.nu,
                                                 r.lb, r.le, r.row) == K.CUDA_ERROR_INVALID_VALUE
    assert K.launch_count() == before
    past = [(tb, te, m) for tb, te, m in r.seqs]
    assert K.repage_route_anypage_units(past, 46354, 46337) is None
    _sync()

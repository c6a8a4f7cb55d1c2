"""GPU parity of re-paging with the gather's head windows (kvbm_kernels_paged_repage_gather, TransferManager.execute_repage_gather)
with tests/repage_gather_oracle.py.  Pools start from random bytes and every destination pool holds a guard block that no id
names; whole destination pools are compared, so every byte that must keep its value (heads no window covers, slots outside the
token range, other layers, the guard block) is checked too."""
import itertools

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import TransferManager, TransferOptions, tp_reshard_plan
from oracle import oracle as O
from tests.gpu_util import DevicePool, ids_dev, randomize, stream_ptr
from tests.repage_gather_oracle import repage_gather
from tests.repage_oracle import table_slice
from tests.test_gpu_permute import _host, _Pool

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
ALL = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]
UNIVERSAL = (KV.UniversalTP, KV.UniversalPP)
ELEMS = {CM.NONE: (2, 2), CM.FP8E4M3_TO_BF16: (1, 2), CM.BF16_TO_FP8E4M3: (2, 1)}   # (source, destination) element bytes
PLANS = [(8, 1), (4, 2), (2, 8), (1, 4)]                                          # (source TP, destination TP) on 8 KV heads
PAGES = [(1, 16), (16, 1), (16, 64), (64, 16), (48, 16), (16, 16)]


def _ranges(ps, pd):
    """Token ranges for a page pair: whole blocks, starting mid-block, starting and ending mid-block on both sides, one token,
    empty."""
    L, s = max(ps, pd), min(ps, pd)
    return {"whole": (0, 2 * L), "start_mid": (3, 2 * L), "both_mid": (s + 1 if s > 1 else 7, 2 * L - 3), "one_token": (L + 1, L + 2),
            "empty": (5, 5)}


def _kind(kv, pref):
    return "FC" if kv in UNIVERSAL else pref


class _Group:
    """Host twins of a prefill TP group's source pools (page ps, one per rank the plan names) and of a decode rank's destination
    pool (page pd, plus a guard block no table names), their block tables over a sequence of te tokens, and the plan."""

    def __init__(self, tp, ps, pd, te, src_kvs, dst_kv, geom, cast, seed, src_kind="LWs", dst_kind="LWf", dst_rank=0):
        self.H, self.nl, self.no, self.hd = geom
        src_tp, dst_tp = tp
        se, de = ELEMS[cast]
        rng = np.random.default_rng(seed)
        self.plan = tp_reshard_plan(self.H, src_tp, dst_tp, dst_rank)
        self.ranks = sorted({w.src_rank for w in self.plan})
        self.snh, self.dnh = max(1, self.H // src_tp), max(1, self.H // dst_tp)
        ns, nd = max(1, -(-te // ps)), max(1, -(-te // pd))
        self.src_kv = {r: src_kvs[i % len(src_kvs)] for i, r in enumerate(self.ranks)}
        self.src, self.src_tab = {}, {}
        for r in self.ranks:
            self.src[r] = _host(_kind(self.src_kv[r], src_kind), ns + 2, self.nl, self.no, ps, self.snh, self.hd, se)
            randomize(self.src[r], seed + 10 + r)
            self.src_tab[r] = [int(x) for x in rng.permutation(ns + 2)[:ns]]
        self.dst_kv = dst_kv
        self.dst = _host(_kind(dst_kv, dst_kind), nd + 1, self.nl, self.no, pd, self.dnh, self.hd, de)
        self.ref = _host(_kind(dst_kv, dst_kind), nd + 1, self.nl, self.no, pd, self.dnh, self.hd, de)
        randomize(self.dst, seed + 1)
        for a, b in zip(self.ref.buffers, self.dst.buffers):
            a[:] = b
        guard = int(rng.integers(0, nd + 1))
        self.dst_tab = [b for b in rng.permutation(nd + 1).tolist() if b != guard][:nd]
        self.ps, self.pd, self.cast = ps, pd, cast
        self.src_row = self.hd * se

    def ids(self, tb, te):
        return {r: table_slice(self.src_tab[r], tb, te, self.ps) for r in self.ranks}, table_slice(self.dst_tab, tb, te, self.pd)

    def expect(self, tb, te, scales=None, layers=None):
        sids, dids = self.ids(tb, te)
        index = {r: i for i, r in enumerate(self.ranks)}
        sources = [([O.read_logical_block(self.src[r], b) for b in sids[r]], int(self.src_kv[r]), self.snh) for r in self.ranks]
        windows = [(index[w.src_rank], w.src_head_begin, w.dst_head_begin, w.head_count) for w in self.plan]
        new = repage_gather(sources, windows, [O.read_logical_block(self.ref, b) for b in dids], int(self.dst_kv), self.dnh, self.nl, self.no,
                            self.ps, self.pd, self.src_row, tb, te, int(self.cast), scales, layers)
        for b, blk in zip(dids, new):
            O.write_logical_block(self.ref, b, blk)

    def check(self):
        for got, want in zip(self.dst.buffers, self.ref.buffers):
            assert np.array_equal(got, want)


def _run(g, tb, te, lb=0, le=None, scales=None, done=0, epoch=0, completion=0, value=0):
    S = {r: DevicePool(g.src[r]) for r in g.ranks}
    D = DevicePool(g.dst)
    sids, dids = g.ids(tb, te)
    si = {r: ids_dev(sids[r] or [0]) for r in g.ranks}
    di = ids_dev(dids or [0])
    srcs = [K.PermuteSource(K.PermuteSide(S[w.src_rank].desc, si[w.src_rank].data_ptr(), int(g.src_kv[w.src_rank])), g.snh, w.src_head_begin,
                            w.dst_head_begin, w.head_count) for w in g.plan]
    sc = None if scales is None else torch.from_numpy(scales).cuda()
    rc = K.paged_repage_gather(srcs, g.ps, K.PermuteSide(D.desc, di.data_ptr(), int(g.dst_kv)), g.dnh, g.pd, tb, te, lb, g.nl if le is None else le,
                               g.src_row, int(g.cast), sc, done, epoch, completion, value, stream_ptr())
    torch.cuda.synchronize()
    if rc == 0:
        D.download()
    return rc


@pytest.mark.parametrize("rng_name", ["whole", "start_mid", "both_mid", "one_token", "empty"])
@pytest.mark.parametrize("ps,pd", PAGES, ids=lambda p: str(p))
@pytest.mark.parametrize("tp", PLANS, ids=lambda t: f"tp{t[0]}_to_tp{t[1]}")
def test_plans_page_pairs_and_token_ranges(tp, ps, pd, rng_name):
    tb, te = _ranges(ps, pd)[rng_name]
    g = _Group(tp, ps, pd, te, [KV.OperationalNHD, KV.OperationalHND], KV.OperationalNHD, (8, 2, 2, 64), CM.NONE, 7 * ps + pd + tp[0])
    assert _run(g, tb, te) == 0
    g.expect(tb, te)
    g.check()


@pytest.mark.parametrize("src_kv,dst_kv", list(itertools.product(ALL, ALL)), ids=lambda k: k.name)
@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16)], ids=lambda p: str(p))
def test_every_pair_of_formats(ps, pd, src_kv, dst_kv):
    """TP4 -> TP2: two sources of src_kv into dst_kv, layer-separate pools where the format allows, else fully contiguous."""
    tb, te = 5, 2 * max(ps, pd) - 3
    g = _Group((4, 2), ps, pd, te, [src_kv], dst_kv, (8, 2, 2, 32), CM.NONE, int(src_kv) * 5 + int(dst_kv), src_kind="LWf", dst_kind="LWs")
    assert _run(g, tb, te) == 0
    g.expect(tb, te)
    g.check()


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16)], ids=lambda p: str(p))
def test_layer_ranges(ps, pd):
    tb, te = 9, 150
    g = _Group((8, 2), ps, pd, te, [KV.OperationalNHD, KV.UniversalPP], KV.OperationalHND, (8, 4, 2, 64), CM.NONE, 77, src_kind="FC")
    assert _run(g, tb, te, lb=1, le=3) == 0
    g.expect(tb, te, layers=range(1, 3))
    g.check()


@pytest.mark.parametrize("scaled", [False, True], ids=["unscaled", "scaled"])
@pytest.mark.parametrize("cast", [CM.FP8E4M3_TO_BF16, CM.BF16_TO_FP8E4M3], ids=lambda c: c.name)
@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (1, 16)], ids=lambda p: str(p))
def test_casts(ps, pd, cast, scaled):
    tb, te = 7, 2 * max(ps, pd) - 5
    g = _Group((8, 1), ps, pd, te, [KV.OperationalHND, KV.OperationalNHD], KV.UniversalTP, (8, 2, 2, 64), cast, 31 + int(cast))
    scales = np.array([0.5, 2.0, 0.037, 3.5], dtype=np.float32) if scaled else None
    assert _run(g, tb, te, scales=scales) == 0
    g.expect(tb, te, scales=scales)
    g.check()


@pytest.mark.parametrize("hd", [80, 96])
@pytest.mark.parametrize("ps,pd", [(48, 16), (16, 64)], ids=lambda p: str(p))
def test_non_pow2_rows(ps, pd, hd):
    tb, te = 17, 3 * max(ps, pd) - 2
    g = _Group((4, 2), ps, pd, te, [KV.OperationalNHD], KV.OperationalHND, (8, 2, 2, hd), CM.NONE, hd + ps)
    assert _run(g, tb, te) == 0
    g.expect(tb, te)
    g.check()


@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16], ids=lambda c: c.name)
@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (1, 16)], ids=lambda p: str(p))
def test_mla_geometry(ps, pd, cast):
    """MLA: one outer index, one 576-wide head replicated over the source ranks; the plan takes it from one replica."""
    tb, te = 3, 2 * max(ps, pd) - 1
    g = _Group((2, 1), ps, pd, te, [KV.OperationalNHD], KV.OperationalNHD, (1, 2, 1, 576), cast, 99, dst_rank=0)
    assert len(g.plan) == 1 and g.snh == 1 and g.dnh == 1
    assert _run(g, tb, te) == 0
    g.expect(tb, te)
    g.check()


def test_signals_and_empty_ranges():
    flags = torch.zeros(4, dtype=torch.int32, device="cuda")
    g = _Group((4, 2), 16, 64, 200, [KV.OperationalNHD], KV.OperationalNHD, (8, 2, 2, 64), CM.NONE, 5, src_kind="FC", dst_kind="FC")
    before = K.launch_count()
    assert _run(g, 10, 200, done=flags[0:].data_ptr(), epoch=7, completion=flags[1:].data_ptr(), value=9) == 0
    assert K.launch_count() == before + 2        # one launch for all the sources, and one signal launch
    g.expect(10, 200)
    g.check()
    assert flags[:2].tolist() == [7, 9]
    before = K.launch_count()
    assert _run(g, 50, 50, done=flags[2:].data_ptr(), epoch=3) == 0   # empty: signals only
    assert _run(g, 10, 20, lb=1, le=1, completion=flags[3:].data_ptr(), value=4) == 0
    assert K.launch_count() == before + 2 and flags[2:].tolist() == [3, 4]
    assert _run(g, 50, 50) == 0 and K.launch_count() == before + 2
    g.check()


# ---------------------------------------------------------------------------------------------------------------------
# TransferManager.execute_repage_gather
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=41)
    yield m
    torch.cuda.synchronize()
    m.close()


class _Managed:
    """A TP group's source pools and a decode rank's destination pool registered with a manager, with host twins."""

    def __init__(self, m, tp, ps, pd, te, cast, src_kv, dst_kv, geom=(8, 2, 2, 64), device=(0, 0), dst_rank=0):
        self.H, self.nl, self.no, self.hd = geom
        se, de = ELEMS[cast]
        self.plan = tp_reshard_plan(self.H, tp[0], tp[1], dst_rank)
        self.ranks = sorted({w.src_rank for w in self.plan})
        self.snh, self.dnh = max(1, self.H // tp[0]), max(1, self.H // tp[1])
        ns, nd = -(-te // ps), -(-te // pd)
        self.src = {r: _Pool(m, _kind(src_kv, "LWs"), ns + 2, self.nl, self.no, ps, self.snh, self.hd, se, kv=src_kv, device=device[0])
                    for r in self.ranks}
        self.dst = _Pool(m, _kind(dst_kv, "LWs"), nd + 1, self.nl, self.no, pd, self.dnh, self.hd, de, kv=dst_kv, device=device[1])
        for r in self.ranks:
            randomize(self.src[r].twin, 3 + r)
            self.src[r].upload()
        randomize(self.dst.twin, 4)
        self.dst.upload()
        self.ref = _host(_kind(dst_kv, "LWs"), nd + 1, self.nl, self.no, pd, self.dnh, self.hd, de)
        for a, b in zip(self.ref.buffers, self.dst.twin.buffers):
            a[:] = b
        self.stab = {r: list(range(ns + 1, 0, -1))[:ns] if r % 2 == 0 else list(range(ns))[::-1] for r in self.ranks}
        self.dtab = list(range(1, nd + 1))     # block 0 of the destination is the guard
        self.ps, self.pd, self.cast, self.src_kv, self.dst_kv = ps, pd, cast, src_kv, dst_kv

    def sources(self, tb, te):
        return {r: (self.src[r].h, table_slice(self.stab[r], tb, te, self.ps)) for r in self.ranks}

    def dids(self, tb, te):
        return table_slice(self.dtab, tb, te, self.pd)

    def expect(self, tb, te, scales=None, layers=None, dst_kv=None):
        index = {r: i for i, r in enumerate(self.ranks)}
        srcs = [([O.read_logical_block(self.src[r].twin, b) for b in table_slice(self.stab[r], tb, te, self.ps)], int(self.src_kv), self.snh)
                for r in self.ranks]
        windows = [(index[w.src_rank], w.src_head_begin, w.dst_head_begin, w.head_count) for w in self.plan]
        dids = self.dids(tb, te)
        dkv = self.dst_kv if dst_kv is None else dst_kv
        new = repage_gather(srcs, windows, [O.read_logical_block(self.ref, b) for b in dids], int(dkv), self.dnh, self.nl, self.no, self.ps,
                            self.pd, self.hd * ELEMS[self.cast][0], tb, te, int(self.cast), scales, layers)
        for b, blk in zip(dids, new):
            O.write_logical_block(self.ref, b, blk)

    def check(self):
        self.dst.download()
        for a, b in zip(self.dst.twin.buffers, self.ref.buffers):
            assert np.array_equal(a, b)


@pytest.mark.parametrize("cast,scaled", [(CM.NONE, False), (CM.FP8E4M3_TO_BF16, True), (CM.BF16_TO_FP8E4M3, False)],
                         ids=["plain", "fp8_to_bf16_scaled", "bf16_to_fp8"])
@pytest.mark.parametrize("tp,ps,pd", [((8, 1), 1, 16), ((4, 2), 64, 16), ((2, 8), 16, 64)], ids=lambda x: str(x))
def test_manager_repage_gather(mgr, tp, ps, pd, cast, scaled):
    tb, te = 5, 2 * max(ps, pd) + 7
    c = _Managed(mgr, tp, ps, pd, te, cast, KV.OperationalNHD, KV.UniversalTP)
    done = torch.zeros(1, dtype=torch.int32, device="cuda")
    scales = torch.tensor([0.25, 4.0, 1.5, 0.75], dtype=torch.float32, device="cuda") if scaled else None
    b0, h0, l0 = mgr.bytes_moved(), mgr.h2d_bytes(), K.launch_count()
    sources, dids = c.sources(tb, te), c.dids(tb, te)
    o = TransferOptions(cast_mode=int(cast), cast_scales=scales, done_flag=done.data_ptr(), epoch=11)
    note = mgr.execute_repage_gather(sources, c.dst.h, dids, c.plan, range(tb, te), o)
    note.wait(20.0)
    torch.cuda.synchronize()
    assert done.item() == 11
    assert K.launch_count() - l0 == 2                    # one launch and one signal launch: the flag is written once
    covered = sum(w.head_count for w in c.plan)
    assert mgr.bytes_moved() - b0 == (te - tb) * c.nl * c.no * covered * c.hd * ELEMS[cast][1]
    n_src = len(next(iter(sources.values()))[1])
    assert mgr.h2d_bytes() - h0 == 4 * (len(c.ranks) * n_src + len(dids))
    c.expect(tb, te, None if scales is None else scales.cpu().numpy())
    c.check()


def test_manager_repage_gather_caller_stream_layer_range_and_overrides(mgr):
    tb, te = 20, 100
    c = _Managed(mgr, (4, 2), 16, 32, te, CM.NONE, KV.OperationalHND, KV.OperationalNHD, geom=(8, 4, 2, 64), dst_rank=1)
    s = torch.cuda.Stream()
    # the destination is registered NHD; the override reads it as HND (a layer-separate pool takes either operational format)
    o = TransferOptions(layer_range=range(1, 3), cuda_stream=int(s.cuda_stream), dst_kv_layout=int(KV.OperationalHND))
    note = mgr.execute_repage_gather(c.sources(tb, te), c.dst.h, c.dids(tb, te), c.plan, range(tb, te), o)
    assert note.is_complete()                              # the caller's stream: the caller synchronises
    s.synchronize()
    c.expect(tb, te, layers=range(1, 3), dst_kv=KV.OperationalHND)
    c.check()


@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16], ids=lambda c: c.name)
@pytest.mark.parametrize("tp,ps,pd", [((8, 1), 1, 16), ((4, 2), 64, 16), ((2, 8), 16, 64), ((1, 4), 48, 16)], ids=lambda x: str(x))
def test_one_launch_equals_the_two_pass_workaround(mgr, tp, ps, pd, cast):
    """Over a range that starts and ends on destination page boundaries, the one launch leaves the same bytes as execute_repage per
    source into a staging pool with the destination's page and the source's heads, then execute_gather out of the staging pools."""
    tb, te = pd, 4 * max(ps, pd)
    tb, te = -(-tb // pd) * pd, te // pd * pd
    c = _Managed(mgr, tp, ps, pd, te, cast, KV.OperationalNHD, KV.OperationalHND)
    sources, dids = c.sources(tb, te), c.dids(tb, te)
    mgr.execute_repage_gather(sources, c.dst.h, dids, c.plan, range(tb, te), TransferOptions(cast_mode=int(cast))).wait(20.0)
    torch.cuda.synchronize()
    c.dst.download()
    one = [b.copy() for b in c.dst.twin.buffers]
    c.expect(tb, te)
    c.check()
    # the workaround, on pools that start from the same bytes
    c2 = _Managed(mgr, tp, ps, pd, te, cast, KV.OperationalNHD, KV.OperationalHND)
    de = ELEMS[cast][1]
    n = len(dids)
    staging = {r: _Pool(mgr, "LWs", n, c2.nl, c2.no, pd, c2.snh, c2.hd, de, kv=KV.OperationalNHD) for r in c2.ranks}
    for r in c2.ranks:
        h, sids = c2.sources(tb, te)[r]
        mgr.execute_repage(h, sids, staging[r].h, list(range(n)), range(tb, te), TransferOptions(cast_mode=int(cast))).wait(20.0)
    mgr.execute_gather({r: (staging[r].h, list(range(n))) for r in c2.ranks}, c2.dst.h, c2.dids(tb, te), c2.plan).wait(20.0)
    torch.cuda.synchronize()
    c2.dst.download()
    for a, b in zip(one, c2.dst.twin.buffers):
        assert np.array_equal(a, b)


@pytest.mark.multigpu
def test_manager_repage_gather_across_gpus():
    """The decode GPU pulls every source rank's heads from pools on the other GPU over NVLink."""
    m = TransferManager(device=1, worker_id=42)
    m.enable_peer_access(0)
    tb, te = 3, 150
    c = _Managed(m, (4, 2), 16, 64, te, CM.NONE, KV.OperationalNHD, KV.OperationalHND, device=(0, 1))
    m.execute_repage_gather(c.sources(tb, te), c.dst.h, c.dids(tb, te), c.plan, range(tb, te)).wait(20.0)
    torch.cuda.synchronize(0)
    torch.cuda.synchronize(1)
    c.expect(tb, te)
    c.check()
    m.close()

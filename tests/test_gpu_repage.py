"""GPU parity of re-paging (kvbm_kernels_paged_repage, TransferManager.execute_repage) with tests/repage_oracle.py.  Pools start from
random bytes and every destination pool holds a guard block that no id names; whole destination pools are compared, so every
byte that must keep its value (slots outside the token range, other layers, the guard block) is checked too."""
import itertools

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import TransferManager, TransferOptions
from oracle import oracle as O
from tests.gpu_util import DevicePool, ids_dev, randomize, stream_ptr
from tests.repage_oracle import repage, table_slice
from tests.test_gpu_permute import _host, _Pool

pytestmark = pytest.mark.gpu
KV = K.KvBlockLayout
CM = K.CastMode
ALL = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]
UNIVERSAL = (KV.UniversalTP, KV.UniversalPP)
ELEMS = {CM.NONE: (2, 2), CM.FP8E4M3_TO_BF16: (1, 2), CM.BF16_TO_FP8E4M3: (2, 1)}
PAIRS = [(16, 64), (64, 16), (32, 64), (16, 16), (1, 16), (16, 1), (528, 16)]


def _ranges(ps, pd):
    """Token ranges for a page pair: whole blocks, starting / ending mid-block on either side, one token, inside one block, empty."""
    L, s = max(ps, pd), min(ps, pd)
    r = {"whole": (0, 2 * L), "start_mid": (3, 2 * L), "end_mid": (L, 2 * L + 5), "both_mid": (s + 1 if s > 1 else 7, 2 * L - 3),
         "one_token": (L + 1, L + 2), "in_one_block": (L + 2, L + max(3, L // 2)), "empty": (5, 5)}
    return r


def _kind(kv, pref):
    return "FC" if kv in UNIVERSAL else pref


class _Case:
    """Host twins of a source and a destination pool, their block tables over a sequence and a random start."""

    def __init__(self, ps, pd, te, src_kind, dst_kind, geom, cast, seed):
        self.nl, self.no, self.nh, self.hd = geom
        se, de = ELEMS[cast]
        rng = np.random.default_rng(seed)
        ns, nd = max(1, -(-te // ps)), max(1, -(-te // pd))
        self.src = _host(src_kind, ns + 2, self.nl, self.no, ps, self.nh, self.hd, se)
        self.dst = _host(dst_kind, nd + 1, self.nl, self.no, pd, self.nh, self.hd, de)      # + a guard block no table names
        self.ref = _host(dst_kind, nd + 1, self.nl, self.no, pd, self.nh, self.hd, de)
        randomize(self.src, seed)
        randomize(self.dst, seed + 1)
        for a, b in zip(self.ref.buffers, self.dst.buffers):
            a[:] = b
        self.src_tab = [int(x) for x in rng.permutation(ns + 2)[:ns]]
        guard = int(rng.integers(0, nd + 1))
        self.dst_tab = [b for b in rng.permutation(nd + 1).tolist() if b != guard][:nd]
        self.ps, self.pd, self.cast = ps, pd, cast
        self.src_row = self.hd * se

    def ids(self, tb, te):
        return table_slice(self.src_tab, tb, te, self.ps), table_slice(self.dst_tab, tb, te, self.pd)

    def expect(self, tb, te, src_kv, dst_kv, scales=None, layers=None):
        sids, dids = self.ids(tb, te)
        new = repage([O.read_logical_block(self.src, b) for b in sids], [O.read_logical_block(self.ref, b) for b in dids], int(src_kv),
                     int(dst_kv), self.nl, self.no, self.nh, self.ps, self.pd, self.src_row, tb, te, int(self.cast), scales, layers)
        for b, blk in zip(dids, new):
            O.write_logical_block(self.ref, b, blk)

    def check(self):
        for got, want in zip(self.dst.buffers, self.ref.buffers):
            assert np.array_equal(got, want)


def _run(c, tb, te, src_kv, dst_kv, lb=0, le=None, scales=None, done=0, epoch=0, completion=0, value=0):
    S, D = DevicePool(c.src), DevicePool(c.dst)
    sids, dids = c.ids(tb, te)
    si, di = ids_dev(sids or [0]), ids_dev(dids or [0])
    sc = None if scales is None else torch.from_numpy(scales).cuda()
    rc = K.paged_repage(K.PermuteSide(S.desc, si.data_ptr(), int(src_kv)), c.ps, K.PermuteSide(D.desc, di.data_ptr(), int(dst_kv)), c.pd,
                        tb, te, lb, c.nl if le is None else le, c.nh, c.src_row, int(c.cast), sc, done, epoch, completion, value, stream_ptr())
    torch.cuda.synchronize()
    if rc == 0:
        D.download()
    return rc


@pytest.mark.parametrize("rng_name", ["whole", "start_mid", "end_mid", "both_mid", "one_token", "in_one_block", "empty"])
@pytest.mark.parametrize("ps,pd", PAIRS + [(16, 528)], ids=lambda p: str(p))
def test_page_pairs_and_token_ranges(ps, pd, rng_name):
    tb, te = _ranges(ps, pd)[rng_name]
    c = _Case(ps, pd, te, "FC", "LWs", (2, 2, 2, 64), CM.NONE, 7 * ps + pd)
    assert _run(c, tb, te, KV.OperationalNHD, KV.OperationalHND) == 0
    c.expect(tb, te, KV.OperationalNHD, KV.OperationalHND)
    c.check()


@pytest.mark.parametrize("src_kv,dst_kv", list(itertools.product(ALL, ALL)), ids=lambda k: k.name)
@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16)], ids=lambda p: str(p))
def test_every_pair_of_formats(ps, pd, src_kv, dst_kv):
    tb, te = 5, 2 * max(ps, pd) - 3
    c = _Case(ps, pd, te, _kind(src_kv, "LWf"), _kind(dst_kv, "LWs"), (2, 2, 4, 32), CM.NONE, int(src_kv) * 5 + int(dst_kv))
    assert _run(c, tb, te, src_kv, dst_kv) == 0
    c.expect(tb, te, src_kv, dst_kv)
    c.check()


@pytest.mark.parametrize("scaled", [False, True], ids=["unscaled", "scaled"])
@pytest.mark.parametrize("cast", [CM.FP8E4M3_TO_BF16, CM.BF16_TO_FP8E4M3], ids=lambda c: c.name)
@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (1, 16), (528, 16)], ids=lambda p: str(p))
def test_casts(ps, pd, cast, scaled):
    tb, te = 7, 2 * max(ps, pd) - 5
    c = _Case(ps, pd, te, "LWf", "FC", (2, 2, 4, 64), cast, 31 + int(cast))
    scales = np.array([0.5, 2.0, 0.037, 3.5], dtype=np.float32) if scaled else None
    assert _run(c, tb, te, KV.OperationalHND, KV.UniversalTP, scales=scales) == 0
    c.expect(tb, te, KV.OperationalHND, KV.UniversalTP, scales=scales)
    c.check()


@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16)], ids=lambda p: str(p))
def test_layer_ranges(ps, pd):
    tb, te = 9, 150
    c = _Case(ps, pd, te, "LWs", "LWf", (4, 2, 2, 64), CM.NONE, 77)
    assert _run(c, tb, te, KV.OperationalNHD, KV.OperationalNHD, lb=1, le=3) == 0
    c.expect(tb, te, KV.OperationalNHD, KV.OperationalNHD, layers=range(1, 3))
    c.check()


@pytest.mark.parametrize("cast", [CM.NONE, CM.FP8E4M3_TO_BF16], ids=lambda c: c.name)
@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (1, 16), (16, 1)], ids=lambda p: str(p))
def test_mla_geometry(ps, pd, cast):
    """MLA: one outer index, one 576-wide head (non-power-of-two rows: the multiply-high split)."""
    tb, te = 3, 2 * max(ps, pd) - 1
    c = _Case(ps, pd, te, "LWs", "LWs", (2, 1, 1, 576), cast, 99)
    assert _run(c, tb, te, KV.OperationalNHD, KV.OperationalNHD) == 0
    c.expect(tb, te, KV.OperationalNHD, KV.OperationalNHD)
    c.check()


@pytest.mark.parametrize("hd", [80, 96])
def test_non_pow2_rows_and_pages(hd):
    tb, te = 17, 1000
    c = _Case(528, 48, te, "FC", "LWs", (2, 2, 3, hd), CM.NONE, hd)
    assert _run(c, tb, te, KV.OperationalNHD, KV.OperationalHND) == 0
    c.expect(tb, te, KV.OperationalNHD, KV.OperationalHND)
    c.check()


def test_signals_and_empty_ranges():
    flags = torch.zeros(4, dtype=torch.int32, device="cuda")
    c = _Case(16, 64, 200, "FC", "FC", (2, 2, 2, 64), CM.NONE, 5)
    before = K.launch_count()
    assert _run(c, 10, 200, KV.OperationalNHD, KV.OperationalNHD, done=flags[0:].data_ptr(), epoch=7, completion=flags[1:].data_ptr(), value=9) == 0
    assert K.launch_count() == before + 2        # the re-paging launch and one signal launch
    c.expect(10, 200, KV.OperationalNHD, KV.OperationalNHD)
    c.check()
    assert flags[:2].tolist() == [7, 9]
    before = K.launch_count()
    assert _run(c, 50, 50, KV.OperationalNHD, KV.OperationalNHD, done=flags[2:].data_ptr(), epoch=3) == 0   # empty: signals only
    assert _run(c, 10, 20, KV.OperationalNHD, KV.OperationalNHD, lb=1, le=1, completion=flags[3:].data_ptr(), value=4) == 0
    assert K.launch_count() == before + 2 and flags[2:].tolist() == [3, 4]
    assert _run(c, 50, 50, KV.OperationalNHD, KV.OperationalNHD) == 0 and K.launch_count() == before + 2
    c.check()


# ---------------------------------------------------------------------------------------------------------------------
# TransferManager.execute_repage
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=31)
    yield m
    torch.cuda.synchronize()
    m.close()


def _manager_case(mgr, ps, pd, te, cast, src_kv, dst_kv, geom=(2, 2, 4, 64), device=(0, 0), dst_kind="LWs"):
    nl, no, nh, hd = geom
    se, de = ELEMS[cast]
    ns, nd = -(-te // ps), -(-te // pd)
    src = _Pool(mgr, _kind(src_kv, "FC"), ns + 2, nl, no, ps, nh, hd, se, kv=src_kv, device=device[0])
    dst = _Pool(mgr, _kind(dst_kv, dst_kind), nd + 1, nl, no, pd, nh, hd, de, kv=dst_kv, device=device[1])
    randomize(src.twin, 3)
    randomize(dst.twin, 4)
    src.upload()
    dst.upload()
    ref = _host(_kind(dst_kv, dst_kind), nd + 1, nl, no, pd, nh, hd, de)
    for a, b in zip(ref.buffers, dst.twin.buffers):
        a[:] = b
    return src, dst, ref, list(range(ns + 1, 0, -1))[:ns], list(range(1, nd + 1))   # block 0 of the destination is the guard


def _expect(src, ref, stab, dtab, ps, pd, tb, te, src_kv, dst_kv, geom, cast, scales=None, layers=None):
    nl, no, nh, hd = geom
    sids, dids = table_slice(stab, tb, te, ps), table_slice(dtab, tb, te, pd)
    new = repage([O.read_logical_block(src.twin, b) for b in sids], [O.read_logical_block(ref, b) for b in dids], int(src_kv), int(dst_kv),
                 nl, no, nh, ps, pd, hd * ELEMS[cast][0], tb, te, int(cast), scales, layers)
    for b, blk in zip(dids, new):
        O.write_logical_block(ref, b, blk)


@pytest.mark.parametrize("cast,scaled", [(CM.NONE, False), (CM.FP8E4M3_TO_BF16, True), (CM.BF16_TO_FP8E4M3, False)],
                         ids=["plain", "fp8_to_bf16_scaled", "bf16_to_fp8"])
@pytest.mark.parametrize("ps,pd", [(16, 64), (64, 16), (1, 16)], ids=lambda p: str(p))
def test_manager_repage(mgr, ps, pd, cast, scaled):
    geom = (2, 2, 4, 64)
    tb, te = 5, 2 * max(ps, pd) + 7
    src, dst, ref, stab, dtab = _manager_case(mgr, ps, pd, te, cast, KV.OperationalNHD, KV.UniversalTP)
    done = torch.zeros(1, dtype=torch.int32, device="cuda")
    scales = torch.tensor([0.25, 4.0, 1.5, 0.75], dtype=torch.float32, device="cuda") if scaled else None
    b0, h0 = mgr.bytes_moved(), mgr.h2d_bytes()
    sids, dids = table_slice(stab, tb, te, ps), table_slice(dtab, tb, te, pd)
    o = TransferOptions(cast_mode=int(cast), cast_scales=scales, done_flag=done.data_ptr(), epoch=11)
    note = mgr.execute_repage(src.h, sids, dst.h, dids, range(tb, te), o)
    note.wait(20.0)
    torch.cuda.synchronize()
    assert done.item() == 11
    d_row = 64 * ELEMS[cast][1]
    assert mgr.bytes_moved() - b0 == (te - tb) * 2 * 2 * 4 * d_row
    assert mgr.h2d_bytes() - h0 == 4 * (len(sids) + len(dids))
    dst.download()
    _expect(src, ref, stab, dtab, ps, pd, tb, te, KV.OperationalNHD, KV.UniversalTP, geom, cast,
            None if scales is None else scales.cpu().numpy())
    for a, b in zip(dst.twin.buffers, ref.buffers):
        assert np.array_equal(a, b)


def test_manager_repage_caller_stream_layer_range_and_overrides(mgr):
    geom = (4, 2, 2, 64)
    tb, te = 20, 100
    src, dst, ref, stab, dtab = _manager_case(mgr, 16, 32, te, CM.NONE, KV.OperationalHND, KV.OperationalNHD, geom=geom)
    s = torch.cuda.Stream()
    sids, dids = table_slice(stab, tb, te, 16), table_slice(dtab, tb, te, 32)
    # the destination is registered NHD; the override reads it as HND (a layer-separate pool takes either operational format)
    o = TransferOptions(layer_range=range(1, 3), cuda_stream=int(s.cuda_stream), dst_kv_layout=int(KV.OperationalHND))
    note = mgr.execute_repage(src.h, sids, dst.h, dids, range(tb, te), o)
    assert note.is_complete()                              # the caller's stream: the caller synchronises
    s.synchronize()
    dst.download()
    _expect(src, ref, stab, dtab, 16, 32, tb, te, KV.OperationalHND, KV.OperationalHND, geom, CM.NONE, layers=range(1, 3))
    for a, b in zip(dst.twin.buffers, ref.buffers):
        assert np.array_equal(a, b)


@pytest.mark.multigpu
@pytest.mark.parametrize("direction", ["pull", "push"])
def test_manager_repage_across_gpus(direction):
    """The decode GPU pulls from (or the prefill GPU pushes into) a pool on the other GPU over NVLink."""
    local, peer = (1, 0) if direction == "pull" else (0, 1)
    m = TransferManager(device=local, worker_id=32)
    m.enable_peer_access(peer)
    geom = (2, 2, 4, 64)
    tb, te = 3, 150
    src, dst, ref, stab, dtab = _manager_case(m, 16, 64, te, CM.NONE, KV.OperationalNHD, KV.OperationalHND, geom=geom, device=(0, 1))
    m.execute_repage(src.h, table_slice(stab, tb, te, 16), dst.h, table_slice(dtab, tb, te, 64), range(tb, te)).wait(20.0)
    torch.cuda.synchronize(0)
    torch.cuda.synchronize(1)
    dst.download()
    _expect(src, ref, stab, dtab, 16, 64, tb, te, KV.OperationalNHD, KV.OperationalHND, geom, CM.NONE)
    for a, b in zip(dst.twin.buffers, ref.buffers):
        assert np.array_equal(a, b)
    m.close()

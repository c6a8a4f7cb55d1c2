"""The option space of the paged copy (kvbm_kernels_paged_copy_v2), byte for byte against the CPU oracle.

The launcher routes every transfer to one of eight ring instantiations, kvbm_paged_copy_kernel<CAST, FAST, SCALED>, and inside
the consumer each one branches again on TMA vs SIMT pieces, `variant`, `cache_hint`, `stores_in_flight` and per-layer
publishing.  The cases here walk that space where the other files do not: casts with several destinations, destinations of
different kinds and strides in one launch, the general ring's run-time options, the FAST cast kernels at piece edges, gated
casts with fan-out, and a profiler run that shows all eight instantiations are reached.

Every destination pool starts from random bytes and is compared whole with the oracle (`O.execute_memcpy_transfer` on its host
twin), so a region that was never written, or written twice, shows up.  The last block of every destination pool is a guard
that no block id names: a store sent to another item's address, which can be larger than that item's piece, then still lands
inside the pool, and the guard must come back unchanged."""
import itertools
import os
import re
import time

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import TransferOptions, TransferManager
from oracle import oracle as O
from tests.gpu_util import DevicePool, ids_dev, paged_dst, randomize, stream_ptr

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")
NONE, UP, DOWN = int(K.CastMode.NONE), int(K.CastMode.FP8E4M3_TO_BF16), int(K.CastMode.BF16_TO_FP8E4M3)
CASTS = [UP, DOWN]
CAST_IDS = {NONE: "none", UP: "fp8_to_bf16", DOWN: "bf16_to_fp8"}
ELEMS = {NONE: (2, 2), UP: (1, 2), DOWN: (2, 1)}   # (source, destination) element bytes
KINDS = {"FC": (O.FC, O.BLOCK_IS_FIRST_DIM), "LWf": (O.LW, O.BLOCK_IS_FIRST_DIM), "LWs": (O.LW, O.BLOCK_IS_SECOND_DIM)}


def _layout(kind, nb, nl, no, page, inner, elem, seed):
    k, bd = KINDS[kind]
    h = O.Layout(k, nb, nl, no, page, inner, elem, block_dim=bd, allow_fp8=elem == 1)
    randomize(h, seed)
    return h


def _mixed(ndst, nb0=9):
    """`ndst` destination geometries: FC, LW block-first and LW block-second in turn, each with its own num_blocks (so its own
    block and outer strides)."""
    return [(("FC", "LWf", "LWs")[d % 3], nb0 + 2 * d) for d in range(ndst)]


def _region_offset(h, buf_index_of, b, l, o):
    a, s = h.memory_region(b, l, o)
    i = buf_index_of(l)
    return i, a - h.buffers[i].ctypes.data, s


class Fanout:
    """One paged copy from a source pool to `len(geoms)` destination pools, each (kind, num_blocks).  Destination block ids
    never name a pool's last block (the guard).  `flags`: per-destination done flags and per-layer done flags."""

    def __init__(self, cast, geoms, n, replicate, nl=3, no=2, page=16, inner=64, src_kind="LWs", src_nb=None, flags=False, seed=0,
                 dids=None):
        se, de = ELEMS[cast]
        self.cast, self.nl, self.replicate = cast, nl, replicate
        self.src_h = _layout(src_kind, src_nb or n + 3, nl, no, page, inner, se, seed)
        self.src = DevicePool(self.src_h)
        self.dst_h = [_layout(kind, nb, nl, no, page, inner, de, seed + 1 + d) for d, (kind, nb) in enumerate(geoms)]
        self.dst = [DevicePool(h) for h in self.dst_h]
        self.initial = [[b.copy() for b in h.buffers] for h in self.dst_h]
        rng = np.random.default_rng(seed)
        nbs = self.src_h.num_blocks
        if replicate:
            self.sids = [rng.permutation(nbs)[:n]] * len(geoms)
        else:
            self.sids = [rng.permutation(nbs)[:n] for _ in geoms]
        self.dids = dids if dids is not None else [rng.permutation(nb - 1)[:n] for _, nb in geoms]
        assert all(max(did) < nb - 1 for did, (_, nb) in zip(self.dids, geoms))
        nd = len(geoms)
        self.done = torch.zeros(nd, dtype=torch.int32, device="cuda") if flags else None
        self.layer_done = torch.zeros(nd, nl, dtype=torch.int32, device="cuda") if flags else None
        shared = ids_dev(self.sids[0])
        self._keep, self.dsts = [], []
        for d in range(nd):
            s = shared if replicate else ids_dev(self.sids[d])
            t = ids_dev(self.dids[d])
            self._keep += [s, t]
            df = self.done[d:].data_ptr() if flags else 0
            lf = self.layer_done[d].data_ptr() if flags else 0
            self.dsts.append(paged_dst(self.dst[d], s, t, df, lf))

    def upload_src(self):
        for t, b in zip(self.src.bufs, self.src_h.buffers):
            t.copy_(torch.from_numpy(b))
        torch.cuda.synchronize()

    def launch(self, layers=None, opts=None, stream=None):
        lb, le = (0, self.nl) if layers is None else (layers.start, layers.stop)
        return K.paged_copy(self.src.desc, self.dsts, len(self.sids[0]), lb, le, self.cast, opts, stream_ptr(stream))

    def run(self, layers=None, **opt):
        assert self.launch(layers, K.PagedCopyOpts(**opt) if opt else None) == 0
        torch.cuda.synchronize()
        self.check(layers)

    def check(self, layers=None):
        """Every destination pool equals the oracle's result, and its guard block is untouched."""
        for d, (h, pool) in enumerate(zip(self.dst_h, self.dst)):
            got = pool.snapshot()
            O.execute_memcpy_transfer(self.src_h, h, self.sids[d], self.dids[d], layers, cast_mode=self.cast)
            bad = _bad_regions(h, got)
            assert not bad, f"destination {d} ({h.num_blocks} blocks): {len(bad)} regions differ from the oracle, first {bad[:6]}"
            guard = h.num_blocks - 1
            for l in range(h.num_layers):
                for o in range(h.outer_dim):
                    i, off, s = _region_offset(h, self._buf_of(h), guard, l, o)
                    assert np.array_equal(got[i][off:off + s], self.initial[d][i][off:off + s]), f"destination {d}: guard block written"

    @staticmethod
    def _buf_of(h):
        return (lambda l: 0) if h.kind == O.FC else (lambda l: l)


def _bad_regions(h, got):
    """(block, layer, outer) of every region where `got` (device buffers) differs from the host twin `h`, plus a marker when
    bytes outside every region differ."""
    if all(np.array_equal(w, g) for w, g in zip(h.buffers, got)):
        return []
    buf_of = Fanout._buf_of(h)
    bad = []
    for b, l, o in itertools.product(range(h.num_blocks), range(h.num_layers), range(h.outer_dim)):
        i, off, s = _region_offset(h, buf_of, b, l, o)
        if not np.array_equal(h.buffers[i][off:off + s], got[i][off:off + s]):
            bad.append((b, l, o))
    return bad or ["bytes outside every region"]


# ---------------------------------------------------------------------------------------------------------------------
# A. unscaled casts with several destinations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("force_simt", [0, 1], ids=["tma", "simt"])
@pytest.mark.parametrize("replicate", [True, False], ids=["replicate", "distinct"])
@pytest.mark.parametrize("ndst", [2, 3, 8])
@pytest.mark.parametrize("cast", CASTS, ids=lambda c: CAST_IDS[c])
def test_cast_to_several_destinations(cast, ndst, replicate, force_simt):
    # FC, LW block-first and LW block-second destinations with their own num_blocks in one launch; 1 KiB fp8 / 2 KiB bf16
    # regions, one piece each (the default tile is the region)
    layers = range(1, 3) if ndst == 3 else None
    f = Fanout(cast, _mixed(ndst), n=6, replicate=replicate, seed=10 * ndst + 2 * replicate + force_simt + 100 * cast)
    f.run(layers, force_simt=force_simt)


@pytest.mark.parametrize("cast", CASTS, ids=lambda c: CAST_IDS[c])
def test_cast_replicated_to_eight_destinations_through_two_slot_rings(cast):
    """Two slots per ring, eight destinations, 2 048 items over 8 rings: every ring hands each slot back ~128 times, each time
    while its producer waits for that slot.  A consumer that read an item's destinations from the slot after handing it back
    would store some of them at the next item's addresses."""
    f = Fanout(cast, _mixed(8, nb0=260), n=256, replicate=True, nl=4, no=2, page=16, inner=16, seed=7 + cast)
    f.run(stages=2, max_ctas=4, warps_per_cta=4)


@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=23)
    yield m
    torch.cuda.synchronize()
    m.close()


@pytest.mark.parametrize("cast", CASTS, ids=lambda c: CAST_IDS[c])
def test_manager_replicated_fanout_with_a_cast(mgr, cast):
    from tests.test_gpu_permute import _Pool
    nl, no, nt, nh, hd = 3, 2, 16, 2, 64
    se, de = ELEMS[cast]
    src = _Pool(mgr, "LWs", 10, nl, no, nt, nh, hd, se, kv=None)
    randomize(src.twin, 61 + cast)
    src.upload()
    dsts, refs = [], []
    for d, (kind, nb) in enumerate(_mixed(4)):
        p = _Pool(mgr, kind, nb, nl, no, nt, nh, hd, de, kv=None)
        randomize(p.twin, 70 + d)
        p.upload()
        ref = _layout(kind, nb, nl, no, nt, nh * hd, de, 0)
        for r, t in zip(ref.buffers, p.twin.buffers):
            r[:] = t
        dsts.append(p)
        refs.append(ref)
    sids = [9, 2, 5, 0, 7]
    dids = [[int(x) for x in np.random.default_rng(80 + d).permutation(p.twin.num_blocks - 1)[:5]] for d, p in enumerate(dsts)]
    mgr.execute_fanout(src.h, [p.h for p in dsts], [sids] * 4, dids, replicate=True,
                       options=TransferOptions(cast_mode=cast)).wait(20.0)
    for p, ref, did in zip(dsts, refs, dids):
        p.download()
        O.execute_memcpy_transfer(src.twin, ref, sids, did, cast_mode=cast)
        assert not _bad_regions(ref, p.twin.buffers)


# ---------------------------------------------------------------------------------------------------------------------
# B. eight destinations of different geometry, no cast
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layers", [None, range(1, 3)], ids=["all_layers", "layers_1_3"])
@pytest.mark.parametrize("replicate", [True, False], ids=["replicate", "distinct"])
def test_eight_destinations_each_with_its_own_strides(replicate, layers):
    # distinct: the producer picks destination d's base table and strides by an unrolled select; replicate: all eight per item
    f = Fanout(NONE, _mixed(8), n=7, replicate=replicate, nl=4, inner=128, seed=30 + 2 * replicate + (layers is None))
    f.run(layers, tile_bytes=0 if layers is None else 1536)


# ---------------------------------------------------------------------------------------------------------------------
# C. the general ring's run-time options (no cast)
# ---------------------------------------------------------------------------------------------------------------------
RING_DEPTHS = [(2, 1), (3, 1), (3, 2), (16, 1), (16, 2), (16, 15)]   # (stages, stores_in_flight): 1, 2 and S - 1 per depth
RING_CASES = ([(0, i % 4, s, p, fl, nd) for i, ((s, p), fl, nd) in enumerate(itertools.product(RING_DEPTHS, (True, False), (1, 3)))] +
              [(1, h, *RING_DEPTHS[(2 * h + fl) % 6], fl, (1, 3)[(h + fl) % 2]) for h in range(4) for fl in (True, False)])


@pytest.mark.parametrize("variant,cache_hint,stages,in_flight,flags,ndst", RING_CASES,
                         ids=[f"v{v}-hint{h}-S{s}-P{p}-{'flags' if fl else 'noflags'}-ndst{nd}" for v, h, s, p, fl, nd in RING_CASES])
def test_general_ring_options(variant, cache_hint, stages, in_flight, flags, ndst):
    """variant 0 = TMA load + TMA store with deferred slot release (stores_in_flight of them), 1 = TMA load + SIMT store from
    shared memory; cache_hint bit 0 / bit 1 = evict-first loads / stores.  With per-layer flags the consumer publishes each
    layer when it would stall or moves on (publish -> release_upto over the deferred slots).  4 KiB regions in 1 KiB tiles,
    4 layers, 4 rings over 2 CTAs: every ring crosses layers many times."""
    nl, epoch = 4, 5
    f = Fanout(NONE, _mixed(ndst, nb0=14) if ndst > 1 else [("LWs", 14)], n=10, replicate=True, nl=nl, inner=128, flags=flags,
               seed=stages * 31 + in_flight + 7 * variant + cache_hint)
    ws = torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device="cuda") if flags else None
    opts = K.PagedCopyOpts(variant=variant, cache_hint=cache_hint, stages=stages, stores_in_flight=in_flight, tile_bytes=1024,
                           max_ctas=2, warps_per_cta=4, epoch=epoch, sync_workspace=ws.data_ptr() if flags else None)
    assert f.launch(None, opts) == 0
    torch.cuda.synchronize()
    f.check()
    if flags:
        assert f.done.tolist() == [epoch] * ndst
        assert f.layer_done.tolist() == [[epoch] * nl] * ndst
        assert ws.tolist() == [0] * K.sync_workspace_words(nl)


# ---------------------------------------------------------------------------------------------------------------------
# D. the FAST cast kernels at piece edges
# ---------------------------------------------------------------------------------------------------------------------
def _round32(x):
    return (x + 31) // 32 * 32


def _pieces(f, tile, layers=None):
    """{(i, layer, outer): [(source offset, source bytes, TMA?)]} of a single-destination launch of `f`, by the producer's rule
    (copy_engine.cuh): TMA when source, destination and size are multiples of 16 B and, for a cast, the size of whole 32 B."""
    src, dst, cast = f.src, f.dst[0], f.cast
    num, den = {NONE: (1, 1), UP: (2, 1), DOWN: (1, 2)}[cast]
    region = f.src_h.region_size
    tile = _round32(tile if tile else min(max(region, 16), 32768))
    out = {}
    for i, (s, d) in enumerate(zip(f.sids[0], f.dids[0])):
        for l in (layers or range(f.nl)):
            for o in range(f.src_h.outer_dim):
                ps = []
                for soff in range(0, region, tile):
                    n = min(tile, region - soff)
                    sa, da = src.region_addr(int(s), l, o) + soff, dst.region_addr(int(d), l, o) + soff * num // den
                    ps.append((soff, n, ((sa | da | n) & 15) == 0 and (cast == NONE or n & 31 == 0)))
                out[(i, l, o)] = ps
    return out


def test_fast_up_cast_mixes_tma_and_simt_pieces_and_moves_every_code():
    # 1296 B fp8 regions in 1024 B tiles: a TMA piece and a 272 B tail (not whole 32 B vectors) that the consumer converts SIMT;
    # all 256 e4m3 codes sit in both pieces of one region
    f = Fanout(UP, [("LWs", 9)], n=6, replicate=True, page=16, inner=81, seed=41)
    pieces = _pieces(f, 1024)
    assert all([t for _, _, t in ps] == [True, False] for ps in pieces.values())
    codes = np.arange(256, dtype=np.uint8)
    s0 = int(f.sids[0][0])
    f.src_h.region_bytes(s0, 1, 0)[0:256] = codes
    f.src_h.region_bytes(s0, 1, 0)[1024:1280] = codes
    f.upload_src()
    f.run(tile_bytes=1024)
    table = np.load(os.path.join(GOLD, "fp8_e4m3_to_bf16_torch.npy"))
    got = f.dst_h[0].region_bytes(int(f.dids[0][0]), 1, 0).view(np.uint16)
    assert np.array_equal(got[0:256], table) and np.array_equal(got[1024:1280], table)


def test_fast_down_cast_mixes_tma_and_simt_pieces_and_moves_every_pattern():
    # 16 400 B bf16 -> 8 200 B fp8 regions in 4 KiB tiles: four TMA pieces and a 16 B SIMT tail where the fp8 region starts on
    # 16 B, every piece SIMT where it starts 8 B off.  All 65 536 bf16 patterns go through TMA pieces (eight regions' first
    # 16 KiB) and through SIMT pieces (eight misaligned regions).
    f = Fanout(DOWN, [("LWs", 9)], n=6, replicate=True, nl=2, no=2, page=8, inner=1025, seed=43, dids=[np.array([5, 0, 3, 2, 1, 4])])
    pieces = _pieces(f, 4096)
    tma = [k for k, ps in pieces.items() if [t for _, _, t in ps] == [True] * 4 + [False]]
    simt = [k for k, ps in pieces.items() if not any(t for _, _, t in ps)]
    assert len(tma) >= 8 and len(simt) >= 8 and len(tma) + len(simt) == len(pieces)
    pats = np.arange(65536, dtype=np.uint16)
    for j, (i, l, o) in enumerate(tma[:8]):
        f.src_h.region_bytes(int(f.sids[0][i]), l, o).view(np.uint16)[:8192] = pats[j * 8192:(j + 1) * 8192]
    for j, (i, l, o) in enumerate(simt[:8]):
        n = min(8200, 65536 - j * 8200)
        f.src_h.region_bytes(int(f.sids[0][i]), l, o).view(np.uint16)[:n] = pats[j * 8200:j * 8200 + n]
    f.upload_src()
    f.run(tile_bytes=4096)
    # torch's table, except that |x| > 464 (and inf) saturates to +-448 where torch gives NaN (tests/test_oracle_kernels.py)
    table = np.load(os.path.join(GOLD, "bf16_to_fp8_e4m3_torch.npy")).copy()
    overflow = ((table & 0x7F) == 0x7F) & ((pats & 0x7FFF) <= 0x7F80)
    table[overflow] = ((pats[overflow] >> 8) & 0x80).astype(np.uint8) | 0x7E
    via_tma = np.concatenate([f.dst_h[0].region_bytes(int(f.dids[0][i]), l, o)[:8192] for i, l, o in tma[:8]])
    via_simt = np.concatenate([f.dst_h[0].region_bytes(int(f.dids[0][i]), l, o) for i, l, o in simt[:8]])[:65536]
    assert np.array_equal(via_tma, table) and np.array_equal(via_simt, table)


@pytest.mark.parametrize("tile", [0, 32], ids=["whole_region", "tile32"])
@pytest.mark.parametrize("cast", CASTS, ids=lambda c: CAST_IDS[c])
def test_fast_cast_of_odd_regions(cast, tile):
    # page 3 x inner 37: 111 B fp8 / 222 B bf16 regions, every piece SIMT; the up-cast converts an odd number of fp8 bytes
    # (the whole region, or a 15 B last piece in 32 B tiles)
    f = Fanout(cast, [("LWs", 11)], n=7, replicate=True, nl=2, page=3, inner=37, seed=47 + cast + tile)
    assert not any(t for ps in _pieces(f, tile).values() for _, _, t in ps)
    if cast == UP:
        assert any(n & 1 for ps in _pieces(f, tile).values() for _, n, _ in ps)
    f.run(tile_bytes=tile)


# ---------------------------------------------------------------------------------------------------------------------
# E. gated casts with fan-out
# ---------------------------------------------------------------------------------------------------------------------
def _poll(fn, timeout_s=10.0):
    t0 = time.monotonic()
    while not fn():
        if time.monotonic() - t0 > timeout_s:
            return False
        time.sleep(0.002)
    return True


@pytest.mark.parametrize("replicate", [True, False], ids=["replicate", "distinct"])
@pytest.mark.parametrize("gate_mode", [K.GATE_SPIN, K.GATE_STREAM_WAIT], ids=["spin", "stream_wait"])
@pytest.mark.parametrize("cast", CASTS, ids=lambda c: CAST_IDS[c])
def test_gated_cast_fanout_publishes_by_absolute_layer(cast, gate_mode, replicate):
    """Layers [1, nl) of a cast to three destinations, released one at a time.  Each released layer's flag must reach every
    destination at index l; no later layer's flag, no done flag and no completion word may appear before its layer is released."""
    nl, epoch = 5, 3
    f = Fanout(cast, _mixed(3), n=8, replicate=replicate, nl=nl, flags=True, seed=50 + 2 * cast + gate_mode + 5 * replicate)
    ready = torch.zeros(nl, dtype=torch.int32, device="cuda")
    ws = torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device="cuda")
    word = torch.zeros(16, dtype=torch.int32).pin_memory()
    opts = K.PagedCopyOpts(epoch=epoch, layer_ready_flags=ready.data_ptr(), sync_workspace=ws.data_ptr(), gate_mode=gate_mode,
                           completion_flag=word.data_ptr(), completion_value=91, max_ctas=4)
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    assert f.launch(range(1, nl), opts, side) == 0
    completion = lambda: int(word[0])  # noqa: E731
    # while the transfer waits, flags are read with device-to-host copies only (no kernel joins the waiting one)
    seen = []
    try:
        for l in range(1, nl):
            seen.append((l, f.layer_done.cpu()[:, l:].tolist(), f.done.cpu().tolist(), completion()))
            assert K.set_flags(ready.data_ptr(), l, 1, epoch, stream_ptr()) == 0
            if l + 1 < nl:
                assert _poll(lambda: bool((f.layer_done.cpu()[:, l] == epoch).all())), f"layer {l} was never published"
    finally:
        K.set_flags(ready.data_ptr(), 0, nl, epoch, stream_ptr())   # a failed check must not leave the launch waiting
        side.synchronize()
        torch.cuda.synchronize()
    assert all(not np.any(a) and not np.any(b) and c == 0 for _, a, b, c in seen), seen
    assert f.layer_done.tolist() == [[0] + [epoch] * (nl - 1)] * 3
    assert f.done.tolist() == [epoch] * 3 and completion() == 91
    assert ws.tolist() == [0] * K.sync_workspace_words(nl)
    f.check(range(1, nl))


# ---------------------------------------------------------------------------------------------------------------------
# F. routing: every instantiation is reached
# ---------------------------------------------------------------------------------------------------------------------
INSTANTIATION = re.compile(r"kvbm_paged_copy_kernel<\s*(?:\(int\))?(\d)\s*,\s*(true|false)\s*,\s*(true|false)\s*>")


def test_the_matrix_reaches_all_eight_ring_instantiations():
    """One representative case per kvbm_paged_copy_kernel<CAST, FAST, SCALED> under torch.profiler (CUDA activity).  The
    scaled ones run with all-ones scales, whose result is the unscaled oracle's."""
    from torch.profiler import ProfilerActivity, profile
    ones = torch.ones(4 * 2, dtype=torch.float32, device="cuda")
    runs = []
    for cast in (NONE, UP, DOWN):
        runs.append((Fanout(cast, [("LWs", 9)], n=5, replicate=True, nl=4, seed=90 + cast), {}))                # FAST
        runs.append((Fanout(cast, _mixed(2), n=5, replicate=True, nl=4, seed=93 + cast), {}))                   # general
        if cast != NONE:
            runs.append((Fanout(cast, [("LWs", 9)], n=5, replicate=True, nl=4, seed=96 + cast), {"cast_scales": ones.data_ptr()}))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for f, opt in runs:
            assert f.launch(None, K.PagedCopyOpts(**opt) if opt else None) == 0
        torch.cuda.synchronize()
    for f, _ in runs:
        f.check()
    names = {e.name for e in prof.events()}
    found = {(int(m.group(1)), m.group(2) == "true", m.group(3) == "true") for n in names for m in [INSTANTIATION.search(n)] if m}
    want = {(c, fast, False) for c in (NONE, UP, DOWN) for fast in (True, False)} | {(UP, False, True), (DOWN, False, True)}
    assert any("kvbm_paged_copy_kernel" in n for n in names), f"the profiler recorded no paged-copy kernel: {sorted(names)[:20]}"
    assert found == want, f"missing {sorted(want - found)}, names {sorted(n for n in names if 'paged_copy' in n)}"

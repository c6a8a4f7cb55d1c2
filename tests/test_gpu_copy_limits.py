"""The paged copy (kvbm_kernels_paged_copy_v2) and the reference ABI kernels (K1, the v1 fatbin's vectorised_copy, K2 / K3) at
the limits their launchers accept, each next to its first rejected neighbour, and past 4 GiB, against the oracles:

A. regions at the 32-bit top: one region of 2^32 - 16 and 2^32 - 32 768 bytes (TMA and SIMT pieces), below and inside the last
   tile of the largest tile the launcher settles on, both casts, and the manager's largest region (2^32 is refused);
B. the scaled cast's packing of (layer, outer) into one word: 65 536 layers and 32 768 outer indices (plain and gated in both
   gate modes), 65 537 and 32 769 rejected, and a 65 537-layer scaled transfer through the manager;
C. 8 destinations with the scaled casts (9 rejected), and the ring options at their clamps (stages 1 / 17, 16+ warps, stores in
   flight >= stages, 1 and 33 B tiles, one CTA with tickets and with the static schedule) over regions of k tiles, +-16 and +-1 B;
D. the item-count bound: exactly 2^31 items is rejected before any launch.  Its accepted neighbour, 2^31 - 1 items, needs
   about 64 GiB of regions and is not run;
E. K1 and the fatbin on one pair of 4 GiB + 48 B, K2 / K3 on universal blocks of 2^32 - 262 144 B (2^32 is rejected).

The > 4 GiB cases share two device buffers of 4 GiB + 64 KiB: sources are filled from a hash of the word offset, every
destination starts from another fill, and the whole destination buffer, guard bytes past the last region included, is
compared on the device in chunks of 64 MiB (casts through a device lookup table of tests/cast_oracle.py's cast of every fp8 code
and every bf16 pattern).  The small cases compare whole host twins with the numpy oracles.  A rejected neighbour returns
cudaErrorInvalidValue (the manager: its error code) before any launch, so K.launch_count() stays put."""
import os

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import ErrorCode, KvbmError, LayoutConfig, StorageKind, TransferManager, TransferOptions
from tests.cast_oracle import cast_bytes
from tests.gpu_util import dev_ptr_table, ids_dev, stream_ptr
from tests.scaled_cast_oracle import bf16_to_e4m3_scaled, e4m3_to_bf16_scaled
from tests.test_gpu_transform_limits import _fill_words

pytestmark = pytest.mark.gpu
CM = K.CastMode
NONE, UP, DOWN = int(CM.NONE), int(CM.FP8E4M3_TO_BF16), int(CM.BF16_TO_FP8E4M3)
INVAL = K.CUDA_ERROR_INVALID_VALUE
NUM_DEN = {NONE: (1, 1), UP: (2, 1), DOWN: (1, 2)}      # destination bytes = source bytes * num / den
CAST_IDS = {NONE: "none", UP: "fp8_to_bf16", DOWN: "bf16_to_fp8"}


def _rejected(run):
    """run() returns cudaErrorInvalidValue and launches nothing."""
    before = K.launch_count()
    assert run() == INVAL
    assert K.launch_count() == before


# ---------------------------------------------------------------------------------------------------------------------
# two buffers past 4 GiB: A is every source, B every destination
# ---------------------------------------------------------------------------------------------------------------------
GUARD = 1 << 16
BIG = (1 << 32) + GUARD
CHUNK = 1 << 26                     # 64 MiB per device-side fill or comparison
SRC_SALT, DST_SALT = 0, 2 << 30     # word offsets of the two fills' hash (every word index stays below 2^32)


class _Big:
    def __init__(self):
        self.a = torch.empty(BIG, dtype=torch.uint8, device="cuda")
        self.b = torch.empty(BIG, dtype=torch.uint8, device="cuda")
        self.fill(self.a, SRC_SALT)
        self.a_base = torch.tensor([self.a.data_ptr()], dtype=torch.int64, device="cuda")
        self.b_base = torch.tensor([self.b.data_ptr()], dtype=torch.int64, device="cuda")
        codes = np.arange(256, dtype=np.uint8)
        pats = np.arange(65536, dtype=np.uint16)
        self.up = torch.from_numpy(cast_bytes(codes, UP).view(np.int16).copy()).cuda()        # fp8 code -> bf16 bits
        self.down = torch.from_numpy(cast_bytes(pats.view(np.uint8), DOWN).copy()).cuda()    # bf16 bits -> fp8 code

    @staticmethod
    def fill(t, salt):
        w = t.view(torch.int32)
        for s in range(0, w.numel(), CHUNK // 4):
            n = min(CHUNK // 4, w.numel() - s)
            w[s:s + n] = _fill_words(salt + s, n)
        torch.cuda.synchronize()      # the manager's streams do not wait for torch's

    @staticmethod
    def assert_filled(t, lo, salt):
        """Bytes [lo, end) of t (lo a multiple of 4) still hold the fill."""
        w = t.view(torch.int32)
        for s in range(lo // 4, w.numel(), CHUNK // 4):
            n = min(CHUNK // 4, w.numel() - s)
            if not torch.equal(w[s:s + n], _fill_words(salt + s, n)):
                bad = int((w[s:s + n] != _fill_words(salt + s, n)).nonzero()[0]) + s
                raise AssertionError(f"byte {4 * bad} past the last region ({lo}) changed")

    def assert_moved(self, n_src, cast):
        """B's first n_src * num / den bytes are the cast of A's first n_src bytes, and the rest of B keeps its fill."""
        num, den = NUM_DEN[cast]
        n_dst = n_src * num // den
        for s in range(0, n_src, CHUNK):
            e = min(n_src, s + CHUNK)
            src, dst = self.a[s:e], self.b[s * num // den:e * num // den]
            if cast == NONE:
                want = src
            elif cast == UP:
                want = self.up.index_select(0, src.int()).view(torch.uint8)
            else:
                want = self.down.index_select(0, src.view(torch.int16).int() & 0xFFFF)
            if not torch.equal(dst, want):
                bad = int((dst != want).nonzero()[0])
                raise AssertionError(f"destination byte {s * num // den + bad} differs from the oracle")
        self.assert_filled(self.b, n_dst, DST_SALT)

    def region(self, which, nbytes):
        """A one-block, one-layer, one-outer paged layout whose region is A's or B's first nbytes."""
        base = self.a_base if which == "a" else self.b_base
        return K.PagedLayout(base.data_ptr(), nbytes, nbytes, nbytes, 1, 1, 1)


@pytest.fixture(scope="module")
def big():
    free, _ = torch.cuda.mem_get_info()
    if free < 12 * 2**30:
        pytest.skip(f"two {BIG / 2**30:.2f} GiB buffers and their checks want about 12 GiB free; {free / 2**30:.1f} GiB are")
    b = _Big()
    yield b
    b.a = b.b = b.a_base = b.b_base = None
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _one_region_copy(big, n_src, cast, **opt):
    big.fill(big.b, DST_SALT)
    num, den = NUM_DEN[cast]
    ids = ids_dev([0])
    dst = K.PagedDst(big.region("b", n_src * num // den), ids.data_ptr(), ids.data_ptr(), 0, 0)
    rc = K.paged_copy(big.region("a", n_src), [dst], 1, 0, 1, cast, K.PagedCopyOpts(**opt) if opt else None, stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, f"paged copy of one {n_src} B region returned cudaError_t {rc}"
    big.assert_moved(n_src, cast)


# ---------------------------------------------------------------------------------------------------------------------
# A. regions at the 32-bit top
# ---------------------------------------------------------------------------------------------------------------------
def _settled_tile(tile_bytes):
    """The tile make_ring (kvbm_kernels.cu) settles on for an uncast copy asking for tile_bytes: rounded up to 32 B, then halved
    while one ring's slots (at least 2) and control block (1 536 B) do not fit the opt-in shared memory less 1 KiB."""
    budget = torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 1024
    t = (tile_bytes + 31) // 32 * 32
    rings = max(1, min(4, 32768 // t))
    while rings * (1536 + 2 * t) > budget and t > 1024:
        t = (t // 2 + 31) // 32 * 32
    return t


LARGE_TILE = 1 << 20


@pytest.mark.parametrize("force_simt", [0, 1], ids=["tma", "simt"])
@pytest.mark.parametrize("n", [2**32 - 16, 2**32 - 32768], ids=["4GiB_minus_16", "4GiB_minus_32KiB"])
def test_region_at_the_32_bit_top(big, n, force_simt):
    """The default 32 KiB tile: 2^32 - 16 has a last piece of 32 752 B inside the region's last tile (its tile count,
    ceil(n / tile), is 2^17); 2^32 - 32 768 ends on a tile."""
    _one_region_copy(big, n, NONE, force_simt=force_simt)


@pytest.mark.parametrize("where", ["below_the_last_tile", "inside_the_last_tile"])
def test_region_at_the_32_bit_top_with_the_largest_tile(big, where):
    """tile_bytes = 1 MiB settles on 64 KiB on an H100 (two 128 KiB slots do not fit a CTA).  Regions just below 2^32 minus that
    tile, and inside the last tile (2^32 - 32 768, a whole number of default tiles but not of these)."""
    t = _settled_tile(LARGE_TILE)
    n = 2**32 - t - 16 if where == "below_the_last_tile" else 2**32 - t // 2
    assert n % t != 0
    _one_region_copy(big, n, NONE, tile_bytes=LARGE_TILE)


def test_bf16_to_fp8_from_a_region_at_the_32_bit_top(big):
    """A 2^32 - 32 B bf16 region (2^31 - 16 fp8 bytes): its last piece is 32 736 B."""
    _one_region_copy(big, 2**32 - 32, DOWN)


def test_fp8_to_bf16_into_a_region_at_the_32_bit_top(big):
    """A 2^31 - 16 B fp8 region: the destination offsets (twice the source's) pass 2^31 and end at 2^32 - 32; the last piece,
    32 752 B, is not whole 32 B vectors and is converted SIMT."""
    _one_region_copy(big, 2**31 - 16, UP)


@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=61)
    yield m
    torch.cuda.synchronize()
    m.close()


def test_manager_moves_the_largest_region(big, mgr):
    """register_fully_contiguous takes a region of 2^32 - 16 B (one block, layer and outer index of 2^31 - 8 bf16 elements), and
    execute_transfer moves it; bytes_moved counts it."""
    n = 2**32 - 16
    cfg = LayoutConfig(1, 1, 1, 1, n // 2, dtype_width_bytes=2)
    ha = mgr.register_fully_contiguous(cfg, big.a.data_ptr(), BIG, StorageKind.Device, 0)
    hb = mgr.register_fully_contiguous(cfg, big.b.data_ptr(), BIG, StorageKind.Device, 0)
    big.fill(big.b, DST_SALT)
    moved = mgr.bytes_moved()
    mgr.execute_transfer(ha, [0], hb, [0]).wait(60.0)
    torch.cuda.synchronize()
    big.assert_moved(n, NONE)
    assert mgr.bytes_moved() == moved + n


def test_manager_refuses_a_4_gib_region(mgr):
    mem = torch.empty(16, dtype=torch.uint8, device="cuda")
    before = K.launch_count()
    with pytest.raises(KvbmError) as e:
        mgr.register_fully_contiguous(LayoutConfig(1, 1, 1, 1, 2**31, dtype_width_bytes=2), mem.data_ptr(), 2**32,
                                      StorageKind.Device, 0)
    assert e.value.code == ErrorCode.CONFIG and "< 4 GiB" in e.value.msg
    assert K.launch_count() == before


# ---------------------------------------------------------------------------------------------------------------------
# small pools: a fully contiguous pool [block, layer, outer, region] and its host twin
# ---------------------------------------------------------------------------------------------------------------------
class _Fc:
    def __init__(self, nb, nl, no, region, rng, bf16=False):
        shape = (nb, nl, no, region)
        if bf16:                          # a quarter random patterns, the rest values within the scaled casts' reach
            moderate = (rng.standard_normal(shape[:3] + (region // 2,)) * 2.0 ** rng.integers(-6, 7, shape[:3] + (region // 2,)))
            bits = (moderate.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
            mix = rng.random(bits.shape) < 0.25
            bits[mix] = rng.integers(0, 65536, int(mix.sum()), dtype=np.uint16)
            self.host = bits.view(np.uint8).reshape(shape)
        else:
            self.host = rng.integers(0, 256, shape, dtype=np.uint8)
        self.nb, self.nl, self.no, self.region = shape
        self.mem = torch.from_numpy(self.host.reshape(-1).copy()).cuda()
        base = self.mem.data_ptr()
        self.layer_base = torch.tensor([base + l * no * region for l in range(nl)], dtype=torch.int64, device="cuda")
        self.desc = K.PagedLayout(self.layer_base.data_ptr(), nl * no * region, region, region, nl, no, nb)

    def got(self):
        return self.mem.cpu().numpy().reshape(self.host.shape)


def _scales(nl, no, rng):
    """One log-uniform scale in [2^-4, 2^4] per (layer, outer)."""
    return (2.0 ** rng.uniform(-4, 4, nl * no)).astype(np.float32)


def _moved(src, cast, scales):
    """The oracle's bytes of source regions src[..., nl, no, region] after the cast (scales[l * no + o] per region)."""
    if cast == NONE:
        return src
    if scales is None:
        return cast_bytes(src, cast)
    s = scales.reshape(1, src.shape[1], src.shape[2], 1)
    if cast == UP:
        return e4m3_to_bf16_scaled(src, s).view(np.uint8)
    return bf16_to_e4m3_scaled(src.view(np.uint16), s)


class _Copy:
    """One paged copy from a source pool into destination pools of their own block counts (the last block of each is a guard
    no id names).  replicate: every destination takes the same source ids."""

    def __init__(self, cast, region, ndst=1, replicate=True, nl=2, no=2, n=5, seed=0):
        rng = np.random.default_rng(seed)
        num, den = NUM_DEN[cast]
        self.cast, self.n = cast, n
        self.src = _Fc(n + 2, nl, no, region, rng, bf16=cast == DOWN)
        self.dst = [_Fc(n + 1 + 2 * d, nl, no, region * num // den, rng) for d in range(ndst)]
        sids = [int(x) for x in rng.permutation(n + 2)[:n]]
        self.sids = [sids if replicate or d == 0 else [int(x) for x in rng.permutation(n + 2)[:n]] for d in range(ndst)]
        self.dids = [[int(x) for x in rng.permutation(p.nb - 1)[:n]] for p in self.dst]
        s_t = [ids_dev(self.sids[0])] * ndst if replicate else [ids_dev(x) for x in self.sids]
        d_t = [ids_dev(x) for x in self.dids]
        self._keep = s_t + d_t
        self.dsts = [K.PagedDst(p.desc, s.data_ptr(), d.data_ptr(), 0, 0) for p, s, d in zip(self.dst, s_t, d_t)]

    def launch(self, opts=None, dsts=None):
        rc = K.paged_copy(self.src.desc, self.dsts if dsts is None else dsts, self.n, 0, self.src.nl, self.cast, opts, stream_ptr())
        torch.cuda.synchronize()
        return rc

    def check(self, scales=None):
        for d, p in enumerate(self.dst):
            want = p.host.copy()
            want[self.dids[d]] = _moved(self.src.host[self.sids[d]], self.cast, scales)
            got = p.got()
            if not np.array_equal(got, want):
                bad = sorted({tuple(int(v) for v in x[:3]) for x in np.argwhere(got != want)})
                raise AssertionError(f"destination {d}: {len(bad)} (block, layer, outer) regions differ, first {bad[:6]}")


# ---------------------------------------------------------------------------------------------------------------------
# B. the scaled cast's packing bounds: Piece::layer = layer | outer << 16
# ---------------------------------------------------------------------------------------------------------------------
PACKING = {"65536_layers": ((65536, 1), (65537, 1)), "32768_outers": ((1, 32768), (1, 32769))}   # (accepted, rejected)


@pytest.mark.parametrize("cast", [UP, DOWN], ids=lambda c: CAST_IDS[c])
@pytest.mark.parametrize("dims", list(PACKING))
def test_scaled_cast_at_its_packing_bounds(dims, cast):
    """32 B fp8 / 64 B bf16 regions, two blocks; a distinct scale per (layer, outer).  One more layer or outer index is
    rejected."""
    (nl, no), past = PACKING[dims]
    c = _Copy(cast, 32 if cast == UP else 64, nl=nl, no=no, n=2, seed=nl + no + cast)
    scales = _scales(nl, no, np.random.default_rng(cast))
    sc = torch.from_numpy(scales).cuda()
    assert c.launch(K.PagedCopyOpts(cast_scales=sc.data_ptr())) == 0
    c.check(scales)
    nl, no = past
    n = _Copy(cast, 32 if cast == UP else 64, nl=nl, no=no, n=2, seed=3)
    big_sc = torch.ones(nl * no, dtype=torch.float32, device="cuda")
    _rejected(lambda: n.launch(K.PagedCopyOpts(cast_scales=big_sc.data_ptr())))


@pytest.mark.parametrize("gate_mode", [K.GATE_SPIN, K.GATE_STREAM_WAIT], ids=["spin", "stream_wait"])
@pytest.mark.parametrize("cast", [UP, DOWN], ids=lambda c: CAST_IDS[c])
def test_gated_scaled_cast_over_65536_layers(cast, gate_mode):
    """The 65 536-layer scaled cast behind per-layer ready flags, all released before the launch (a stream-wait gate holds its
    hardware queue while it waits).  Every layer_done flag, the done flag and the completion word arrive; the workspace is
    left zeroed."""
    nl, epoch = 65536, 7
    c = _Copy(cast, 32 if cast == UP else 64, nl=nl, no=1, n=2, seed=40 + cast + gate_mode)
    scales = _scales(nl, 1, np.random.default_rng(50 + cast))
    sc = torch.from_numpy(scales).cuda()
    ready = torch.full((nl,), epoch, dtype=torch.int32, device="cuda")
    ws = torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device="cuda")
    layer_done = torch.zeros(nl, dtype=torch.int32, device="cuda")
    done = torch.zeros(1, dtype=torch.int32, device="cuda")
    word = torch.zeros(16, dtype=torch.int32).pin_memory()
    d = c.dsts[0]
    flagged = K.PagedDst(d.layout, d.src_block_ids, d.dst_block_ids, done.data_ptr(), layer_done.data_ptr())
    torch.cuda.synchronize()
    opts = K.PagedCopyOpts(epoch=epoch, layer_ready_flags=ready.data_ptr(), sync_workspace=ws.data_ptr(), gate_mode=gate_mode,
                           completion_flag=word.data_ptr(), completion_value=77, cast_scales=sc.data_ptr())
    assert c.launch(opts, [flagged]) == 0
    c.check(scales)
    assert bool((layer_done == epoch).all()), f"{int((layer_done != epoch).sum())} layer_done flags missing"
    assert int(done[0]) == epoch and int(word[0]) == 77
    assert not bool(ws.any())


def test_manager_reports_a_scaled_transfer_past_the_packing_bound(mgr):
    """The manager does not check the packing bound itself: a 65 537-layer scaled cast stages its tables, then the kernel
    rejects it.  The error is the kernel's, nothing is launched or moved, and the next transfer on the manager completes."""
    nl, rng = 65537, np.random.default_rng(60)
    src, dst = _Fc(3, nl, 1, 32, rng), _Fc(4, nl, 1, 64, rng)
    hs = mgr.register_fully_contiguous(LayoutConfig(3, nl, 1, 16, 2, dtype_width_bytes=1, allow_fp8=True), src.mem.data_ptr(),
                                       src.mem.numel(), StorageKind.Device, 0)
    hd = mgr.register_fully_contiguous(LayoutConfig(4, nl, 1, 16, 2, dtype_width_bytes=2), dst.mem.data_ptr(), dst.mem.numel(),
                                       StorageKind.Device, 0)
    scales = torch.ones(nl, dtype=torch.float32, device="cuda")
    sids, dids = [2, 0], [1, 0]
    moved, launches = mgr.bytes_moved(), K.launch_count()
    with pytest.raises(KvbmError) as e:
        mgr.execute_transfer(hs, sids, hd, dids, options=TransferOptions(cast_mode=UP, cast_scales=scales))
    assert e.value.code == ErrorCode.CUDA
    assert e.value.msg == "kvbm_kernels_paged_copy_v2 failed: cudaErrorInvalidValue (1)"
    torch.cuda.synchronize()
    assert mgr.bytes_moved() == moved and K.launch_count() == launches
    assert np.array_equal(dst.got(), dst.host)
    mgr.execute_transfer(hs, sids, hd, dids, options=TransferOptions(cast_mode=UP)).wait(30.0)
    torch.cuda.synchronize()
    want = dst.host.copy()
    want[dids] = _moved(src.host[sids], UP, None)
    assert np.array_equal(dst.got(), want)
    assert mgr.bytes_moved() == moved + 2 * nl * 64


# ---------------------------------------------------------------------------------------------------------------------
# C. destinations and ring options at their clamps
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("replicate", [True, False], ids=["replicate", "distinct"])
@pytest.mark.parametrize("cast", [UP, DOWN], ids=lambda c: CAST_IDS[c])
def test_scaled_cast_to_eight_destinations(cast, replicate):
    """Eight destinations of their own block counts; 3 056 B regions in 1 KiB tiles (two whole tiles and a 1 008 B piece).
    A ninth destination is rejected."""
    c = _Copy(cast, 3056, ndst=8, replicate=replicate, nl=3, seed=70 + cast + replicate)
    scales = _scales(3, 2, np.random.default_rng(71))
    sc = torch.from_numpy(scales).cuda()
    opts = K.PagedCopyOpts(cast_scales=sc.data_ptr(), tile_bytes=1024)
    assert c.launch(opts) == 0
    c.check(scales)
    _rejected(lambda: c.launch(opts, c.dsts + c.dsts[:1]))


@pytest.mark.parametrize("cast", [NONE, UP, DOWN], ids=lambda c: CAST_IDS[c])
def test_nine_destinations_are_rejected(cast):
    c = _Copy(cast, 64, ndst=1, seed=80 + cast)
    sids = [ids_dev([i] * 5) for i in range(9)]
    distinct = [K.PagedDst(c.dsts[0].layout, t.data_ptr(), c.dsts[0].dst_block_ids, 0, 0) for t in sids]
    _rejected(lambda: c.launch(None, c.dsts * 9))
    _rejected(lambda: c.launch(None, distinct))


# (options, the tile they settle on): every clamp of make_ring and of the launcher
RING_CLAMPS = {
    "stages_1": (dict(stages=1, tile_bytes=1024), 1024),                           # -> 2
    "stages_17": (dict(stages=17, tile_bytes=1024), 1024),                         # -> 16
    "warps_16": (dict(warps_per_cta=16, tile_bytes=1024), 1024),                   # 8 rings
    "warps_17": (dict(warps_per_cta=17, tile_bytes=1024), 1024),                   # -> 16
    "warps_64": (dict(warps_per_cta=64, tile_bytes=1024), 1024),                   # -> 16
    "in_flight_eq_stages": (dict(stages=4, stores_in_flight=4, tile_bytes=1024), 1024),   # -> stages - 1
    "in_flight_past_stages": (dict(stages=3, stores_in_flight=99, tile_bytes=1024), 1024),
    "tile_1": (dict(tile_bytes=1), 32),
    "tile_33": (dict(tile_bytes=33), 64),
    "one_cta_tickets": (dict(max_ctas=1, tile_bytes=1024), 1024),
    "one_cta_static": (dict(max_ctas=1, static_schedule=1, tile_bytes=1024), 1024),
}
CASTS_SCALED = [(NONE, False), (UP, False), (DOWN, False), (UP, True), (DOWN, True)]


@pytest.mark.parametrize("cast,scaled", CASTS_SCALED, ids=[CAST_IDS[c] + ("_scaled" if s else "") for c, s in CASTS_SCALED])
@pytest.mark.parametrize("setting", list(RING_CLAMPS))
def test_ring_options_at_their_clamps(setting, cast, scaled):
    """Regions of 3 tiles, +-16 B and +-1 B (bf16 -> fp8 regions are whole bf16 elements: +-1 is skipped), one destination: the
    unscaled casts run the FAST rings, the scaled ones the general rings."""
    opt, tile = RING_CLAMPS[setting]
    deltas = (-16, 0, 16) if cast == DOWN else (-16, -1, 0, 1, 16)
    for k, delta in enumerate(deltas):
        c = _Copy(cast, 3 * tile + delta, seed=1000 * list(RING_CLAMPS).index(setting) + 100 * cast + 10 * scaled + k)
        scales = _scales(2, 2, np.random.default_rng(k)) if scaled else None
        sc = torch.from_numpy(scales).cuda() if scaled else None
        assert c.launch(K.PagedCopyOpts(**opt, cast_scales=sc.data_ptr() if scaled else None)) == 0, (3 * tile + delta)
        c.check(scales)


# ---------------------------------------------------------------------------------------------------------------------
# D. the item-count bound: items = layers * blocks * outer * (destinations unless replicated) * tiles per region < 2^31
# ---------------------------------------------------------------------------------------------------------------------
ITEMS = {   # (num_layers, num_blocks, outer, distinct destinations, region bytes, tile_bytes)
    "layers_blocks_outer": (2**16, 2**14, 2, 1, 32, 0),
    "destinations": (2**14, 2**14, 1, 8, 32, 0),
    "tiles": (1, 2**16, 1, 1, 2**20, 32),
}


@pytest.mark.parametrize("case", list(ITEMS))
def test_exactly_2_pow_31_items_is_rejected(case):
    """Exactly 2^31 items is rejected before any launch.  Every block and outer index of both sides aliases one region
    (block and outer strides 0, id tables of zeros, every layer at one base), so the launch a wrong bound would let through
    still stays inside its allocations.  The accepted neighbour (2^31 - 1 items) needs about 64 GiB of regions and is not run."""
    nl, nb, no, fan, region, tile = ITEMS[case]
    assert nl * nb * no * fan * -(-region // (tile or 32768)) == 2**31
    mem = torch.zeros(2 * region, dtype=torch.uint8, device="cuda")
    src_base = torch.full((nl,), mem.data_ptr(), dtype=torch.int64, device="cuda")
    dst_base = torch.full((nl,), mem.data_ptr() + region, dtype=torch.int64, device="cuda")
    src = K.PagedLayout(src_base.data_ptr(), 0, 0, region, nl, no, nb)
    dst = K.PagedLayout(dst_base.data_ptr(), 0, 0, region, nl, no, nb)
    ids = [torch.zeros(nb, dtype=torch.int32, device="cuda") for _ in range(fan + 1)]
    dsts = [K.PagedDst(dst, i.data_ptr(), ids[-1].data_ptr(), 0, 0) for i in ids[:fan]]
    _rejected(lambda: K.paged_copy(src, dsts, nb, 0, nl, NONE, K.PagedCopyOpts(tile_bytes=tile), stream_ptr()))


# ---------------------------------------------------------------------------------------------------------------------
# E. K1, the v1 fatbin and K2 / K3 past their 32-bit offsets
# ---------------------------------------------------------------------------------------------------------------------
PAIR = 2**32 + 48


def test_k1_pair_past_4_gib(big):
    """One pair of 4 GiB + 48 B: 131 073 chunks of 32 KiB, the last at byte offset 2^32."""
    big.fill(big.b, DST_SALT)
    st, dt = dev_ptr_table([big.a.data_ptr()]), dev_ptr_table([big.b.data_ptr()])
    assert K.vectorized_copy(st.data_ptr(), dt.data_ptr(), PAIR, 1, stream_ptr()) == 0
    torch.cuda.synchronize()
    big.assert_moved(PAIR, NONE)


def test_v1_fatbin_pair_past_4_gib(big):
    """The same pair through dynamo_b200/vectorized_copy.fatbin, loaded and launched as the v1 block manager does (one CTA for
    one pair, pinned pointer tables)."""
    from cuda.bindings import driver as drv
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dynamo_b200", "vectorized_copy.fatbin")
    big.fill(big.b, DST_SALT)
    err, mod = drv.cuModuleLoadData(open(path, "rb").read())
    assert err == drv.CUresult.CUDA_SUCCESS, err
    try:
        err, fn = drv.cuModuleGetFunction(mod, b"vectorised_copy")
        assert err == drv.CUresult.CUDA_SUCCESS, err
        st = torch.tensor([big.a.data_ptr()], dtype=torch.int64).pin_memory()
        dt = torch.tensor([big.b.data_ptr()], dtype=torch.int64).pin_memory()
        a0, a1, a2 = (np.array([v], dtype=np.uint64) for v in (st.data_ptr(), dt.data_ptr(), PAIR))
        a3 = np.array([1], dtype=np.int32)
        params = np.array([a.ctypes.data for a in (a0, a1, a2, a3)], dtype=np.uint64)
        (err,) = drv.cuLaunchKernel(fn, 1, 1, 1, 256, 1, 1, 0, 0, params.ctypes.data, 0)
        assert err == drv.CUresult.CUDA_SUCCESS, err
        torch.cuda.synchronize()
    finally:
        drv.cuModuleUnload(mod)
    big.assert_moved(PAIR, NONE)


NH, NL, NO, HD = 8, 64, 2, 128
NT = 16383                                    # bf16: 2^32 - 262 144 B per universal block; NT + 1 makes exactly 2^32


@pytest.mark.parametrize("layout", [K.BlockLayout.NHD, K.BlockLayout.HND], ids=["NHD", "HND"])
@pytest.mark.parametrize("to_universal", [True, False], ids=["universal_from_block", "block_from_universal"])
def test_k2_k3_universal_block_at_the_32_bit_top(big, to_universal, layout):
    """One universal block [nh, nl, no, nt, hd] of 2^32 - 262 144 B and its nl * no chunks, laid out back to back in the other
    buffer: A holds the source side, B the destination.  nt = 16 384 (exactly 2^32 B per block) is rejected; the buffers would
    hold that launch too."""
    U = NH * NL * NO * NT * HD * 2
    assert U == 2**32 - 262144
    chunk = U // (NL * NO)
    big.fill(big.b, DST_SALT)
    uni_buf, chunk_buf = (big.b, big.a) if to_universal else (big.a, big.b)
    ut = dev_ptr_table([uni_buf.data_ptr()])
    bt = dev_ptr_table([chunk_buf.data_ptr() + i * chunk for i in range(NL * NO)])
    run = K.universal_from_block if to_universal else K.block_from_universal
    assert run(ut.data_ptr(), bt.data_ptr(), 1, NH, NL, NO, NT, HD, K.TensorDataType.BF16, layout, stream_ptr()) == 0
    torch.cuda.synchronize()
    uni = uni_buf[:U].view(torch.int16).view(NH, NL, NO, NT, HD)
    if layout == K.BlockLayout.NHD:
        chunks = chunk_buf[:U].view(torch.int16).view(NL, NO, NT, NH, HD).permute(3, 0, 1, 2, 4)
    else:
        chunks = chunk_buf[:U].view(torch.int16).view(NL, NO, NH, NT, HD).permute(2, 0, 1, 3, 4)
    for h in range(NH):
        for l0 in range(0, NL, 8):                # 64 MiB of the universal block per comparison
            assert torch.equal(uni[h, l0:l0 + 8], chunks[h, l0:l0 + 8]), f"head {h}, layers {l0}..{l0 + 7}"
    _Big.assert_filled(big.b, U, DST_SALT)
    _Big.assert_filled(big.a, 0, SRC_SALT)
    _rejected(lambda: run(ut.data_ptr(), bt.data_ptr(), 1, NH, NL, NO, NT + 1, HD, K.TensorDataType.BF16, layout, stream_ptr()))

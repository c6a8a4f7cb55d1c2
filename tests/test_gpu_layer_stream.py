"""Layer streaming against a producer that writes the source after the launch.

A gated paged copy is launched once, before the forward pass.  It reads layer l only after layer_ready_flags[l] has reached
`epoch` (the cyclic order (int32)(flag - epoch) >= 0, include/kvbm_kernels.h) and publishes layer_done_flags[l] once layer l
has landed in a destination.  Every case here models the engine that produces the layers:

  * the source pool starts as poison, a seeded pattern whose copy (and cast) differs from the final bytes in every layer;
  * each layer's final bytes are staged on the device beforehand;
  * the gated transfer is launched first, on its own non-blocking stream, with few CTAs so the producer gets SMs;
  * then a producer stream, for each layer in order, sleeps, copies the layer's final bytes into the source (whole buffers of a
    layer-separate pool, a strided view of a fully contiguous one) and releases the layer's ready flag.

The oracle runs on the final source, so a gate that lets a read through early moves poison and the whole-pool comparison (guard
blocks included, as in test_gpu_paged_matrix.Fanout) sees it.  State is observed only through a checker stream that waits for a
flag (kvbm_kernels_wait_flag) and copies the destination aside: the host never synchronizes the device while a ready flag is
unreleased, every host wait has a deadline, and a `finally` releases every flag a launch or the checker could still be waiting
for.  Every torch kernel the producer and the checker use runs once before the first gated launch, so no lazily loaded kernel
waits for a device that a spinning gate keeps busy."""
import time

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from dynamo_b200.physical import ErrorCode, KvbmError, StorageKind, TransferManager, TransferOptions
from oracle import oracle as O
from tests.gpu_util import stream_ptr
from tests.scaled_cast_oracle import cast_bytes_scaled
from tests.test_gpu_manager import Pool
from tests.test_gpu_paged_matrix import CAST_IDS, DOWN, ELEMS, NONE, UP, Fanout, _bad_regions, _layout, _mixed

pytestmark = pytest.mark.gpu

MASK = 0xFFFFFFFF
GATES = [K.GATE_SPIN, K.GATE_STREAM_WAIT]
GATE_IDS = ["spin", "stream_wait"]
GATE_TIMEOUT_MS = 10000
HOST_TIMEOUT_S = 15.0     # longer than the gate timeout: a spinning launch that gave up has finished by then
LAYER_SLEEP = 500_000     # cycles the producer sleeps before each layer's bytes (~0.25 ms at H100 clocks)
CHECKER_SLEEP = 2_000_000  # ~1 ms
# 512 B tiles over 7 blocks x 2 outer: 28 (fp8 source) or 56 (bf16 source) items per layer and destination, not a multiple of
# the tile scheduler's 8-item tickets, so a ring's ticket crosses layers and a ring that waited for one layer meets the next
TILE = 512


def _i32(v):
    """A uint32 value as the int32 a torch.int32 tensor holds."""
    v &= MASK
    return v - (1 << 32) if v >= 1 << 31 else v


def _u32(t):
    """Values of an int32 tensor as uint32, nested like tolist()."""
    x = t.tolist()
    return [_u32_list(r) for r in x] if x and isinstance(x[0], list) else _u32_list(x)


def _u32_list(r):
    return [v & MASK for v in r]


def _layer_t(h, bufs, l):
    """Layer l of a pool on the device: its own buffer when the pool is layer-separate, a strided view [block, layer bytes]
    of a fully contiguous one (blocks outermost)."""
    if h.kind != O.FC:
        return bufs[l]
    return bufs[0].view(h.num_blocks, h.num_layers, -1)[:, l]


def _layer_np(h, bufs, l):
    if h.kind != O.FC:
        return bufs[l]
    return bufs[0].reshape(h.num_blocks, h.num_layers, -1)[:, l]


def _check_fc_order(h):
    if h.kind == O.FC:
        a0, s = h.memory_region(0, 0, 0)
        assert h.memory_region(0, 1, 0)[0] - a0 == h.outer_dim * s and h.memory_region(1, 0, 0)[0] - a0 == h.num_layers * h.outer_dim * s


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


def _scales(nl, no, seed):
    """Distinct scales per (layer, outer): a scale read at the relative layer, or at another outer index, shows up."""
    rng = np.random.default_rng(seed)
    host = (rng.uniform(0.05, 4.0, nl * no) * (1 + np.arange(nl * no) * 1e-2)).astype(np.float32)
    assert len(set(host.tolist())) == nl * no
    return torch.from_numpy(host).to("cuda"), host


def _oracle(src_h, ref, sids, dids, layers, cast, scales=None):
    """The transfer on host twins: `ref` (holding the destination's initial bytes) receives layers `layers` of the blocks."""
    if scales is None:
        O.execute_memcpy_transfer(src_h, ref, [int(x) for x in sids], [int(x) for x in dids], layers, cast_mode=cast)
        return
    no = src_h.outer_dim
    for s, d in zip(sids, dids):
        for l in layers:
            for o in range(no):
                ref.region_bytes(int(d), l, o)[:] = cast_bytes_scaled(src_h.region_bytes(int(s), l, o), cast, float(scales[l * no + o]))


class Producer:
    """The engine side of a source pool: poison and final bytes on the device, the ready flags, and the streams that write the
    layers, observe the destinations and launch the gated transfer."""

    def __init__(self, src_h, src_bufs, poison_h, nl):
        _check_fc_order(src_h)
        self.src_h, self.src_bufs, self.nl = src_h, src_bufs, nl
        self.final = [torch.from_numpy(b.copy()).to("cuda") for b in src_h.buffers]
        self.poison = [torch.from_numpy(b.copy()).to("cuda") for b in poison_h.buffers]
        self.ready = torch.zeros(nl, dtype=torch.int32, device="cuda")
        self.side, self.producer, self.checker = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()

    def poison_source(self):
        for t, p in zip(self.src_bufs, self.poison):
            t.copy_(p)

    def produce(self, layers, epoch):
        """On the producer stream: for each layer, sleep, copy its final bytes into the source, release its flag."""
        with torch.cuda.stream(self.producer):
            for l in layers:
                torch.cuda._sleep(LAYER_SLEEP)
                _layer_t(self.src_h, self.src_bufs, l).copy_(_layer_t(self.src_h, self.final, l))
                K.check(K.set_flags(self.ready.data_ptr(), l, 1, epoch, stream_ptr(self.producer)), "set_flags")

    def warm(self, copies):
        """Run the producer's and the checker's torch kernels once (sleep, each layer copy, and `copies`: (dst, src) pairs the
        checker will copy), then put the poison back."""
        for s in (self.producer, self.checker):
            with torch.cuda.stream(s):
                torch.cuda._sleep(100)
                for l in range(self.nl):
                    _layer_t(self.src_h, self.src_bufs, l).copy_(_layer_t(self.src_h, self.final, l))
                for a, b in copies:
                    a.copy_(b)
        torch.cuda.synchronize()
        self.poison_source()
        torch.cuda.synchronize()

    def wait(self, flag_ptr, value):
        K.check(K.wait_flag(flag_ptr, value, stream_ptr(self.checker)), "wait_flag")

    def rescue(self, epoch, waited_flags=()):
        """Release every ready flag at `epoch` from a fresh stream and let the launch drain.  When the checker still waits
        afterwards (the launch gave up and never published), the flags it waits for ((pointer, count) pairs) are set too."""
        s = torch.cuda.Stream()
        K.set_flags(self.ready.data_ptr(), 0, self.nl, epoch, stream_ptr(s))
        drained = _finish(self.side) and _finish(self.producer)
        if not _finish(self.checker, 1.0 if drained else 0.0):
            for p, c in waited_flags:
                K.set_flags(p, 0, c, epoch, stream_ptr(s))
        assert _finish(self.side) and _finish(self.checker) and _finish(s), "a gated launch or the checker is still waiting"
        torch.cuda.synchronize()


class Rig:
    """A gated kernel-API paged copy (K.paged_copy) from a poisoned source to `geoms` destinations (test_gpu_paged_matrix's
    Fanout: random block tables, a guard block no id names), with its layer_done / done flags, workspace and completion word,
    and the oracle of every destination pool."""

    def __init__(self, cast, geoms, replicate, nl=4, layers=None, scaled=False, src_kind="LWs", seed=0, n=7, no=2, page=16,
                 inner=64):
        self.f = f = Fanout(cast, geoms, n, replicate, nl=nl, no=no, page=page, inner=inner, src_kind=src_kind, flags=True, seed=seed)
        self.cast, self.nl, self.nd, self.geoms, self.shape = cast, nl, len(geoms), geoms, (no, page, inner)
        self.layers = range(nl) if layers is None else layers
        self.scales_t, self.scales_h = _scales(nl, no, seed) if scaled else (None, None)
        for h in f.dst_h:
            _check_fc_order(h)
        poison_h = _layout(src_kind, f.src_h.num_blocks, nl, no, page, inner, ELEMS[cast][0], seed + 977)
        self.p = Producer(f.src_h, f.src.bufs, poison_h, nl)
        self.p.poison_source()
        self.ws = torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device="cuda")
        self.word = torch.zeros(16, dtype=torch.int32).pin_memory()
        self.initial_t = [[t.clone() for t in pool.bufs] for pool in f.dst]
        self.want = [self._expected(f.src_h, d) for d in range(self.nd)]
        for d in range(self.nd):   # the poison is distinct from the final bytes in every streamed layer, also after the cast
            bad = self._expected(poison_h, d)
            for l in self.layers:
                assert not np.array_equal(_layer_np(bad, bad.buffers, l), _layer_np(self.want[d], self.want[d].buffers, l))
        # checker buffers: whole pools, each layer of each pool, the flags
        self.snap = [[torch.empty_like(t) for t in pool.bufs] for pool in f.dst]
        self.lsnap = [[torch.empty(_layer_t(h, pool.bufs, l).shape, dtype=torch.uint8, device="cuda") for l in range(nl)]
                      for h, pool in zip(f.dst_h, f.dst)]
        self.layer_done_snap = torch.empty_like(f.layer_done)
        self.done_snap = torch.empty_like(f.done)
        copies = [(self.layer_done_snap, f.layer_done), (self.done_snap, f.done)]
        for d, (h, pool) in enumerate(zip(f.dst_h, f.dst)):
            copies += list(zip(self.snap[d], pool.bufs))
            copies += [(self.lsnap[d][l], _layer_t(h, pool.bufs, l)) for l in range(nl)]
        self.p.warm(copies)

    def _expected(self, src_h, d):
        """Destination d's pool after the transfer from `src_h`: a host twin holding its initial bytes, through the oracle."""
        kind, nb = self.geoms[d]
        ref = _layout(kind, nb, self.nl, *self.shape, ELEMS[self.cast][1], 0)
        for r, b in zip(ref.buffers, self.f.initial[d]):
            r[:] = b
        _oracle(src_h, ref, self.f.sids[d], self.f.dids[d], self.layers, self.cast, self.scales_h)
        return ref

    # -- flags -----------------------------------------------------------------------------------------------------------
    def set_all_flags(self, value):
        """ready, layer_done and done flags to `value` (the previous round's epoch)."""
        self.p.ready.fill_(_i32(value))
        self.f.layer_done.fill_(_i32(value))
        self.f.done.fill_(_i32(value))

    def layer_done_ptr(self, d, l):
        return self.f.layer_done[d][l:].data_ptr()

    def done_ptr(self, d):
        return self.f.done[d:].data_ptr()

    def waited(self):
        return [(self.f.layer_done.data_ptr(), self.nd * self.nl), (self.f.done.data_ptr(), self.nd)]

    # -- one round ---------------------------------------------------------------------------------------------------------
    def reset(self):
        """Poison the source and put every destination back to its initial bytes (no gated launch is in flight)."""
        self.p.poison_source()
        for pool, init in zip(self.f.dst, self.initial_t):
            for t, u in zip(pool.bufs, init):
                t.copy_(u)
        torch.cuda.synchronize()

    def launch(self, epoch, gate_mode, value, force_simt=0):
        opts = K.PagedCopyOpts(epoch=epoch & MASK, layer_ready_flags=self.p.ready.data_ptr(), sync_workspace=self.ws.data_ptr(),
                               gate_mode=gate_mode, gate_timeout_ms=GATE_TIMEOUT_MS, completion_flag=self.word.data_ptr(),
                               completion_value=value, max_ctas=8, tile_bytes=TILE, force_simt=force_simt,
                               cast_scales=self.scales_t.data_ptr() if self.scales_t is not None else None)
        K.check(self.f.launch(self.layers, opts, self.p.side), "gated paged_copy")

    def snapshot(self, pools=True):
        """On the checker stream: every destination pool and the flags."""
        with torch.cuda.stream(self.p.checker):
            if pools:
                for d, pool in enumerate(self.f.dst):
                    for a, b in zip(self.snap[d], pool.bufs):
                        a.copy_(b)
            self.layer_done_snap.copy_(self.f.layer_done)
            self.done_snap.copy_(self.f.done)

    def snapped(self):
        return [[t.cpu().numpy() for t in s] for s in self.snap]

    # -- checks ------------------------------------------------------------------------------------------------------------
    def check_pools(self, got=None):
        got = got or [pool.snapshot() for pool in self.f.dst]
        for d in range(self.nd):
            bad = _bad_regions(self.want[d], got[d])
            assert not bad, f"destination {d}: {len(bad)} regions differ from the oracle, first {bad[:6]}"

    def check_layers(self, got, released, state):
        """Layers in `released` equal the oracle, every other layer still holds its initial bytes."""
        for d in range(self.nd):
            h = self.f.dst_h[d]
            for l in range(self.nl):
                want = self.want[d].buffers if l in released else self.f.initial[d]
                assert np.array_equal(_layer_np(h, got[d], l), _layer_np(h, want, l)), f"{state}: destination {d} layer {l}"

    def check_end(self, epoch, value, prev=0):
        epoch &= MASK
        f = self.f
        assert _u32(f.layer_done) == [[epoch if l in self.layers else prev for l in range(self.nl)]] * self.nd
        assert _u32(f.done) == [epoch] * self.nd
        assert int(self.word[0]) & MASK == value
        assert self.ws.tolist() == [0] * K.sync_workspace_words(self.nl)
        self.check_pools()

    def stream_all(self, epoch, gate_mode, value, force_simt=0):
        """Launch, produce every layer of the range, finish; the checks are the caller's."""
        try:
            self.launch(epoch, gate_mode, value, force_simt)
            self.p.produce(self.layers, epoch)
            assert _finish(self.p.producer) and _finish(self.p.side), "the gated launch did not finish"
        finally:
            self.p.rescue(epoch & MASK, self.waited())


def _rig_geoms(dsts):
    return {"one": ([("LWs", 11)], True), "three_replicated": (_mixed(3, nb0=11), True), "three_distinct": (_mixed(3, nb0=11), False)}[dsts]


# ---------------------------------------------------------------------------------------------------------------------
# A. an honoured gate through the kernel API
# ---------------------------------------------------------------------------------------------------------------------
# (cast, scaled) x destinations in full, under both gate modes; force_simt, the layer range and the source kind alternate so
# that each value of each appears under both gate modes (30 cases)
CAST_CASES = [(NONE, False), (UP, False), (UP, True), (DOWN, False), (DOWN, True)]
DST_CASES = ["one", "three_replicated", "three_distinct"]
A_CASES = [(g, c, s, dsts, i % 2, (i // 2) % 2 == 1, ("LWs", "FC", "LWf")[i % 3])
           for g in GATES for i, ((c, s), dsts) in enumerate((cs, d) for cs in CAST_CASES for d in DST_CASES)]


@pytest.mark.parametrize("gate_mode,cast,scaled,dsts,force_simt,inner_layers,src_kind", A_CASES,
                         ids=[f"{GATE_IDS[GATES.index(g)]}-{CAST_IDS[c]}{'-scaled' if s else ''}-{d}-{'simt' if fs else 'tma'}-"
                              f"{'layers_1_3' if il else 'all_layers'}-src{k}" for g, c, s, d, fs, il, k in A_CASES])
def test_layers_written_after_the_launch_arrive_whole(gate_mode, cast, scaled, dsts, force_simt, inner_layers, src_kind):
    nl, epoch = 4, 5
    geoms, replicate = _rig_geoms(dsts)
    r = Rig(cast, geoms, replicate, nl=nl, layers=range(1, nl - 1) if inner_layers else None, scaled=scaled, src_kind=src_kind,
            seed=A_CASES.index((gate_mode, cast, scaled, dsts, force_simt, inner_layers, src_kind)))
    r.stream_all(epoch, gate_mode, 61, force_simt)
    r.check_end(epoch, 61)


# ---------------------------------------------------------------------------------------------------------------------
# B. partial release
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 3], ids=["k1", "k_nl_minus_1"])
@pytest.mark.parametrize("cast", [NONE, DOWN], ids=lambda c: CAST_IDS[c])
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_only_released_layers_move(gate_mode, cast, k):
    """Layers < k released: once every destination has published them, they equal the oracle and every later layer still holds
    its initial bytes; no done flag and no completion word has appeared.  Then the rest is released and everything checked."""
    nl, epoch = 4, 9
    r = Rig(cast, _mixed(3, nb0=11), False, nl=nl, seed=200 + 10 * gate_mode + cast + k)
    try:
        r.launch(epoch, gate_mode, 77)
        r.p.produce(range(k), epoch)
        for l in range(k):
            for d in range(r.nd):
                r.p.wait(r.layer_done_ptr(d, l), epoch)
        r.snapshot()
        assert _finish(r.p.checker), f"layers < {k} were never published"
        word_then = int(r.word[0])
        r.p.produce(range(k, nl), epoch)
        assert _finish(r.p.producer) and _finish(r.p.side), "the gated launch did not finish"
    finally:
        r.p.rescue(epoch, r.waited())
    r.check_layers(r.snapped(), range(k), f"after releasing layers < {k}")
    assert _u32(r.layer_done_snap) == [[epoch if l < k else 0 for l in range(nl)]] * r.nd
    assert _u32(r.done_snap) == [0] * r.nd and word_then == 0
    r.check_end(epoch, 77)


# ---------------------------------------------------------------------------------------------------------------------
# C. arrival order
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cast,scaled", [(NONE, False), (UP, True)], ids=["none", "fp8_to_bf16-scaled"])
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_a_layer_has_landed_when_its_flag_appears(gate_mode, cast, scaled):
    """The checker waits for layer_done[d][l] and at once copies destination d's layer l aside; that copy must equal the
    oracle's layer l.  Likewise the whole pool when done_flag[d] appears.  This is timing evidence: a flag published before
    its stores landed is only caught when the copy overtakes the stores, so it can miss such a bug, but a correct kernel
    cannot fail it."""
    nl, epoch = 4, 3
    r = Rig(cast, _mixed(3, nb0=11), False, nl=nl, scaled=scaled, seed=300 + gate_mode + cast)
    try:
        r.launch(epoch, gate_mode, 5)
        with torch.cuda.stream(r.p.checker):
            for l in range(nl):
                for d, (h, pool) in enumerate(zip(r.f.dst_h, r.f.dst)):
                    r.p.wait(r.layer_done_ptr(d, l), epoch)
                    r.lsnap[d][l].copy_(_layer_t(h, pool.bufs, l))
            for d, pool in enumerate(r.f.dst):
                r.p.wait(r.done_ptr(d), epoch)
                for a, b in zip(r.snap[d], pool.bufs):
                    a.copy_(b)
        r.p.produce(range(nl), epoch)
        assert _finish(r.p.producer) and _finish(r.p.side) and _finish(r.p.checker), "the gated launch did not finish"
    finally:
        r.p.rescue(epoch, r.waited())
    for d, h in enumerate(r.f.dst_h):
        for l in range(nl):
            assert np.array_equal(r.lsnap[d][l].cpu().numpy(), _layer_np(h, r.want[d].buffers, l)), f"destination {d} layer {l} at its flag"
    r.check_pools(r.snapped())
    r.check_end(epoch, 5)


# ---------------------------------------------------------------------------------------------------------------------
# D. epoch sequences on the same flags, workspace and pools
# ---------------------------------------------------------------------------------------------------------------------
SEQUENCES = {"1_2_3": (0, [1, 2, 3], NONE), "wrap": (0xFFFFFFFD, [0xFFFFFFFE, 0xFFFFFFFF, 0, 1], DOWN),
             "window_edge": (0, [0x7FFFFFFF], UP)}


@pytest.mark.parametrize("seq", list(SEQUENCES))
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_rounds_of_epochs_on_the_same_flags(gate_mode, seq):
    """Each round launches while the ready and layer-done flags still hold the previous round's epoch and the source is poison
    again.  Before any release a checker that slept ~1 ms must see every destination unchanged and no flag at the new epoch;
    then the round streams as in A.  The wrap crosses 0xFFFFFFFF -> 0; window_edge starts from zeroed flags at 0x7FFFFFFF,
    the largest lag the epoch order allows."""
    prev, epochs, cast = SEQUENCES[seq]
    nl = 4
    r = Rig(cast, _mixed(2, nb0=11), True, nl=nl, seed=400 + gate_mode + cast)
    r.set_all_flags(prev)
    torch.cuda.synchronize()
    for i, epoch in enumerate(epochs):
        value = 100 + i
        r.reset()
        try:
            r.launch(epoch, gate_mode, value)
            with torch.cuda.stream(r.p.checker):
                torch.cuda._sleep(CHECKER_SLEEP)
            r.snapshot()
            assert _finish(r.p.checker), "the checker did not finish"
            word_then = int(r.word[0]) & MASK
            r.p.produce(range(nl), epoch)
            assert _finish(r.p.producer) and _finish(r.p.side), "the gated launch did not finish"
        finally:
            r.p.rescue(epoch, r.waited())
        r.check_layers(r.snapped(), (), f"epoch {epoch:#x} before any release")
        assert _u32(r.layer_done_snap) == [[prev] * nl] * r.nd and _u32(r.done_snap) == [prev] * r.nd, f"epoch {epoch:#x}"
        assert word_then == (value - 1 if i else 0), f"epoch {epoch:#x}: completion word before any release"
        assert _u32(r.p.ready) == [epoch] * nl
        r.check_end(epoch, value)
        prev = epoch


# ---------------------------------------------------------------------------------------------------------------------
# E. the manager path
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def mgr():
    m = TransferManager(device=0, worker_id=31)
    yield m
    torch.cuda.synchronize()
    m.close()


def _mgr_pools(mgr, cast, src_kind, dst_geoms, nl, seed, inner=128):
    se, de = ELEMS[cast]
    src = Pool(mgr, src_kind, 24, StorageKind.Device, nl=nl, inner=inner, dt=se, allow_fp8=se == 1)
    rng = np.random.default_rng(seed)
    for b in src.twin.buffers:
        b[:] = rng.integers(0, 256, b.size, dtype=np.uint8)
    poison = O.Layout(src.twin.kind, 24, nl, 2, 16, inner, se, block_dim=src.twin.c.block_dim, allow_fp8=se == 1)
    for b in poison.buffers:
        b[:] = rng.integers(0, 256, b.size, dtype=np.uint8)
    dsts, refs = [], []
    for kind, nb in dst_geoms:
        p = Pool(mgr, kind, nb, StorageKind.Device, nl=nl, inner=inner, dt=de)
        for b in p.twin.buffers:
            b[:] = rng.integers(0, 256, b.size, dtype=np.uint8)
        p.upload()
        ref = O.Layout(p.twin.kind, nb, nl, 2, 16, inner, de, block_dim=p.twin.c.block_dim)
        for a, b in zip(ref.buffers, p.twin.buffers):
            a[:] = b
        dsts.append(p)
        refs.append(ref)
    prod = Producer(src.twin, src.mem, poison, nl)
    prod.poison_source()
    return src, dsts, refs, prod


@pytest.mark.parametrize("how", ["manager_streams", "caller_stream", "scaled_cast"])
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_manager_transfer_streams_layers(mgr, gate_mode, how):
    """execute_transfer with layer_ready_flags, layer_done_flags and done_flag.  Until the last layer is released the
    notification is not complete (on the manager's streams) and the done flag has not appeared."""
    nl, epoch = 4, 12
    cast = UP if how == "scaled_cast" else NONE
    src, (dst,), (ref,), p = _mgr_pools(mgr, cast, "FC" if how == "caller_stream" else "LWs", [("LWf", 20)], nl, 500 + gate_mode)
    scales_t, scales_h = _scales(nl, 2, 7) if how == "scaled_cast" else (None, None)
    sids, dids = [3, 17, 0, 9, 22, 5], [19, 2, 11, 7, 0, 14]
    _oracle(src.twin, ref, sids, dids, range(nl), cast, scales_h)
    ldone = torch.zeros(nl, dtype=torch.int32, device="cuda")
    done = torch.zeros(1, dtype=torch.int32, device="cuda")
    done_snap = torch.empty_like(done)
    p.warm([(done_snap, done)])
    opts = TransferOptions(layer_ready_flags=p.ready.data_ptr(), layer_done_flags=ldone.data_ptr(), done_flag=done.data_ptr(), epoch=epoch,
                           gate_mode=gate_mode, gate_timeout_ms=GATE_TIMEOUT_MS, max_ctas=8, cast_mode=cast, cast_scales=scales_t,
                           cuda_stream=int(p.side.cuda_stream) if how == "caller_stream" else None)
    try:
        note = mgr.execute_transfer(src.h, sids, dst.h, dids, opts)
        p.produce(range(nl - 1), epoch)
        p.wait(ldone[nl - 2:].data_ptr(), epoch)
        with torch.cuda.stream(p.checker):
            done_snap.copy_(done)
        assert _finish(p.checker), f"layer {nl - 2} was never published"
        complete_early = how != "caller_stream" and note.is_complete()
        p.produce([nl - 1], epoch)
        if how == "caller_stream":
            assert note.is_complete() and _finish(p.side)      # the caller's stream carries the transfer
        else:
            note.wait(HOST_TIMEOUT_S)
        assert _finish(p.producer)
    finally:
        p.rescue(epoch, [(ldone.data_ptr(), nl), (done.data_ptr(), 1)])
    assert not complete_early, "the notification completed before the last layer was released"
    assert done_snap.tolist() == [0]
    assert ldone.tolist() == [epoch] * nl and done.tolist() == [epoch]
    for got, want in zip(dst.bytes(), ref.buffers):
        assert np.array_equal(got, want)


@pytest.mark.parametrize("replicate", [True, False], ids=["replicate", "distinct"])
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
def test_manager_fanout_streams_layers(mgr, gate_mode, replicate):
    """execute_fanout with per_dst_layer_done_flags and per_dst_done_flags to three destinations of different kinds."""
    nl, epoch, nd = 4, 6, 3
    geoms = _mixed(nd, nb0=20)
    src, dsts, refs, p = _mgr_pools(mgr, NONE, "LWs", geoms, nl, 600 + gate_mode + 2 * replicate)
    rng = np.random.default_rng(61)
    base = [int(x) for x in rng.permutation(24)[:7]]
    sids = [base] * nd if replicate else [[int(x) for x in rng.permutation(24)[:7]] for _ in range(nd)]
    dids = [[int(x) for x in rng.permutation(nb - 1)[:7]] for _, nb in geoms]
    for d in range(nd):
        _oracle(src.twin, refs[d], sids[d], dids[d], range(nl), NONE)
    ldone = torch.zeros(nd, nl, dtype=torch.int32, device="cuda")
    done = torch.zeros(nd, dtype=torch.int32, device="cuda")
    done_snap = torch.empty_like(done)
    p.warm([(done_snap, done)])
    opts = TransferOptions(layer_ready_flags=p.ready.data_ptr(), per_dst_layer_done_flags=[ldone[d].data_ptr() for d in range(nd)],
                           per_dst_done_flags=[done[d:].data_ptr() for d in range(nd)], epoch=epoch, gate_mode=gate_mode,
                           gate_timeout_ms=GATE_TIMEOUT_MS, max_ctas=8)
    try:
        note = mgr.execute_fanout(src.h, [q.h for q in dsts], sids, dids, replicate=replicate, options=opts)
        p.produce(range(nl - 1), epoch)
        for d in range(nd):
            p.wait(ldone[d][nl - 2:].data_ptr(), epoch)
        with torch.cuda.stream(p.checker):
            done_snap.copy_(done)
        assert _finish(p.checker), f"layer {nl - 2} was never published"
        complete_early = note.is_complete()
        p.produce([nl - 1], epoch)
        note.wait(HOST_TIMEOUT_S)
        assert _finish(p.producer)
    finally:
        p.rescue(epoch, [(ldone.data_ptr(), nd * nl), (done.data_ptr(), nd)])
    assert not complete_early, "the notification completed before the last layer was released"
    assert done_snap.tolist() == [0] * nd
    assert ldone.tolist() == [[epoch] * nl] * nd and done.tolist() == [epoch] * nd
    for q, ref in zip(dsts, refs):
        bad = _bad_regions(ref, q.bytes())
        assert not bad, bad[:6]


# ---------------------------------------------------------------------------------------------------------------------
# F. two-hop plans
# ---------------------------------------------------------------------------------------------------------------------
def _two_hop(mgr, n, nb, bounce_blocks, seed):
    """test_gpu_manager.test_two_hop_through_a_pinned_bounce_buffer's setup: the destination is registered as another GPU's so
    that disallowing GPU RDMA selects TwoHop{D2H, Pinned, H2D}."""
    src, dst = Pool(mgr, "LWs", nb, StorageKind.Device, nl=3), Pool(mgr, "FC", nb, StorageKind.Device, nl=3)
    far = mgr.register_fully_contiguous(dst.cfg, dst.mem[0].data_ptr(), dst.mem[0].numel(), StorageKind.Device, 1)
    bounce = Pool(mgr, "FC", max(bounce_blocks, 2), StorageKind.Pinned, nl=3)
    rng = np.random.default_rng(seed)
    for b in src.twin.buffers:
        b[:] = rng.integers(0, 256, b.size, dtype=np.uint8)
    src.upload()
    sid, did = [int(x) for x in rng.permutation(nb)[:n]], [int(x) for x in rng.permutation(nb)[:n]]
    ref = O.Layout(O.FC, nb, 3, 2, 16, 128, 2)
    O.execute_memcpy_transfer(src.twin, ref, sid, did)
    return src, dst, far, bounce, sid, did, ref


def test_two_hop_rejects_layer_streaming(mgr):
    """Each chunk's first hop would be a whole gated launch, and each chunk's second hop would announce layers that later
    chunks have not landed: the plan takes no per-layer flag at all."""
    src, dst, far, bounce, sid, did, _ = _two_hop(mgr, 8, 16, 2, 1)
    ready = torch.zeros(3, dtype=torch.int32, device="cuda")
    layer_done = torch.zeros(3, dtype=torch.int32, device="cuda")
    mgr.set_capabilities(allow_gpu_rdma=False)
    try:
        for opt in ({"layer_ready_flags": ready.data_ptr()}, {"layer_done_flags": layer_done.data_ptr()},
                    {"per_dst_layer_done_flags": [layer_done.data_ptr()]}):
            before = K.launch_count()
            with pytest.raises(KvbmError) as e:
                mgr.execute_transfer(src.h, sid, far, did, TransferOptions(bounce_buffer=(bounce.h, [0, 1]), epoch=1, **opt))
            assert e.value.code == ErrorCode.UNSUPPORTED and "layer streaming is not available on two-hop transfers" in e.value.msg, opt
            assert K.launch_count() == before, opt
    finally:
        mgr.set_capabilities(allow_gpu_rdma=True)
        K.set_flags(ready.data_ptr(), 0, 3, 1, stream_ptr(torch.cuda.Stream()))   # a transfer accepted by mistake must not wait
        torch.cuda.synchronize()
    assert layer_done.tolist() == [0] * 3


@pytest.mark.parametrize("flag", ["per_dst_done_flags", "done_flag"])
def test_two_hop_done_flag_follows_the_last_chunk(mgr, flag):
    """64 blocks through 2 bounce blocks: 64 chunks.  A checker that is already waiting for the done flag when the transfer is
    submitted, and then copies the destination, must see every chunk landed."""
    n, nb, epoch = 64, 72, 9
    src, dst, far, bounce, sid, did, ref = _two_hop(mgr, n, nb, 2, 2 + len(flag))
    done = torch.zeros(2, dtype=torch.int32, device="cuda")
    snap = torch.empty_like(dst.mem[0])
    checker = torch.cuda.Stream()
    with torch.cuda.stream(checker):
        snap.copy_(dst.mem[0])
    torch.cuda.synchronize()
    opt = {"per_dst_done_flags": [done[1:].data_ptr()]} if flag == "per_dst_done_flags" else {"done_flag": done[1:].data_ptr()}
    mgr.set_capabilities(allow_gpu_rdma=False)
    try:
        K.check(K.wait_flag(done[1:].data_ptr(), epoch, stream_ptr(checker)))
        with torch.cuda.stream(checker):
            snap.copy_(dst.mem[0])
        note = mgr.execute_transfer(src.h, sid, far, did, TransferOptions(bounce_buffer=(bounce.h, [0, 1]), epoch=epoch, **opt))
        assert _finish(checker), "the done flag never appeared"
        note.wait(HOST_TIMEOUT_S)
    finally:
        mgr.set_capabilities(allow_gpu_rdma=True)
        if not _finish(checker, 5.0):
            K.set_flags(done[1:].data_ptr(), 0, 1, epoch, stream_ptr(torch.cuda.Stream()))
        torch.cuda.synchronize()
    assert done.tolist() == [0, epoch]
    got = snap.cpu().numpy()
    bad = [b for b in range(nb) if not np.array_equal(got.reshape(nb, -1)[b], ref.buffers[0].reshape(nb, -1)[b])]
    assert not bad, f"blocks {bad[:8]} ({len(bad)} of {nb}) had not landed when the done flag appeared"

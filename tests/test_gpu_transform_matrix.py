"""Every instantiation of the permuting and re-paging transform kernels, reached and checked against the oracle; the gated ones
against producers that write the sources after the launch, with batches that span layers; and the scaled cast over the whole
range of scales its header promises.

A. One case per instantiation (100: the paged permute, gather, re-page and re-paging gather, their gated forms, and K2 / K3's
   table and VEC kernels), each built so that the launchers' selection rules must route it there, all launched under
   torch.profiler and compared with the oracle; the kernel names the profiler saw must be exactly the expected set.  A CPU test
   holds the same set against the instantiations the built library contains, so a kernel added later without a case fails.
B. tests/test_gpu_transform_stream.py's Rig discipline (poisoned sources, the launch first, per-layer writes and flag releases,
   the checker stream only, host deadlines, every flag released in a `finally`) for every gated instantiation, for batches of the
   spinning form that cross a layer boundary (the batch formula of gate_args is restated here and each case asserts it spans),
   for a producer that writes layer l + 1 only after the destination published layer l, and for 16 sources over 256 heads.
C. The scaled fp8 <-> bf16 cast at about a thousand scales from 2^-60 to 2^60 (include/kvbm_kernels.h, ptx.cuh make_scale /
   div_by), every bf16 pattern or every fp8 code per scale, through the scaled paged permute and the scaled gated gather.

Every comparison is bit-exact over whole destination pools, guard blocks included."""
import os
import re
import shutil
import subprocess
from functools import lru_cache

import numpy as np
import pytest
import torch

from dynamo_b200 import kernels as K
from oracle import oracle as O
from tests.gpu_util import dev_ptr_table, stream_ptr
from tests.scaled_cast_oracle import cast_bytes_scaled
from tests.test_gpu_layer_stream import _finish
from tests.test_gpu_transform_stream import GATE_IDS, GATES, LAYER_SLEEP, MASK, Rig, _i32

KV = K.KvBlockLayout
CM = K.CastMode
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = [KV.UniversalTP, KV.UniversalPP, KV.OperationalHND, KV.OperationalNHD]
CAST_IDS = {0: "none", 1: "fp8_to_bf16", 2: "bf16_to_fp8"}

# ---------------------------------------------------------------------------------------------------------------------
# the expected instantiations
# ---------------------------------------------------------------------------------------------------------------------
# <CAST, POW2, SCALED> of the walk: scaled only with a cast (with_walk_kernel)
WALKS = [(0, p, False) for p in (True, False)] + [(c, p, s) for c in (1, 2) for p in (True, False) for s in (False, True)]
WALK_FAMILIES = ("kvbm_paged_permute_kernel", "kvbm_paged_gather_kernel", "kvbm_gated_gather_kernel")
REPAGE_FAMILIES = ("kvbm_paged_repage_kernel", "kvbm_paged_repage_gather_kernel", "kvbm_gated_repage_gather_kernel")
EXPECTED = ({(f, w) for f in WALK_FAMILIES for w in WALKS}
            | {(f, w + (pp,)) for f in REPAGE_FAMILIES for w in WALKS for pp in (True, False)}
            | {("kvbm_permute_table_kernel", (p,)) for p in (True, False)}
            | {("kvbm_permute_kernel", (v, t)) for v in (16, 8, 4, 2) for t in (True, False)})
FAMILIES = set(WALK_FAMILIES + REPAGE_FAMILIES + ("kvbm_permute_table_kernel", "kvbm_permute_kernel"))

DEMANGLED = re.compile(r"(kvbm_\w+?_kernel)<([^<>]*)>")
MANGLED = re.compile(r"(kvbm_[a-z0-9_]+?_kernel)I((?:L[ib]\d+E)+)E")


def _arg(a):
    a = a.strip().replace("(int)", "")
    return {"true": True, "false": False}[a] if a in ("true", "false") else int(a)


def _demangled(names):
    """(family, template arguments) of every transform kernel among profiler event names."""
    out = set()
    for n in names:
        for m in DEMANGLED.finditer(n):
            if m.group(1) in FAMILIES:
                out.add((m.group(1), tuple(_arg(a) for a in m.group(2).split(","))))
    return out


def _mangled(names):
    """The same from Itanium-mangled symbol names (L<i|b><value>E per template argument)."""
    out = set()
    for n in names:
        m = MANGLED.search(n)
        if m and m.group(1) in FAMILIES:
            out.add((m.group(1), tuple(int(v) if t == "i" else v == "1" for t, v in re.findall(r"L([ib])(\d+)E", m.group(2)))))
    return out


def _describe(s):
    return sorted(f"{f}<{', '.join(str(a).lower() for a in args)}>" for f, args in s)


def test_the_expected_set_is_what_the_library_contains():
    """The 100 instantiations the profiler test expects are exactly those compiled into libkvbm_kernels.so (cuobjdump, as
    benchmarks/dump_sass.py reads them), and no kernel of the library is a staged twin of one of them."""
    assert len(EXPECTED) == 100
    so = os.path.join(ROOT, "dynamo_b200", "libkvbm_kernels.so")
    tool = shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)
    if not os.path.exists(so) or tool is None:
        pytest.skip("needs the built libkvbm_kernels.so and cuobjdump")
    txt = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    functions = re.findall(r"Function : (\S+)", txt)
    found = _mangled(functions)
    assert found == EXPECTED, f"in the library only: {_describe(found - EXPECTED)}; expected only: {_describe(EXPECTED - found)}"
    # the staged gathers are these gathers with a stage table: no second family of them
    assert not [n for n in functions if "_stage_" in n]


# ---------------------------------------------------------------------------------------------------------------------
# shapes
# ---------------------------------------------------------------------------------------------------------------------
def _hd(pow2, i, mla=False):
    """A head_dim whose walk row (the fp8 side's under a cast) is a power of two of 16 B vectors (64), or is not (80, 96, 48 /
    MLA's 576)."""
    return 64 if pow2 else (80, 96, 576 if mla else 48)[i % 3]


def _mla(hd):
    return dict(srcs=[(1, KV.OperationalNHD)], windows=[(0, 0, 0, 1)], dst_nh=1, no=1)


def gather_spec(i, cast, pow2, scaled, sources, mla=False):
    """sources 1: one source, alternately every head or a window (the paged permute); 2: two sources over a partial cover of
    the destination's heads (the gather)."""
    hd = _hd(pow2, i, mla)
    if hd == 576:
        geo = _mla(hd)
    elif sources == 1:
        geo = dict(srcs=[(4, KV.OperationalHND if i % 2 else KV.OperationalNHD)], windows=[(0, 0, 0, 4)] if i % 2 else [(0, 1, 0, 2)],
                   dst_nh=4 if i % 2 else 3)
    else:
        geo = dict(srcs=[(2, KV.OperationalHND), (3, KV.OperationalNHD)], windows=[(0, 0, 1, 2), (1, 1, 3, 2)], dst_nh=6)
    return dict(geo, dst_kv=KINDS[i % 4], hd=hd, cast=CM(cast), scaled=scaled, seed=100 + i)


def repage_spec(i, cast, pow2, scaled, ppow2, src_small, sources, mla=False):
    """Pages whose smaller one is a power of two (48 / 16) or not (96 / 48, 48 / 6), the source on the small or the big side;
    a token range that starts and ends inside big blocks.  sources 0: a plain re-page (one source, every head of both sides);
    1: one source's window; 2: two sources."""
    big, small = (48, 16) if ppow2 else ((96, 48) if i % 2 else (48, 6))
    ps, pd = (small, big) if src_small else (big, small)
    hd = _hd(pow2, i, mla)
    if hd == 576:
        geo = _mla(hd)
    elif sources == 0:
        geo = dict(srcs=[(3, KV.OperationalNHD)], windows=[(0, 0, 0, 3)], dst_nh=3)
    elif sources == 1:
        geo = dict(srcs=[(4, KV.OperationalHND)], windows=[(0, 1, 0, 3)], dst_nh=3)
    else:
        geo = dict(srcs=[(2, KV.OperationalNHD), (2, KV.OperationalHND)], windows=[(0, 0, 0, 2), (1, 0, 2, 2)], dst_nh=5)
    return dict(geo, dst_kv=KINDS[(i + 1) % 4], hd=hd, cast=CM(cast), scaled=scaled, ps=ps, pd=pd, tokens=(5, 2 * big + big // 2 + 3),
                seed=200 + i)


def gate_grid_batch(per_layer, nlayers, max_ctas):
    """gate_args (kvbm_kernels.cu): the spinning form's grid, min(units, max_ctas), and its batch of consecutive layer-major
    units per ticket, min(8, max(1, ceil(per_layer / (2 grid))))."""
    grid = min(per_layer * nlayers, max_ctas)
    return grid, min(8, max(1, -(-per_layer // (2 * grid))))


def spans_layers(per_layer, nlayers, batch):
    """Whether some batch of `batch` units, claimed in layer-major order, holds units of two layers."""
    total = per_layer * nlayers
    return any(k // per_layer != (min(k + batch, total) - 1) // per_layer for k in range(0, total, batch))


class MRig(Rig):
    """Rig with the unstreamed launch, a spinning launch with every ready flag released before it, and the unit count of a layer."""

    @property
    def per_layer(self):
        if not self.repage:
            return len(self.dids) * self.no
        big = max(self.ps, self.pd)
        return (-(-self.te // big) - self.tb // big) * self.no

    def sources_final(self):
        for p in self.srcs:
            p.buf.copy_(p.final)
        torch.cuda.synchronize()

    def check_pool(self, what):
        got, want = self.dst.buf.cpu().numpy(), self.expected()
        bad = [b for b in range(len(got)) if not np.array_equal(got[b], want[b])]
        assert not bad, f"{what}: destination blocks {bad} differ from the oracle (ids {self.dids.tolist()})"

    def run_unstreamed(self, what):
        self.sources_final()
        dside = self.dst.side(self.dids_t)
        srcs = [K.PermuteSource(self.srcs[s].side(self.sids_t[s]), self.srcs[s].nh, sb, db, k) for s, sb, db, k in self.windows]
        sp = stream_ptr(self.side_stream)
        if self.repage:
            rc = K.paged_repage_gather(srcs, self.ps, dside, self.dst_nh, self.pd, self.tb, self.te, self.lb, self.le, self.row, self.cast,
                                       self.scales, stream=sp)
        else:
            rc = K.paged_permute_gather(srcs, dside, self.dst_nh, len(self.dids), self.lb, self.le, self.ps, self.row, self.cast,
                                        stream=sp, cast_scales=self.scales)
        K.check(rc, what)
        assert _finish(self.side_stream), f"{what} did not finish"
        self.check_pool(what)

    def run_released(self, what, epoch=3, value=4):
        self.sources_final()
        for p in self.srcs:
            p.ready.fill_(epoch)
        torch.cuda.synchronize()
        try:
            self.launch(epoch, K.GATE_SPIN, value)
            assert _finish(self.side_stream), f"{what} did not finish"
        finally:
            self.rescue(epoch)
        self.check_pool(what)
        self.check_end(epoch, value)


# ---------------------------------------------------------------------------------------------------------------------
# A. every instantiation reached and checked
# ---------------------------------------------------------------------------------------------------------------------
def a_cases():
    """(family, template arguments, how, Rig arguments) per instantiation of the walk and re-paging families."""
    out = []
    for i, w in enumerate(WALKS):
        c, p, s = w
        out.append(("kvbm_paged_permute_kernel", w, "unstreamed", gather_spec(i, c, p, s, 1)))
        out.append(("kvbm_paged_gather_kernel", w, "unstreamed", gather_spec(i + 1, c, p, s, 2)))
        out.append(("kvbm_gated_gather_kernel", w, "released", gather_spec(i + 2, c, p, s, 1 + i % 2)))
        for pp in (True, False):
            ss = (i + pp) % 2 == 1   # the source on either side, for both kinds of small page, in every family
            out.append(("kvbm_paged_repage_kernel", w + (pp,), "unstreamed", repage_spec(i, c, p, s, pp, ss, 0)))
            out.append(("kvbm_paged_repage_gather_kernel", w + (pp,), "unstreamed", repage_spec(i + 1, c, p, s, pp, not ss, 1 + i % 2)))
            out.append(("kvbm_gated_repage_gather_kernel", w + (pp,), "released", repage_spec(i + 2, c, p, s, pp, ss, i % 3)))
    return out


# K2 / K3 on pointer tables: (kernel, template arguments without TO_UNIVERSAL) -> head_dim in F16 (dims nh, nl, no, nt).  The
# table kernel takes rows of whole 16 B vectors up to 64 KiB; past that, or on other rows, the VEC kernel of the widest vector
# dividing the row.
K23 = {("kvbm_permute_table_kernel", (True,)): (64, (3, 2, 2, 16)), ("kvbm_permute_table_kernel", (False,)): (80, (3, 2, 2, 16)),
       ("kvbm_permute_kernel", (16,)): (32776, (1, 1, 2, 1)), ("kvbm_permute_kernel", (8,)): (4, (3, 2, 2, 5)),
       ("kvbm_permute_kernel", (4,)): (6, (3, 2, 2, 5)), ("kvbm_permute_kernel", (2,)): (3, (3, 2, 2, 5))}


def run_k23(hd, dims, layout, seed):
    """universal_from_block then block_from_universal over two blocks of F16, each result against the oracle (kv_layout_permute:
    a block's chunks in (layer, outer) order are an operational block, its universal buffer UniversalTP)."""
    nh, nl, no, nt = dims
    row, nb = 2 * hd, 2
    chunk = nt * nh * row
    kvc = O.KV_OPERATIONAL_NHD if layout == K.BlockLayout.NHD else O.KV_OPERATIONAL_HND
    rng = np.random.default_rng(seed)
    blocks = rng.integers(0, 256, (nb, nl * no * chunk), dtype=np.uint8)
    unis = np.stack([O.kv_layout_permute(b, kvc, O.KV_UNIVERSAL_TP, nl, no, nt, nh, row) for b in blocks])
    d_chunks = torch.from_numpy(blocks).cuda()
    d_unis = torch.full(unis.shape, 0xDE, dtype=torch.uint8, device="cuda")
    bt = dev_ptr_table([d_chunks.data_ptr() + i * chunk for i in range(nb * nl * no)])
    ut = dev_ptr_table([d_unis[b].data_ptr() for b in range(nb)])
    sp = stream_ptr()
    K.check(K.universal_from_block(ut.data_ptr(), bt.data_ptr(), nb, nh, nl, no, nt, hd, K.TensorDataType.F16, layout, sp), "K2")
    torch.cuda.synchronize()
    assert np.array_equal(d_unis.cpu().numpy(), unis), f"K2 head_dim {hd}"
    d_chunks.fill_(0xDE)
    K.check(K.block_from_universal(ut.data_ptr(), bt.data_ptr(), nb, nh, nl, no, nt, hd, K.TensorDataType.F16, layout, sp), "K3")
    torch.cuda.synchronize()
    assert np.array_equal(d_chunks.cpu().numpy(), blocks), f"K3 head_dim {hd}"


@pytest.mark.gpu
def test_every_transform_instantiation_is_reached_and_matches_the_oracle():
    from torch.profiler import ProfilerActivity, profile
    cases = a_cases()
    assert {(f, a) for f, a, _, _ in cases} | {(f, a + (t,)) if f == "kvbm_permute_kernel" else (f, a) for f, a in K23
                                                for t in (True, False)} == EXPECTED
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for f, args, how, spec in cases:
            what = f"{f}<{', '.join(str(a).lower() for a in args)}>"
            r = MRig(**spec)
            if how == "unstreamed":
                r.run_unstreamed(what)
            else:
                r.run_released(what)
            del r
        for i, ((f, args), (hd, dims)) in enumerate(K23.items()):
            run_k23(hd, dims, (K.BlockLayout.NHD, K.BlockLayout.HND)[i % 2], 300 + i)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    found = _demangled(names)
    assert found, f"the profiler recorded no transform kernel: {sorted(names)[:20]}"
    assert found == EXPECTED, f"never reached: {_describe(EXPECTED - found)}; unexpected: {_describe(found - EXPECTED)}"


# ---------------------------------------------------------------------------------------------------------------------
# B. the gated kernels against producers that write after the launch
# ---------------------------------------------------------------------------------------------------------------------
def b1_cases():
    """One case per gated instantiation: head_dim 64 or 80 / 96 / MLA's 576 (one head, one outer index), scaled casts over an
    inner layer range (scales differ per (layer, outer), so one read at the relative layer shows), 1 .. 3 CTAs."""
    out = []
    for i, w in enumerate(WALKS):
        c, p, s = w
        extra = dict(layers=range(1, 4), nl=4) if s else {}
        spec = dict(gather_spec(i, c, p, s, 1 + (i + 1) % 2, mla=True), n=5, max_ctas=1 + i % 3, **extra)
        out.append(("gather", w, spec))
        for pp in (True, False):
            spec = dict(repage_spec(i, c, p, s, pp, (i + pp) % 2 == 0, 1 + i % 2, mla=True), max_ctas=1 + (i + pp) % 3, **extra)
            out.append(("repage_gather", w + (pp,), spec))
    return out


B1 = b1_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("kind,args,spec", B1, ids=[f"{k}-{CAST_IDS[a[0]]}-{'pow2' if a[1] else 'mulhi'}{'-scaled' if a[2] else ''}"
                                                     f"{('-page_pow2' if a[3] else '-page_mulhi') if len(a) > 3 else ''}" for k, a, _ in B1])
def test_every_gated_instantiation_under_a_late_producer(gate_mode, kind, args, spec):
    r = MRig(**spec)
    r.warm()
    r.run(5, gate_mode, 77)
    r.check_end(5, 77)


# per_layer 3 / 5 / 7 (and 14 with two outer indices) at 1 .. 3 CTAs, an inner layer range, and a grid clamped to the units
SPAN = {
    "gather_pl3_ctas1": dict(gather_spec(0, 0, True, False, 2), n=3, no=1, max_ctas=1),
    "gather_pl5_ctas2": dict(gather_spec(1, 2, False, False, 2), n=5, no=1, max_ctas=2),
    "gather_pl7_ctas3": dict(gather_spec(2, 1, True, False, 1), n=7, no=1, max_ctas=3),
    "gather_pl14_ctas2_layers_1_4_scaled": dict(gather_spec(3, 1, False, True, 2), n=7, no=2, nl=5, layers=range(1, 4), max_ctas=2),
    "gather_clamped": dict(gather_spec(4, 0, True, False, 2), n=3, no=1, nl=2, max_ctas=64),
    "repage_48_16_pl3_ctas1": dict(repage_spec(0, 0, True, False, True, False, 2), no=1, tokens=(5, 2 * 48 + 29), max_ctas=1),
    "repage_16_48_pl5_ctas2": dict(repage_spec(1, 2, True, False, True, True, 2), no=1, tokens=(20, 4 * 48 + 30), max_ctas=2),
    "repage_6_48_pl7_ctas3_layers_1_4_scaled": dict(repage_spec(2, 2, False, True, False, True, 2), ps=6, pd=48, no=1, nl=5,
                                                    tokens=(7, 6 * 48 + 11), layers=range(1, 4), max_ctas=3),
    "repage_96_48_pl3_ctas1_scaled": dict(repage_spec(3, 1, True, True, False, False, 1), ps=96, pd=48, no=1, tokens=(50, 2 * 96 + 40),
                                          max_ctas=1),
    "repage_clamped": dict(repage_spec(4, 0, False, False, True, False, 2), no=1, nl=2, tokens=(5, 40), max_ctas=64),
}


@pytest.mark.gpu
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("name", list(SPAN))
def test_batches_that_span_layers(gate_mode, name):
    """A CTA whose batch crosses from layer l into l + 1 must publish its units of l, gate on l + 1 for every source, then go on;
    the producers release layers ~0.15 ms apart, so a batch that reads l + 1 before its flags moves poison.  A clamped grid
    (more CTAs allowed than units) always takes batches of one unit."""
    r = MRig(**SPAN[name])
    nlay = r.le - r.lb
    grid, batch = gate_grid_batch(r.per_layer, nlay, r.max_ctas)
    if "clamped" in name:
        assert grid == r.per_layer * nlay < r.max_ctas and batch == 1
    else:
        assert spans_layers(r.per_layer, nlay, batch), f"per_layer {r.per_layer}, grid {grid}, batch {batch}: no batch spans layers"
    r.warm()
    r.run(6, gate_mode, 88)
    r.check_end(6, 88)


class LockstepRig(MRig):
    """One producer stream for every source that writes layer l + 1 only after its stream waited for the destination's
    layer_done[l]: a receiver that releases layer l + 1 only after seeing layer l done.  The producer stream is created right
    after a fresh launch stream, so the two sit on different hardware queues (the stream-wait form's wait holds its queue)."""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.side_stream = torch.cuda.Stream()
        self.producer = torch.cuda.Stream()

    def warm(self):
        super().warm()
        with torch.cuda.stream(self.producer):
            torch.cuda._sleep(100)
            for p in self.srcs:
                for l in range(self.nl):
                    p.layer(p.buf, l).copy_(p.layer(p.final, l))
        torch.cuda.synchronize()
        self.reset()

    def run_lockstep(self, epoch, gate_mode, value):
        sp = stream_ptr(self.producer)
        try:
            self.launch(epoch, gate_mode, value)
            with torch.cuda.stream(self.producer):
                for l in range(self.nl):
                    if l > self.lb:
                        K.check(K.wait_flag(self.layer_done.data_ptr() + 4 * (l - 1), epoch, sp), "wait_flag")
                    torch.cuda._sleep(LAYER_SLEEP)
                    for p in self.srcs:
                        p.layer(p.buf, l).copy_(p.layer(p.final, l))
                        K.check(K.set_flags(p.ready.data_ptr(), l, 1, epoch, sp), "set_flags")
            assert _finish(self.producer) and _finish(self.side_stream), "the lockstep transfer did not finish"
        finally:
            s = torch.cuda.Stream()
            for p in self.srcs:
                K.set_flags(p.ready.data_ptr(), 0, self.nl, epoch & MASK, stream_ptr(s))
            if not (_finish(self.side_stream) and _finish(self.producer, 2.0)):
                K.set_flags(self.layer_done.data_ptr(), 0, self.nl, epoch & MASK, stream_ptr(s))
            assert _finish(s) and _finish(self.producer) and _finish(self.side_stream), "a launch or the producer is still waiting"
            torch.cuda.synchronize()


LOCKSTEP = {
    "gather_3_sources_pl5_ctas2": dict(srcs=[(2, KV.OperationalNHD), (1, KV.OperationalHND), (2, KV.OperationalHND)],
                                       windows=[(0, 0, 0, 2), (1, 0, 2, 1), (2, 0, 3, 2)], dst_nh=5, dst_kv=KV.UniversalPP, n=5, no=1,
                                       nl=5, max_ctas=2, cast=CM.FP8E4M3_TO_BF16, scaled=True),
    "repage_gather_6_48_2_sources_pl7_ctas3": dict(srcs=[(2, KV.OperationalHND), (2, KV.OperationalNHD)],
                                                   windows=[(0, 0, 0, 2), (1, 0, 2, 2)], dst_nh=4, dst_kv=KV.OperationalNHD, ps=6, pd=48,
                                                   tokens=(7, 6 * 48 + 11), no=1, nl=5, hd=80, max_ctas=3),
}


@pytest.mark.gpu
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("name", list(LOCKSTEP))
def test_a_lockstep_producer_never_waits_forever(gate_mode, name):
    r = LockstepRig(**LOCKSTEP[name], seed=len(name))
    grid, batch = gate_grid_batch(r.per_layer, r.le - r.lb, r.max_ctas)
    assert spans_layers(r.per_layer, r.le - r.lb, batch)
    r.warm()
    r.run_lockstep(9, gate_mode, 90)
    r.check_end(9, 90)


# 16 sources of 16 heads each, 256 covered heads: 8 warps loop 32 heads each
MAXIMA = {
    "gather": dict(srcs=[(16, KV.OperationalNHD if s % 2 else KV.OperationalHND) for s in range(16)],
                   windows=[(s, 0, 16 * s, 16) for s in range(16)], dst_nh=256, dst_kv=KV.UniversalTP, n=5, no=1, nl=4, max_ctas=2),
    "repage_gather_16_48": dict(srcs=[(16, KV.OperationalHND if s % 2 else KV.OperationalNHD) for s in range(16)],
                                windows=[(s, 0, 16 * s, 16) for s in range(16)], dst_nh=256, dst_kv=KV.OperationalNHD, ps=16, pd=48,
                                tokens=(5, 2 * 48 + 29), no=1, nl=4, max_ctas=1, cast=CM.BF16_TO_FP8E4M3, scaled=True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("gate_mode", GATES, ids=GATE_IDS)
@pytest.mark.parametrize("name", list(MAXIMA))
def test_sixteen_sources_over_256_heads_on_skewed_schedules(gate_mode, name):
    r = MRig(**MAXIMA[name], seed=7 + len(name))
    grid, batch = gate_grid_batch(r.per_layer, r.le - r.lb, r.max_ctas)
    assert spans_layers(r.per_layer, r.le - r.lb, batch)
    r.warm()
    r.run(11, gate_mode, 12, lag=[s % 4 for s in range(16)])
    r.check_end(11, 12)


# ---------------------------------------------------------------------------------------------------------------------
# C. the scaled cast from 2^-60 to 2^60
# ---------------------------------------------------------------------------------------------------------------------
NL_SWEEP, NO_SWEEP = 256, 4


@lru_cache(maxsize=None)
def sweep_scales():
    """1024 float32 scales, one per (layer, outer): both ends of [2^-60, 2^60] and the float just inside each, every power of two
    between them, 1 +- 1 ulp, and log-uniform values with full random mantissas from a fixed seed."""
    f = np.float32
    lo, hi = f(2.0 ** -60), f(2.0 ** 60)
    fixed = [lo, hi, np.nextafter(lo, f(np.inf)), np.nextafter(hi, f(0))] + [f(2.0 ** e) for e in range(-60, 61)]
    fixed += [np.nextafter(f(1), f(2)), np.nextafter(f(1), f(0))]
    vals = list(dict.fromkeys(float(v) for v in fixed))
    rng = np.random.default_rng(2026)
    while len(vals) < NL_SWEEP * NO_SWEEP:
        bits = ((rng.integers(-60, 60) + 127) << 23) | int(rng.integers(0, 1 << 23))
        v = float(np.array([bits], dtype=np.uint32).view(np.float32)[0])
        if v not in vals:
            vals.append(v)
    out = np.array(vals, dtype=np.float32)
    assert out.min() == lo and out.max() == hi and len(out) == NL_SWEEP * NO_SWEEP
    return out


def _sweep_geometry(cast):
    """(head_dim, source bytes of one region): every bf16 pattern (16 tokens x 4096) or every fp8 code (16 tokens x 16)."""
    if cast == CM.BF16_TO_FP8E4M3:
        return 4096, np.arange(1 << 16, dtype=np.uint16).view(np.uint8)
    return 16, np.arange(256, dtype=np.uint8)


@lru_cache(maxsize=None)
def sweep_expected(cast):
    """The destination regions, [nl * no, region bytes], through scaled_cast_oracle (numpy's IEEE float32 product / quotient)."""
    _, region = _sweep_geometry(cast)
    return np.stack([cast_bytes_scaled(region, int(cast), float(s)) for s in sweep_scales()])


class _Flat:
    """One fully contiguous pool of nb blocks [nl, no, region] with one head, as a PermuteSide over block ids `ids`."""

    def __init__(self, data, nl, no, ids, page, row):
        self.buf = data
        self.region = page * row
        base = data.data_ptr()
        self.layer_base = torch.tensor([base + l * no * self.region for l in range(nl)], dtype=torch.int64, device="cuda")
        self.ids = torch.tensor(ids, dtype=torch.int32, device="cuda")
        self.side = K.PermuteSide(K.PagedLayout(self.layer_base.data_ptr(), nl * no * self.region, self.region, self.region, nl, no,
                                                data.shape[0]), self.ids.data_ptr(), KV.OperationalNHD)


def _sweep_check(cast, got, guard):
    want = sweep_expected(cast)
    blk = got[1].reshape(want.shape)
    assert np.array_equal(got[0], guard), "the guard block changed"
    bad = [i for i in range(len(want)) if not np.array_equal(blk[i], want[i])]
    if bad:
        s = sweep_scales()
        detail = [(float(s[i]), int(np.count_nonzero(blk[i] != want[i]))) for i in bad[:8]]
        pytest.fail(f"{len(bad)} of {len(want)} scales give codes other than IEEE division's; (scale, differing bytes): {detail}")


@pytest.mark.gpu
@pytest.mark.parametrize("gated", [False, True], ids=["paged_permute", "gated_gather"])
@pytest.mark.parametrize("cast", [CM.BF16_TO_FP8E4M3, CM.FP8E4M3_TO_BF16], ids=["bf16_to_fp8", "fp8_to_bf16"])
def test_the_scaled_cast_over_the_whole_documented_range(cast, gated):
    """One scaled launch over 1024 (layer, outer) regions, each with its own scale and every input pattern; the gated form runs
    the kvbm_gated_gather_kernel instantiation with every ready flag released."""
    hd, region = _sweep_geometry(cast)
    se, de = {CM.BF16_TO_FP8E4M3: (2, 1), CM.FP8E4M3_TO_BF16: (1, 2)}[cast]
    nl, no, page = NL_SWEEP, NO_SWEEP, 16
    src_data = torch.from_numpy(np.tile(region, nl * no)).cuda().view(1, -1)
    rng = np.random.default_rng(5)
    dst_init = rng.integers(0, 256, (2, nl * no * page * hd * de), dtype=np.uint8)
    dst_data = torch.from_numpy(dst_init).cuda()
    src, dst = _Flat(src_data, nl, no, [0], page, hd * se), _Flat(dst_data, nl, no, [1], page, hd * de)
    scales = torch.from_numpy(sweep_scales()).cuda()
    torch.cuda.synchronize()
    if not gated:
        K.check(K.paged_permute_heads(src.side, dst.side, 1, 0, nl, 1, 0, 1, 0, 1, page, hd * se, int(cast), stream=stream_ptr(),
                                      cast_scales=scales), "scaled paged permute")
        torch.cuda.synchronize()
    else:
        epoch, value = 2, 3
        ready = torch.full((nl,), epoch, dtype=torch.int32, device="cuda")
        layer_done = torch.zeros(nl, dtype=torch.int32, device="cuda")
        flags = torch.zeros(2, dtype=torch.int32, device="cuda")
        ws = torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device="cuda")
        st = K.PermuteStream()
        st.layer_ready_flags[0] = ready.data_ptr()
        st.layer_done_flags, st.done_flag, st.completion_flag = layer_done.data_ptr(), flags.data_ptr(), flags[1:].data_ptr()
        st.epoch, st.completion_value, st.sync_workspace = epoch, value, ws.data_ptr()
        st.gate_mode, st.gate_timeout_ms = K.GATE_SPIN, 10000
        side = torch.cuda.Stream()
        torch.cuda.synchronize()
        K.check(K.paged_permute_gather_streamed([K.PermuteSource(src.side, 1, 0, 0, 1)], dst.side, 1, 1, 0, nl, page, hd * se, int(cast),
                                                scales, st, stream_ptr(side)), "scaled gated gather")
        assert _finish(side), "the gated gather did not finish"
        torch.cuda.synchronize()
        assert layer_done.tolist() == [epoch] * nl and flags.tolist() == [epoch, value]
        assert not ws.any().item()
    _sweep_check(cast, dst_data.cpu().numpy(), dst_init[0])

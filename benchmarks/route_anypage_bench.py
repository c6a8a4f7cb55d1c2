"""Routed re-paging between pages that need not divide (kvbm_kernels_paged_repage_scatter_routed_anypage and
kvbm_kernels_paged_stage_repage_gather_routed_anypage), timed against the workarounds the library offered before them.

Shapes: Llama-3-70B (80 layers, K/V, 8 KV heads of 128) and an MLA latent head (61 layers, one 576-wide head), every pool on one
GPU, fully contiguous OperationalNHD with random block tables, bf16.  Sequence i of a batch belongs to worker i % W.
  push  prefill rank 0 into W decode workers: TP2 -> 2 x TP16 (8 windows per worker, 16 targets), TP1 -> 2 x TP8 (16 targets),
        MLA to 8 DP ranks (one window each);
  pull  decode rank 0 from W prefill workers: 8 x TP2 -> TP16 and 8 x TP1 -> TP8 (one window per worker), MLA from 8 DP ranks;
  pages 544 -> 64, 48 -> 64 and 24 -> 16 (the pull: the reverse of the decode side's page); batches 8 x 2048, 32 x 512,
  128 x 128 and a mixed batch (1 to 4000 tokens, each starting inside a block).
Arms, alternating inside each of --rounds rounds, timed with CUDA events (median of --iters calls per round):
  routed     one routed anypage launch
  per_worker one anypage launch per worker over its sequences (kvbm_kernels_paged_repage_scatter_anypage /
             kvbm_kernels_paged_stage_repage_gather_anypage), each with its own tables
  two_pass   two dividing launches through a staging pool of page gcd(Ps, Pd): push, a batch re-page Ps -> gcd then the routed
             scatter gcd -> Pd; pull, the routed gather Ps -> gcd then a batch re-page gcd -> Pd.  Every byte moves twice.
Two more comparisons: with every mask full, the routed push against kvbm_kernels_paged_repage_scatter_anypage (the cost of
routing); at the dividing pair 512 -> 64, the routed anypage push against kvbm_kernels_paged_repage_scatter_routed (the cost of
the phase).
Tail (TP2 -> 2 x TP16, 8 x 2048, 544 -> 64 and 48 -> 64; --no-tail skips it): the exposed tail behind an emulated prefill that runs
--layer-us of busy kernel per layer, enqueued from its own host thread, from its last ready flag to the end of the transfer, in both
gate forms: the routed push streamed against one streamed anypage push per worker on one stream.  Ready flags live in mapped pinned
host memory; a transfer not finished after --deadline-s is released from the host and fails the run.
Manager (TP2 -> 2 x TP16, 32 x 512, 544 -> 64): TransferManager.execute_repage_scatter_routed_anypage against one
execute_repage_scatter_anypage per worker, each call waited on.
Printed: one JSON line per (shape, arm) with the median of the round medians, their min-max, the bytes the routed arm reads and
writes, the card's name and power limit read in this run; then markdown tables.  Every shape checks the routed arm's whole
destination pools against the per-worker arm's.  Needs a GPU; there is no fallback."""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from dynamo_b200 import kernels as K  # noqa: E402
from dynamo_b200.physical import (LayoutConfig, ScatterWindow, StorageKind, TransferManager, tp_pp_reshard_plan,  # noqa: E402
                                  tp_pp_scatter_plan)

p = argparse.ArgumentParser()
p.add_argument("--iters", type=int, default=5, help="calls per arm per round")
p.add_argument("--rounds", type=int, default=5)
p.add_argument("--only", default=None, help="comma-separated shape names")
p.add_argument("--no-tail", action="store_true")
p.add_argument("--layer-us", type=float, default=100.0, help="busy time of one emulated prefill layer (tail)")
p.add_argument("--lead-us", type=float, default=1000.0, help="busy time before the emulated prefill's first layer (tail)")
p.add_argument("--deadline-s", type=float, default=60.0)
a = p.parse_args()
if not torch.cuda.is_available():
    sys.exit("route_anypage_bench.py needs a GPU")
dev = torch.device("cuda:0")
torch.cuda.set_device(0)
sp = int(torch.cuda.current_stream().cuda_stream)
NHD = int(K.KvBlockLayout.OperationalNHD)
LLAMA, MLA = (80, 8, 128, 2), (61, 1, 576, 1)   # layers, KV heads, head_dim, outer dim


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "not read")
    return {"name": name, "power_limit": limit}


class Pool:
    """A fully contiguous pool of nb blocks [nl, no, page * nh * row] of random bytes."""

    def __init__(self, nb, nl, no, page, nh, row, seed):
        self.nb, self.nl, self.no, self.page, self.nh, self.row = nb, nl, no, page, nh, row
        self.region = page * nh * row
        self.block = nl * no * self.region
        g = torch.Generator(device=dev).manual_seed(seed)
        self.buf = torch.randint(0, 256, (nb * self.block,), dtype=torch.uint8, device=dev, generator=g)
        self.layer_base = torch.tensor([self.buf.data_ptr() + l * no * self.region for l in range(nl)], dtype=torch.int64, device=dev)
        self.desc = K.PagedLayout(self.layer_base.data_ptr(), self.block, self.region, self.region, nl, no, nb)

    def side(self, ids):
        return K.PermuteSide(self.desc, ids.data_ptr(), NHD)


def nblocks(tb, te, page):
    return 0 if tb == te else -(-te // page) - tb // page


def dev_i32(x):
    return torch.from_numpy(np.concatenate([np.ascontiguousarray(x).view(np.int32).reshape(-1), np.zeros(4, np.int32)])).to(dev)


def units(helper, seqs, ps, pd):
    u = helper(seqs, ps, pd)
    return dev_i32(u[0]), len(u[0])


class Tables:
    """Batch-layout id tables of one side at page `page`: every sequence's positions; those of sequences the side does not take
    name block 0 (never read or written).  Blocks are drawn without repeats for the sequences in `mine`."""

    def __init__(self, seqs, page, mine, rng):
        self.spans, ids, n = [], [], sum(nblocks(tb, te, page) for i, (tb, te) in enumerate(seqs) if i in mine)
        perm = iter(rng.permutation(n + 1)[:n] if n else [])
        for i, (tb, te) in enumerate(seqs):
            k = nblocks(tb, te, page)
            self.spans.append((len(ids), k))
            ids += [int(next(perm)) if i in mine else 0 for _ in range(k)]
        self.ids, self.nb = np.array(ids, dtype=np.int32), n + 1
        self.t = dev_i32(self.ids)

    def subset(self, idx):
        return dev_i32(np.concatenate([self.ids[s:s + k] for s, k in (self.spans[i] for i in idx)] or [np.zeros(0, np.int32)]))


class Push:
    """Prefill rank 0 of src_tp into `workers` decode workers of dst_tp; sequence i to worker i % workers (or every worker)."""

    def __init__(self, name, model, src_tp, dst_tp, workers, seqs, ps, pd, ones=False):
        nl, h, hd, no = model
        self.name, self.nl, self.no, self.ps, self.pd, self.seqs, self.g = name, nl, no, ps, pd, seqs, math.gcd(ps, pd)
        self.row = hd * 2
        one = tp_pp_scatter_plan(h, nl, src_tp, 1, dst_tp, 1, 0)
        ranks = sorted({w.dst_rank for w in one})
        self.per = len(ranks)
        self.windows = [(k * self.per + ranks.index(w.dst_rank), w.src_head_begin, w.dst_head_begin, w.head_count) for k in range(workers)
                        for w in one]
        self.src_nh, self.dst_nh, self.workers = max(1, h // src_tp), max(1, h // dst_tp), workers
        self.owner = [None if ones else i % workers for i in range(len(seqs))]
        rng = np.random.default_rng(len(name))
        everyone = set(range(len(seqs)))
        self.stab = Tables(seqs, ps, everyone, rng)
        self.src = Pool(self.stab.nb, nl, no, ps, self.src_nh, self.row, 10)
        self.mine = [{i for i, o in enumerate(self.owner) if o in (None, k)} for k in range(workers)]
        self.dtab = [Tables(seqs, pd, self.mine[d // self.per], rng) for d in range(workers * self.per)]
        self.dsts = [Pool(t.nb, nl, no, pd, self.dst_nh, self.row, 20 + d) for d, t in enumerate(self.dtab)]
        self.masks = [sum(1 << t for t, w in enumerate(self.windows) if o is None or w[0] // self.per == o) for o in self.owner]
        self.rseqs = [(tb, te, m) for (tb, te), m in zip(seqs, self.masks)]
        self.ru, self.nru = units(K.repage_route_anypage_units, self.rseqs, ps, pd)
        # read once, written to every routed window
        self.bytes = sum((te - tb) * nl * no * self.row * (self.src_nh + sum(w[3] for t, w in enumerate(self.windows) if (m >> t) & 1))
                         for tb, te, m in self.rseqs)
        self.initial = [d.buf.clone() for d in self.dsts]

    def targets(self, pools=None, ids=None, only=None):
        pools, ids = pools or self.dsts, ids or [t.t for t in self.dtab]
        return [K.ScatterTarget(pools[d].side(ids[d]), self.dst_nh, sb, db, k, 0, 0, self.nl, 0)
                for d, sb, db, k in self.windows if only is None or d // self.per == only]

    def routed(self):
        K.check(K.paged_repage_scatter_routed_anypage(self.src.side(self.stab.t), self.src_nh, self.ps, self.targets(), self.pd, self.rseqs,
                                                      self.ru.data_ptr(), self.nru, 0, self.nl, self.row, stream=sp), "routed anypage push")

    def prepare_per_worker(self):
        self.pw = []
        for k in range(self.workers):
            idx = sorted(self.mine[k])
            seqs = [self.seqs[i] for i in idx]
            u, n = units(K.repage_anypage_units, seqs, self.ps, self.pd)
            ids = [t.subset(idx) for t in self.dtab]
            self.pw.append((seqs, self.stab.subset(idx), ids, u, n, k))

    def per_worker(self):
        for seqs, sid, ids, u, n, k in self.pw:
            K.check(K.paged_repage_scatter_anypage(self.src.side(sid), self.src_nh, self.ps, self.targets(ids=ids, only=k), self.pd, seqs,
                                                   u.data_ptr(), n, 0, self.nl, self.row, stream=sp), "per-worker anypage push")

    def prepare_two_pass(self):
        g = self.g
        self.gtab = Tables(self.seqs, g, set(range(len(self.seqs))), np.random.default_rng(5))
        self.stage = Pool(self.gtab.nb, self.nl, self.no, g, self.src_nh, self.row, 30)
        self.bu1, self.nbu1 = units(K.repage_batch_units, self.seqs, self.ps, g)
        self.ru2, self.nru2 = units(K.repage_route_units, self.rseqs, g, self.pd)

    def two_pass(self):
        src = [K.StageSource(K.PermuteSource(self.src.side(self.stab.t), self.src_nh, 0, 0, self.src_nh), 0, 0, self.nl)]
        K.check(K.paged_stage_repage_gather_batch(src, self.ps, self.stage.side(self.gtab.t), self.src_nh, self.g, self.seqs, self.bu1.data_ptr(),
                                                  self.nbu1, 0, self.nl, self.row, stream=sp), "two-pass: Ps -> gcd")
        K.check(K.paged_repage_scatter_routed(self.stage.side(self.gtab.t), self.src_nh, self.g, self.targets(), self.pd, self.rseqs,
                                              self.ru2.data_ptr(), self.nru2, 0, self.nl, self.row, stream=sp), "two-pass: gcd -> Pd")

    def anypage(self):
        """Every mask full: the anypage scatter on the same inputs."""
        K.check(K.paged_repage_scatter_anypage(self.src.side(self.stab.t), self.src_nh, self.ps, self.targets(), self.pd, self.seqs,
                                               self.au.data_ptr(), self.nau, 0, self.nl, self.row, stream=sp), "anypage push")

    def routed_dividing(self):
        K.check(K.paged_repage_scatter_routed(self.src.side(self.stab.t), self.src_nh, self.ps, self.targets(), self.pd, self.rseqs,
                                              self.du.data_ptr(), self.ndu, 0, self.nl, self.row, stream=sp), "routed push")

    def reset(self):
        for d, x in zip(self.dsts, self.initial):
            d.buf.copy_(x)

    def verify(self, other):
        self.reset()
        self.routed()
        torch.cuda.synchronize()
        got = [d.buf.clone() for d in self.dsts]
        self.reset()
        other()
        torch.cuda.synchronize()
        for d, (x, y) in enumerate(zip(got, self.dsts)):
            assert torch.equal(x, y.buf), f"{self.name}: destination {d} differs between the routed launch and {other.__name__}"


class Pull:
    """Decode rank 0 of dst_tp from `workers` prefill workers of src_tp; sequence i from worker i % workers."""

    def __init__(self, name, model, src_tp, dst_tp, workers, seqs, ps, pd):
        nl, h, hd, no = model
        self.name, self.nl, self.no, self.ps, self.pd, self.seqs, self.g = name, nl, no, ps, pd, seqs, math.gcd(ps, pd)
        self.row = hd * 2
        one = tp_pp_reshard_plan(h, nl, src_tp, 1, dst_tp, 1, 0)
        ranks = sorted({w.src_rank for w in one})
        self.per = len(ranks)
        self.windows = [(k * self.per + ranks.index(w.src_rank), w.src_head_begin, w.dst_head_begin, w.head_count) for k in range(workers)
                        for w in one]
        self.src_nh, self.dst_nh, self.workers = max(1, h // src_tp), max(1, h // dst_tp), workers
        rng = np.random.default_rng(len(name))
        self.mine = [{i for i in range(len(seqs)) if i % workers == k} for k in range(workers)]
        self.stabs = [Tables(seqs, ps, self.mine[s // self.per], rng) for s in range(workers * self.per)]
        self.srcs = [Pool(t.nb, nl, no, ps, self.src_nh, self.row, 10 + s) for s, t in enumerate(self.stabs)]
        self.dtab = Tables(seqs, pd, set(range(len(seqs))), rng)
        self.dst = Pool(self.dtab.nb, nl, no, pd, self.dst_nh, self.row, 40)
        self.rseqs = [(tb, te, sum(1 << j for j, w in enumerate(self.windows) if w[0] // self.per == i % workers))
                      for i, (tb, te) in enumerate(seqs)]
        self.ru, self.nru = units(K.repage_route_anypage_units, self.rseqs, ps, pd)
        self.bytes = sum(te - tb for tb, te in seqs) * nl * no * self.dst_nh * self.row * 2   # each destination head read once, written once
        self.initial = self.dst.buf.clone()

    def sources(self, ids=None, only=None):
        ids = ids or [t.t for t in self.stabs]
        return [K.StageSource(K.PermuteSource(self.srcs[s].side(ids[s]), self.src_nh, sb, db, k), 0, 0, self.nl)
                for s, sb, db, k in self.windows if only is None or s // self.per == only]

    def routed(self):
        K.check(K.paged_stage_repage_gather_routed_anypage(self.sources(), self.ps, self.dst.side(self.dtab.t), self.dst_nh, self.pd, self.rseqs,
                                                           self.ru.data_ptr(), self.nru, 0, self.nl, self.row, stream=sp), "routed anypage pull")

    def prepare_per_worker(self):
        self.pw = []
        for k in range(self.workers):
            idx = sorted(self.mine[k])
            seqs = [self.seqs[i] for i in idx]
            u, n = units(K.repage_anypage_units, seqs, self.ps, self.pd)
            self.pw.append((seqs, [t.subset(idx) for t in self.stabs], self.dtab.subset(idx), u, n, k))

    def per_worker(self):
        for seqs, ids, did, u, n, k in self.pw:
            K.check(K.paged_stage_repage_gather_anypage(self.sources(ids, only=k), self.ps, self.dst.side(did), self.dst_nh, self.pd, seqs,
                                                        u.data_ptr(), n, 0, self.nl, self.row, stream=sp), "per-worker anypage pull")

    def prepare_two_pass(self):
        g = self.g
        self.gtab = Tables(self.seqs, g, set(range(len(self.seqs))), np.random.default_rng(5))
        self.stage = Pool(self.gtab.nb, self.nl, self.no, g, self.dst_nh, self.row, 50)
        self.ru1, self.nru1 = units(K.repage_route_units, self.rseqs, self.ps, g)
        self.bu2, self.nbu2 = units(K.repage_batch_units, self.seqs, g, self.pd)

    def two_pass(self):
        K.check(K.paged_stage_repage_gather_routed(self.sources(), self.ps, self.stage.side(self.gtab.t), self.dst_nh, self.g, self.rseqs,
                                                   self.ru1.data_ptr(), self.nru1, 0, self.nl, self.row, stream=sp), "two-pass: Ps -> gcd")
        src = [K.StageSource(K.PermuteSource(self.stage.side(self.gtab.t), self.dst_nh, 0, 0, self.dst_nh), 0, 0, self.nl)]
        K.check(K.paged_stage_repage_gather_batch(src, self.g, self.dst.side(self.dtab.t), self.dst_nh, self.pd, self.seqs, self.bu2.data_ptr(),
                                                  self.nbu2, 0, self.nl, self.row, stream=sp), "two-pass: gcd -> Pd")

    def reset(self):
        self.dst.buf.copy_(self.initial)

    def verify(self, other):
        self.reset()
        self.routed()
        torch.cuda.synchronize()
        got = self.dst.buf.clone()
        self.reset()
        other()
        torch.cuda.synchronize()
        assert torch.equal(got, self.dst.buf), f"{self.name}: the routed launch differs from {other.__name__}"


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1e3


def mixed(seed=7):
    rng = np.random.default_rng(seed)
    lens = [1, 4000] + [int(x) for x in rng.integers(1, 4001, 6)]
    return [(int(s), int(s) + n) for s, n in zip(rng.integers(1, 600, len(lens)), lens)]


def batch(n, length):
    return [(3 + 11 * i, 3 + 11 * i + length) for i in range(n)]


BATCHES = {"8x2048": batch(8, 2048), "32x512": batch(32, 512), "128x128": batch(128, 128), "mixed": mixed()}
PUSH_PAIRS = ((544, 64), (48, 64), (24, 16))


def shapes():
    specs = []
    for ps, pd in PUSH_PAIRS:
        for b in BATCHES:
            specs.append((f"push_tp2_to_2xtp16_{b}_{ps}to{pd}", lambda b=b, ps=ps, pd=pd: Push("", LLAMA, 2, 16, 2, BATCHES[b], ps, pd)))
    specs += [("push_tp1_to_2xtp8_32x512_544to64", lambda: Push("", LLAMA, 1, 8, 2, BATCHES["32x512"], 544, 64)),
              ("push_mla_to_8dp_32x512_544to64", lambda: Push("", MLA, 1, 1, 8, BATCHES["32x512"], 544, 64)),
              ("pull_8xtp2_to_tp16_32x512_64to544", lambda: Pull("", LLAMA, 2, 16, 8, BATCHES["32x512"], 64, 544)),
              ("pull_8xtp1_to_tp8_128x128_64to48", lambda: Pull("", LLAMA, 1, 8, 8, BATCHES["128x128"], 64, 48)),
              ("pull_8xtp1_to_tp8_mixed_16to24", lambda: Pull("", LLAMA, 1, 8, 8, BATCHES["mixed"], 16, 24)),
              ("pull_mla_from_8dp_32x512_64to544", lambda: Pull("", MLA, 1, 1, 8, BATCHES["32x512"], 64, 544))]
    for name, make in specs:
        if not a.only or name in a.only.split(","):
            sh = make()
            sh.name = name
            yield sh


def run_arms(sh, arms, info, rows, ref):
    for fn in arms.values():       # warm-up
        fn()
    torch.cuda.synchronize()
    per = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, fn in arms.items():
            per[k].append(statistics.median(timed(fn) for _ in range(a.iters)))
    med = {k: statistics.median(v) for k, v in per.items()}
    for k, v in per.items():
        r = {"shape": sh.name, "arm": k, "us": round(med[k], 1), "min_us": round(min(v), 1), "max_us": round(max(v), 1), "bytes": sh.bytes,
             "GBps": round(sh.bytes / med[k] / 1e3, 1), f"vs_{ref}": round(med[k] / med[ref], 3), **info}
        print(json.dumps(r), flush=True)
        rows.append(r)


# ---- the streamed tail ---------------------------------------------------------------------------------------------------------
def layer_cycles(us):
    props = torch.cuda.get_device_properties(0)
    return int(us * props.clock_rate / 1e3) if hasattr(props, "clock_rate") else int(us * 1980)


def tails(sh, info, out):
    ready = torch.zeros(sh.nl, dtype=torch.int32).pin_memory()
    n = sh.workers
    ws = [torch.zeros(K.sync_workspace_words(sh.nl), dtype=torch.int32, device=dev) for _ in range(n)]
    comp = torch.zeros(n, dtype=torch.int32, device=dev)
    xfer, prod = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(prod):
        torch.cuda._sleep(100)
        K.check(K.set_flags(ready.data_ptr(), 0, 1, 0, int(prod.cuda_stream)), "set_flags")
    torch.cuda.synchronize()
    cycles, lead = layer_cycles(a.layer_us), layer_cycles(a.lead_us)
    epoch = [0]

    def desc(i, gate):
        st = K.PermuteStream()
        st.layer_ready_flags[0] = ready.data_ptr()
        st.epoch, st.sync_workspace, st.completion_flag, st.completion_value = epoch[0], ws[i].data_ptr(), comp[i:].data_ptr(), epoch[0]
        st.gate_mode, st.gate_timeout_ms = gate, int(a.deadline_s * 1000)
        return st

    def enqueue(arm, gate):
        s = int(xfer.cuda_stream)
        if arm == "routed":
            K.check(K.paged_repage_scatter_routed_anypage_streamed(sh.src.side(sh.stab.t), sh.src_nh, sh.ps, sh.targets(), sh.pd, sh.rseqs,
                                                                   sh.ru.data_ptr(), sh.nru, 0, sh.nl, sh.row, 0, None, desc(0, gate), s),
                    "streamed routed push")
            return 1
        for i, (seqs, sid, ids, u, nu, k) in enumerate(sh.pw):
            K.check(K.paged_repage_scatter_anypage_streamed(sh.src.side(sid), sh.src_nh, sh.ps, sh.targets(ids=ids, only=k), sh.pd, seqs,
                                                            u.data_ptr(), nu, 0, sh.nl, sh.row, 0, None, desc(i, gate), s), "streamed push")
        return n

    def one(arm, gate):
        epoch[0] += 1
        ready.zero_()
        comp.zero_()
        torch.cuda.synchronize()
        last, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def produce():
            with torch.cuda.stream(prod):
                torch.cuda._sleep(lead)
                for l in range(sh.nl):
                    torch.cuda._sleep(cycles)
                    K.check(K.set_flags(ready.data_ptr(), l, 1, epoch[0], int(prod.cuda_stream)), "set_flags")
                last.record(prod)
        th = threading.Thread(target=produce)
        th.start()
        k = enqueue(arm, gate)
        end.record(xfer)
        th.join()
        t0 = time.monotonic()
        while not end.query():
            if time.monotonic() - t0 > a.deadline_s:
                ready.numpy()[:] = epoch[0]
                torch.cuda.synchronize()
                raise AssertionError(f"{sh.name} {arm}: not finished after {a.deadline_s} s; flags released from the host")
            time.sleep(1e-4)
        torch.cuda.synchronize()
        assert comp[:k].tolist() == [epoch[0]] * k, f"{sh.name} {arm}: completion words {comp[:k].tolist()}"
        return last.elapsed_time(end) * 1e3

    for gate, gname in ((K.GATE_STREAM_WAIT, "stream_wait"), (K.GATE_SPIN, "spin")):
        one("routed", gate)
        per = {"routed": [], "per_worker": []}
        for _ in range(a.rounds):
            for arm in per:
                per[arm].append(one(arm, gate))
        for arm, v in per.items():
            r = {"shape": sh.name, "tail": arm, "gate": gname, "us": round(statistics.median(v), 1), "min_us": round(min(v), 1),
                 "max_us": round(max(v), 1), "layer_us": a.layer_us, **info}
            print(json.dumps(r), flush=True)
            out.append(r)


# ---- the manager ---------------------------------------------------------------------------------------------------------------
def manager(sh, info, rows):
    mgr = TransferManager(device=0, worker_id=91)
    try:
        def reg(pool):
            cfg = LayoutConfig(pool.nb, pool.nl, pool.no, pool.page, pool.nh * (pool.row // 2), dtype_width_bytes=2, num_heads=pool.nh)
            h = mgr.register_fully_contiguous(cfg, pool.buf.data_ptr(), pool.buf.numel(), StorageKind.Device, 0)
            mgr.set_kv_block_layout(h, K.KvBlockLayout.OperationalNHD)
            return h
        sh_h, dhs = reg(sh.src), [reg(d) for d in sh.dsts]
        plan = [ScatterWindow(d, 0, 0, sh.nl, sb, db, k) for d, sb, db, k in sh.windows]
        reqs, per_worker = [], [[] for _ in range(sh.workers)]
        for i, (tb, te) in enumerate(sh.seqs):
            s, k = sh.stab.spans[i]
            src_ids = [int(x) for x in sh.stab.ids[s:s + k]]
            o = sh.owner[i]
            dst = {d: [int(x) for x in sh.dtab[d].ids[sh.dtab[d].spans[i][0]:sh.dtab[d].spans[i][0] + sh.dtab[d].spans[i][1]]]
                   for d in range(len(sh.dsts)) if d // sh.per == o}
            reqs.append((range(tb, te), src_ids, dst))
            per_worker[o].append((range(tb, te), src_ids, [dst[d] for d in sorted(dst)]))
        wplans = [[ScatterWindow(d - k * sh.per, 0, 0, sh.nl, sb, db, kk) for d, sb, db, kk in sh.windows if d // sh.per == k]
                  for k in range(sh.workers)]
        wdsts = [[dhs[d] for d in range(k * sh.per, (k + 1) * sh.per)] for k in range(sh.workers)]
        arms = {"manager_routed": lambda: mgr.execute_repage_scatter_routed_anypage(sh_h, dhs, reqs, plan).wait(60.0),
                "manager_per_worker": lambda: [mgr.execute_repage_scatter_anypage(sh_h, wdsts[k], per_worker[k], wplans[k]).wait(60.0)
                                               for k in range(sh.workers)]}
        for fn in arms.values():
            fn()
        per = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                t = []
                for _ in range(a.iters):
                    t0 = time.perf_counter()
                    fn()
                    t.append((time.perf_counter() - t0) * 1e6)
                per[k].append(statistics.median(t))
        for k, v in per.items():
            r = {"shape": sh.name, "arm": k, "us": round(statistics.median(v), 1), "min_us": round(min(v), 1), "max_us": round(max(v), 1),
                 "bytes": sh.bytes, "GBps": round(sh.bytes / statistics.median(v) / 1e3, 1), **info}
            print(json.dumps(r), flush=True)
            rows.append(r)
    finally:
        mgr.close()


def main():
    info = card()
    rows, extra, tail_rows = [], [], []
    for sh in shapes():
        sh.prepare_per_worker()
        sh.prepare_two_pass()
        sh.verify(sh.per_worker)
        run_arms(sh, {"routed": sh.routed, "per_worker": sh.per_worker, "two_pass": sh.two_pass}, info, rows, "routed")
        if not a.no_tail and sh.name in ("push_tp2_to_2xtp16_8x2048_544to64", "push_tp2_to_2xtp16_8x2048_48to64"):
            tails(sh, info, tail_rows)
        if sh.name == "push_tp2_to_2xtp16_32x512_544to64":
            manager(sh, info, extra)
        del sh
        torch.cuda.empty_cache()
    # the cost of routing: every mask full, against the anypage scatter
    if not a.only or "ones" in a.only:
        sh = Push("push_tp2_to_2xtp16_32x512_544to64_all_masks_full", LLAMA, 2, 16, 2, BATCHES["32x512"], 544, 64, ones=True)
        sh.au, sh.nau = units(K.repage_anypage_units, sh.seqs, sh.ps, sh.pd)
        sh.verify(sh.anypage)
        run_arms(sh, {"routed": sh.routed, "anypage": sh.anypage}, info, extra, "routed")
        del sh
        torch.cuda.empty_cache()
    # the cost of the phase: a dividing pair, against the routed scatter
    if not a.only or "dividing" in a.only:
        sh = Push("push_tp2_to_2xtp16_32x512_512to64_dividing", LLAMA, 2, 16, 2, BATCHES["32x512"], 512, 64)
        sh.du, sh.ndu = units(K.repage_route_units, sh.rseqs, sh.ps, sh.pd)
        sh.verify(sh.routed_dividing)
        run_arms(sh, {"routed": sh.routed, "routed_dividing_entry": sh.routed_dividing}, info, extra, "routed")
        del sh
        torch.cuda.empty_cache()
    print(f"\n{info['name']}, power limit {info['power_limit']}\n")
    print("| shape | arm | median us | min-max us | GB/s | time / routed |")
    print("|---|---|---|---|---|---|")
    for r in rows + extra:
        print(f"| {r['shape']} | {r['arm']} | {r['us']} | {r['min_us']}-{r['max_us']} | {r['GBps']} | {r.get('vs_routed', '')} |")
    if tail_rows:
        print("\n| shape | gate | arm | exposed tail us (median, min-max) |")
        print("|---|---|---|---|")
        for r in tail_rows:
            print(f"| {r['shape']} | {r['gate']} | {r['tail']} | {r['us']} ({r['min_us']}-{r['max_us']}) |")


if __name__ == "__main__":
    main()

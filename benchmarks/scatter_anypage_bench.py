"""The re-paging scatter between pages that need not divide (kvbm_kernels_paged_repage_scatter_anypage), timed against the
single-pass workaround the library offered before it: one kvbm_kernels_paged_stage_repage_gather_anypage launch per target, which
reads replicated heads once per target.

Shapes: Llama-3-70B (80 layers, K/V, 8 KV heads of 128), every pool on one GPU, fully contiguous OperationalNHD with random block
tables, bf16 unless named:
  TP2 -> TP16 prefill rank 0: 4 source heads into 8 decode ranks of one head each (every head to two ranks of the 16);
  TP1 -> TP8: 8 source heads into 8 decode ranks of one head;
  pages 544 -> 64 and 48 -> 64; batches 8 x 2048, 32 x 512 and a mixed batch (1 to 4000 tokens, each starting inside a block);
  fp8 -> bf16 on TP2 -> TP16, 544 -> 64, 8 x 2048.
Arms, alternating inside each of --rounds rounds, timed with CUDA events (median of --iters single launches per round):
  (a) anypage  one kvbm_kernels_paged_repage_scatter_anypage launch
  (b) gathers  n kvbm_kernels_paged_stage_repage_gather_anypage launches, one per target
  (c) ceiling  kvbm_kernels_paged_repage_scatter_batch Ps -> gcd(Ps, Pd) over the same sequences into pools of page gcd: the same
               bytes read and written at a dividing pair
Tail (on TP2 -> TP16, 8 x 2048, both page pairs; --no-tail skips it): the exposed tail behind an emulated prefill, from the
producer's last ready flag to the end of the transfer, in both gate forms: the anypage scatter streamed, against n streamed
anypage gathers on one stream.  The producer runs --layer-us of busy kernel per source layer and then writes that layer's ready
flag; it is enqueued from its own host thread, as an engine's forward is, and starts with --lead-us of busy time, so the
transfer is enqueued and waiting when layer 0 lands.  Ready flags live in mapped pinned host memory, so the host can release
them without a CUDA call: a transfer that has not finished after --deadline-s is released, reported and fails the run.
Enqueue probe (with the tail): each streamed arm in the stream-wait form is enqueued with no producer at all, and a watchdog
thread reads the library's launch count after 3 s, then releases the flags from the host.  It shows whether the enqueue returns
while the stream waits on layer 0, or blocks inside a launch (and after how many), which is why the producer gets its own thread.
Printed: one JSON line per (shape, arm) with the median of the round medians and their min-max, the bytes read + written, the
card's name and power limit read in this run; then a markdown table.  Every run checks (a)'s whole target pools against (b)'s and
the first and last target block of sequence 0 against tests/scatter_oracle.py.  Needs a GPU; there is no fallback."""
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
from dynamo_b200.physical import tp_pp_scatter_plan  # noqa: E402
from tests.scatter_oracle import repage_scatter  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--iters", type=int, default=5, help="single launches per arm per round")
p.add_argument("--rounds", type=int, default=5)
p.add_argument("--only", default=None, help="comma-separated shape names")
p.add_argument("--no-tail", action="store_true")
p.add_argument("--layer-us", type=float, default=100.0, help="busy time of one emulated prefill layer (tail)")
p.add_argument("--lead-us", type=float, default=1000.0, help="busy time before the emulated prefill's first layer (tail)")
p.add_argument("--deadline-s", type=float, default=60.0, help="a streamed transfer not finished by then is released and fails the run")
a = p.parse_args()
if not torch.cuda.is_available():
    sys.exit("scatter_anypage_bench.py needs a GPU")
dev = torch.device("cuda:0")
torch.cuda.set_device(0)
sp = int(torch.cuda.current_stream().cuda_stream)
NL, H, NO, HD = 80, 8, 2, 128
NHD = int(K.KvBlockLayout.OperationalNHD)
CM = K.CastMode


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "not read")
    return {"name": name, "power_limit": limit}


class Pool:
    """A fully contiguous pool of nb blocks [NL, NO, page * nh * row] of random bytes."""

    def __init__(self, nb, page, nh, row, seed):
        self.nb, self.page, self.nh, self.row = nb, page, nh, row
        self.region = page * nh * row
        self.block = NL * NO * self.region
        g = torch.Generator(device=dev).manual_seed(seed)
        self.buf = torch.randint(0, 256, (nb * self.block,), dtype=torch.uint8, device=dev, generator=g)
        self.layer_base = torch.tensor([self.buf.data_ptr() + l * NO * self.region for l in range(NL)], dtype=torch.int64, device=dev)
        self.desc = K.PagedLayout(self.layer_base.data_ptr(), self.block, self.region, self.region, NL, NO, nb)

    def side(self, ids):
        return K.PermuteSide(self.desc, ids.data_ptr(), NHD)

    def blocks(self, ids):
        v = self.buf.view(self.nb, self.block)
        return [v[int(b)].cpu().numpy() for b in ids]


def nblocks(tb, te, page):
    return 0 if tb == te else -(-te // page) - tb // page


def table(seqs, page, rng):
    n = sum(nblocks(tb, te, page) for tb, te in seqs)
    return rng.permutation(n + 1)[:n].astype(np.int32), n + 1


def dev_i32(x):
    return torch.from_numpy(np.concatenate([np.ascontiguousarray(x).view(np.int32).reshape(-1), np.zeros(4, np.int32)])).to(dev)


class Shape:
    def __init__(self, name, src_tp, dst_tp, seqs, ps, pd, cast=CM.NONE):
        self.name, self.ps, self.pd, self.seqs, self.cast = name, ps, pd, seqs, int(cast)
        self.g = math.gcd(ps, pd)
        se, de = (1, 2) if cast == CM.FP8E4M3_TO_BF16 else (2, 2)
        self.srow, self.drow = HD * se, HD * de
        plan = tp_pp_scatter_plan(H, NL, src_tp, 1, dst_tp, 1, 0)
        self.src_nh, self.dst_nh = H // src_tp, max(1, H // dst_tp)
        self.windows = [(w.src_head_begin, w.dst_head_begin, w.head_count) for w in plan]
        rng = np.random.default_rng(len(name))
        self.sids, nbs = table(seqs, ps, rng)
        self.src = Pool(nbs, ps, self.src_nh, self.srow, 10)
        self.dsts, self.dids, self.stages, self.gids = [], [], [], []
        for t in range(len(plan)):
            ids, nbd = table(seqs, pd, rng)
            self.dids.append(ids)
            self.dsts.append(Pool(nbd, pd, self.dst_nh, self.drow, 20 + t))
            gids, nbg = table(seqs, self.g, rng)
            self.gids.append(gids)
            self.stages.append(Pool(nbg, self.g, self.dst_nh, self.drow, 40 + t))
        self.initial = [d.buf.clone() for d in self.dsts]
        self.sids_t = dev_i32(self.sids)
        self.dids_t, self.gids_t = [dev_i32(x) for x in self.dids], [dev_i32(x) for x in self.gids]
        any_u = K.repage_anypage_units(seqs, ps, pd)[0]
        ceil_u = K.repage_batch_units(seqs, ps, self.g)[0]
        self.any_u, self.n_any, self.ceil_u, self.n_ceil = dev_i32(any_u), len(any_u), dev_i32(ceil_u), len(ceil_u)
        tokens = sum(te - tb for tb, te in seqs)
        # read once, written to every target
        self.bytes = tokens * NL * NO * (self.src_nh * self.srow + sum(k for _sb, _db, k in self.windows) * self.drow)

    def targets(self, pools=None, ids=None, flags=None):
        pools, ids = pools or self.dsts, ids or self.dids_t
        return [K.ScatterTarget(pools[t].side(ids[t]), self.dst_nh, sb, db, k, 0, 0, NL, flags[t].data_ptr() if flags else 0)
                for t, (sb, db, k) in enumerate(self.windows)]

    def source(self, t):
        sb, db, k = self.windows[t]
        return [K.StageSource(K.PermuteSource(self.src.side(self.sids_t), self.src_nh, sb, db, k), 0, 0, NL)]

    def anypage(self):
        K.check(K.paged_repage_scatter_anypage(self.src.side(self.sids_t), self.src_nh, self.ps, self.targets(), self.pd, self.seqs,
                                               self.any_u.data_ptr(), self.n_any, 0, NL, self.srow, self.cast, stream=sp), "anypage scatter")

    def gathers(self):
        for t in range(len(self.windows)):
            K.check(K.paged_stage_repage_gather_anypage(self.source(t), self.ps, self.dsts[t].side(self.dids_t[t]), self.dst_nh, self.pd,
                                                        self.seqs, self.any_u.data_ptr(), self.n_any, 0, NL, self.srow, self.cast, stream=sp),
                    "anypage gather")

    def ceiling(self):
        K.check(K.paged_repage_scatter_batch(self.src.side(self.sids_t), self.src_nh, self.ps, self.targets(self.stages, self.gids_t), self.g,
                                             self.seqs, self.ceil_u.data_ptr(), self.n_ceil, 0, NL, self.srow, self.cast, stream=sp),
                "ceiling")

    def reset(self):
        for d, x in zip(self.dsts, self.initial):
            d.buf.copy_(x)

    def verify(self):
        """(a)'s whole target pools against (b)'s, and the first and last target block of sequence 0 against the oracle."""
        self.reset()
        self.anypage()
        torch.cuda.synchronize()
        got = [d.buf.clone() for d in self.dsts]
        self.reset()
        self.gathers()
        torch.cuda.synchronize()
        for t, (g, d) in enumerate(zip(got, self.dsts)):
            assert torch.equal(g, d.buf), f"{self.name}: target {t} differs between the scatter and the gathers"
        tb, te = self.seqs[0]
        nd = nblocks(tb, te, self.pd)
        sb, db, k = self.windows[0]
        for i in (0, nd - 1):
            lo, hi = max(tb, (tb // self.pd + i) * self.pd), min(te, (tb // self.pd + i + 1) * self.pd)
            s0 = lo // self.ps - tb // self.ps
            src = (self.src.blocks(self.sids[s0:s0 + nblocks(lo, hi, self.ps)]), NHD, self.src_nh, NL)
            pool = np.stack([self.initial[0].view(self.dsts[0].nb, self.dsts[0].block)[int(self.dids[0][i])].cpu().numpy()])
            repage_scatter(src, [(0, [0], NHD, self.dst_nh, NL, (0, 0, NL, sb, db, k))], [pool], NO, self.ps, self.pd, self.srow, lo, hi,
                           self.cast)
            assert np.array_equal(got[0].view(self.dsts[0].nb, self.dsts[0].block)[int(self.dids[0][i])].cpu().numpy(), pool[0]), \
                f"{self.name}: target block {i} of sequence 0 differs from the oracle"


    # ---- streamed: the exposed tail behind an emulated prefill ----------------------------------------------------------
    def streamed(self, arm, gate_mode, ready, epoch, ws, comp, stream):
        """Enqueue arm "anypage" (one streamed scatter) or "gathers" (one streamed anypage gather per target) on `stream`, waiting
        on the host-memory `ready` flags at `epoch`; each launch's completion word comp[i] becomes `epoch`."""
        def desc(i):
            st = K.PermuteStream()
            st.layer_ready_flags[0] = ready.data_ptr()
            st.epoch = epoch
            st.sync_workspace = ws[i].data_ptr()
            st.completion_flag = comp[i:].data_ptr()
            st.completion_value = epoch
            st.gate_mode = gate_mode
            st.gate_timeout_ms = int(a.deadline_s * 1000)
            return st
        if arm == "anypage":
            K.check(K.paged_repage_scatter_anypage_streamed(self.src.side(self.sids_t), self.src_nh, self.ps, self.targets(), self.pd, self.seqs,
                                                            self.any_u.data_ptr(), self.n_any, 0, NL, self.srow, self.cast, None, desc(0),
                                                            stream), "streamed scatter")
            return
        for t in range(len(self.windows)):
            K.check(K.paged_stage_repage_gather_anypage_streamed(self.source(t), self.ps, self.dsts[t].side(self.dids_t[t]), self.dst_nh,
                                                                 self.pd, self.seqs, self.any_u.data_ptr(), self.n_any, 0, NL, self.srow,
                                                                 self.cast, None, desc(t), stream), "streamed gather")


class Streamed:
    """The flags, workspaces and streams of one shape's streamed arms: ready flags in mapped pinned host memory."""

    def __init__(self, sh):
        self.sh, self.n = sh, len(sh.windows)
        self.ready = torch.zeros(NL, dtype=torch.int32).pin_memory()
        self.ws = [torch.zeros(K.sync_workspace_words(NL), dtype=torch.int32, device=dev) for _ in range(self.n)]
        self.comp = torch.zeros(self.n, dtype=torch.int32, device=dev)
        self.xfer, self.prod = torch.cuda.Stream(), torch.cuda.Stream()
        self.epoch = 0
        with torch.cuda.stream(self.prod):    # every kernel the producer takes, loaded before anything waits on it
            torch.cuda._sleep(100)
            K.check(K.set_flags(self.ready.data_ptr(), 0, 1, 0, int(self.prod.cuda_stream)), "set_flags")
        torch.cuda.synchronize()

    def _begin(self):
        self.epoch += 1
        self.ready.zero_()
        self.comp.zero_()
        torch.cuda.synchronize()
        return self.epoch

    def _drain(self, end, epoch, what):
        """Wait for `end` until the deadline; past it, release every flag from the host and fail."""
        t0 = time.monotonic()
        while not end.query():
            if time.monotonic() - t0 > a.deadline_s:
                self.ready.numpy()[:] = epoch
                torch.cuda.synchronize()
                raise AssertionError(f"{self.sh.name} {what}: not finished after {a.deadline_s} s; flags released from the host")
            time.sleep(1e-4)
        torch.cuda.synchronize()
        n = 1 if what.startswith("anypage") else self.n
        assert self.comp[:n].tolist() == [epoch] * n, f"{self.sh.name} {what}: completion words {self.comp[:n].tolist()}"

    def tail(self, arm, gate_mode, cycles, lead):
        """The producer's last ready flag to the end of the transfer, in us, and the transfer's host enqueue time, in us."""
        epoch = self._begin()
        last, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        go = threading.Event()

        def produce():
            go.wait()
            with torch.cuda.stream(self.prod):
                ps = int(self.prod.cuda_stream)
                torch.cuda._sleep(lead)
                for l in range(NL):
                    torch.cuda._sleep(cycles)
                    K.check(K.set_flags(self.ready.data_ptr(), l, 1, epoch, ps), "set_flags")
                last.record(self.prod)
        prod = threading.Thread(target=produce)
        prod.start()
        go.set()
        t0 = time.perf_counter()
        self.sh.streamed(arm, gate_mode, self.ready, epoch, self.ws, self.comp, int(self.xfer.cuda_stream))
        enqueue = (time.perf_counter() - t0) * 1e6
        end.record(self.xfer)
        prod.join()
        self._drain(end, epoch, f"{arm} tail")
        return last.elapsed_time(end) * 1e3, enqueue

    def probe(self, arm):
        """Enqueue `arm` in the stream-wait form with no producer.  A watchdog reads the launch count after 3 s and then releases
        the flags from the host.  Returns whether the enqueue had returned by then, the launches it had made, and the total."""
        epoch = self._begin()
        before, seen = K.launch_count(), {}
        done = threading.Event()

        def watchdog():
            done.wait(3.0)
            seen["returned"], seen["launches"] = done.is_set(), K.launch_count() - before
            self.ready.numpy()[:] = epoch
        w = threading.Thread(target=watchdog)
        w.start()
        self.sh.streamed(arm, K.GATE_STREAM_WAIT, self.ready, epoch, self.ws, self.comp, int(self.xfer.cuda_stream))
        done.set()
        w.join()
        end = torch.cuda.Event()
        end.record(self.xfer)
        self._drain(end, epoch, f"{arm} probe")
        return seen["returned"], seen["launches"], K.launch_count() - before


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


def layer_cycles(us):
    """Clock cycles of a busy kernel that runs `us` microseconds on device 0."""
    props = torch.cuda.get_device_properties(0)
    return int(us * props.clock_rate / 1e3) if hasattr(props, "clock_rate") else int(us * 1980)


TAIL_SHAPES = ("tp2_to_tp16_8x2048_544to64", "tp2_to_tp16_8x2048_48to64")
BATCHES = {"8x2048": batch(8, 2048), "32x512": batch(32, 512), "mixed": mixed()}


def shapes():
    specs = [(f"tp2_to_tp16_{b}_{ps}to{pd}", 2, 16, b, ps, pd, CM.NONE) for ps, pd in ((544, 64), (48, 64)) for b in BATCHES]
    specs += [("tp1_to_tp8_8x2048_544to64", 1, 8, "8x2048", 544, 64, CM.NONE), ("tp1_to_tp8_32x512_48to64", 1, 8, "32x512", 48, 64, CM.NONE),
              ("tp2_to_tp16_8x2048_544to64_fp8_to_bf16", 2, 16, "8x2048", 544, 64, CM.FP8E4M3_TO_BF16)]
    for name, s, d, b, ps, pd, cast in specs:
        if not a.only or name in a.only.split(","):
            yield Shape(name, s, d, BATCHES[b], ps, pd, cast)


def main():
    info = card()
    rows, tails, probes = [], [], []
    for sh in shapes():
        sh.verify()
        arms = {"anypage": sh.anypage, "gathers": sh.gathers, "ceiling": sh.ceiling}
        for fn in arms.values():       # warm-up
            fn()
        torch.cuda.synchronize()
        per = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                per[k].append(statistics.median(timed(fn) for _ in range(a.iters)))
        med = {k: statistics.median(v) for k, v in per.items()}
        for k, v in per.items():
            r = {"shape": sh.name, "arm": k, "us": round(med[k], 1), "min_us": round(min(v), 1), "max_us": round(max(v), 1),
                 "bytes": sh.bytes, "GBps": round(sh.bytes / med[k] / 1e3, 1), "vs_anypage": round(med[k] / med["anypage"], 3), **info}
            print(json.dumps(r), flush=True)
            rows.append(r)
        if not a.no_tail and sh.name in TAIL_SHAPES:
            s = Streamed(sh)
            for arm in ("anypage", "gathers"):
                returned, at, total = s.probe(arm)
                r = {"shape": sh.name, "probe": arm, "enqueue_returned_before_release": returned, "launches_when_read": at,
                     "launches_total": total, **info}
                print(json.dumps(r), flush=True)
                probes.append(r)
            cycles, lead = layer_cycles(a.layer_us), layer_cycles(a.lead_us)
            for gate, gname in ((K.GATE_STREAM_WAIT, "stream_wait"), (K.GATE_SPIN, "spin")):
                per = {"anypage": [], "gathers": []}
                enq = {"anypage": [], "gathers": []}
                s.tail("anypage", gate, cycles, lead)     # warm-up
                sh.reset()
                for _ in range(a.rounds):
                    for arm in per:
                        t, e = s.tail(arm, gate, cycles, lead)
                        per[arm].append(t)
                        enq[arm].append(e)
                        sh.reset()
                for arm, v in per.items():
                    r = {"shape": sh.name, "tail": arm, "gate": gname, "us": round(statistics.median(v), 1), "min_us": round(min(v), 1),
                         "max_us": round(max(v), 1), "enqueue_us": round(statistics.median(enq[arm]), 1), "layer_us": a.layer_us, **info}
                    print(json.dumps(r), flush=True)
                    tails.append(r)
            del s
        del sh, arms
        torch.cuda.empty_cache()
    print(f"\n{info['name']}, power limit {info['power_limit']}\n")
    print("| shape | arm | median us | min-max us | GB/s | time / anypage |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['shape']} | {r['arm']} | {r['us']} | {r['min_us']}-{r['max_us']} | {r['GBps']} | {r['vs_anypage']} |")
    if tails:
        print("\n| shape | gate | arm | exposed tail us (median, min-max) | host enqueue us |")
        print("|---|---|---|---|---|")
        for r in tails:
            print(f"| {r['shape']} | {r['gate']} | {r['tail']} | {r['us']} ({r['min_us']}-{r['max_us']}) | {r['enqueue_us']} |")
    for r in probes:
        print(f"probe {r['shape']} {r['probe']}: enqueue returned before release {r['enqueue_returned_before_release']}, "
              f"{r['launches_when_read']} of {r['launches_total']} launches made")


if __name__ == "__main__":
    main()

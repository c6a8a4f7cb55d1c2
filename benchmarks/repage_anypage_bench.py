"""Re-paging between pages that need not divide (kvbm_kernels_paged_stage_repage_gather_anypage), timed against the two-pass
workaround the library offered before it: re-page the source into a staging pool whose page is gcd(Ps, Pd) with today's batch
entry, then that pool into the destination.

Shapes, on fully contiguous OperationalNHD pools with random block tables (K/V, head_dim 128, bf16 unless named):
  Llama-3-8B (32 layers, 8 KV heads), one 4096-token sequence at pages 544 -> 64, 64 -> 544, 24 -> 16 and 48 -> 64;
  Llama-3-70B (80 layers, 8 KV heads) TP4 -> TP2 at 544 -> 64: a decode rank's 4 heads from two prefill ranks of 2;
  Llama-3-8B, a batch of 32 x 512 tokens, each starting inside a block, at 544 -> 64;
  Llama-3-8B, fp8 -> bf16 at 544 -> 64 (the cast runs in the first leg of the two-pass).
Arms, alternating inside each round, timed with CUDA events over --iters launches:
  (a) anypage   one kvbm_kernels_paged_stage_repage_gather_anypage launch
  (b) two-pass  kvbm_kernels_paged_stage_repage_gather_batch Ps -> gcd, then gcd -> Pd
  (c) ceiling   the first leg of (b) alone: the same bytes read and written, between dividing pages
and on one dividing pair (16 -> 64) the anypage entry against kvbm_kernels_paged_stage_repage_gather_batch on the same inputs.
Printed: one JSON line per (shape, arm) with the median of the round medians and their min-max, bytes read + written from the
shapes, the card's name and power limit read in this run; then a markdown table.  Every run checks (a)'s whole destination
against (b)'s and two sampled destination blocks against tests/stage_repage_oracle.py.  Needs a GPU; there is no fallback."""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from dynamo_b200 import kernels as K  # noqa: E402
from tests.stage_repage_oracle import stage_repage_gather  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--iters", type=int, default=10, help="launches per arm per round")
p.add_argument("--rounds", type=int, default=5)
p.add_argument("--only", default=None, help="comma-separated shape names")
a = p.parse_args()
if not torch.cuda.is_available():
    sys.exit("repage_anypage_bench.py needs a GPU")
dev = torch.device("cuda:0")
torch.cuda.set_device(0)
sp = int(torch.cuda.current_stream().cuda_stream)
NO, HD = 2, 128
NHD = int(K.KvBlockLayout.OperationalNHD)
CM = K.CastMode


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "not read")
    return {"name": name, "power_limit": limit}


class Pool:
    """A fully contiguous pool of nb blocks [nl, NO, page * nh * row] of random bytes."""

    def __init__(self, nb, nl, page, nh, row, seed):
        self.nb, self.nl, self.page, self.nh, self.row = nb, nl, page, nh, row
        self.region = page * nh * row
        self.block = nl * NO * self.region
        g = torch.Generator(device=dev).manual_seed(seed)
        self.buf = torch.randint(0, 256, (nb * self.block,), dtype=torch.uint8, device=dev, generator=g)
        self.layer_base = torch.tensor([self.buf.data_ptr() + l * NO * self.region for l in range(nl)], dtype=torch.int64, device=dev)
        self.desc = K.PagedLayout(self.layer_base.data_ptr(), self.block, self.region, self.region, nl, NO, nb)

    def side(self, ids):
        return K.PermuteSide(self.desc, ids.data_ptr(), NHD)

    def blocks(self, ids):
        v = self.buf.view(self.nb, self.block)
        return [v[int(b)].cpu().numpy() for b in ids]


def nblocks(tb, te, page):
    return 0 if tb == te else -(-te // page) - tb // page


def tables(seqs, page, rng):
    n = [nblocks(tb, te, page) for tb, te in seqs]
    perm = rng.permutation(sum(n) + 1).astype(np.int32)
    return [perm[s - c:s] for s, c in zip(np.cumsum(n), n)], sum(n) + 1


def dev_ids(parts):
    return torch.from_numpy(np.concatenate(list(parts) + [np.zeros(1, np.int32)])).to(dev)


def dev_units(u):
    return torch.from_numpy(np.concatenate([u, np.zeros((1, 4), np.uint32)]).view(np.int32)).to(dev)


class Shape:
    """src_nh heads per source over `windows` (source, src_head_begin, dst_head_begin, head_count) into dst_nh heads."""

    def __init__(self, name, nl, src_nh, dst_nh, windows, seqs, ps, pd, cast=CM.NONE):
        self.name, self.nl, self.ps, self.pd, self.seqs, self.cast, self.windows = name, nl, ps, pd, seqs, int(cast), windows
        self.g = math.gcd(ps, pd)
        se, de = (1, 2) if cast == CM.FP8E4M3_TO_BF16 else (2, 2)
        self.srow, self.drow = HD * se, HD * de
        rng = np.random.default_rng(len(name))
        n_src = 1 + max(w[0] for w in windows)
        self.sids, nbs = zip(*[tables(seqs, ps, rng) for _ in range(n_src)])
        self.dids, nbd = tables(seqs, pd, rng)
        self.gids, nbg = tables(seqs, self.g, rng)
        self.srcs = [Pool(nbs[s], nl, ps, src_nh, self.srow, 10 + s) for s in range(n_src)]
        self.dst = Pool(nbd, nl, pd, dst_nh, self.drow, 1)
        self.stage = Pool(nbg, nl, self.g, dst_nh, self.drow, 2)
        self.initial = self.dst.buf.clone()
        self.sids_t, self.dids_t, self.gids_t = [dev_ids(x) for x in self.sids], dev_ids(self.dids), dev_ids(self.gids)
        self.any_u = dev_units(K.repage_anypage_units(seqs, ps, pd)[0])
        self.leg1_u = dev_units(K.repage_batch_units(seqs, ps, self.g)[0])
        self.leg2_u = dev_units(K.repage_batch_units(seqs, self.g, pd)[0])
        self.n_any, self.n1, self.n2 = (len(K.repage_anypage_units(seqs, ps, pd)[0]), len(K.repage_batch_units(seqs, ps, self.g)[0]),
                                        len(K.repage_batch_units(seqs, self.g, pd)[0]))
        tokens = sum(te - tb for tb, te in seqs)
        self.bytes = tokens * nl * NO * sum(w[3] for w in windows) * (self.srow + self.drow)

    def sources(self):
        return [K.StageSource(K.PermuteSource(self.srcs[s].side(self.sids_t[s]), self.srcs[s].nh, sb, db, k), 0, 0, self.nl)
                for s, sb, db, k in self.windows]

    def anypage(self):
        K.check(K.paged_stage_repage_gather_anypage(self.sources(), self.ps, self.dst.side(self.dids_t), self.dst.nh, self.pd, self.seqs,
                                                    self.any_u.data_ptr(), self.n_any, 0, self.nl, self.srow, self.cast, stream=sp), "anypage")

    def leg1(self):
        K.check(K.paged_stage_repage_gather_batch(self.sources(), self.ps, self.stage.side(self.gids_t), self.stage.nh, self.g, self.seqs,
                                                  self.leg1_u.data_ptr(), self.n1, 0, self.nl, self.srow, self.cast, stream=sp), "leg 1")

    def two_pass(self):
        self.leg1()
        whole = [K.StageSource(K.PermuteSource(self.stage.side(self.gids_t), self.dst.nh, 0, 0, self.dst.nh), 0, 0, self.nl)]
        K.check(K.paged_stage_repage_gather_batch(whole, self.g, self.dst.side(self.dids_t), self.dst.nh, self.pd, self.seqs,
                                                  self.leg2_u.data_ptr(), self.n2, 0, self.nl, self.drow, 0, stream=sp), "leg 2")

    def batch(self):
        if not hasattr(self, "batch_u"):
            self.batch_u = dev_units(K.repage_batch_units(self.seqs, self.ps, self.pd)[0])
        K.check(K.paged_stage_repage_gather_batch(self.sources(), self.ps, self.dst.side(self.dids_t), self.dst.nh, self.pd, self.seqs,
                                                  self.batch_u.data_ptr(), self.n_any, 0, self.nl, self.srow, self.cast, stream=sp), "batch")

    def verify(self, other):
        """(a)'s destination against `other`'s (the two-pass, or the batch entry), and two sampled blocks against the oracle."""
        self.dst.buf.copy_(self.initial)
        self.anypage()
        torch.cuda.synchronize()
        got = self.dst.buf.clone()
        self.dst.buf.copy_(self.initial)
        other()
        torch.cuda.synchronize()
        assert torch.equal(got, self.dst.buf), f"{self.name}: the anypage launch differs from the reference arm"
        tb, te = self.seqs[0]
        ids = self.dids[0]
        for i in (0, len(ids) - 1):           # the first and last destination block of sequence 0
            lo, hi = max(tb, (tb // self.pd + i) * self.pd), min(te, (tb // self.pd + i + 1) * self.pd)
            srcs = [(self.srcs[s].blocks(self.sids[s][0][lo // self.ps - tb // self.ps:-(-hi // self.ps) - tb // self.ps]), NHD,
                     self.srcs[s].nh, self.nl) for s in range(len(self.srcs))]
            before = [self.initial.view(self.dst.nb, self.dst.block)[int(ids[i])].cpu().numpy()]
            want = stage_repage_gather(srcs, [(s, 0, 0, self.nl, sb, db, k) for s, sb, db, k in self.windows], before, NHD, self.dst.nh,
                                       self.nl, NO, self.ps, self.pd, self.srow, lo, hi, self.cast)[0]
            assert np.array_equal(got.view(self.dst.nb, self.dst.block)[int(ids[i])].cpu().numpy(), want), f"{self.name}: block {i}"


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


def shapes():
    one8 = dict(nl=32, src_nh=8, dst_nh=8, windows=[(0, 0, 0, 8)])
    rng = np.random.default_rng(3)
    starts = [int(x) for x in rng.integers(1, 2000, 32)]
    out = [Shape(f"8b_4096_{ps}to{pd}", seqs=[(0, 4096)], ps=ps, pd=pd, **one8) for ps, pd in ((544, 64), (64, 544), (24, 16), (48, 64))]
    out.append(Shape("70b_tp4_to_tp2_544to64", 80, 2, 4, [(0, 0, 0, 2), (1, 0, 2, 2)], [(0, 4096)], 544, 64))
    out.append(Shape("8b_32x512_544to64", seqs=[(s, s + 512) for s in starts], ps=544, pd=64, **one8))
    out.append(Shape("8b_4096_fp8_to_bf16_544to64", seqs=[(0, 4096)], ps=544, pd=64, cast=CM.FP8E4M3_TO_BF16, **one8))
    out.append(Shape("8b_4096_16to64_dividing", seqs=[(0, 4096)], ps=16, pd=64, **one8))
    return [s for s in out if not a.only or s.name in a.only.split(",")]


def main():
    info = card()
    rows = []
    for sh in shapes():
        dividing = sh.pd % sh.ps == 0 or sh.ps % sh.pd == 0
        arms = {"anypage": sh.anypage, "batch": sh.batch} if dividing else {"anypage": sh.anypage, "two-pass": sh.two_pass, "ceiling": sh.leg1}
        sh.verify(sh.batch if dividing else sh.two_pass)
        for fn in arms.values():       # warm-up
            fn()
        torch.cuda.synchronize()
        per = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                per[k].append(statistics.median(timed(fn, 1) for _ in range(a.iters)))
        med = {k: statistics.median(v) for k, v in per.items()}
        for k, v in per.items():
            r = {"shape": sh.name, "arm": k, "us": round(med[k], 1), "min_us": round(min(v), 1), "max_us": round(max(v), 1),
                 "bytes": sh.bytes, "GBps": round(sh.bytes / med[k] / 1e3, 1), "vs_anypage": round(med[k] / med["anypage"], 3), **info}
            print(json.dumps(r))
            rows.append(r)
        del sh
        torch.cuda.empty_cache()
    print(f"\n{info['name']}, power limit {info['power_limit']}\n")
    print("| shape | arm | median us | min-max us | GB/s | time / anypage |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['shape']} | {r['arm']} | {r['us']} | {r['min_us']}-{r['max_us']} | {r['GBps']} | {r['vs_anypage']} |")


if __name__ == "__main__":
    main()

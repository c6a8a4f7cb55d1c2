"""Re-paging hand-off, timed: kvbm_kernels_paged_repage moving a 4k-token sequence between block tables of different page sizes,
against (a) the paged permute of the same bytes with equal pages (the rate to approach) and (b) what a caller has to do without
it: K1 (kvbm_kernels_launch_vectorized_copy) over host-built pointer tables of min(Ps, Pd)-token runs, timed as the whole host
flow (build the tables, upload them, launch, wait).  K1 cannot cast, so it runs only without --cast.

Llama-3-8B KV geometry (32 layers, K/V, 8 heads x 128, bf16) on vLLM-style layer-separate NHD pools with random block tables,
plus MLA (one outer index, one 576-wide head).  One JSON line per arm with the card's name and power limit; sample destination
blocks of every arm are compared with tests/repage_oracle.py.

--reshard S:D times kvbm_kernels_paged_repage_gather instead: decode rank 0 of TP D (page Pd) assembling its heads from the ranks
of TP S (page Ps) that hold them, over the whole sequence, in one launch.  Its arms, alternated within each of the --iters rounds
and timed with CUDA events (median): the one launch; the two-pass workaround without it (kvbm_kernels_paged_repage per source
into a staging pool with page Pd and the source's heads, then kvbm_kernels_paged_permute_gather out of the staging pools), timed
whole; and the same-page gather of the same bytes from sources that already have page Pd (the rate to approach).  The pages
default to 8:1 -> 1:16, 4:2 -> 64:16, 2:8 -> 16:64; --pages Ps:Pd overrides them.  Sample destination blocks of every arm are
compared with tests/repage_gather_oracle.py.

--pp SRC_PP:SRC_TP:DST_TP times kvbm_kernels_paged_stage_repage_gather on a 4k-token Llama-3-70B sequence (80 layers, 8 KV heads
x 128): decode rank 0 of TP DST_TP (page Pd) from a SRC_PP x SRC_TP prefill group (page Ps, each source pool holding only its
stage's layers), against the two-pass workaround, the re-paging gather from sources that hold every layer and the same-page
staged gather (run_pp).  --pages Ps:Pd, default 16:64."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from dynamo_b200 import kernels as K  # noqa: E402
from tests.repage_oracle import repage, table_slice  # noqa: E402
from tests.repage_gather_oracle import repage_gather  # noqa: E402
from tests.reshard_oracle import reshard_plan  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--tokens", type=int, default=4096)
p.add_argument("--iters", type=int, default=20)
p.add_argument("--cast", choices=["none", "fp8-to-bf16"], default="none")
p.add_argument("--only", default=None, help="comma-separated config names to run")
p.add_argument("--reshard", default=None, help="S:D -- time the re-paging gather from TP S to rank 0 of TP D")
p.add_argument("--pages", default=None, help="Ps:Pd for --reshard (default: 8:1 1:16, 4:2 64:16, 2:8 16:64) or --pp (default 16:64)")
p.add_argument("--pp", default=None, metavar="SRC_PP:SRC_TP:DST_TP",
               help="time kvbm_kernels_paged_stage_repage_gather: decode rank 0 of TP DST_TP from a SRC_PP x SRC_TP prefill group")
a = p.parse_args()
CAST = K.CastMode.FP8E4M3_TO_BF16 if a.cast == "fp8-to-bf16" else K.CastMode.NONE
SE, DE = (1, 2) if CAST else (2, 2)
NHD = int(K.KvBlockLayout.OperationalNHD)
dev = torch.device("cuda:0")
torch.cuda.set_device(0)
stream = torch.cuda.current_stream()
sp = int(stream.cuda_stream)

# name: (src page, dst page, token_begin, token_end, outer, heads, head_dim)
T = a.tokens
CONFIGS = {"16to64": (16, 64, 0, T, 2, 8, 128), "64to16": (64, 16, 0, T, 2, 8, 128), "16to16_partial": (16, 16, 0, T - 5, 2, 8, 128),
           "1to16": (1, 16, 0, T, 2, 8, 128), "16to1": (16, 1, 0, T, 2, 8, 128), "mla_16to64": (16, 64, 0, T, 1, 1, 576)}
NL = 32


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "not read")
    return {"name": name, "power_limit": limit}


class Pool:
    """A vLLM-style layer-separate pool (block is the second dimension), NHD regions of `page` tokens."""

    def __init__(self, nb, page, no, nh, hd, elem, seed, nl=None):
        self.nb, self.page, self.no, self.region, self.nl = nb, page, no, page * nh * hd * elem, nl or NL
        g = torch.Generator(device=dev).manual_seed(seed)
        self.layers = [torch.randint(0, 256, (no * nb * self.region,), dtype=torch.uint8, device=dev, generator=g) for _ in range(self.nl)]
        self.base = torch.tensor([t.data_ptr() for t in self.layers], dtype=torch.int64, device=dev)
        self.desc = K.PagedLayout(self.base.data_ptr(), self.region, nb * self.region, self.region, self.nl, no, nb)

    def block(self, b):
        return np.concatenate([self.layers[l][o * self.nb * self.region + b * self.region:][:self.region].cpu().numpy()
                               for l in range(self.nl) for o in range(self.no)])


def timed(fn, iters=a.iters, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def wall(fn, iters=a.iters, warm=3):
    for _ in range(warm):
        fn()
        torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def run(name, ps, pd, tb, te, no, nh, hd):
    rng = np.random.default_rng(0)
    ns, nd = -(-te // ps), -(-te // pd)
    src, dst = Pool(ns + 8, ps, no, nh, hd, SE, 1), Pool(nd + 8, pd, no, nh, hd, DE, 2)
    stab, dtab = rng.permutation(ns + 8)[:ns].tolist(), rng.permutation(nd + 8)[:nd].tolist()
    sids, dids = table_slice(stab, tb, te, ps), table_slice(dtab, tb, te, pd)
    si, di = torch.tensor(sids, dtype=torch.int32, device=dev), torch.tensor(dids, dtype=torch.int32, device=dev)
    s_row = hd * SE
    moved = (te - tb) * NL * no * nh * hd * (SE + DE)          # bytes read + written
    # sample destination blocks: the first, one in the middle, the last; their bytes before any arm ran
    sample = sorted({0, len(dids) // 2, len(dids) - 1})
    before = {j: dst.block(dids[j]) for j in sample}

    def expected(j):
        lo, hi = max(tb, (tb // pd + j) * pd), min(te, (tb // pd + j + 1) * pd)
        s = table_slice(stab, lo, hi, ps)
        return repage([src.block(b) for b in s], [before[j]], NHD, NHD, NL, no, nh, ps, pd, s_row, lo, hi, int(CAST))[0]

    def check(arm):
        torch.cuda.synchronize()
        for j in sample:
            assert np.array_equal(dst.block(dids[j]), expected(j)), (name, arm, j)
            for l in range(NL):           # restore the sample so the next arm starts from the same bytes
                for o in range(no):
                    off = (l * no + o) * dst.region
                    dst.layers[l][o * dst.nb * dst.region + dids[j] * dst.region:][:dst.region].copy_(
                        torch.from_numpy(before[j][off:off + dst.region]))

    out = []
    info = card()

    def emit(arm, ms, **kw):
        r = {"config": name, "arm": arm, "src_page": ps, "dst_page": pd, "tokens": te - tb, "layers": NL, "outer": no, "heads": nh,
             "head_dim": hd, "cast": a.cast, "ms": round(ms, 4), "GBps": round(moved / ms / 1e6, 1), "card": info}
        r.update(kw)
        print(json.dumps(r), flush=True)
        out.append(r)

    S = K.PermuteSide(src.desc, si.data_ptr(), NHD)
    D = K.PermuteSide(dst.desc, di.data_ptr(), NHD)
    fn = lambda: K.check(K.paged_repage(S, ps, D, pd, tb, te, 0, NL, nh, s_row, int(CAST), stream=sp), "paged_repage")  # noqa: E731
    ms = timed(fn)
    check("repage")
    emit("repage", ms)

    # the same bytes with equal pages: the paged permute of the big page's blocks (NHD -> NHD, fused cast as asked)
    big = max(ps, pd)
    nbig = -(-(te - tb) // big)
    eq_src, eq_dst = Pool(nbig + 8, big, no, nh, hd, SE, 3), Pool(nbig + 8, big, no, nh, hd, DE, 4)
    es = torch.tensor(rng.permutation(nbig + 8)[:nbig].tolist(), dtype=torch.int32, device=dev)
    ed = torch.tensor(rng.permutation(nbig + 8)[:nbig].tolist(), dtype=torch.int32, device=dev)
    ES, ED = K.PermuteSide(eq_src.desc, es.data_ptr(), NHD), K.PermuteSide(eq_dst.desc, ed.data_ptr(), NHD)
    ms_eq = timed(lambda: K.check(K.paged_permute_cast(ES, ED, nbig, 0, NL, nh, big, s_row, int(CAST), stream=sp), "paged_permute_cast"))
    torch.cuda.synchronize()
    b0 = int(es[0].item()), int(ed[0].item())
    want = repage([eq_src.block(b0[0])], [eq_dst.block(b0[1])], NHD, NHD, NL, no, nh, big, big, s_row, 0, big, int(CAST))[0]
    assert np.array_equal(eq_dst.block(b0[1]), want), (name, "same_page")
    emit("same_page_permute", ms_eq, page=big, blocks=nbig)
    del eq_src, eq_dst

    if CAST == K.CastMode.NONE:
        # K1 over host-built pointer tables of min(Ps, Pd)-token runs: NHD keeps a run of tokens contiguous inside a region
        run_t = min(ps, pd)
        runs = [(t, min(t + run_t - (t % run_t), te)) for t in range(tb, te, run_t)] if tb % run_t == 0 else None
        assert runs is not None
        full = [r for r in runs if r[1] - r[0] == run_t]
        tok_b = nh * hd * SE
        stab_a, dtab_a = np.array(stab, dtype=np.int64), np.array(dtab, dtype=np.int64)
        s_lay = np.array([t.data_ptr() for t in src.layers], dtype=np.int64)
        d_lay = np.array([t.data_ptr() for t in dst.layers], dtype=np.int64)
        t0s = np.array([r[0] for r in full], dtype=np.int64)

        def k1_flow():
            # (layer, outer, run) -> the run's address on each side
            s_blk, s_slot = stab_a[t0s // ps], t0s % ps
            d_blk, d_slot = dtab_a[t0s // pd], t0s % pd
            lo = np.arange(NL * no, dtype=np.int64)
            l_idx, o_idx = lo // no, lo % no
            sp_tab = (s_lay[l_idx][:, None] + (o_idx * src.nb * src.region)[:, None] + (s_blk * src.region + s_slot * tok_b)[None, :]).reshape(-1)
            dp_tab = (d_lay[l_idx][:, None] + (o_idx * dst.nb * dst.region)[:, None] + (d_blk * dst.region + d_slot * tok_b)[None, :]).reshape(-1)
            tab = torch.from_numpy(np.concatenate([sp_tab, dp_tab])).pin_memory().to(dev, non_blocking=True)
            n = sp_tab.size
            K.check(K.vectorized_copy(tab.data_ptr(), tab.data_ptr() + 8 * n, run_t * tok_b, n, sp), "vectorized_copy")

        if len(full) == len(runs):
            ms_k1 = wall(k1_flow)
            check("k1")
            ms_rp_wall = wall(fn)
            emit("k1_pointer_tables", ms_k1, run_tokens=run_t, pairs=NL * no * len(full), timed_as="host flow (tables, upload, launch, wait)")
            emit("repage_host_flow", ms_rp_wall, timed_as="host flow (launch, wait)")
    return out


def run_reshard(src_tp, dst_tp, ps, pd, H=8, hd=128, no=2):
    """Decode rank 0 of TP dst_tp (page pd) from the TP src_tp ranks (page ps) that hold its heads: one launch, the two-pass
    workaround and the same-page gather, alternated."""
    name = f"tp{src_tp}_p{ps}_to_tp{dst_tp}_p{pd}"
    plan = reshard_plan(H, src_tp, dst_tp, 0)             # (src_rank, src_head_begin, dst_head_begin, head_count)
    ranks = sorted({w[0] for w in plan})
    index = {r: i for i, r in enumerate(ranks)}
    snh, dnh = max(1, H // src_tp), max(1, H // dst_tp)
    covered = sum(w[3] for w in plan)
    tb, te = 0, a.tokens
    ns, nd = -(-te // ps), -(-te // pd)
    rng = np.random.default_rng(0)
    src = {r: Pool(ns + 8, ps, no, snh, hd, SE, 10 + r) for r in ranks}
    stab = {r: rng.permutation(ns + 8)[:ns].tolist() for r in ranks}
    dst = Pool(nd + 8, pd, no, dnh, hd, DE, 2)
    dtab = rng.permutation(nd + 8)[:nd].tolist()
    si = {r: torch.tensor(stab[r], dtype=torch.int32, device=dev) for r in ranks}
    di = torch.tensor(dtab, dtype=torch.int32, device=dev)
    s_row = hd * SE
    moved = (te - tb) * NL * no * covered * hd * (SE + DE)    # bytes read + written
    D = K.PermuteSide(dst.desc, di.data_ptr(), NHD)
    srcs = [K.PermuteSource(K.PermuteSide(src[r].desc, si[r].data_ptr(), NHD), snh, sb, db, k) for r, sb, db, k in plan]

    def one():
        K.check(K.paged_repage_gather(srcs, ps, D, dnh, pd, tb, te, 0, NL, s_row, int(CAST), stream=sp), "paged_repage_gather")

    # the workaround: each source re-paged into a staging pool of page pd with its own heads (the cast in this pass), then the
    # gather out of the staging pools; staging block i is destination block i
    stage = {r: Pool(nd, pd, no, snh, hd, DE, 20 + r) for r in ranks}
    ident = torch.arange(nd, dtype=torch.int32, device=dev)
    st_src = {r: K.PermuteSide(stage[r].desc, ident.data_ptr(), NHD) for r in ranks}
    st_gather = [K.PermuteSource(st_src[r], snh, sb, db, k) for r, sb, db, k in plan]

    def two_pass():
        for r in ranks:
            K.check(K.paged_repage(K.PermuteSide(src[r].desc, si[r].data_ptr(), NHD), ps, st_src[r], pd, tb, te, 0, NL, snh, s_row, int(CAST),
                                   stream=sp), "paged_repage")
        K.check(K.paged_permute_gather(st_gather, D, dnh, nd, 0, NL, pd, hd * DE, stream=sp), "paged_permute_gather")

    # the same bytes with equal pages: sources that already have page pd
    eq = {r: Pool(nd + 8, pd, no, snh, hd, SE, 30 + r) for r in ranks}
    etab = {r: rng.permutation(nd + 8)[:nd].tolist() for r in ranks}
    ei = {r: torch.tensor(etab[r], dtype=torch.int32, device=dev) for r in ranks}
    eq_dst = Pool(nd + 8, pd, no, dnh, hd, DE, 5)
    edi = torch.tensor(rng.permutation(nd + 8)[:nd].tolist(), dtype=torch.int32, device=dev)
    ED = K.PermuteSide(eq_dst.desc, edi.data_ptr(), NHD)
    eq_srcs = [K.PermuteSource(K.PermuteSide(eq[r].desc, ei[r].data_ptr(), NHD), snh, sb, db, k) for r, sb, db, k in plan]

    def same_page():
        K.check(K.paged_permute_gather(eq_srcs, ED, dnh, nd, 0, NL, pd, s_row, int(CAST), stream=sp), "paged_permute_gather")

    sample = sorted({0, nd // 2, nd - 1})
    windows = [(index[r], sb, db, k) for r, sb, db, k in plan]

    def host_blocks(pool, ids):    # one download per layer, then the blocks' regions in (layer, outer) order
        h = [t.cpu().numpy() for t in pool.layers]
        return [np.concatenate([h[l][o * pool.nb * pool.region + b * pool.region:][:pool.region] for l in range(NL) for o in range(pool.no)])
                for b in ids]

    def check(arm, pool, tables, page, d_pool, d_ids):
        torch.cuda.synchronize()
        for j in sample:            # every covered head of every token is overwritten: the old bytes do not show through
            lo, hi = j * pd, (j + 1) * pd
            sources = [(host_blocks(pool[r], table_slice(tables[r], lo, hi, page)), NHD, snh) for r in ranks]
            got = host_blocks(d_pool, [d_ids[j]])
            want = repage_gather(sources, windows, got, NHD, dnh, NL, no, page, pd, s_row, lo, hi, int(CAST))[0]
            assert np.array_equal(got[0], want), (name, arm, j)

    arms = {"repage_gather": one, "two_pass": two_pass, "same_page_gather": same_page}
    for fn in arms.values():
        for _ in range(3):
            fn()
    check("repage_gather", src, stab, ps, dst, dtab)
    two_pass()
    check("two_pass", src, stab, ps, dst, dtab)
    check("same_page_gather", eq, etab, pd, eq_dst, edi.tolist())
    times = {k: [] for k in arms}
    for _ in range(a.iters):           # the arms alternate within every round
        for k, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            fn()
            e1.record(stream)
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1))
    info = card()
    ref = statistics.median(times["same_page_gather"])
    for k in arms:
        ms = statistics.median(times[k])
        print(json.dumps({"config": name, "arm": k, "src_tp": src_tp, "dst_tp": dst_tp, "src_page": ps, "dst_page": pd, "sources": len(ranks),
                          "tokens": te - tb, "layers": NL, "outer": no, "covered_heads": covered, "head_dim": hd, "cast": a.cast,
                          "ms": round(ms, 4), "GBps": round(moved / ms / 1e6, 1), "vs_same_page": round(ref / ms, 3),
                          "timed_as": "all launches of the arm, CUDA events, median of %d alternated rounds" % a.iters, "card": info}),
              flush=True)


def run_pp(src_pp, src_tp, dst_tp, ps, pd, H=8, hd=128, no=2, nl=80):
    """Decode rank 0 (PP1, TP dst_tp, page pd) of a Llama-3-70B sequence (80 layers, 8 KV heads x 128) from a src_pp x src_tp
    prefill group (page ps), every source pool holding only its stage's layers.  Arms, alternated within each of 5 rounds of
    --iters launches (CUDA events): the one launch; the two-pass workaround (the staged gather at ps into a staging pool that
    holds every decode layer, then kvbm_kernels_paged_repage out of it); the re-paging gather of the same bytes from sources that
    hold every layer (the ceiling); the staged gather from sources that already have page pd.  Median of the round medians, with
    their range.  Sample destination blocks of every arm are compared with tests/stage_repage_oracle.py."""
    from dynamo_b200.physical import tp_pp_reshard_plan, tp_reshard_plan
    from tests.stage_repage_oracle import stage_repage_gather
    name = f"pp{src_pp}tp{src_tp}_p{ps}_to_tp{dst_tp}_p{pd}"
    plan = tp_pp_reshard_plan(H, nl, src_tp, src_pp, dst_tp, 1, 0)
    ranks = sorted({w.src_rank for w in plan})
    snh, dnh, snl = max(1, H // src_tp), max(1, H // dst_tp), nl // src_pp
    tb, te = 0, a.tokens
    ns, nd = -(-te // ps), -(-te // pd)
    rng = np.random.default_rng(0)
    s_row, d_row = hd * SE, hd * DE
    moved = (te - tb) * nl * no * dnh * hd * (SE + DE)    # bytes read + written: every head of every decode layer

    def side(pool, ids):
        return K.PermuteSide(pool.desc, ids.data_ptr(), NHD)

    def tables(n_ids):
        tab = {r: rng.permutation(n_ids + 8)[:n_ids].tolist() for r in ranks}
        return tab, {r: torch.tensor(tab[r], dtype=torch.int32, device=dev) for r in ranks}

    src = {r: Pool(ns + 8, ps, no, snh, hd, SE, 10 + r, nl=snl) for r in ranks}
    stab, si = tables(ns)
    dst = Pool(nd + 8, pd, no, dnh, hd, DE, 2, nl=nl)
    dtab = rng.permutation(nd + 8)[:nd].tolist()
    di = torch.tensor(dtab, dtype=torch.int32, device=dev)
    D = side(dst, di)
    staged = [K.StageSource(K.PermuteSource(side(src[w.src_rank], si[w.src_rank]), snh, w.src_head_begin, w.dst_head_begin, w.head_count),
                            w.src_layer_begin, w.dst_layer_begin, w.layer_count) for w in plan]

    def one():
        K.check(K.paged_stage_repage_gather(staged, ps, D, dnh, pd, tb, te, 0, nl, s_row, int(CAST), stream=sp), "paged_stage_repage_gather")

    # the workaround: the staged gather (with the cast) into a staging pool of page ps over every decode layer, staging block i
    # holding tokens [i * ps, (i + 1) * ps), then the plain re-page of the staging pool into the destination
    staging = Pool(ns, ps, no, dnh, hd, DE, 3, nl=nl)
    ident = torch.arange(ns, dtype=torch.int32, device=dev)
    st_d = side(staging, ident)

    def two_pass():
        K.check(K.paged_stage_gather(staged, st_d, dnh, ns, 0, nl, ps, s_row, int(CAST), stream=sp), "paged_stage_gather")
        K.check(K.paged_repage(st_d, ps, D, pd, tb, te, 0, nl, dnh, d_row, 0, stream=sp), "paged_repage")

    # the ceiling: the same bytes re-page-gathered from TP sources that hold every layer
    tp_plan = tp_reshard_plan(H, src_tp, dst_tp, 0)
    full = {w.src_rank: Pool(ns + 8, ps, no, snh, hd, SE, 40 + w.src_rank, nl=nl) for w in tp_plan}
    ftab = {r: rng.permutation(ns + 8)[:ns].tolist() for r in full}
    fi = {r: torch.tensor(ftab[r], dtype=torch.int32, device=dev) for r in full}
    full_srcs = [K.PermuteSource(side(full[w.src_rank], fi[w.src_rank]), snh, w.src_head_begin, w.dst_head_begin, w.head_count) for w in tp_plan]

    def ceiling():
        K.check(K.paged_repage_gather(full_srcs, ps, D, dnh, pd, tb, te, 0, nl, s_row, int(CAST), stream=sp), "paged_repage_gather")

    # the staged gather of the same bytes from sources that already have page pd, into a destination of its own
    eq = {r: Pool(nd + 8, pd, no, snh, hd, SE, 30 + r, nl=snl) for r in ranks}
    etab, ei = tables(nd)
    eq_dst = Pool(nd + 8, pd, no, dnh, hd, DE, 5, nl=nl)
    edtab = rng.permutation(nd + 8)[:nd].tolist()
    edi = torch.tensor(edtab, dtype=torch.int32, device=dev)
    eq_staged = [K.StageSource(K.PermuteSource(side(eq[w.src_rank], ei[w.src_rank]), snh, w.src_head_begin, w.dst_head_begin, w.head_count),
                               w.src_layer_begin, w.dst_layer_begin, w.layer_count) for w in plan]

    def same_page():
        K.check(K.paged_stage_gather(eq_staged, side(eq_dst, edi), dnh, nd, 0, nl, pd, s_row, int(CAST), stream=sp), "paged_stage_gather")

    sample = sorted({0, nd // 2, nd - 1})

    def check(arm, pools, tabs, page, d_pool, d_ids, windows):
        torch.cuda.synchronize()
        for j in sample:            # every head of every token is overwritten: the old bytes do not show through
            lo, hi = j * pd, min((j + 1) * pd, te)
            order = sorted(pools)
            sources = [([pools[r].block(b) for b in table_slice(tabs[r], lo, hi, page)], NHD, snh, pools[r].nl) for r in order]
            got = d_pool.block(d_ids[j])
            win = [(order.index(w[0]),) + tuple(w[1:]) for w in windows]
            want = stage_repage_gather(sources, win, [got], NHD, dnh, nl, no, page, pd, s_row, lo, hi, int(CAST))[0]
            assert np.array_equal(got, want), (name, arm, j)

    stage_windows = [(w.src_rank, w.src_layer_begin, w.dst_layer_begin, w.layer_count, w.src_head_begin, w.dst_head_begin, w.head_count)
                     for w in plan]
    full_windows = [(w.src_rank, 0, 0, nl, w.src_head_begin, w.dst_head_begin, w.head_count) for w in tp_plan]
    arms = {"stage_repage_one_launch": one, "two_pass_stage_gather_then_repage": two_pass, "repage_gather_from_full_layer_sources": ceiling,
            "same_page_stage_gather": same_page}
    for k, fn in arms.items():
        for t in (eq_dst if k == "same_page_stage_gather" else dst).layers:   # the arm alone decides the bytes it is checked on
            t.fill_(0x5A)
        for _ in range(3):
            fn()
        if k == "same_page_stage_gather":
            check(k, eq, etab, pd, eq_dst, edtab, stage_windows)
        elif k == "repage_gather_from_full_layer_sources":
            check(k, full, ftab, ps, dst, dtab, full_windows)
        else:
            check(k, src, stab, ps, dst, dtab, stage_windows)
    rounds = {k: [] for k in arms}
    for _ in range(5):                 # the arms alternate within every round
        for k, fn in arms.items():
            rounds[k].append(timed(fn))
    info = card()
    for k in arms:
        ms = statistics.median(rounds[k])
        print(json.dumps({"config": name, "arm": k, "src_pp": src_pp, "src_tp": src_tp, "dst_tp": dst_tp, "src_page": ps, "dst_page": pd,
                          "sources": len(ranks), "tokens": te - tb, "layers": nl, "outer": no, "heads": dnh, "head_dim": hd, "cast": a.cast,
                          "ms": round(ms, 4), "ms_range": [round(min(rounds[k]), 4), round(max(rounds[k]), 4)],
                          "GBps": round(moved / ms / 1e6, 1),
                          "timed_as": "CUDA events, median of 5 alternated rounds of median-of-%d launches" % a.iters, "card": info}),
              flush=True)


if a.pp:
    s_pp, s_tp, d_tp = (int(x) for x in a.pp.split(":"))
    run_pp(s_pp, s_tp, d_tp, *(tuple(int(x) for x in a.pages.split(":")) if a.pages else (16, 64)))
elif a.reshard:
    s_tp, d_tp = (int(x) for x in a.reshard.split(":"))
    default_pages = {(8, 1): (1, 16), (4, 2): (64, 16), (2, 8): (16, 64)}
    pages = tuple(int(x) for x in a.pages.split(":")) if a.pages else default_pages[(s_tp, d_tp)]
    run_reshard(s_tp, d_tp, *pages)
else:
    for name, cfg in CONFIGS.items():
        if a.only and name not in a.only.split(","):
            continue
        run(name, *cfg)
        torch.cuda.empty_cache()

"""Decode-visible TTFT of a disaggregated deployment under the reference's own hand-off model (SURVEY.md §8 f4).

A small discrete-event replay in the shape of the reference's offline disagg replay
(/root/reference/lib/mocker/src/replay/offline/disagg.rs: arrival -> prefill worker -> `handoff_delay_ms` event ->
decode enqueue -> first token) and of the PrefillRouter flow (lib/llm/src/kv_router/prefill_router/execution.rs:124-220:
pick a prefill worker, prefill, hand the KV to the decode worker the KV router chose).  As in the mocker,

    TTFT = queueing + T_prefill + T_transfer + T_first_decode            (lib/mocker/src/common/utils.rs:14-40)

and ONLY `T_transfer` differs between the data planes compared:

  mocker64   tokens * kv_bytes_per_token / 64 GB/s     the mocker's default `--kv-transfer-bandwidth`
             (components/src/dynamo/mocker/utils/kv_cache.py:30-33), a pure delay
  cpu        the reference's CPU memcpy path at the rate of a bench.py cpu_baseline (--cpu-bench),
             one transfer at a time per prefill host
  ours       latency + bytes / BW fitted to measured 1 -> 1 NVLink pushes (--sweep, benchmarks/fanout_sweep.py output),
             one transfer at a time per prefill GPU (its NVLink egress is the shared resource)
  ours_pull  with --pull-bench (a bench.py --gpus 2 line): the same latency, the pull direction's measured rate
Without those files the model falls back to the H100 SXM data sheet's NVLink rate and an assumed CPU rate, and says so.

The decode worker is chosen by the KV router restated in libkvbm_router.so (`RadixTree.find_matches`, XXH3 block hashes):
best prefix overlap wins, ties go to the least loaded worker -- and only the NON-HIT suffix of the block table is moved
(`prefix_hit_block_table`), so the prefix-hit rate is an outcome of the request mix, not a knob.

    python benchmarks/ttft_sim.py [--sweep fanout_n2.jsonl] [--cpu-bench bench_n1.json] [--pull-bench bench_n2.json] --out sim.json
"""
import argparse
import heapq
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dynamo_b200 import router as R  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--requests", type=int, default=2000)
ap.add_argument("--rate", type=float, default=25.0, help="Poisson arrival rate, requests/s")
ap.add_argument("--prefill-workers", type=int, default=4)
ap.add_argument("--decode-workers", type=int, default=4)
ap.add_argument("--prompt-tokens", type=int, nargs="+", default=[1024, 4096, 4096, 8192, 16384])
ap.add_argument("--families", type=int, default=16, help="distinct shared prefixes (system prompts / documents)")
ap.add_argument("--shared-fraction", type=float, default=0.5, help="fraction of a prompt that is its family's shared prefix")
ap.add_argument("--block-size", type=int, default=16)
ap.add_argument("--kv-bytes-per-token", type=int, default=32 * 2 * 8 * 128 * 2)   # Llama-3-8B bf16 (docs/mocker/mocker.md:447)
ap.add_argument("--prefill-tok-per-s", type=float, default=60000.0)
ap.add_argument("--first-decode-ms", type=float, default=8.0)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--out", default="")
ap.add_argument("--sweep", default="", help="fanout_sweep.py jsonl of 1 -> 1 pushes to fit `ours` to")
ap.add_argument("--cpu-bench", default="", help="bench.py result line with a cpu_baseline")
ap.add_argument("--pull-bench", default="", help="bench.py --gpus 2 result line (pull direction)")
a = ap.parse_args()


def fit_ours():
    """latency_ms + bytes / BW from the measured 1 -> 1 pushes (least squares over the sweep's sizes)."""
    pts = []
    if a.sweep:
        for line in open(a.sweep):
            d = json.loads(line)
            if d["mode"] == "distinct" and d["max_ctas"] == 0 and d["cast"] == "none":
                pts.append((d["blocks_moved"] * 2 * 1024 * 1024, d["ms"]))
    if len(pts) < 2:
        return 0.02, 450.0, "fallback: assumed 20 us launch latency + H100 SXM data-sheet NVLink 4 rate (450 GB/s per direction), not measured"
    x = np.array([p[0] for p in pts], dtype=np.float64)
    y = np.array([p[1] for p in pts], dtype=np.float64)
    slope, icpt = np.polyfit(x, y, 1)
    return max(0.0, float(icpt)), 1e-6 / slope, f"fit over {len(pts)} measured 1->1 pushes"


def _bench_line(path):
    for line in open(path):
        if line.startswith("{"):
            return json.loads(line)
    raise ValueError(path)


def cpu_rate():
    if a.cpu_bench:
        return float(_bench_line(a.cpu_bench)["cpu_baseline"]["value"]), f"{a.cpu_bench} cpu_baseline"
    return 47.0, "fallback: assumed 47 GB/s, not measured"


def pull_rate():
    """the decode GPU pulls (reads the prefill pool over NVLink) -- measured 1 -> 1 rate of the bench line"""
    if a.pull_bench:
        return float(_bench_line(a.pull_bench)["value"]), a.pull_bench
    return None, "no pull bench line"


LAT_MS, BW_GBS, ours_src = fit_ours()
CPU_GBS, cpu_src = cpu_rate()
PULL_GBS, pull_src = pull_rate()
PLANES = {
    "mocker64": dict(serial=False, ms=lambda b: b / 64e9 * 1e3),
    "cpu": dict(serial=True, ms=lambda b: b / (CPU_GBS * 1e9) * 1e3),
    "ours": dict(serial=True, ms=lambda b: (LAT_MS + b / (BW_GBS * 1e9) * 1e3) if b else 0.0),
}
if PULL_GBS:
    # same launch latency as the fitted push, the pull direction's bandwidth; the prefill GPU's port stays the shared resource
    PLANES["ours_pull"] = dict(serial=True, ms=lambda b: (LAT_MS + b / (PULL_GBS * 1e9) * 1e3) if b else 0.0)

# ---- request trace (identical for every data plane) ----
rng = np.random.default_rng(a.seed)
arrivals = np.cumsum(rng.exponential(1.0 / a.rate, a.requests)) * 1e3   # ms
families = [rng.integers(1, 50000, max(a.prompt_tokens), dtype=np.int64) for _ in range(a.families)]
reqs = []
for i in range(a.requests):
    n = int(rng.choice(a.prompt_tokens))
    fam = int(rng.integers(0, a.families))
    shared = int(n * a.shared_fraction) // a.block_size * a.block_size
    toks = np.concatenate([families[fam][:shared], rng.integers(50000, 100000, n - shared, dtype=np.int64)])
    reqs.append((float(arrivals[i]), toks))


def simulate(plane):
    tree = R.RadixTree()
    prefill_free = [0.0] * a.prefill_workers      # time each prefill worker finishes its queue
    link_free = [0.0] * a.prefill_workers         # the prefill GPU's egress (serial planes)
    decode_load = [0] * a.decode_workers
    ttft, moved, total, xfer = [], 0, 0, []
    pending = []                                  # (time the KV becomes resident on the decode worker, worker, hashes)
    for t_arr, toks in reqs:
        # KV events of finished transfers reach the router before later arrivals are routed
        while pending and pending[0][0] <= t_arr:
            _, w, bh, sh = heapq.heappop(pending)
            tree.apply_stored(w, sh, bh)
            decode_load[w] -= 1
        bh = R.compute_block_hash_for_seq(toks.tolist(), a.block_size)
        sh = R.compute_seq_hash_for_block(bh)
        scores = tree.find_matches(bh).scores
        best = max(range(a.decode_workers), key=lambda w: (scores.get((w, 0), 0), -decode_load[w]))
        hit = min(scores.get((best, 0), 0), len(bh))
        nbytes = (len(bh) - hit) * a.block_size * a.kv_bytes_per_token
        moved += len(bh) - hit
        total += len(bh)
        p = min(range(a.prefill_workers), key=lambda k: prefill_free[k])
        start = max(t_arr, prefill_free[p])
        done_prefill = start + len(toks) / a.prefill_tok_per_s * 1e3
        prefill_free[p] = done_prefill
        t_x = PLANES[plane]["ms"](nbytes)
        if PLANES[plane]["serial"]:
            x_start = max(done_prefill, link_free[p])
            link_free[p] = x_start + t_x
            landed = x_start + t_x
        else:
            landed = done_prefill + t_x
        xfer.append(landed - done_prefill)
        first = landed + a.first_decode_ms
        ttft.append(first - t_arr)
        decode_load[best] += 1
        heapq.heappush(pending, (landed, best, bh, sh))
    tree.close()
    q = lambda v, p: float(np.percentile(v, p))
    return {"ttft_ms": {"p50": q(ttft, 50), "p90": q(ttft, 90), "p99": q(ttft, 99)},
            "handoff_ms": {"p50": q(xfer, 50), "p90": q(xfer, 90), "p99": q(xfer, 99)},
            "prefix_hit_rate": 1.0 - moved / total, "blocks_moved": moved}


res = {"config": {k: getattr(a, k) for k in ("requests", "rate", "prefill_workers", "decode_workers", "prompt_tokens", "families",
                                             "shared_fraction", "block_size", "kv_bytes_per_token", "prefill_tok_per_s", "first_decode_ms", "seed")},
       "ours_model": {"latency_ms": LAT_MS, "bandwidth_gbs": BW_GBS, "source": ours_src},
       "cpu_model": {"bandwidth_gbs": CPU_GBS, "source": cpu_src},
       "planes": {name: simulate(name) for name in PLANES}}
base = res["planes"]["ours"]["ttft_ms"]
res["ttft_drop_ms_vs_ours"] = {name: {k: r["ttft_ms"][k] - base[k] for k in base} for name, r in res["planes"].items() if name != "ours"}
if a.out:
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    json.dump(res, open(a.out, "w"), indent=1)

c = res["config"]
print("# Decode-visible TTFT over a request stream, only the hand-off data plane changes (`benchmarks/ttft_sim.py`)\n")
print(f"{c['requests']} requests, Poisson {c['rate']}/s, prompts {c['prompt_tokens']} tokens, {c['families']} shared prefixes covering "
      f"{c['shared_fraction']:.0%} of a prompt, {c['prefill_workers']} prefill + {c['decode_workers']} decode workers, prefill "
      f"{c['prefill_tok_per_s']:.0f} tok/s, first decode step {c['first_decode_ms']} ms, {c['kv_bytes_per_token'] // 1024} KiB of KV per token.")
print(f"Decode worker = best prefix overlap in the RadixTree (libkvbm_router.so); prefix-hit rate that results: "
      f"{res['planes']['ours']['prefix_hit_rate']:.1%} of blocks never move.\n")
print(f"`ours` = {LAT_MS * 1e3:.0f} us + bytes / {BW_GBS:.0f} GB/s ({ours_src}); `cpu` = {CPU_GBS:.1f} GB/s ({cpu_src})"
      + (f"; `ours_pull` = the same latency + bytes / {PULL_GBS:.0f} GB/s ({pull_src})" if PULL_GBS else "") + ".\n")
print("| data plane | hand-off p50 / p90 / p99 (ms) | TTFT p50 (ms) | TTFT p90 | TTFT p99 | TTFT p50 above `ours` (ms) |")
print("|---|---|---:|---:|---:|---:|")
for name, r in res["planes"].items():
    h, t = r["handoff_ms"], r["ttft_ms"]
    print(f"| {name} | {h['p50']:.2f} / {h['p90']:.2f} / {h['p99']:.2f} | {t['p50']:.1f} | {t['p90']:.1f} | {t['p99']:.1f} | {t['p50'] - base['p50']:.1f} |")

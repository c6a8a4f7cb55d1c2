"""Decode-visible TTFT under the reference's own hand-off model, from bench.py result lines.

The mocker models the prefill->decode hand-off as  delay_ms = tokens * kv_bytes_per_token / (bw * 1e9) * 1e3
(lib/mocker/src/common/utils.rs:14-40; default bw 64 GB/s "inter-node InfiniBand",
components/src/dynamo/mocker/utils/kv_cache.py:30-33) and TTFT = T_prefill + T_transfer + T_first_decode.
Only T_transfer differs between data planes, so the TTFT drop of a decode worker is the difference of transfer
times.  This script tabulates it for the measured fan-outs.

    python benchmarks/ttft_model.py bench_n1.json bench_n2.json ... > ttft.md
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
rows = []
for f in sys.argv[1:]:
    try:
        d = json.loads(open(f).read().strip().splitlines()[-1])
    except Exception:
        continue
    if "config" not in d or "pairs" in d["config"].get("topology", "") or "fp8" in d["config"]["workload"]:
        continue
    rows.append((d["n_gpus"], os.path.basename(f), d))
best = {}
for n, name, d in rows:           # keep the latest file per N and per replicate flag
    key = (n, "identical" in d["config"]["workload"])
    best[key] = (name, d)

tokens, kv_bytes_per_token = 4096, 32 * 2 * 8 * 128 * 2          # Llama-3-8B bf16: 128 KiB per token (docs/mocker/mocker.md:447)
B = tokens * kv_bytes_per_token
cpu1 = cpu_all = None
for (n, rep), (name, d) in best.items():
    if n == 1 and "cpu_baseline" in d:
        cpu_all = d["cpu_baseline"]["value"]
        cpu1 = d["cpu_baseline"].get("single_thread_value")
print("# Decode-visible TTFT change from the KV hand-off alone (Llama-3-8B bf16, 4 k-token prompt, 512 MiB of KV per decode worker)\n")
print("`T_transfer = tokens * kv_bytes_per_token / BW` (lib/mocker/src/common/utils.rs:14-40); measured columns are the p50 of the")
print("end-to-end step (`e2e.p50_ms`, host API, host block tables) of the bench lines given.\n")
print("| fan-out | payload | ours: all destinations complete (ms, p50) | mocker default 64 GB/s, per destination (ms) | NVLink figure of the docs 450 GB/s (ms) | "
      "reference CPU path, all host threads, destinations one after another (ms) | TTFT drop of the LAST decode worker vs CPU path (ms) | file |")
print("|---|---|---:|---:|---:|---:|---:|---|")
for (n, rep), (name, d) in sorted(best.items()):
    nd = max(1, n - 1)
    ours = d["e2e"]["p50_ms"]
    mock = B / 64e9 * 1e3
    nvl = B / 450e9 * 1e3
    cpu = (B / (cpu_all * 1e9) * 1e3 * nd) if cpu_all else float("nan")
    topo = "same GPU" if n == 1 else f"1 -> {nd}"
    print(f"| {topo} | {'identical' if rep else 'distinct'} | {ours:.3f} | {mock:.2f} | {nvl:.2f} | {cpu:.1f} | {cpu - ours:.1f} | {name} |")
if cpu1:
    print(f"\nThe reference's memcpy executor is a single-threaded loop: {cpu1:.2f} GB/s on one core of this host, i.e. {B / (cpu1 * 1e9) * 1e3:.0f} ms per "
          f"destination; the table uses the stronger all-threads figure ({cpu_all:.1f} GB/s).")

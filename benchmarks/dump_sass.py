"""Writes the SASS of the library's kernels under profiles/ (no GPU needed: cuobjdump reads the sm_90a cubin in the .so).

    python benchmarks/dump_sass.py            -> profiles/sass_<kernel>.txt + profiles/sass_summary.md
The summary counts the mnemonics that show what the kernel is built from: UBLKCP = cp.async.bulk (TMA 1-D bulk),
SYNCS = mbarrier, UTMACMDFLUSH / fences, F2FP = fp8<->bf16 converts, LDG/STG widths for the SIMT kernels."""
import collections
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "dynamo_b200", "libkvbm_kernels.so")
WANT = {"paged_copy_kernelILi0": "paged_copy_cast0", "paged_copy_kernelILi1": "paged_copy_fp8_to_bf16", "paged_copy_kernelILi2": "paged_copy_bf16_to_fp8",
        "pair_copy_kernel": "pair_copy_k1", "permute_rows_kernelILb1": "permute_rows_to_universal", "permute_rows_kernelILb0": "permute_rows_from_universal",
        "paged_permute_kernel": "paged_permute"}
KEYS = ["UBLKCP.S.G", "UBLKCP.G.S", "SYNCS.ARRIVE.TRANS64", "SYNCS.PHASECHK.TRANS64.TRYWAIT", "SYNCS.ARRIVE", "UTMACMDFLUSH", "FENCE.VIEW.ASYNC",
            "F2FP", "ATOMG", "LDG.E.NA.128", "STG.E.NA.128", "LDS.128", "STS.128", "NANOSLEEP", "SHFL"]


def main():
    txt = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
    out = os.path.join(ROOT, "profiles")
    os.makedirs(out, exist_ok=True)
    parts = re.split(r"\n\s*Function : ", txt)
    rows = []
    for p in parts[1:]:
        name = p.split("\n", 1)[0].strip()
        tag = next((v for k, v in WANT.items() if k in name), None)
        if not tag:
            continue
        body = p
        ops = collections.Counter(m.group(1) for m in re.finditer(r"^\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d\s+)?([A-Z][A-Z0-9_.]+)", body, re.M))
        regs = re.search(r"REG:(\d+)", body)
        with open(os.path.join(out, f"sass_{tag}.txt"), "w") as f:
            f.write("Function : " + p)
        rows.append((tag, name, sum(ops.values()), {k: sum(v for o, v in ops.items() if o.startswith(k)) for k in KEYS}))
    with open(os.path.join(out, "sass_summary.md"), "w") as f:
        f.write("# SASS of the sm_90a kernels in dynamo_b200/libkvbm_kernels.so (`python benchmarks/dump_sass.py`)\n\n")
        f.write("| kernel | instructions | " + " | ".join(KEYS) + " |\n|---|---:|" + "---:|" * len(KEYS) + "\n")
        for tag, name, total, c in rows:
            f.write(f"| `{tag}` | {total} | " + " | ".join(str(c[k]) for k in KEYS) + " |\n")
        f.write("\nUBLKCP.S.G / UBLKCP.G.S = cp.async.bulk global->shared / shared->global (TMA 1-D bulk copies); SYNCS.* = mbarrier "
                "arrive / expect_tx / try_wait; F2FP = e4m3<->f16/f32 converts of the fused cast; the K1 and permute kernels are SIMT "
                "(128-bit LDG/STG with L1 no-allocate).\n")
    for r in rows:
        print(r[0], r[2], {k: v for k, v in r[3].items() if v})


if __name__ == "__main__":
    main()

"""The literal drop-in (INTEGRATION.md §1, lib/kvbm-kernels/cuda/stubs.c:4-7): ONE C binary built against the six reference
symbols runs with this repo's libkvbm_kernels.so and with the reference's own kernels compiled unmodified under the same
file name, and must print the same bytes.  The reference's output is stored in tests/golden/ref_kernels_dropin.txt
(make_ref_outputs.py); when oracle/_ref is built the reference also runs live.  No Python in the data path."""
import os
import shutil
import subprocess

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_kernels_dropin.txt")


def build_dropin(exe):
    """Compiles tests/c/kernels_dropin.c against this repo's libkvbm_kernels.so into `exe`; None when gcc/cudart are absent."""
    gcc = shutil.which("gcc")
    if not gcc or not os.path.exists(os.path.join(CUDA, "lib64", "libcudart.so")):
        return None
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-I", os.path.join(CUDA, "include"), os.path.join(ROOT, "tests", "c", "kernels_dropin.c"),
                        "-o", str(exe), "-L", os.path.join(ROOT, "dynamo_b200"), "-lkvbm_kernels", "-L", os.path.join(CUDA, "lib64"), "-lcudart"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def run_dropin(exe, libdir):
    """Runs the drop-in binary with `libdir`'s libkvbm_kernels.so; returns (exit code, stdout + stderr)."""
    env = dict(os.environ, LD_LIBRARY_PATH=f"{libdir}:{os.path.join(CUDA, 'lib64')}:" + os.environ.get("LD_LIBRARY_PATH", ""))
    p = subprocess.run([str(exe)], capture_output=True, text=True, env=env, timeout=120)
    return p.returncode, p.stdout + p.stderr


def ref_libdir(tmp_path):
    """A directory holding oracle/_ref's reference kernels under the product's file name, or None when not built."""
    ref_so = os.path.join(ROOT, "oracle", "_ref", "libkvbm_kernels_ref.so")
    if not os.path.exists(ref_so):
        return None
    refdir = tmp_path / "ref"
    refdir.mkdir()
    os.symlink(ref_so, refdir / "libkvbm_kernels.so")
    return str(refdir)


def test_same_binary_same_output_with_either_library(tmp_path):
    exe = build_dropin(tmp_path / "dropin")
    if exe is None:
        pytest.skip("gcc or libcudart are not installed")
    rc, out = run_dropin(exe, os.path.join(ROOT, "dynamo_b200"))
    assert rc == 0 and out.strip().endswith("done") and "k3_roundtrip 1" in out, out
    assert "k1_edges 0 0 1" in out and "k4_edges 0 1" in out and "k2_bad_dtype 1" in out, out
    with open(GOLDEN) as f:
        want = f.read()
    assert out == want, f"ours:\n{out}\nreference (stored):\n{want}"
    refdir = ref_libdir(tmp_path)
    if refdir is not None:
        rc2, out2 = run_dropin(exe, refdir)
        assert rc2 == 0, out2
        assert out2 == out, f"ours:\n{out}\nreference:\n{out2}"

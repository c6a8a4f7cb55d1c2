"""Records what the reference's own kernels compute for the GPU tests that compare with them, so that those tests run
without the reference.  Needs a GPU and oracle/_ref/libkvbm_kernels_ref.so (build() with the reference tree present):

    python tests/golden/make_ref_outputs.py

Writes, next to this file:
  ref_k1_rows_sha256.npy                       SHA-256 of every destination row of the seeded K1 case (test_gpu_kernels)
  ref_block_from_universal_{nhd,hnd}.npy       K3 on the position-encoded F32 KAT, chunks as float32 (test_gpu_kernels)
  ref_kernels_dropin.txt                       stdout of tests/c/kernels_dropin.c linked to the reference (test_gpu_zz_c_dropin)
"""
import os
import pathlib
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import kats  # noqa: E402
from tests import test_gpu_kernels as T  # noqa: E402
from tests import test_gpu_zz_c_dropin as D  # noqa: E402

R = T.ref_lib()
if R is None:
    raise SystemExit("oracle/_ref/libkvbm_kernels_ref.so is not built")
np.save(os.path.join(HERE, "ref_k1_rows_sha256.npy"), T.row_sha256(T.k1_reference_case(R.kvbm_kernels_launch_vectorized_copy)))
for layout in (kats.NHD, kats.HND):
    np.save(T.permute_golden_path(layout), T.permute_position_encoded_chunks(R, layout))
with tempfile.TemporaryDirectory() as tmp:
    tmp = pathlib.Path(tmp)
    exe = D.build_dropin(tmp / "dropin")
    rc, out = D.run_dropin(exe, D.ref_libdir(tmp))
    if rc != 0:
        raise SystemExit("drop-in binary failed with the reference:\n" + out)
    with open(D.GOLDEN, "w") as f:
        f.write(out)
print("wrote reference outputs under", HERE)

"""Generates the golden tables of the SCALED fp8(e4m3fn) <-> bf16 cast from torch CPU (run in the build container).

    python tests/golden/make_scaled_cast_tables.py

For each scale s of SCALES, in fp32 on both sides, as vLLM's fp8 KV cache does (dequantise multiplies, quantise divides):
    scaled_fp8_e4m3_to_bf16_torch.npy  uint16[len(SCALES), 256]    (code.to(float32) * s).to(bfloat16)
    scaled_bf16_to_fp8_e4m3_torch.npy  uint8[len(SCALES), 65536]   (bf16.to(float32) / s).to(float8_e4m3fn)
The scale is a full float32 tensor, so torch divides element by element (no reciprocal of a scalar divisor).  torch's
down-cast maps overflow to NaN; the transfer kernels saturate to +-448 -- tests compare wherever torch's answer is not an
overflow-NaN, as for the unscaled tables.
SCALES: 1 (the unscaled cast), a power of two, two calibrated-looking values, one that overflows e4m3 for most of the bf16
range (s = 2^-12: |x| > 0.11 saturates) and one that sends much of it into the e4m3 subnormals (s = 600).
"""
import os

import numpy as np
import torch

SCALES = np.array([1.0, 0.25, 0.0173, 3.9, 2.0**-12, 600.0], dtype=np.float32)

if __name__ == "__main__":
    here = os.path.dirname(os.path.abspath(__file__))
    codes = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).to(torch.float32)
    bits = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).to(torch.float32)
    up, down = [], []
    for s in SCALES.tolist():
        up.append((codes * torch.full_like(codes, s)).to(torch.bfloat16).view(torch.int16).numpy().astype(np.uint16))
        down.append((bits / torch.full_like(bits, s)).to(torch.float8_e4m3fn).view(torch.uint8).numpy())
    np.save(os.path.join(here, "scaled_fp8_e4m3_to_bf16_torch.npy"), np.stack(up))
    np.save(os.path.join(here, "scaled_bf16_to_fp8_e4m3_torch.npy"), np.stack(down))
    print("torch", torch.__version__, "scales", SCALES.tolist())

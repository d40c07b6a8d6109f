"""The chain kernel's lighter instruction stream keeps every bit:

* bsb_div6 (bsb_common.h), the hard-swish's division by 6 without the IEEE divide subroutine, equals v / 6 for every
  float32 bit pattern: on the CPU under FTZ + DAZ (tests/emu/div6_check.cpp) and on the H100 against __fdiv_rn;
* the compile-time-geometry instantiations of k_chain (Meet full 9x16, MLKit 16x16) and the runtime-shape ones (Meet
  lite 6x10, and every geometry when the emulator forces them) give the bits of the stand-alone kernels and the oracle
  (the fixed shapes and Meet lite on the emulator: test_emu_pipeline.py, test_chain_two_per_sm.py)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import parity_common as pc
from tests.conftest import model_path

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "backscrub_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def test_div6_every_float_on_the_cpu(tmp_path):
    exe = str(tmp_path / "div6_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DBSB_EMU", "-I" + os.path.join(HERE, "emu"), "-I" + CSRC,
                           "-ffp-contract=off", "-fno-fast-math", "-mfma", "-msse4.1", "-Wall", "-Wno-misleading-indentation",
                           "-Wno-unused-function", "-pthread", "-o", exe, os.path.join(HERE, "emu", "div6_check.cpp")])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "mismatches 0" in r.stdout, r.stdout + r.stderr


GPU_CHECK = r"""
#include <cstdio>
#include "bsb_common.h"
__global__ void k_div6_check(unsigned hi, unsigned long long* bad, unsigned* first) {
  const unsigned u = (hi << 24) | (blockIdx.x << 10) | threadIdx.x;   // 2^14 blocks of 1024 threads per call
  const float v = __uint_as_float(u);
  const float ref = __fdiv_rn(v, 6.f), got = bsb::bsb_div6(v);
  if (__float_as_uint(ref) != __float_as_uint(got) && !(ref != ref && got != got)) {
    if (atomicAdd(bad, 1ull) == 0) *first = u;
  }
}
int main() {
  unsigned long long* bad; unsigned* first;
  if (cudaMallocManaged(&bad, 8) != cudaSuccess || cudaMallocManaged(&first, 4) != cudaSuccess) return 2;
  *bad = 0; *first = 0;
  for (unsigned hi = 0; hi < 256; ++hi) k_div6_check<<<1u << 14, 1024>>>(hi, bad, first);
  if (cudaDeviceSynchronize() != cudaSuccess) return 2;
  printf("patterns 4294967296 mismatches %llu first 0x%08x\n", *bad, *first);
  return *bad != 0;
}
"""


@pytest.mark.gpu
def test_div6_every_float_on_the_gpu(tmp_path):
    """The device's FTZ comparisons and fmaf agree with __fdiv_rn over all 2^32 inputs (the library's nvcc flags)."""
    src = tmp_path / "div6_gpu_check.cu"
    src.write_text(GPU_CHECK)
    exe = str(tmp_path / "div6_gpu_check")
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false", "-ftz=true",
                           "-prec-div=true", "-prec-sqrt=true", "-I" + CSRC, "-o", exe, str(src)])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "mismatches 0" in r.stdout, r.stdout + r.stderr


@pytest.mark.parametrize("key", ["meet_full", "mlkit"])
def test_runtime_shape_chain_on_the_emulator(key):
    """The runtime-shape instantiations, which no bundled graph but Meet lite reaches, for the geometries of the others."""
    from tests.emu.emu_lib import emu
    lib = emu()
    flag = ctypes.c_int.in_dll(lib, "bsb_emu_chain_runtime_shape")
    flag.value = 1
    try:
        pc.check_chain(lib, key, n=2)
    finally:
        flag.value = 0


@pytest.mark.gpu
@pytest.mark.parametrize("key", ["meet_lite", "mlkit"])
def test_chain_two_waves(key):
    """2 x SMs + 3 frames in one call (Meet lite 6x10: two CTAs per SM; MLKit 16x16: one), bit for bit against the
    stand-alone kernels, and a few frames against the oracle."""
    import torch

    import backscrub_b200 as bs
    from backscrub_b200 import api
    lib = bs.lib()
    assert lib.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    n = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 3
    rng = np.random.default_rng(53)
    outs, x = {}, None
    try:
        for chain in (1, 0):
            assert lib.bsb_set_tuning(b"cnn_chain", chain)
            g = api.MaskGen(lib, model_path(key), 1280, 720, max_batch=n)
            if x is None:
                x = rng.uniform(0, 1, (n, *g.in_hwc)).astype(np.float32)
            outs[chain] = g.infer(x)
            g.close()
    finally:
        lib.bsb_set_tuning(b"cnn_chain", 1)
    for b in range(n):
        assert np.array_equal(outs[1][b].view(np.uint32), outs[0][b].view(np.uint32)), f"{key} frame {b}: chain and stand-alone kernels differ"
    m = po.Model(model_path(key))
    for b in (0, n // 2, n - 1):
        assert np.array_equal(outs[1][b].view(np.uint32), m.invoke(x[b])[0].view(np.uint32)), f"{key} frame {b} differs from the oracle"

"""The two inverted-residual blocks between the encoder entry and the chain (Meet full / lite, MLKit) run as two kernels,
k_enc_block_s2 and k_enc_block_res, instead of eight.  They must give the bits of the oracle and of a KEEP_TENSORS
context (every step stand-alone), on the kernel-logic emulator and, with several waves of CTAs, on the H100.  The
18x32, 12x20 and 32x32 block outputs leave partial 4x16 tiles in both directions."""
import numpy as np
import pytest

from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path

KEEP_TENSORS = 1
LAUNCHES = {"meet_full": 19, "meet_lite": 19, "mlkit": 22}


def run(lib, key, W, H, n, x, frames, flags):
    g = api.MaskGen(lib, model_path(key), W, H, max_batch=n, flags=flags)
    out = g.infer(x)
    g.set_background(synth.background())
    comp = g.composite(frames)
    launches = g.launches_per_call
    g.close()
    return out, comp, launches


def check_against_stand_alone(lib, key, W, H, n, oracle_frames, seed):
    rng = np.random.default_rng(seed)
    in_hwc = api.MaskGen(lib, model_path(key), W, H, max_batch=1).in_hwc
    x = rng.uniform(0, 1, (n, *in_hwc)).astype(np.float32)
    base = np.stack([synth.frame(W, H, t=t) for t in range(min(n, 8))])
    frames = np.ascontiguousarray(np.resize(base, (n, *base.shape[1:])))
    fused, fused_comp, fused_launches = run(lib, key, W, H, n, x, frames, 0)
    keep, keep_comp, keep_launches = run(lib, key, W, H, n, x, frames, KEEP_TENSORS)
    assert fused_launches == LAUNCHES[key] and keep_launches > fused_launches, (key, fused_launches, keep_launches)
    assert np.array_equal(fused.view(np.uint32), keep.view(np.uint32)), f"{key}: fused blocks and stand-alone kernels differ"
    for a, b, what in zip(fused_comp, keep_comp, ("composite", "YUYV", "mask")):
        assert np.array_equal(a, b), f"{key}: {what} differs from the KEEP_TENSORS context"
    m = po.Model(model_path(key))
    for b in oracle_frames:
        assert np.array_equal(fused[b].view(np.uint32), m.invoke(x[b])[0].view(np.uint32)), f"{key}: frame {b} differs from the oracle"


@pytest.mark.parametrize("key", ["meet_full", "meet_lite", "mlkit"])
def test_encoder_blocks_on_the_emulator(key):
    from tests.emu.emu_lib import emu
    check_against_stand_alone(emu(), key, 640, 480, 3, (0, 1, 2), seed=61)


@pytest.mark.gpu
@pytest.mark.parametrize("key,W,H,n", [("meet_full", 1280, 720, None), ("mlkit", 640, 480, 32)])
def test_encoder_blocks_on_the_gpu(key, W, H, n):
    """Meet: 2 x SMs + 3 frames in one call (co-resident CTAs, a partial last wave); MLKit: 32 frames."""
    import torch

    import backscrub_b200 as bs
    lib = bs.lib()
    assert lib.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    if n is None:
        n = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 3
    check_against_stand_alone(lib, key, W, H, n, (0, n // 2, n - 1), seed=67)

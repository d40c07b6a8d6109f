"""The Meet full chain (9x16 pixels) runs two frames per SM: 16-channel E slices, 384 threads, __launch_bounds__(384, 2).
It must give the bits of the stand-alone kernels it replaces and of the oracle, on the kernel-logic emulator and, with
co-resident CTAs and a partial last wave, on the H100."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import parity_common as pc
from tests.conftest import model_path


def test_meet_full_chain_on_the_emulator():
    from tests.emu.emu_lib import emu
    pc.check_chain(emu(), "meet_full", n=2)


@pytest.mark.gpu
def test_meet_full_chain_two_waves():
    """2 x SMs + 3 frames in one call: every SM holds two chain CTAs, and a last partial wave follows."""
    import torch

    import backscrub_b200 as bs
    from backscrub_b200 import api
    lib = bs.lib()
    assert lib.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    n = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 3
    rng = np.random.default_rng(47)
    outs, x = {}, None
    try:
        for chain in (1, 0):
            assert lib.bsb_set_tuning(b"cnn_chain", chain)
            g = api.MaskGen(lib, model_path("meet_full"), 1280, 720, max_batch=n)
            if x is None:
                x = rng.uniform(0, 1, (n, *g.in_hwc)).astype(np.float32)
            outs[chain] = g.infer(x)
            g.close()
    finally:
        lib.bsb_set_tuning(b"cnn_chain", 1)
    for b in range(n):
        assert np.array_equal(outs[1][b].view(np.uint32), outs[0][b].view(np.uint32)), f"frame {b}: chain and stand-alone kernels differ"
    m = po.Model(model_path("meet_full"))
    for b in (0, n // 2, n - 1):
        assert np.array_equal(outs[1][b].view(np.uint32), m.invoke(x[b])[0].view(np.uint32)), f"frame {b} differs from the oracle"

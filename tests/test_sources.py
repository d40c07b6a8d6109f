"""Independent sources: one frame from each of several cameras per call (bsb_set_sources, bsb_composite_sources,
bsb_composite_sources_yuyv_device).  Every frame must equal what a context of its own — or the oracle fed that camera's
frames in order — produces: per-source smoother state, per-source background, no leaks between sources or into the
plain (one-stream) state of the same context.

`-m "not gpu"`: the kernel-logic emulator build vs the oracle.  `-m gpu`: the sm_90a library vs plain contexts."""
import numpy as np
import pytest

from backscrub_b200 import api
from oracle import pyoracle as po
from tests import synth
from tests.conftest import model_path

FLAG_EXACT = 16


def _frame(W, H, src, t):
    return synth.frame(W, H, t=t, stream=src)


def _backgrounds():
    bg = synth.background()
    return {"ctx": bg[::-1].copy(), 0: bg, 2: np.roll(bg, 200, axis=1)[:600, :1000].copy()}


class _Feeds:
    """per-source oracles and frame counters"""

    def __init__(self, key, W, H, n):
        self.W, self.H = W, H
        self.o = [po.MaskGen(model_path(key), W, H) for _ in range(n)]
        self.t = [0] * n

    def next_frames(self, ids):
        fr = np.stack([_frame(self.W, self.H, s, self.t[s]) for s in ids])
        return fr

    def check(self, g, ids, frames, res, bg_of, **kw):
        out, yuyv, mask = res
        for b, s in enumerate(ids):
            ro, ry, rm = self.o[s].composite_ex(frames[b], bg_of(s), **kw)
            tag = (ids, b, s, self.t[s])
            assert np.array_equal(g.stage_u8(2, b), self.o[s].ofinal), f"smoother state differs {tag}"
            assert np.array_equal(mask[b], rm), f"mask differs {tag}"
            assert np.array_equal(out[b], ro), f"composite differs {tag}"
            assert np.array_equal(yuyv[b], ry), f"YUYV differs {tag}"
            self.t[s] += 1

    def restart(self, key, s):
        self.o[s] = po.MaskGen(model_path(key), self.W, self.H)


# ---------------------------------------------------------------------------------------------------------------------
# kernel-logic emulator
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


def _sources_ctx(lib, key, W, H, n_sources, max_batch, bgs, flags=0):
    g = api.MaskGen(lib, model_path(key), W, H, max_batch=max_batch, flags=flags)
    g.set_background(bgs["ctx"])
    g.set_sources(n_sources)
    for s in range(n_sources):
        if s in bgs:
            g.set_source_background(s, bgs[s])
    return g


def test_interleaved_sources_match_the_oracle(emu_lib):
    key, W, H = "meet_lite", 320, 240
    bgs = _backgrounds()
    g = _sources_ctx(emu_lib, key, W, H, 3, 3, bgs)
    f = _Feeds(key, W, H, 3)
    for ids in ([0, 1, 2], [2, 0], [1], [1, 0, 2], [0]):
        fr = f.next_frames(ids)
        f.check(g, ids, fr, g.composite_sources(fr, ids), lambda s: bgs.get(s, bgs["ctx"]))
    g.close()


@pytest.mark.slow
def test_deeplab_sources(emu_lib):
    """the DeepLab decision kernel with the 33 -> 257 resize folded in (k_decision_up_sources)"""
    key, W, H = "deeplab", 160, 120
    bgs = _backgrounds()
    g = _sources_ctx(emu_lib, key, W, H, 2, 2, bgs, flags=FLAG_EXACT)
    f = _Feeds(key, W, H, 2)
    for ids in ([1, 0], [0, 1]):
        fr = f.next_frames(ids)
        f.check(g, ids, fr, g.composite_sources(fr, ids), lambda s: bgs.get(s, bgs["ctx"]))
    g.close()


def test_bgblur_camera_blur_slot(emu_lib):
    """bgblur on, no context background: source 0 blends its own (blurred) background, source 1 its own blurred camera
    frame; the blur strength is switched after the source background was set, and once more between calls."""
    key, W, H = "meet_lite", 320, 240
    bg = synth.background()
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=2)
    g.set_sources(2)
    g.set_source_background(0, bg)
    g.set_bgblur(7)
    f = _Feeds(key, W, H, 2)
    bg_of = lambda s: bg if s == 0 else None
    for ids in ([0, 1], [1, 0]):
        fr = f.next_frames(ids)
        f.check(g, ids, fr, g.composite_sources(fr, ids), bg_of, bgblur=7)
    g.set_bgblur(25)
    fr = f.next_frames([1, 0])
    f.check(g, [1, 0], fr, g.composite_sources(fr, [1, 0]), bg_of, bgblur=25)
    # a call whose frames all have a background of their own: source 1 gets one now
    g.set_source_background(1, bg[::-1].copy())
    fr = f.next_frames([1, 0])
    f.check(g, [1, 0], fr, g.composite_sources(fr, [1, 0]), lambda s: bg if s == 0 else bg[::-1].copy(), bgblur=25)
    g.close()


def test_plain_and_sources_calls_are_isolated(emu_lib):
    """plain calls on a sources context see only their own stream; reset_source restarts one source alone; clearing a
    source background falls back to the context background"""
    key, W, H = "meet_lite", 320, 240
    bgs = _backgrounds()
    g = _sources_ctx(emu_lib, key, W, H, 3, 3, bgs)
    f = _Feeds(key, W, H, 3)
    plain = po.MaskGen(model_path(key), W, H)
    pt = [0]

    def plain_call():
        fr = _frame(W, H, 7, pt[0])
        out, yuyv, mask = g.composite(fr)
        ro, ry, rm = plain.composite(fr, bgs["ctx"])
        assert np.array_equal(out, ro) and np.array_equal(yuyv, ry) and np.array_equal(mask, rm), ("plain", pt[0])
        assert np.array_equal(g.stage_u8(2, 0), plain.ofinal)
        pt[0] += 1

    bg_of = lambda s: bgs.get(s, bgs["ctx"])
    plain_call()
    for ids in ([0, 1, 2], [2, 1]):
        fr = f.next_frames(ids)
        f.check(g, ids, fr, g.composite_sources(fr, ids), bg_of)
    plain_call()
    g.reset_source(1)
    f.restart(key, 1)
    for ids in ([1, 0, 2], [0, 2, 1]):
        fr = f.next_frames(ids)
        f.check(g, ids, fr, g.composite_sources(fr, ids), bg_of)
    plain_call()
    g.set_source_background(2, None)
    fr = f.next_frames([2])
    f.check(g, [2], fr, g.composite_sources(fr, [2]), lambda s: bgs["ctx"])
    plain_call()
    g.close()


def test_sources_errors(emu_lib):
    key, W, H = "meet_lite", 320, 240
    g = api.MaskGen(emu_lib, model_path(key), W, H, max_batch=3)
    fr = lambda n: np.stack([_frame(W, H, s, 0) for s in range(n)]) if n else np.zeros((0, H, W, 3), np.uint8)
    with pytest.raises(api.BackscrubError, match="set_sources"):
        g.composite_sources(fr(1), [0])
    with pytest.raises(api.BackscrubError, match="set_sources"):
        g.set_source_background(0, synth.background())
    with pytest.raises(api.BackscrubError, match="out of range"):
        g.set_sources(0)
    g.set_sources(3)
    bad = [([0, 0], "distinct"), ([1, 2, 1], "distinct"), ([-1], "out of range"), ([3], "out of range"), ([0, 1, 2, 0], "n_frames"),
           ([], "n_frames")]
    for ids, msg in bad:
        with pytest.raises(api.BackscrubError, match=msg):
            g.composite_sources(fr(len(ids)), ids)
    for s in (-1, 3):
        with pytest.raises(api.BackscrubError, match="out of range"):
            g.set_source_background(s, synth.background())
        with pytest.raises(api.BackscrubError, match="out of range"):
            g.reset_source(s)
    bg = synth.background()
    g.set_background_ring(np.stack([bg, bg[::-1].copy()]), advance=1)
    with pytest.raises(api.BackscrubError, match="still context background"):
        g.composite_sources(fr(2), [0, 1])
    g.set_background(bg)
    # the context is still usable, and nothing above advanced a source: every source is at its first frame
    o = [po.MaskGen(model_path(key), W, H) for _ in range(3)]
    ids = [2, 0, 1]
    frames = np.stack([_frame(W, H, s, 0) for s in ids])
    out, yuyv, mask = g.composite_sources(frames, ids)
    for b, s in enumerate(ids):
        ro, ry, rm = o[s].composite(frames[b], bg)
        assert np.array_equal(out[b], ro) and np.array_equal(yuyv[b], ry) and np.array_equal(mask[b], rm), s
    g.close()


# ---------------------------------------------------------------------------------------------------------------------
# H100
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu_lib():
    import backscrub_b200 as bs
    L = bs.lib()
    assert L.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
    return L


class _DeviceSources:
    """camera YUYV frames of each source on the device, and one plain batch-1 context per source as the reference"""

    def __init__(self, lib, key, W, H, n_sources, max_batch, own_bg, flags=0):
        import torch
        self.torch, self.W, self.H = torch, W, H
        bg = synth.background()
        self.ctx_bg = bg[::-1].copy()
        self.src_bg = {s: np.roll(bg, 37 * s, axis=1) for s in own_bg}
        self.g = api.MaskGen(lib, model_path(key), W, H, max_batch=max_batch, flags=flags)
        self.g.set_background(self.ctx_bg)
        self.g.set_sources(n_sources)
        for s, b in self.src_bg.items():
            self.g.set_source_background(s, b)
        self.lib, self.key, self.flags = lib, key, flags
        self.ref = {}
        self.t = [0] * n_sources
        dev = "cuda:0"
        self.d_in = torch.empty((max_batch, H, W, 2), dtype=torch.uint8, device=dev)
        self.d_out = torch.empty((max_batch, H, W, 3), dtype=torch.uint8, device=dev)
        self.d_yuyv = torch.empty((max_batch, H, W, 2), dtype=torch.uint8, device=dev)
        self.d_mask = torch.empty((max_batch, H, W), dtype=torch.uint8, device=dev)

    def plain(self, s):
        if s not in self.ref:
            import torch
            c = api.MaskGen(self.lib, model_path(self.key), self.W, self.H, max_batch=1, flags=self.flags)
            c.set_background(self.src_bg.get(s, self.ctx_bg))
            bufs = [torch.empty(shape, dtype=torch.uint8, device="cuda:0")
                    for shape in ((1, self.H, self.W, 2), (1, self.H, self.W, 3), (1, self.H, self.W, 2), (1, self.H, self.W))]
            self.ref[s] = (c, bufs)
        return self.ref[s]

    def yuyv_of(self, s, t):
        return synth.yuyv_frame(self.W, self.H, t=t, stream=s)

    def load(self, ids):
        host = np.stack([self.yuyv_of(s, self.t[s]) for s in ids])
        self.d_in[:len(ids)].copy_(self.torch.from_numpy(host))
        return host

    def run(self, ids, sync=True):
        n = len(ids)
        self.g.composite_sources_yuyv_device(n, ids, self.d_in.data_ptr(), self.d_out.data_ptr(), self.d_yuyv.data_ptr(),
                                             self.d_mask.data_ptr(), sync=sync)

    def results(self, n):
        return self.d_out[:n].cpu().numpy(), self.d_yuyv[:n].cpu().numpy(), self.d_mask[:n].cpu().numpy()

    def check(self, ids, got, frames=None, sample=None):
        out, yuyv, mask = got
        for b, s in enumerate(ids):
            if sample is not None and s not in sample:
                self.t[s] += 1
                continue
            c, (r_in, r_out, r_yuyv, r_mask) = self.plain(s)
            fr = frames[b] if frames is not None else self.yuyv_of(s, self.t[s])
            r_in.copy_(self.torch.from_numpy(fr[None]))
            c.composite_yuyv_device(1, r_in.data_ptr(), r_out.data_ptr(), r_yuyv.data_ptr(), r_mask.data_ptr(), sync=True)
            tag = (ids, b, s, self.t[s])
            assert np.array_equal(mask[b], r_mask[0].cpu().numpy()), f"mask differs {tag}"
            assert np.array_equal(out[b], r_out[0].cpu().numpy()), f"composite differs {tag}"
            assert np.array_equal(yuyv[b], r_yuyv[0].cpu().numpy()), f"YUYV differs {tag}"
            self.t[s] += 1

    def step(self, ids, sample=None):
        self.load(ids)
        self.run(ids)
        self.check(ids, self.results(len(ids)), sample=sample)

    def close(self):
        self.g.close()
        for c, _ in self.ref.values():
            c.close()


@pytest.mark.gpu
def test_gpu_meet_720p_sources_match_plain_contexts(gpu_lib):
    """Meet full 1280x720 through the TMA post kernel reading camera YUYV in place: 8 sources, half with their own
    background, six calls of varying subsets and orders == 8 plain contexts fed batch-1 calls."""
    d = _DeviceSources(gpu_lib, "meet_full", 1280, 720, 8, 8, own_bg=(0, 2, 4, 6))
    for ids in ([0, 1, 2, 3, 4, 5, 6, 7], [7, 5, 3, 1], [2], [6, 0, 4, 1, 7], [3, 2, 1, 0, 4, 5, 6, 7], [5, 4]):
        d.step(ids)
        assert d.g.yuyv_native, "the sources call should read the camera YUYV in place (TMA post kernel)"
    d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("key,W,H", [("deeplab", 1280, 720), ("bodypix", 640, 480)])
def test_gpu_tensor_core_models_match_plain_contexts(gpu_lib, key, W, H):
    """default flags (tensor-core 1x1 convs): a frame's rows accumulate the same way whatever the batch, so the sources
    call must give the bytes of a batch-1 plain context"""
    d = _DeviceSources(gpu_lib, key, W, H, 3, 3, own_bg=(1,))
    assert d.g.uses_tensor_cores
    for ids in ([0, 1, 2], [2, 0], [1, 2, 0]):
        d.step(ids)
    d.close()


@pytest.mark.gpu
def test_gpu_graph_replayed_for_new_ids(gpu_lib):
    """two asynchronous calls, same n and buffers, different ids, no sync in between: one captured graph (no launches
    issued by the second call), and each call read its own id table"""
    d = _DeviceSources(gpu_lib, "meet_lite", 640, 480, 4, 2, own_bg=(3,))
    d.step([0, 1])                              # captures the graph for n = 2 and these buffers
    # the first frames of sources 2 and 3, fed from the same buffer to sources 0 / 1 (as their second frames) and then to
    # sources 2 / 3
    frames01 = d.load([2, 3])
    l0 = gpu_lib.bsb_total_launches()
    d.run([0, 1], sync=False)
    l1 = gpu_lib.bsb_total_launches()
    d.run([2, 3], sync=False)
    l2 = gpu_lib.bsb_total_launches()
    assert l1 == l0 and l2 == l1, (l0, l1, l2)
    d.g.synchronize()
    got = d.results(2)
    d.check([2, 3], got)                        # the second call's outputs
    # the first call advanced sources 0 and 1 with frames01: replay it on their references, then a synced call proves
    # the states they carry
    for b, s in enumerate([0, 1]):
        c, (r_in, r_out, r_yuyv, r_mask) = d.plain(s)
        r_in.copy_(d.torch.from_numpy(frames01[b][None]))
        c.composite_yuyv_device(1, r_in.data_ptr(), r_out.data_ptr(), r_yuyv.data_ptr(), r_mask.data_ptr(), sync=True)
        d.t[s] += 1
    d.step([1, 0])
    d.close()


@pytest.mark.gpu
def test_gpu_host_bgr_entry_matches_device_path(gpu_lib):
    """MLKit 640x480: bsb_composite_sources (host BGR frames) == bsb_composite_sources_yuyv_device on the same frames"""
    key, W, H = "mlkit", 640, 480
    d = _DeviceSources(gpu_lib, key, W, H, 3, 3, own_bg=(0,))
    h = api.MaskGen(gpu_lib, model_path(key), W, H, max_batch=3)
    h.set_background(d.ctx_bg)
    h.set_sources(3)
    h.set_source_background(0, d.src_bg[0])
    for ids in ([0, 1, 2], [2, 1], [1, 0, 2]):
        yin = d.load(ids)
        d.run(ids)
        dev = d.results(len(ids))
        bgr = np.stack([api.convert_yuyv_to_bgr(gpu_lib, y) for y in yin])
        host = h.composite_sources(bgr, ids)
        for a, b, what in zip(dev, host, ("composite", "YUYV", "mask")):
            assert np.array_equal(a, b), (ids, what)
    h.close()
    d.close()


@pytest.mark.gpu
def test_gpu_64_sources_in_one_call(gpu_lib):
    """max_batch = 64, one call with a frame of each of 64 sources, then the reverse order: sampled sources == plain
    batch-1 contexts"""
    d = _DeviceSources(gpu_lib, "meet_lite", 640, 480, 64, 64, own_bg=range(0, 64, 3))
    sample = {0, 1, 17, 42, 62, 63}
    d.step(list(range(64)), sample=sample)
    d.step(list(range(63, -1, -1)), sample=sample)
    d.close()

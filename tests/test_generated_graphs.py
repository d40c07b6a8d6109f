"""The CNN planner and its kernels on generated TFLite graphs (tests/tflite_writer.py), not only on the five bundled
models: each operator at shapes of its own, each fusion detector on both sides of its eligibility test, BodyPix-shaped
MobileNetV1 graphs, and the constructs the planner must refuse.

Every graph is checked three ways:
  - the oracle, bit for bit, on every frame of a batch of distinct frames (BSB_FLAG_EXACT);
  - float64 (tests/torch_graph.py): |device - f64| <= 16 n_ops EPS M, where M is the same graph evaluated in float64
    on |input| with |weights| (an upper bound of sum |a||w| through every layer);
  - for graphs of linear ops, ReLU / ReLU6, power-of-two global pools, transposed convs, ADD / MUL and exact-2x
    half-pixel resizes, on dyadic fixtures (inputs multiples of 2^-4, weights small multiples of 2^-3): every partial
    sum is exact in fp32, so the device output must equal the float64 result rounded once, bit for bit.

Each fusion case proves which path it took: the kernels it launches (counted around the call) must be fewer than
those of the same graph with that fusion switched off, a near-miss's exactly as many; and the kernel trace must show,
or not show, the kernel the fusion replaces.  The trace is the emulator's (CUEMU_TRACE, which names a kernel by the
expression launched, so only kernels launched by name are seen) on the CPU and torch.profiler's on the H100 (every
kernel, demangled), where the stem, strip and chain variants are told apart too.

Every test that takes the `runner` fixture runs twice: on the kernel-logic emulator and, under -m gpu, on the H100.

The model family comes from the file's whole path, so graphs are written to a directory whose path contains none of
the family names, under a name that starts with the family the output channel count requires."""
import json
import os
import shutil
import subprocess
import sys
import re
import tempfile
import zlib

import numpy as np
import pytest

from backscrub_b200 import api
from oracle import pyoracle as po
from tests import tflite_writer as tw
from tests import torch_graph
from tests.conftest import ROOT

FAMILIES = ("body-pix", "deeplab", "segm_", "selfie")
KEEP, NO_GRAPH, TENSOR_CORES, FUSE_BLOCKS, EXACT = 1, 2, 4, 8, 16
EPS = 2.0 ** -24

# run one context on the emulator in a subprocess, so that its launch trace names the kernels that ran
_EMU_RUN = """
import json, sys
import numpy as np
from backscrub_b200 import api
from tests.emu.emu_lib import emu
spec = json.loads(sys.argv[1])
lib = emu()
for k, v in spec["tuning"].items():
    assert lib.bsb_set_tuning(k.encode(), v)
x = np.load(spec["x"])
g = api.MaskGen(lib, spec["path"], spec["W"], spec["H"], max_batch=x.shape[0], flags=spec["flags"])
n0 = lib.bsb_total_launches()
y = g.infer(x)
print("launches", lib.bsb_total_launches() - n0)
np.save(spec["y"], y)
g.close()
"""


# ---------------------------------------------------------------------------------------------------- runners
class Emu:
    name = "emu"

    def __init__(self):
        from tests.emu.emu_lib import emu
        self.lib = emu()
        self.tmp = tempfile.mkdtemp(prefix="bsb-run-")

    def close(self):
        shutil.rmtree(self.tmp, ignore_errors=True)

    def run(self, path, x, flags=EXACT, tuning=None, trace=False):
        """(outputs, kernels launched by the call, names of the kernels launched or None)"""
        if not trace:
            return _run_in_process(self.lib, path, x, flags, tuning)
        xp, yp = os.path.join(self.tmp, "x.npy"), os.path.join(self.tmp, "y.npy")
        np.save(xp, x)
        h, w = x.shape[1:3]
        spec = dict(path=path, x=xp, y=yp, flags=flags, tuning=tuning or {}, W=4 * w, H=4 * h)
        r = subprocess.run([sys.executable, "-c", _EMU_RUN, json.dumps(spec)], cwd=ROOT, capture_output=True, text=True,
                           env=dict(os.environ, CUEMU_TRACE="1", PYTHONPATH=ROOT), timeout=600)
        assert r.returncode == 0, r.stderr[-3000:]
        kernels = {ln.split("cuemu: launch ", 1)[1].strip() for ln in r.stderr.splitlines() if "cuemu: launch " in ln}
        launches = int(r.stdout.split("launches", 1)[1].split()[0])
        return np.load(yp), launches, kernels


class Gpu:
    name = "gpu"

    def __init__(self):
        import backscrub_b200 as bs
        self.lib = bs.lib()
        assert self.lib.bsb_device_count() > 0, "no CUDA device: the gpu tests must run on an H100"
        import torch
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count

    def close(self):
        pass

    def run(self, path, x, flags=EXACT, tuning=None, trace=False):
        if not trace:
            return _run_in_process(self.lib, path, x, flags, tuning)
        (y, launches, _), kernels = gpu_kernels(lambda: _run_in_process(self.lib, path, x, flags, tuning))
        return y, launches, kernels


def _short_name(name):
    """'void bsb::(anonymous namespace)::k_chain<3, 16, 384, 2, 0, 0>(bsb::ChainOp const*, ...)' -> 'k_chain<3, 16, ...>'"""
    n = name[5:] if name.startswith("void ") else name
    depth = 0
    for i, ch in enumerate(n):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0 and i > 0:
            n = n[:i]
            break
    base, sep, targs = n.partition("<")
    return base.split("::")[-1] + sep + targs


def gpu_kernels(fn):
    """(fn(), short names of the CUDA kernels it ran), from torch.profiler (CUPTI sees the library's launches too)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r = fn()
        torch.cuda.synchronize()
    return r, {_short_name(e.key) for e in prof.key_averages()}


def _tuning_defaults():
    """the shipped values of the launcher switches, read from struct Tuning in kernels.h"""
    with open(os.path.join(ROOT, "backscrub_b200", "csrc", "kernels.h")) as f:
        src = f.read()
    body = src[src.index("struct Tuning {"):]
    body = body[:body.index("};")]
    return {k: int(v) for k, v in re.findall(r"int (\w+) = (-?\d+);", body)}


TUNING_DEFAULTS = _tuning_defaults()


def _run_in_process(lib, path, x, flags, tuning):
    tuning = tuning or {}
    try:
        for k, v in tuning.items():
            assert lib.bsb_set_tuning(k.encode(), v)
        h, w = x.shape[1:3]
        g = api.MaskGen(lib, path, 4 * w, 4 * h, max_batch=x.shape[0], flags=flags)
        try:
            n0 = lib.bsb_total_launches()
            y = g.infer(x)
            return y, lib.bsb_total_launches() - n0, None
        finally:
            g.close()
    finally:
        for k in tuning:
            lib.bsb_set_tuning(k.encode(), TUNING_DEFAULTS[k])


@pytest.fixture(scope="module")
def gen_dir():
    d = tempfile.mkdtemp(prefix="bsb-graphs-")
    assert not any(f in d for f in FAMILIES), d
    yield d
    shutil.rmtree(d, ignore_errors=True)


def test_tuning_defaults_read_from_the_header():
    assert {"dw_px", "dw_plane", "dw_plane_cs", "cnn_chain", "head", "pw_dws2", "up_pw", "up_staged", "pool_merge",
            "stem_x2"} <= set(TUNING_DEFAULTS)


@pytest.fixture(scope="module", params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def runner(request):
    r = Emu() if request.param == "emu" else Gpu()
    yield r
    r.close()


@pytest.fixture(scope="module")
def gpu_runner():
    return Gpu()


# ---------------------------------------------------------------------------------------------------- graphs
def write(b, d, name, family="selfie"):
    assert not any(f in name for f in FAMILIES), name
    return b.write(os.path.join(d, f"{family}-{name}.tflite"))


def inputs(b, n, seed, dyadic=False):
    h, w, _ = b.shape(b.x)
    rng = np.random.default_rng(seed)
    if dyadic:
        return (rng.integers(0, 17, (n, h, w, 3)) / 16).astype(np.float32)
    return rng.uniform(0, 1, (n, h, w, 3)).astype(np.float32)


def absolute_graph(b, path):
    """the same graph with |weights|: evaluated on |input| in float64 it bounds sum |a||w| through every layer"""
    saved = [t["data"] for t in b.tensors]
    for t in b.tensors:
        if t["data"] is not None and t["dtype"] != "i32":
            t["data"] = np.abs(t["data"])
    try:
        return b.write(path[:-len(".tflite")] + "-abs.tflite")
    finally:
        for t, d in zip(b.tensors, saved):
            t["data"] = d


def check(runner, b, path, n=3, flags=EXACT, tuning=None, dyadic=False, trace=False, seed=0, frames=None):
    """device vs oracle (every frame, bits), vs float64 (bound) and, for dyadic graphs, vs float64 rounded once (bits)"""
    x = inputs(b, n, seed, dyadic)
    y, launches, kernels = runner.run(path, x, flags, tuning, trace)
    m = po.Model(path)
    frames = range(n) if frames is None else frames
    for i in frames:
        ref = m.invoke(x[i])[0]
        assert np.array_equal(y[i].view(np.uint32), ref.view(np.uint32)), \
            f"{os.path.basename(path)}: frame {i} differs from the oracle (max |d| {np.abs(y[i] - ref).max()})"
    m.close()
    n_ops = sum(op["kind"] not in ("DEQUANTIZE",) for op in b.ops)
    abs_path = absolute_graph(b, path)
    for i in sorted({0, n - 1}):
        f64 = torch_graph.run(path, x[i])
        if dyadic:
            assert np.array_equal(y[i].view(np.uint32), f64.astype(np.float32).view(np.uint32)), \
                f"{os.path.basename(path)}: frame {i} differs from the exact result (max |d| {np.abs(y[i] - f64).max()})"
        M = torch_graph.run(abs_path, np.abs(x[i]))
        err = np.abs(y[i].astype(np.float64) - f64)
        tol = 16 * n_ops * EPS * M + 1e-30
        assert (err <= tol).all(), f"{os.path.basename(path)}: frame {i}: |device - f64| {err.max()} over the bound"
    return launches, kernels


def sandwich(h, w, C, op, seed=0, dyadic=False, out_c=1, wmax=2):
    """entry 1x1 (3 -> C), the op under test, exit 1x1 (-> out_c)"""
    b = tw.Builder(h, w, seed=seed, dyadic=dyadic, wmax=wmax)
    x = b.pw(b.x, C)
    x = op(b, x)
    b.pw(x, out_c)
    return b


# ---------------------------------------------------------------------------------------------------- a. op sweep
# (name, h, w, C, k, stride, dil, pad)
DW_CASES = [
    ("k3s1", 9, 13, 8, 3, 1, 1, "SAME"), ("k3s2", 10, 14, 5, 3, 2, 1, "SAME"), ("k3s2v", 9, 13, 21, 3, 2, 1, "VALID"),
    ("k5s1", 1, 17, 24, 5, 1, 1, "SAME"), ("k5s2", 17, 16, 96, 5, 2, 1, "SAME"), ("k5s2v", 12, 11, 8, 5, 2, 1, "VALID"),
    ("k3d2", 12, 11, 24, 3, 1, 2, "SAME"), ("k3d4", 33, 33, 16, 3, 1, 4, "SAME"), ("k3d4v", 19, 21, 5, 3, 1, 4, "VALID"),
    ("k5d2", 14, 15, 21, 5, 1, 2, "SAME"), ("k3d2c96", 21, 18, 96, 3, 1, 2, "SAME"), ("k3s1w1", 7, 1, 24, 3, 1, 1, "SAME"),
    ("k3d4c8", 23, 17, 8, 3, 1, 4, "SAME"),
]
DW_SWITCHES = [{}, {"dw_px": 0}, {"dw_plane": 0}, {"dw_plane_cs": 8}]


def dw_graph(case, dyadic=False):
    name, h, w, C, k, s, d, pad = case
    return sandwich(h, w, C, lambda b, x: b.dw(x, k, s, d, pad, act="RELU6"), seed=zlib.crc32(name.encode()) % 1000, dyadic=dyadic)


# emulator time, one after another on an 8-core CPU: about 6 s each; the switched variants are marked slow
@pytest.mark.parametrize("sw", [s if not s else pytest.param(s, marks=pytest.mark.slow) for s in DW_SWITCHES], ids=lambda s: ",".join(f"{k}{v}" for k, v in s.items()) or "default")
def test_depthwise_sweep(runner, gen_dir, sw):
    for case in DW_CASES:
        b = dw_graph(case)
        path = write(b, gen_dir, "dw-" + case[0])
        _, kernels = check(runner, b, path, n=2, tuning=sw, trace=True)
        name, h, w, C, k, s, d, pad = case
        plane = d > 1 and pad == "SAME" and sw.get("dw_plane", 1) and C % sw.get("dw_plane_cs", 16) == 0
        assert any(kn.startswith("k_depthwise_plane") for kn in kernels) == bool(plane), (case, sw, kernels)
        generic = not plane and (C % 4 or not sw.get("dw_px", 1))
        if generic:
            assert any(kn.startswith("k_depthwise<") for kn in kernels), (case, sw, kernels)


@pytest.mark.parametrize("case", DW_CASES[:6], ids=lambda c: c[0])
def test_depthwise_dyadic(runner, gen_dir, case):
    b = dw_graph(case, dyadic=True)
    check(runner, b, write(b, gen_dir, "dwx-" + case[0]), n=2, dyadic=True)


# (name, h, w, ic, oc, k, stride, pad)
CONV_CASES = [("ic3s2", 17, 18, 3, 16, 3, 2, "SAME"), ("ic8s1", 9, 13, 8, 12, 3, 1, "SAME"),
              ("ic8s2v", 11, 10, 8, 5, 3, 2, "VALID"), ("ic8k5", 8, 9, 8, 8, 5, 1, "SAME")]


@pytest.mark.parametrize("dyadic", [False, True])
def test_dense_conv(runner, gen_dir, dyadic):
    for name, h, w, ic, oc, k, s, pad in CONV_CASES:
        b = tw.Builder(h, w, seed=3, dyadic=dyadic)
        x = b.pw(b.x, ic) if ic != 3 else b.x
        x = b.conv(x, oc, k, s, pad=pad, act="RELU")
        b.pw(x, 1)
        _, kernels = check(runner, b, write(b, gen_dir, f"conv-{name}-{int(dyadic)}"), n=2, dyadic=dyadic, trace=True)
        assert "k_conv_direct" in kernels, kernels


def test_dense_conv_over_the_weight_limit_is_refused(runner, gen_dir):
    # 3 x 3 x 96 x 32 x 4 bytes = 108 KB > 96 KB
    b = sandwich(8, 8, 96, lambda b, x: b.conv(x, 32, 3))
    refused(runner.lib, write(b, gen_dir, "conv-big"), "dense KxK conv too large")
    b = sandwich(8, 8, 64, lambda b, x: b.conv(x, 40, 3))          # 3 x 3 x 64 x 40 x 4 = 90 KB: runs
    check(runner, b, write(b, gen_dir, "conv-limit"), n=2)


# (name, h, w, oh, ow, mode, dyadic)
RESIZE_CASES = [("hp2x", 6, 7, 12, 14, "half_pixel", True), ("hpup", 5, 7, 13, 16, "half_pixel", False),
                ("hpdown", 13, 16, 5, 7, "half_pixel", False), ("ac", 7, 11, 20, 30, "align_corners", False),
                ("acdown", 20, 30, 7, 11, "align_corners", False), ("asym", 6, 9, 15, 20, "asymmetric", False),
                ("asym2x", 6, 9, 12, 18, "asymmetric", True), ("asymdown", 12, 18, 5, 7, "asymmetric", False)]


@pytest.mark.parametrize("case", RESIZE_CASES, ids=lambda c: c[0])
def test_resize(runner, gen_dir, case):
    name, h, w, oh, ow, mode, dyadic = case
    # C = 5: the resize stays a stand-alone kernel (the folded resize + 1x1 is pinned in test_fusion_upsample_pw)
    b = sandwich(h, w, 5, lambda b, x: b.resize(x, oh, ow, mode), dyadic=dyadic)
    check(runner, b, write(b, gen_dir, "rs-" + name), n=2, dyadic=dyadic)


@pytest.mark.parametrize("K", [8, 16, 24, 40])
def test_tconv(runner, gen_dir, K):
    for N in (8, 16, 24, 40):
        b = tw.Builder(5, 7, seed=K + N, dyadic=True)
        x = b.pw(b.x, K)
        x = b.tconv(x, N)
        b.pw(x, 1)
        _, kernels = check(runner, b, write(b, gen_dir, f"tc-{K}-{N}"), n=2, dyadic=True, trace=True)
        assert "k_tconv2x2" in kernels


@pytest.mark.parametrize("kind", ["HARD_SWISH", "LOGISTIC", "RELU", "RELU6"])
def test_unary(runner, gen_dir, kind):
    # after an ADD (not folded into a producer) and after a 1x1 (folded into its epilogue)
    b = tw.Builder(7, 9, seed=5)
    x = b.pw(b.x, 12)
    y = b.pw(b.x, 12)
    s = b.unary(kind, b.add(x, y))
    t = b.unary(kind, b.pw(s, 8))
    b.pw(t, 1)
    check(runner, b, write(b, gen_dir, "un-" + kind.lower()), n=3, dyadic=False)


def test_eltwise_folded_and_not(runner, gen_dir):
    """MUL / MUL + ADD folded into a 1x1's prologue, and the same ops left as element-wise steps"""
    out = {}
    for folded in (True, False):
        b = tw.Builder(8, 8, seed=7)
        x = b.pw(b.x, 8)
        y = b.pw(b.x, 8)
        s = b.se(x, 4, gate=None)            # per-channel scale vector (pool: 64 pixels, exact)
        m = b.mul(x, s)                       # channel-broadcast MUL
        a = b.add(m, y)                       # ... + ADD
        if folded:
            z = b.pw(a, 4)                     # 1x1 reads MUL+ADD: both folded into its prologue
        else:
            z = b.pw(b.unary("RELU", a), 4)    # a unary in between: MUL and ADD stay element-wise steps
        v = b.mul(z, b.pw(b.x, 4))             # same-shape MUL
        b.add(b.pw(v, 1), b.pw(b.x, 1))        # ADD of two tensors at the end
        out[folded] = check(runner, b, write(b, gen_dir, f"elt-{int(folded)}"), n=2, trace=True)
    # folded: MUL and ADD are read by the 1x1's prologue; unfolded: MUL, ADD and RELU are three element-wise launches
    assert out[True][0] == out[False][0] - 3, out


@pytest.mark.parametrize("split", [(4, 8), (5, 7), (8, 3), (6, 10)])
def test_concat(runner, gen_dir, split):
    a, c = split
    b = tw.Builder(7, 9, seed=11, dyadic=True)
    x = b.pw(b.x, 8)
    t = b.concat([b.pw(x, a), b.pw(x, c), b.pw(x, 4)])
    b.pw(t, 1)
    _, kernels = check(runner, b, write(b, gen_dir, f"cat-{a}-{c}"), n=2, dyadic=True, trace=True)
    # producers write into the concatenation in place when their channel offset and the total depth are multiples of 4
    total = a + c + 4
    aliased = total % 4 == 0 and a % 4 == 0
    assert ("k_copy_channels" in kernels) == (not aliased or (a + c) % 4 != 0), (split, kernels)


# ---------------------------------------------------------------------------------------------------- b. fusion boundaries
def chain_graph(h=8, w=8, C=16, narrow=16, k=3, stride=2, blocks=1, residual=True, pw_first=True, E=32, seed=0,
                family="segm_"):
    """DW (k, stride, from a larger tensor) -> SE -> scaled 1x1 into X { -> 1x1 -> DW -> SE -> scaled 1x1 [+ X] }*
    -> (1x1 of X, SE of X) -> MUL -> resize back -> 1x1 (2 channels)"""
    ih, iw = (2 * h, 2 * w) if stride == 2 else (h + k - 1, w + k - 1)
    b = tw.Builder(ih, iw, seed=seed)
    x = b.pw(b.x, C, act="RELU")
    d = b.dw(x, k, stride, pad="SAME" if stride == 2 else "VALID", act="RELU")
    X = b.pw(b.mul(d, b.se(d, 8)), narrow)
    for _ in range(blocks):
        e = b.pw(X, E, act="RELU6")
        dd = b.dw(e, 3, act="RELU6")
        q = b.pw(b.mul(dd, b.se(dd, 8)), narrow)
        X = b.add(q, X) if residual else q
    if pw_first:
        t0 = b.pw(X, 16)
        t1 = b.unary("LOGISTIC", b.pw(b.pool(X), 16))
    else:
        t1 = b.unary("LOGISTIC", b.pw(b.pool(X), 16))
        t0 = b.pw(X, 16)
    y = b.mul(t0, t1)
    y = b.resize(y, ih, iw, "half_pixel")
    b.pw(y, 2 if family == "segm_" else 1)
    return b


def launches_off(runner, path, switch):
    return runner.run(path, inputs_for(path, 1), EXACT, {switch: 0})[1]


def inputs_for(path, n):
    m = po.Model(path)
    shp = m.shape(m.input)
    m.close()
    return np.random.default_rng(1).uniform(0, 1, (n, *shp[1:])).astype(np.float32)


def fusion_case(runner, b, path, switch, fuses, saved=None, n=3, flags=EXACT, **kw):
    launches, kernels = check(runner, b, path, n=n, flags=flags, **kw)
    off = launches_off(runner, path, switch) if switch else runner.run(path, inputs_for(path, 1), flags | KEEP)[1]
    if fuses:
        assert launches < off and (saved is None or off - launches == saved), (os.path.basename(path), launches, off)
    else:
        assert launches == off, (os.path.basename(path), "fused where it should not", launches, off)
    return launches, kernels


# (name, kwargs, fuses)
CHAIN_CASES = [
    ("8x8", {}, True), ("7x11", dict(h=7, w=11), True), ("12x20", dict(h=12, w=20, blocks=0), True),
    ("p256", dict(h=16, w=16, blocks=0, C=8), True), ("p257", dict(h=1, w=257, blocks=0, C=8), False),
    ("c128", dict(h=4, w=4, C=128, blocks=0), True), ("c132", dict(h=4, w=4, C=132, blocks=0), False),
    ("n32", dict(narrow=32), True), ("n36", dict(narrow=36), False),
    ("k5s1", dict(k=5, stride=1, h=6, w=10), True), ("b0", dict(blocks=0), True),
    ("b3", dict(blocks=3), True), ("b3nores", dict(blocks=3, residual=False), True),
    ("b1nores", dict(residual=False), True), ("sefirst", dict(pw_first=False), True),
    # P % 3 == 0 and P <= 144: the two-CTAs-per-SM configuration
    ("9x9", dict(h=9, w=9), True), ("3x16", dict(h=3, w=16, blocks=3), True), ("12x12", dict(h=12, w=12, blocks=0), True),
]
TWO_PER_SM = ("9x9", "3x16", "12x12", "k5s1")


@pytest.mark.parametrize("case", CHAIN_CASES, ids=lambda c: c[0])
def test_fusion_chain(runner, gen_dir, case):
    name, kw, fuses = case
    b = chain_graph(**kw)
    path = write(b, gen_dir, "chain-" + name, "segm_")
    saved = None
    if fuses:   # DW + SE + PW, 4 per block, PW + SE + MUL in one launch
        saved = 3 + 4 * kw.get("blocks", 1) + 3 - 1
    _, kernels = fusion_case(runner, b, path, "cnn_chain", fuses, saved=saved, n=2, trace=True)
    if isinstance(runner, Gpu) and fuses:      # k_chain<4, 32, ...>: one CTA per SM; k_chain<3, 16, ...>: two
        chain = [k for k in kernels if k.startswith("k_chain<")]
        assert len(chain) == 1 and chain[0].startswith("k_chain<3, 16," if name in TWO_PER_SM else "k_chain<4, 32,"), chain


def head_graph(C=16, tconv=True, N=2, h=7, w=9):
    b = tw.Builder(h, w, seed=C + N)
    x = b.pw(b.x, C)
    t = b.pw(x, C, act="RELU")
    r = b.add(b.dw(t, 3, act="RELU"), t)
    if tconv:
        r = b.tconv(r, N)
        if N > 2:
            b.pw(r, 2)
    else:
        b.pw(r, 2)
    return b


# (C, with a transposed conv, its N; the 1x1 + depthwise fuse; the transposed conv fuses too)
HEAD_CASES = [(16, True, 2, True, True), (24, True, 2, True, True), (24, True, 1, True, True), (16, False, 0, True, False),
              (24, False, 0, True, False), (16, True, 3, True, False), (20, True, 2, False, False),
              (20, False, 0, False, False)]


@pytest.mark.parametrize("case", HEAD_CASES, ids=lambda c: f"C{c[0]}-t{int(c[1])}-N{c[2]}")
def test_fusion_head(runner, gen_dir, case):
    C, tconv, N, fuses, t_fused = case
    b = head_graph(C, tconv, N)
    family = "selfie" if N == 1 else "segm_"
    path = write(b, gen_dir, f"head-{C}-{int(tconv)}-{N}", family)
    saved = (1 + t_fused) if fuses else None
    _, kernels = fusion_case(runner, b, path, "head", fuses, saved=saved, n=2, trace=True)
    if tconv:
        assert ("k_tconv2x2" in kernels) == (not t_fused), kernels


@pytest.mark.parametrize("case", [(16, 15, 17, "SAME", True), (16, 16, 18, "SAME", True), (16, 15, 17, "VALID", True),
                                  (16, 16, 18, "VALID", True), (16, 33, 20, "SAME", True), (20, 15, 17, "SAME", False)],
                         ids=lambda c: f"C{c[0]}-{c[1]}x{c[2]}-{c[3]}")
def test_fusion_pw_dws2(runner, gen_dir, case):
    C, h, w, pad, fuses = case
    for act in ("RELU6", "RELU"):
        b = tw.Builder(h, w, seed=h + w)
        x = b.pw(b.x, C)
        x = b.dw(b.pw(x, C, act=act), 3, 2, pad=pad, act=act)
        b.pw(x, 1)
        fusion_case(runner, b, write(b, gen_dir, f"pwdw-{C}-{h}x{w}-{pad}-{act}"), "pw_dws2", fuses,
                    saved=1 if fuses else None, n=2)


def enc_graph(h, w, act="RELU6", pad="SAME", seed=0):
    b = tw.Builder(h, w, seed=seed)
    X = b.pw(b.x, 16, act="RELU")
    t25 = b.pw(b.mul(X, b.se(X, 8)), 16)
    t36 = b.pw(b.dw(b.pw(t25, 72, act=act), 3, 2, pad=pad, act=act), 24)
    t48 = b.add(b.pw(b.dw(b.pw(t36, 88, act=act), 3, 1, act=act), 24), t36)
    t52 = b.unary("HARD_SWISH", b.pw(t48, 96))
    b.pw(b.add(b.resize(t52, h, w, "half_pixel"), b.pw(t25, 96)), 1)
    return b


@pytest.mark.parametrize("case", [(14, 18, "RELU6", "SAME", True), (13, 19, "RELU", "SAME", True),
                                  (9, 5, "RELU6", "SAME", True), (13, 19, "RELU6", "VALID", False),
                                  (14, 18, "RELU", "VALID", False)], ids=lambda c: f"{c[0]}x{c[1]}-{c[2]}-{c[3]}")
def test_fusion_encoder_blocks(runner, gen_dir, case):
    h, w, act, pad, fuses = case
    b = enc_graph(h, w, act, pad)
    fusion_case(runner, b, write(b, gen_dir, f"enc-{h}x{w}-{act}-{pad}"), None, fuses, saved=6 if fuses else None, n=2)


@pytest.mark.parametrize("N", [24, 28])
def test_fusion_upsample_pw(runner, gen_dir, N):
    for mode in ("half_pixel", "align_corners", "asymmetric"):
        for staged in (1, 0):
            b = tw.Builder(6, 7, seed=N)
            x = b.pw(b.x, 8)
            x = b.pw(b.resize(x, 15, 17, mode), N, act="RELU")
            b.pw(x, 1)
            path = write(b, gen_dir, f"up-{N}-{mode}-{staged}")
            _, kernels = fusion_case(runner, b, path, "up_pw", N <= 24, saved=1 if N <= 24 else None, n=2,
                                     trace=True, tuning={"up_staged": staged})
            assert ("k_resize_bilinear<4>" in kernels) == (N > 24), kernels


def pool_launches(wbytes, merge):
    """launch_pool_fc: one k_rowsum_fc when pool_merge is on and the folded FC weights fit in 48 KB, else k_rowsum and
    k_pool_fc"""
    return 1 if merge and wbytes <= 48 * 1024 else 2


# (name, C, mid, FC kind, h, w, largest folded FC in bytes (K x N rounded up to 4 x 4 B), both FCs folded)
POOL_SE_CASES = [("c512", 512, 16, "conv", 4, 4, 512 * 16 * 4, True), ("n6", 24, 6, "conv", 4, 4, 24 * 8 * 4, True),
                 ("fc", 24, 6, "fc", 4, 4, 24 * 8 * 4, True), ("w48k", 384, 32, "conv", 4, 4, 384 * 32 * 4, True),
                 ("w52k", 416, 32, "conv", 4, 4, 416 * 32 * 4, True), ("w192k", 512, 96, "conv", 2, 2, 512 * 96 * 4, True),
                 ("w200k", 512, 100, "conv", 2, 2, 16, False)]


@pytest.mark.parametrize("case", POOL_SE_CASES, ids=lambda c: c[0])
@pytest.mark.parametrize("merge", [1, 0])
def test_fusion_pool_se(runner, gen_dir, case, merge):
    """global pool + squeeze-excite FCs in one step: 512 channels, FC N not a multiple of 4, FULLY_CONNECTED and 1x1
    FCs, the 48 KB limit of the one-launch kernel, the 192 KB limit of the fold (512 x 96 x 4 B folds; 512 x 100 x 4 B,
    the first FC of w200k, does not, so neither FC is folded), pool_merge 0 / 1"""
    name, C, mid, fc, h, w, wbytes, folded = case
    b = tw.Builder(h, w, seed=C)
    x = b.pw(b.x, C, act="RELU")
    b.pw(b.mul(x, b.se(x, mid, fc=fc)), 1)
    launches, kernels = check(runner, b, write(b, gen_dir, f"se-{name}-{merge}"), n=2, tuning={"pool_merge": merge},
                              trace=True)
    # entry 1x1, the pool (+ FCs + gate), the exit 1x1 with the channel-scale MUL in its prologue; when the FCs are not
    # folded they are two 1x1 steps of their own (the gate folded into the second)
    p = pool_launches(wbytes, merge)
    assert launches == 2 + p + (0 if folded else 2), (name, merge, launches)
    assert ("k_rowsum_fc" in kernels) == (p == 1), kernels
    assert ("k_rowsum" in kernels and "k_pool_fc" in kernels) == (p == 2), kernels


def test_pool_over_concat(runner, gen_dir):
    b = tw.Builder(8, 8, seed=2, dyadic=True)
    x = b.pw(b.x, 8)
    c = b.concat([b.pw(x, 8), b.pw(x, 12)])
    s = b.pw(b.pool(c), 8, act="RELU")
    b.pw(b.mul(x, s), 1)
    for merge in (1, 0):
        launches, kernels = check(runner, b, write(b, gen_dir, f"catpool-{merge}"), n=2, dyadic=True,
                                  tuning={"pool_merge": merge}, trace=True)
        assert "k_copy_channels" not in kernels, kernels      # the concatenation is never materialised


def test_pool_over_512_channels_is_refused(runner, gen_dir):
    b = tw.Builder(4, 4, seed=1)
    x = b.pw(b.x, 516)
    b.pw(b.mul(x, b.se(x, 8)), 1)
    refused(runner.lib, write(b, gen_dir, "se-c516"), "global pool over more than 512 channels")


def mb_graph(h=8, w=8, C=16, E=64, residual=True):
    b = tw.Builder(h, w, seed=E)
    X = b.pw(b.x, C)
    dd = b.dw(b.pw(X, E, act="RELU6"), 3, act="RELU6")
    q = b.pw(b.mul(dd, b.se(dd, 16)), C)
    b.pw(b.add(q, X) if residual else q, 1)
    return b


@pytest.mark.parametrize("case", [(8, 8, 16, 64, True, True), (7, 9, 16, 64, False, True), (16, 16, 32, 128, True, True),
                                  (16, 17, 16, 64, True, False), (8, 8, 16, 132, True, False)],
                         ids=lambda c: f"{c[0]}x{c[1]}-{c[2]}-{c[3]}-{int(c[4])}")
def test_fusion_mb_block(runner, gen_dir, case):
    h, w, C, E, residual, fuses = case
    b = mb_graph(h, w, C, E, residual)
    path = write(b, gen_dir, f"mb-{h}x{w}-{C}-{E}-{int(residual)}")
    launches, kernels = check(runner, b, path, n=2, flags=EXACT | FUSE_BLOCKS, trace=True)
    off = runner.run(path, inputs_for(path, 1), EXACT)[1]
    assert ("k_mb_block" in kernels) == fuses, kernels
    assert (launches < off) == fuses, (launches, off)


def stem_graph(h, w):
    """3x3 stride-2 16-channel stem (the conv the pipeline runs on the camera bytes), a 1x1, a resize back to the input
    grid and a 1-channel head"""
    b = tw.Builder(h, w, seed=h * w)
    x = b.conv(b.x, 16, 3, 2, act="RELU6")
    x = b.pw(x, 8, act="RELU")
    b.unary("LOGISTIC", b.pw(b.resize(x, h, w, "half_pixel"), 1))
    return b


# (model h, w): stem output widths 16 (even: the two-pixel kernel), 15 (odd: the one-pixel kernel), 16 from an odd 31
@pytest.mark.parametrize("hw", [(24, 32), (24, 30), (23, 31)], ids=lambda c: f"{c[0]}x{c[1]}")
@pytest.mark.parametrize("stem_x2", [1, 0])
def test_stem_through_the_pipeline(runner, gen_dir, hw, stem_x2):
    """the fused u8 stem (k_stem_u8_x2 / k_stem_u8) runs only from camera frames: composite against the oracle's
    pipeline, mask, composite and YUYV bit for bit, every frame; on the H100 the profiler names the stem kernel"""
    from tests import synth
    h, w = hw
    b = stem_graph(h, w)
    path = write(b, gen_dir, f"stem-{h}x{w}")
    W, H, n = 2 * w + 6, 2 * h, 3
    frames = np.stack([synth.frame(W, H, t=t) for t in range(n)])
    bg = synth.background()
    lib = runner.lib

    def run():
        g = api.MaskGen(lib, path, W, H, max_batch=n, flags=EXACT | NO_GRAPH)
        try:
            g.set_background(bg)
            return g.composite(frames)
        finally:
            g.close()
    try:
        assert lib.bsb_set_tuning(b"stem_x2", stem_x2)
        if isinstance(runner, Gpu):
            (out, yuyv, mask), kernels = gpu_kernels(run)
            stems = {k.split("<")[0] for k in kernels if k.startswith("k_stem_u8")}
            assert stems == {"k_stem_u8_x2" if stem_x2 and tw.conv_out(w, 3, 2, 1, "SAME") % 2 == 0 else "k_stem_u8"}, kernels
        else:
            out, yuyv, mask = run()
    finally:
        lib.bsb_set_tuning(b"stem_x2", TUNING_DEFAULTS["stem_x2"])
    ref = po.MaskGen(path, W, H)
    for i in range(n):
        ro, ry, rm = ref.composite(frames[i], bg)
        assert np.array_equal(mask[i], rm), f"frame {i}: mask differs from the oracle"
        assert np.array_equal(out[i], ro), f"frame {i}: composite differs from the oracle"
        assert np.array_equal(yuyv[i], ry), f"frame {i}: YUYV differs from the oracle"
    ref.close()


# ---------------------------------------------------------------------------------------------------- c. BodyPix-shaped
def mobilenet_v1(mult, stride, h=33, w=25, seed=0):
    """MobileNetV1 (BodyPix): 3x3 s2 stem, 13 depthwise-separable blocks; past the output stride the strides become
    dilations (atrous), then a 1x1 segmentation head and a sigmoid"""
    ch = lambda c: max(8, int(c * mult + 4) // 8 * 8)
    b = tw.Builder(h, w, seed=seed)
    x = b.conv(b.x, ch(32), 3, 2, act="RELU6")
    plan = [(64, 1), (128, 2), (128, 1), (256, 2), (256, 1), (512, 2)] + [(512, 1)] * 5 + [(1024, 2), (1024, 1)]
    cur, rate = 2, 1
    for c, s in plan:
        if s == 2 and cur >= stride:
            s, dil, rate = 1, rate, rate * 2
        else:
            dil = rate if cur >= stride else 1
            cur *= s
        x = b.dw(x, 3, s, dil, act="RELU6")
        x = b.pw(x, ch(c), act="RELU6")
    b.unary("LOGISTIC", b.pw(x, 1))
    return b


MOBILENETS = [(0.5, 8), (0.5, 16), (0.75, 8), (0.75, 16), (1.0, 8), (1.0, 16)]


@pytest.mark.parametrize("mult,stride", MOBILENETS)
def test_bodypix_mobilenet(runner, gen_dir, mult, stride):
    """(a 9x9 input on the emulator, whose time grows with the 512- and 1024-channel layers; 33x25 on the H100)"""
    b = mobilenet_v1(mult, stride, h=9, w=9)
    check(runner, b, write(b, gen_dir, f"mnv1-{mult}-{stride}", "body-pix"), n=2)


# ---------------------------------------------------------------------------------------------------- d. refusals
def refused(lib, path, what):
    n0 = lib.bsb_total_launches()
    with pytest.raises(api.BackscrubError) as e:
        api.MaskGen(lib, path, 64, 64)
    msg = str(e.value)
    assert "unsupported model construct" in msg or "unsupported TFLite operator code" in msg or "malformed model" in msg, msg
    assert what in msg, msg
    assert lib.bsb_total_launches() == n0


def _refusal_graphs():
    out = {}
    b = tw.Builder(8, 8); x = b.pw(b.x, 8); b.pw(b.dw(x, 3, mult=2), 1); out["mult2"] = (b, "depthwise multiplier")
    b = tw.Builder(8, 8); x = b.pw(b.x, 8); b.pw(b.add(x, b.pool(x)), 1); out["addbcast"] = (b, "ADD with broadcasting")
    b = tw.Builder(8, 8); x = b.pw(b.x, 8); b.pw(b.pool(x, fh=2, fw=2, stride=2), 1); out["localpool"] = (b, "not global")
    b = tw.Builder(7, 9); x = b.pw(b.x, 8); b.pw(b.tconv(x, 8, out_hw=(13, 17)), 1); out["tconvodd"] = (b, "Convolution2DTransposeBias")
    b = tw.Builder(8, 8); x = b.pw(b.x, 8); b.pw(b.mul(x, b.const(np.ones(8, np.float32), shape=[8])), 1)
    out["mulconst"] = (b, "MUL broadcast")
    b = tw.Builder(8, 8); x = b.pw(b.x, 8); b.pw(b.concat([x, x], axis=1), 1); out["concath"] = (b, "CONCATENATION")
    b = tw.Builder(8, 8); x = b.pw(b.x, 8); b.pw(b.custom("MaxPoolingWithArgmax2D", x), 1); out["custom"] = (b, "unknown custom op")
    return out


@pytest.mark.parametrize("name", ["mult2", "addbcast", "localpool", "tconvodd", "mulconst", "concath", "custom"])
def test_refusals(runner, gen_dir, name):
    b, what = _refusal_graphs()[name]
    refused(runner.lib, write(b, gen_dir, "ref-" + name), what)


# Messages a well-formed but different model may be refused with (a flipped byte can make another op code, shape or
# option); a truncated file must load or be refused as malformed.
REFUSALS = ("malformed model", "model file too short", "unsupported model construct", "unsupported TFLite operator code",
            "model output channel count does not match", "input/output tensor is not", "model input must have 3 channels",
            "degenerate ROI", "ROI outside the frame", "batch dimension must be 1", "graph output is never produced",
            "planner: step reads a tensor that was folded away")

_FUZZ = """
import json, sys
import numpy as np
from backscrub_b200 import api
from tests.emu.emu_lib import emu
lib = emu()
spec = json.load(open(sys.argv[1]))
ran = refused = 0
for p, allowed in spec:
    try:
        g = api.MaskGen(lib, p, 64, 64)
    except api.BackscrubError as e:
        assert any(m in str(e) for m in allowed), (p, str(e))
        refused += 1
        continue
    # a model that loads must also run: one frame through every planned kernel
    x = np.random.default_rng(0).uniform(0, 1, (1, *g.in_hwc)).astype(np.float32)
    g.infer(x)
    g.close()
    ran += 1
print("fuzz", ran, refused)
"""


@pytest.mark.slow
def test_truncated_and_corrupted_models(gen_dir):
    """(about 30 s on the emulator, the slowest case here) every truncation of a small generated model and 300 seeded single-byte corruptions either load and run one
    frame, or are refused with one of the planner's messages (a truncation: only as malformed); none crashes the process
    (run in a subprocess, so a crash fails this test instead of the session)"""
    b = tw.Builder(2, 2, seed=9)
    x = b.pw(b.x, 4)
    b.pw(b.add(b.dw(x, 3), x), 1)
    data = b.bytes()
    d = os.path.join(gen_dir, "fuzz")
    os.makedirs(d, exist_ok=True)
    spec = []
    for n in range(len(data)):
        p = os.path.join(d, f"selfie-trunc{n}.tflite")
        open(p, "wb").write(data[:n])
        spec.append((p, ["malformed model", "model file too short"]))
    rng = np.random.default_rng(5)
    for i in range(300):
        buf = bytearray(data)
        buf[int(rng.integers(0, len(buf)))] = int(rng.integers(0, 256))
        p = os.path.join(d, f"selfie-flip{i}.tflite")
        open(p, "wb").write(bytes(buf))
        spec.append((p, list(REFUSALS)))
    with open(os.path.join(d, "spec.json"), "w") as f:
        json.dump(spec, f)
    r = subprocess.run([sys.executable, "-c", _FUZZ, os.path.join(d, "spec.json")], cwd=ROOT, capture_output=True, text=True,
                       env=dict(os.environ, PYTHONPATH=ROOT), timeout=900)
    assert r.returncode == 0 and "fuzz" in r.stdout, r.stderr[-3000:]
    ran, n_refused = map(int, r.stdout.split("fuzz", 1)[1].split()[:2])
    assert ran > 0 and n_refused >= len(data) - 16, (ran, n_refused)


# ---------------------------------------------------------------------------------------------------- GPU
# (name, h, w, C, k, stride, dil): at 2 x SMs + 3 frames each has more than SMs x 1024 (pixel row-quad, channel quad)
# threads, so launch_depthwise takes the strip kernel (dw_plane off for the atrous ones)
STRIP_CASES = [("k3s1", 12, 16, 48, 3, 1, 1), ("k3s2", 24, 32, 48, 3, 2, 1), ("k5s1", 12, 16, 48, 5, 1, 1),
               ("k5s2", 24, 32, 48, 5, 2, 1), ("k3d2", 12, 16, 48, 3, 1, 2), ("k3d4", 12, 16, 48, 3, 1, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", STRIP_CASES, ids=lambda c: c[0])
def test_gpu_depthwise_strips(gpu_runner, gen_dir, case):
    name, h, w, C, k, s, d = case
    n = 2 * gpu_runner.sms + 3
    oh, ow = tw.conv_out(h, k, s, d, "SAME"), tw.conv_out(w, k, s, d, "SAME")
    assert n * oh * ((ow + 3) // 4) * (C // 4) >= gpu_runner.sms * 1024
    b = sandwich(h, w, C, lambda b, x: b.dw(x, k, s, d, "SAME", act="RELU6"), seed=zlib.crc32(name.encode()) % 1000)
    _, kernels = check(gpu_runner, b, write(b, gen_dir, "dws-" + name), n=n, frames=(0, n // 2, n - 1),
                       tuning={"dw_plane": 0}, trace=True)
    assert f"k_depthwise_strip<{k}, {s}, {d}" in " ".join(kernels), kernels


@pytest.mark.gpu
def test_gpu_fusions_partial_waves(gpu_runner, gen_dir):
    """the fusing cases at 2 x SMs + 3 frames per call: chains, heads, encoder blocks and pw_dws2 run a partial last
    wave; the chain geometries that fit two CTAs per SM among them"""
    n = 2 * gpu_runner.sms + 3
    fr = (0, 1, n // 2, n - 1)
    for name, kw, fuses in CHAIN_CASES:
        b = chain_graph(**kw)
        fusion_case(gpu_runner, b, write(b, gen_dir, "chain-" + name, "segm_"), "cnn_chain", fuses, n=n, frames=fr)
    for C, tconv, N in ((16, True, 2), (24, False, 0), (20, True, 2)):
        b = head_graph(C, tconv, N)
        fusion_case(gpu_runner, b, write(b, gen_dir, f"head-{C}-{int(tconv)}-{N}", "segm_"), "head", C != 20, n=n, frames=fr)
    for h, w, pad in ((15, 17, "SAME"), (16, 18, "VALID")):
        b = tw.Builder(h, w, seed=h + w)
        b.pw(b.dw(b.pw(b.pw(b.x, 16), 16, act="RELU6"), 3, 2, pad=pad, act="RELU6"), 1)
        fusion_case(gpu_runner, b, write(b, gen_dir, f"pwdw-{h}x{w}-{pad}"), "pw_dws2", True, n=n, frames=fr)
    for h, w, act, pad, fuses in ((14, 18, "RELU6", "SAME", True), (13, 19, "RELU", "SAME", True), (13, 19, "RELU6", "VALID", False)):
        b = enc_graph(h, w, act, pad)
        fusion_case(gpu_runner, b, write(b, gen_dir, f"enc-{h}x{w}-{act}-{pad}"), None, fuses, n=n, frames=fr)
    for N in (24, 28):
        b = tw.Builder(6, 7, seed=N)
        b.pw(b.pw(b.resize(b.pw(b.x, 8), 15, 17, "half_pixel"), N, act="RELU"), 1)
        fusion_case(gpu_runner, b, write(b, gen_dir, f"up-{N}"), "up_pw", N <= 24, n=n, frames=fr)
    for mult, stride in MOBILENETS:
        b = mobilenet_v1(mult, stride)
        check(gpu_runner, b, write(b, gen_dir, f"mnv1-{mult}-{stride}", "body-pix"), n=8)


def tc_graph(h, w, K, N, seed=0):
    b = tw.Builder(h, w, seed=seed)
    x = b.pw(b.x, K, act="RELU")
    y = b.pw(x, N, act="RELU6")
    b.pw(y, 1)
    return b, x, y


# (name, h, w, K, N, tensor cores expected on the middle 1x1)
TC_CASES = [("k16n8", 32, 32, 16, 8, True), ("k12", 32, 32, 12, 8, False), ("k18", 32, 32, 18, 8, False),
            ("n7", 32, 32, 16, 7, False), ("px1023", 31, 33, 16, 8, False), ("px1024", 16, 64, 16, 8, True),
            ("k20n40", 33, 33, 20, 40, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", TC_CASES, ids=lambda c: c[0])
def test_gpu_tensor_core_eligibility(gpu_runner, gen_dir, case):
    """engine.cu's tensor-core test (K >= tc_min_k, K % 4, N >= 8, h w >= 1024, ld % 4) on both sides of each boundary,
    under BSB_FLAG_TENSOR_CORES and in a body-pix graph (tensor cores by default); each tensor-core layer against float64
    with tests/tc_reference's bound, in place on its own inputs (KEEP_TENSORS)"""
    from tests import tc_reference as tr
    name, h, w, K, N, want = case
    lib = gpu_runner.lib
    for family, flags in (("selfie", TENSOR_CORES), ("body-pix", 0)):
        b, tin, tout = tc_graph(h, w, K, N)
        path = write(b, gen_dir, f"tce-{name}", family)
        x = inputs(b, 2, 3)
        # the planner's choice, in the context that runs it (KEEP_TENSORS turns the default tensor cores off)
        g = api.MaskGen(lib, path, 4 * w, 4 * h, max_batch=2, flags=flags)
        assert bool([s for s in g.tc_steps() if s["out"] == tout]) == want, (name, family, g.tc_steps())
        g.close()
        y, _, _ = gpu_runner.run(path, x, flags)
        f64 = torch_graph.run(path, x[0])
        assert np.abs(y[0] - f64).max() <= 1e-4 * max(1.0, np.abs(f64).max()), (name, family)
    # each tensor-core layer in place, on its own inputs
    g = api.MaskGen(lib, path, 4 * w, 4 * h, max_batch=2, flags=TENSOR_CORES | KEEP)
    g.infer(x)
    steps = g.tc_steps()
    assert bool([s for s in steps if s["out"] == tout]) == want, (name, steps)
    for s in steps:
        op = next(o for o in b.ops if o["outputs"][0] == s["out"])
        wt = b.tensors[op["inputs"][1]]["data"].reshape(s["N"], s["K"])
        bias = b.tensors[op["inputs"][2]]["data"]
        for f in range(2):
            A = g.tensor(s["in"], h * w * s["K"], f).reshape(-1, s["K"])
            got = g.tensor(s["out"], h * w * s["N"], f).reshape(-1, s["N"])
            ref = tr.r1(A, wt, bias, None, s["act1"], s["act2"], s["act3"])
            assert (np.abs(got - ref) <= tr.bound(A, wt, bias)).all(), (name, s)
    g.close()

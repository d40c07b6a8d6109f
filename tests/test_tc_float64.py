"""The tensor-core (3xTF32 wgmma) 1x1 convolution against float64, the way the engine calls it.

The kernel cannot be bit-identical to the fp32 oracle, so it is pinned two ways (tests/tc_reference.py has the
definitions and the derivation of the bound):
  * exact dyadic fixtures, on which its result does not depend on the order or the rounding of its adds: the device must
    return R2 (the split products summed exactly) bit for bit;
  * wide-range fixtures, mixed and same signs, within the derived bound of R1 (the exact operation).
Every call goes through bsb_pointwise_ex: A and out are sub-matrices of larger buffers (NaN in the pitch gap and in the
rows after M, sentinels around the output), with residual, act1 / act2 / act3, all tile widths, ragged N and M, K that
is not a multiple of the 32-wide chunk, and enough tiles that each persistent CTA walks its tile loop three times or more.
The same grid runs through the exact FFMA kernels against the oracle bit for bit, on the emulator and on the GPU.

The CPU tests first show that the fixtures and the bound can do their job: the fixtures are exact, every summation order
gives R2 on them, each plausible fault of the kernel changes the result on one of them, and fp32 emulations of the kernel
stay within the bound."""
import numpy as np
import pytest

from backscrub_b200 import BackscrubError, api
from oracle import pyoracle as po
from tests import tc_reference as tr

NONE, RELU, N1_TO_1, RELU6 = tr.ACT_NONE, tr.ACT_RELU, tr.ACT_RELU_N1_TO_1, tr.ACT_RELU6
SENTINEL = np.uint32(0x7fcafe00)         # a NaN with a payload: a stray write (of anything) changes its bits


# ---- the CPU side: fixtures, order independence, fault detection, the bound --------------------------------------
DYADIC_SMALL = [("a_lo", 96, 40, 24, 1), ("w_lo", 80, 36, 20, 2), ("both", 64, 8, 16, 3), ("both", 48, 4, 8, 4)]


@pytest.mark.parametrize("kind,M,K,N,seed", DYADIC_SMALL + [("a_lo", 130, 960, 21, 5), ("w_lo", 129, 1024, 33, 6)])
def test_dyadic_fixture_is_exact(kind, M, K, N, seed):
    A, W, b, res = tr.dyadic(kind, M, K, N, seed, residual=True)        # the generator asserts representability
    r2 = tr.r2(A, W, b, res)
    assert np.array_equal(r2.astype(np.float32).astype(np.float64), r2)
    if kind == "both":          # the dropped a_lo * w_lo term is visible: R2 is not the rounded exact result
        assert (tr.r1(A, W, b, res).astype(np.float32) != r2.astype(np.float32)).any()


@pytest.mark.parametrize("kind,M,K,N,seed", DYADIC_SMALL)
@pytest.mark.parametrize("acts", [(RELU6, NONE, NONE), (NONE, RELU, RELU), (N1_TO_1, NONE, NONE)])
def test_dyadic_result_is_independent_of_summation_order(kind, M, K, N, seed, acts):
    A, W, b, res = tr.dyadic(kind, M, K, N, seed, residual=True)
    r2 = tr.r2(A, W, b, res, *acts)
    for order in tr.ORDERS:
        got = tr.emulate(A, W, b, res, *acts, order=order)
        assert np.array_equal(got.astype(np.float64), r2), order


def test_each_fault_changes_a_dyadic_result():
    """Dropping any one of the three split terms, a tensor core that rounds A to tf32 instead of truncating it, a_lo
    taken from the neighbouring row, the residual added before the activation, a missing bias: each moves at least one
    element of one fixture away from R2."""
    caught = {}
    for kind, M, K, N, seed in DYADIC_SMALL:
        for acts in [(RELU6, NONE, NONE), (NONE, NONE, RELU)]:
            A, W, b, res = tr.dyadic(kind, M, K, N, seed, residual=True)
            r2 = tr.r2(A, W, b, res, *acts).astype(np.float32)
            for name, got in tr.mutants(A, W, b, res, *acts).items():
                caught[name] = caught.get(name, False) or bool((got != r2).any())
    assert len(caught) == 7 and all(caught.values()), caught


WIDE_SMALL = [("mixed", 64, 20, 16, 11), ("same", 64, 20, 16, 12), ("mixed", 48, 96, 24, 13), ("same", 48, 96, 24, 14),
              ("same", 16, 480, 8, 15), ("mixed", 16, 480, 8, 16)]


@pytest.mark.parametrize("kind,M,K,N,seed", WIDE_SMALL)
def test_bound_covers_fp32_emulations(kind, M, K, N, seed):
    A, W, b, res = tr.wide(kind, M, K, N, seed, residual=True)
    ref, bnd = tr.r1(A, W, b, res), tr.bound(A, W, b, res)
    for order in tr.ORDERS:
        err = np.abs(tr.emulate(A, W, b, res, order=order) - ref)
        assert (err <= bnd).all(), (order, (err / bnd).max())


@pytest.mark.parametrize("K", [20, 96])
def test_bound_catches_a_dropped_term(K):
    """Not vacuous: on same-sign data (post-ReLU activations times positive weights) at these depths, a kernel that
    drops the a_lo * w_hi or the a_hi * w_lo term leaves the bound."""
    A, W, b, _ = tr.wide("same", 64, K, 32, K)
    ref, bnd = tr.r1(A, W, b), tr.bound(A, W, b)
    for drop in (1, 2):
        got = tr.epilogue(tr.split_matmul(A, W, drop=drop), b.astype(np.float64), None, 0, 0, 0).astype(np.float32)
        assert (np.abs(got - ref) > bnd).any(), drop


# ---- the grid ----------------------------------------------------------------------------------------------------
# name: M, K, N, act1, act2, residual, act3, bias, A pitch pad, out pitch pad, residual pitch pad, out offset, res offset
GRID = {
    "n16_k20_m100_oddout": (100, 20, 16, RELU6, NONE, False, NONE, True, 4, 3, 0, 1, 0),
    "n32_k36_m129_res": (129, 36, 32, NONE, NONE, True, NONE, True, 8, 2, 2, 4, 2),
    "n21_k256_res_relu": (1089, 256, 21, RELU6, NONE, True, RELU, True, 4, 0, 0, 4, 4),
    "n33_k52_relu": (777, 52, 33, RELU, NONE, False, NONE, True, 0, 1, 0, 4, 0),
    "n64_k96_m129": (129, 96, 64, N1_TO_1, NONE, True, NONE, True, 4, 4, 1, 4, 1),
    "n65_k68_act2": (385, 68, 65, NONE, RELU6, False, NONE, False, 4, 0, 0, 4, 0),
    "n96_k40_nobias": (300, 40, 96, RELU, NONE, True, NONE, False, 4, 2, 3, 6, 3),
    "n97_k128": (200, 128, 97, RELU6, NONE, False, NONE, True, 12, 0, 0, 4, 0),
    "n160_k960": (1025, 960, 160, RELU6, NONE, False, NONE, True, 4, 8, 0, 4, 0),
    "n240_k100_act2": (513, 100, 240, NONE, N1_TO_1, True, RELU, True, 4, 0, 0, 4, 2),
    "n480_k32": (257, 32, 480, RELU6, NONE, True, NONE, True, 0, 0, 0, 4, 2),
    "n7_k4_m1": (1, 4, 7, NONE, NONE, False, NONE, True, 4, 1, 0, 4, 0),
    "n128_k160": (1000, 160, 128, RELU6, NONE, False, NONE, True, 4, 0, 0, 4, 0),
    # enough tiles for >= 3 trips of each persistent CTA round the tile loop on a 132-SM H100, with a chunk count the
    # stage count does not divide (the full / empty parities and the stage index carry across tiles)
    "n16_k36_many": (50689, 36, 16, RELU6, NONE, True, NONE, True, 4, 0, 0, 4, 0),
    "n64_k96_many": (50689, 96, 64, RELU, NONE, True, RELU, True, 4, 2, 0, 4, 2),
    "n256_k64_many": (25601, 64, 256, RELU6, NONE, True, NONE, False, 0, 0, 0, 4, 2),
    "n80_k160_many": (40000, 160, 160, NONE, NONE, False, NONE, True, 4, 0, 0, 4, 0),
}
SMALL = [k for k, v in GRID.items() if v[0] <= 1100]


class Layout:
    """The operands as sub-matrices of larger buffers, as the engine passes them (concatenation slices, pitches above
    the width).  NaN fills A's pitch gap, the rows after M and the residual's gaps; SENTINEL fills the output buffer."""

    def __init__(self, case, A, res):
        M, K, N, *_ = case
        a_pad, out_pad, res_pad, out_off, res_off = case[8:]
        self.M, self.N = M, N
        self.ld_a, self.a_off = K + a_pad, 4
        self.a = np.full(self.a_off + (M + 3) * self.ld_a, np.nan, np.float32)
        self.a[self.a_off:self.a_off + M * self.ld_a].reshape(M, self.ld_a)[:, :K] = A
        self.ld_out, self.out_off = N + out_pad, out_off
        self.res = None
        if res is not None:
            self.ld_res, self.res_off = N + res_pad, res_off
            self.res = np.full(res_off + M * self.ld_res + 3, np.nan, np.float32)
            self.res[res_off:res_off + M * self.ld_res].reshape(M, self.ld_res)[:, :N] = res

    def run(self, lib, W, b, acts, variant, out_off=None):
        out_off = self.out_off if out_off is None else out_off
        out = np.full(out_off + self.M * self.ld_out + 5, SENTINEL, np.uint32).view(np.float32)
        kw = dict(residual=self.res, res_off=self.res_off, ld_res=self.ld_res) if self.res is not None else {}
        api.pointwise(lib, self.a, W, b, act=acts[0], act2=acts[1], act3=acts[2], variant=variant, rows=self.M,
                      a_off=self.a_off, ld_a=self.ld_a, out=out, out_off=out_off, ld_out=self.ld_out, **kw)
        bits = out.view(np.uint32).copy()
        got = out[out_off:out_off + self.M * self.ld_out].reshape(self.M, self.ld_out)[:, :self.N].copy()
        bits[out_off:out_off + self.M * self.ld_out].reshape(self.M, self.ld_out)[:, :self.N] = SENTINEL
        assert (bits == SENTINEL).all(), f"{(bits != SENTINEL).sum()} elements outside the output written"
        assert not np.isnan(got).any(), "NaN in the output: a read past K, past M or outside the residual"
        return got


def fixtures(case, seed):
    M, K, N, _, _, residual, _, bias = case[:8]
    out = [("wide-mixed", tr.wide("mixed", M, K, N, seed, bias, residual)),
           ("wide-same", tr.wide("same", M, K, N, seed + 1, bias, residual))]
    if K <= 1024:
        out.append(("dyadic-a_lo", tr.dyadic("a_lo", M, K, N, seed + 2, bias, residual)))
        out.append(("dyadic-w_lo", tr.dyadic("w_lo", M, K, N, seed + 3, bias, residual)))
    if K <= 64:
        out.append(("dyadic-both", tr.dyadic("both", M, K, N, seed + 4, bias, residual)))
    return out


def oracle_exact(A, W, b, res, acts):
    """the oracle's conv2d (k-ascending fmaf, act1) followed by act2 and the fp32 residual add and act3"""
    M, K = A.shape
    N = W.shape[0]
    v = po.conv2d(A.reshape(1, M, K), W.reshape(N, 1, 1, K), b, padding=po.PAD_VALID, act=acts[0]).reshape(M, N)
    v = tr.act(v, acts[1])
    return tr.act((v + res).astype(np.float32), acts[2]) if res is not None else v


def check_exact_variants(lib, name, variants):
    """The exact FFMA kernels on one grid case, through the same strided buffers: the case's first (wide-range, mixed
    sign) fixture only, since bit-exactness against the oracle does not depend on the data."""
    case = GRID[name]
    acts = (case[3], case[4], case[6])
    for fx, (A, W, b, res) in fixtures(case, 100 + sum(map(ord, name)))[:1]:
        lay = Layout(case, A, res)
        ref = oracle_exact(A, W, b, res, acts)
        for v in variants:
            got = lay.run(lib, W, b, acts, v, out_off=4)         # the FFMA kernels store float4 rows: 16-byte aligned out
            assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (name, fx, v)


def check_refusals(lib, tc_present):
    """Operands the tensor-core kernel cannot take are refused on the host, with the reason; nothing is launched."""
    rng = np.random.default_rng(0)
    M, K, N = 64, 32, 16
    A = rng.standard_normal((M, K)).astype(np.float32)
    W = rng.standard_normal((N, K)).astype(np.float32)
    a = np.zeros(8 + M * 36, np.float32)
    res = np.zeros(8 + M * N, np.float32)
    out = np.zeros(8 + M * 17, np.float32)
    refused = [  # (what, kwargs)
        ("16-byte", dict(rows=M, a_off=2, ld_a=K, out=out, ld_out=N, out_off=0)),                 # A 8-byte aligned
        ("multiples of 4", dict(rows=M, a_off=0, ld_a=K + 2, out=out, ld_out=N, out_off=0)),      # pitch of A
        ("8-byte", dict(rows=M, a_off=0, ld_a=K, out=out, ld_out=N, out_off=1)),                  # float2 stores
        ("8-byte", dict(rows=M, a_off=0, ld_a=K, out=out, ld_out=N, out_off=0, residual=res, res_off=1, ld_res=N)),
    ]
    for what, kw in refused:
        with pytest.raises(BackscrubError, match=what):
            api.pointwise(lib, a, W, None, variant=1, **kw)
    with pytest.raises(BackscrubError, match="multiples of 4"):
        api.pointwise(lib, A[:, :30], W[:, :30], None, variant=1)
    # the exact kernels need A and out on 16-byte boundaries (as the engine's arena gives them)
    with pytest.raises(BackscrubError, match="16-byte"):
        api.pointwise(lib, a, W, None, variant=0, rows=M, a_off=0, ld_a=K, out=out, ld_out=N, out_off=2)
    with pytest.raises(BackscrubError, match="outside its buffer"):
        api.pointwise(lib, a, W, None, variant=0, rows=M + 8, a_off=0, ld_a=36, out=out, ld_out=N, out_off=0)
    # odd ld_out: the scalar store path, which takes any alignment
    if tc_present:
        a[:M * K] = A.reshape(-1)
        got = api.pointwise(lib, a, W, None, variant=1, rows=M, a_off=0, ld_a=K, out=out, ld_out=17, out_off=1)
        got = got[1:1 + M * 17].reshape(M, 17)[:, :N]
        assert (np.abs(got - A.astype(np.float64) @ W.T.astype(np.float64)) <= tr.bound(A, W)).all()


# ---- on the emulator (no GPU): the entry, its checks and the exact kernels -------------------------------------
@pytest.fixture(scope="module")
def emu_lib():
    from tests.emu.emu_lib import emu
    return emu()


@pytest.mark.parametrize("name", SMALL)
def test_pointwise_ex_exact_variants_on_the_emulator(emu_lib, name):
    check_exact_variants(emu_lib, name, (0, 3, 5, 16))


def test_pointwise_ex_refusals_on_the_emulator(emu_lib):
    check_refusals(emu_lib, tc_present=False)


def test_pointwise_keywords_are_checked(emu_lib):
    """api.pointwise takes either a plain [M, K] array or a flat buffer described by rows / a_off / ld_a, not a mix"""
    A = np.ones((8, 4), np.float32); W = np.ones((4, 4), np.float32)
    for kw in [dict(ld_a=4), dict(a_off=4), dict(rows=8), dict(ld_out=4), dict(out_off=4), dict(ld_res=4), dict(res_off=2)]:
        with pytest.raises(ValueError):
            api.pointwise(emu_lib, A if "ld_a" not in kw else A.reshape(-1)[None], W, **kw)
    with pytest.raises(ValueError):
        api.pointwise(emu_lib, A.reshape(-1), W, ld_a=4, out=np.zeros(32, np.float64))


# ---- on the GPU ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu_lib():
    import backscrub_b200 as bs
    L = bs.lib()
    assert L.bsb_device_count() > 0
    return L


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GRID))
def test_pointwise_ex_exact_variants(gpu_lib, name):
    check_exact_variants(gpu_lib, name, (0, 2, 3, 4, 5, 8, 16, 32, 64))


@pytest.mark.gpu
def test_pointwise_ex_refusals(gpu_lib):
    check_refusals(gpu_lib, tc_present=True)


@pytest.mark.gpu
@pytest.mark.parametrize("tc_variant,mask_hi", [(2, 0), (2, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("name", list(GRID))
def test_tensor_core_against_float64(gpu_lib, name, tc_variant, mask_hi):
    case = GRID[name]
    acts = (case[3], case[4], case[6])
    try:
        assert gpu_lib.bsb_set_tuning(b"tc_variant", tc_variant) and gpu_lib.bsb_set_tuning(b"tc_mask_hi", mask_hi)
        for fx, (A, W, b, res) in fixtures(case, sum(map(ord, name))):
            got = Layout(case, A, res).run(gpu_lib, W, b, acts, 1)
            if fx.startswith("dyadic"):
                r2 = tr.r2(A, W, b, res, *acts).astype(np.float32)
                bad = got != r2
                assert not bad.any(), (fx, int(bad.sum()), np.argwhere(bad)[:4].tolist())
                print(f"TC {name} v{tc_variant} mask{mask_hi} {fx}: R2 bit for bit")
            else:
                ratio = np.abs(got - tr.r1(A, W, b, res, *acts)) / tr.bound(A, W, b, res)
                print(f"TC {name} v{tc_variant} mask{mask_hi} {fx}: max |got - R1| / bound = {ratio.max():.3g}")
                assert ratio.max() <= 1, (fx, ratio.max(), np.unravel_index(ratio.argmax(), ratio.shape))
    finally:
        gpu_lib.bsb_set_tuning(b"tc_variant", 2)
        gpu_lib.bsb_set_tuning(b"tc_mask_hi", 0)


# ---- each tensor-core layer of DeepLab and BodyPix, checked in place -----------------------------------------------
ACT_CODE = {"NONE": NONE, "RELU": RELU, "RELU_N1_TO_1": N1_TO_1, "RELU6": RELU6}
# the qualifying 1x1 convolutions in the graphs' own 257 x 257 shapes; a 640 x 480 frame only makes BodyPix's layers larger
MIN_TC_LAYERS = {"deeplab": 33, "bodypix": 13}


def tc_candidates(graph, pixels, K_min=16):
    """op indices of the 1x1 convolutions the planner gives the tensor cores: stride 1, K >= tc_min_k (16) and a multiple
    of 4, N >= 8, at least 1024 pixels per frame (engine.cu, Engine::plan).  pixels(t): h * w of tensor t as planned
    (the graph's shapes are those of its nominal input size)."""
    out = set()
    for op in graph.ops:
        if op.kind != "CONV_2D" or op.opts.get("stride_w") != 1 or op.opts.get("stride_h") != 1:
            continue
        N, kh, kw, K = graph.tensors[op.inputs[1]].shape
        if kh == 1 and kw == 1 and K >= K_min and K % 4 == 0 and N >= 8 and pixels(op.inputs[0]) >= 1024:
            out.add(op.idx)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("sub_batch_mb", [0, 1])
@pytest.mark.parametrize("key", ["deeplab", "bodypix"])
def test_model_tensor_core_layers_in_place(gpu_lib, key, sub_batch_mb):
    """Every tensor-core layer of the model, as the engine runs it (concatenation slices, folded residual ADDs, N = 21
    through the generic epilogue, M = n*h*w over many waves, and with sub_batch_mb = 1 frame-offset launches), is
    within the derived bound of R1 computed in float64 from that context's own input and residual tensors and the
    model's weights, in the first and the last frame (the last holds the ragged last tile).  Keeping the tensors must
    not change the logits: they equal those of a plain tensor-core context bit for bit."""
    from tests.conftest import model_path
    from tools import tflite_graph
    n = 6
    graph = tflite_graph.load(model_path(key))
    rng = np.random.default_rng(3)
    try:
        assert gpu_lib.bsb_set_tuning(b"sub_batch_mb", sub_batch_mb)
        g = api.MaskGen(gpu_lib, model_path(key), 640, 480, max_batch=n, flags=1 | 4)    # KEEP_TENSORS | TENSOR_CORES
        plain = api.MaskGen(gpu_lib, model_path(key), 640, 480, max_batch=n, flags=4)
        x = rng.uniform(-1 if key == "deeplab" else 0, 1, (n, *g.in_hwc)).astype(np.float32)
        logits = g.infer(x)
        assert np.array_equal(logits.view(np.uint32), plain.infer(x).view(np.uint32)), "KEEP_TENSORS changes the logits"
        # capacity for tensor t: the model input's pixels times t's channels (no tensor has more pixels than the input)
        size = lambda t: g.in_hwc[0] * g.in_hwc[1] * graph.tensors[t].shape[-1]
        steps = g.tc_steps()
        def pixels(t):       # as planned; a tensor folded into its consumer (a pooled row) keeps the graph's shape
            v = g.tensor(t, size(t))
            return v.size // graph.tensors[t].shape[-1] if v is not None else int(np.prod(graph.tensors[t].shape[1:3]))
        want = tc_candidates(graph, pixels)
        assert {s["op"] for s in steps} == want, (sorted(want - {s["op"] for s in steps}), sorted({s["op"] for s in steps} - want))
        assert len(steps) >= MIN_TC_LAYERS[key]
        worst = 0.0
        for s in steps:
            op = graph.ops[s["op"]]
            K, N = s["K"], s["N"]
            assert s["act1"] == ACT_CODE[op.opts["act"]], s
            W = graph.const_f32(op.inputs[1]).reshape(N, K)
            b = graph.const_f32(op.inputs[2]) if len(op.inputs) > 2 and op.inputs[2] >= 0 else None
            for f in (0, n - 1):
                A = g.tensor(s["in"], size(s["in"]), frame=f).reshape(-1, K)
                res = g.tensor(s["residual"], size(s["residual"]), frame=f).reshape(-1, N) if s["residual"] >= 0 else None
                got = g.tensor(s["out"], size(s["out"]), frame=f).reshape(-1, N)
                acts = (s["act1"], s["act2"], s["act3"])
                ratio = (np.abs(got - tr.r1(A, W, b, res, *acts)) / tr.bound(A, W, b, res)).max()
                print(f"TC-LAYER {key} sub_batch_mb={sub_batch_mb} op {s['op']} K={K} N={N} residual={s['residual'] >= 0} "
                      f"frame {f}: max |got - R1| / bound = {ratio:.3g}")
                assert ratio <= 1, (s, f, ratio)
                worst = max(worst, ratio)
        print(f"TC-LAYER {key} sub_batch_mb={sub_batch_mb}: {len(steps)} layers, worst {worst:.3g}")
        g.close()
        plain.close()
    finally:
        gpu_lib.bsb_set_tuning(b"sub_batch_mb", 0)

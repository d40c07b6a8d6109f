"""float64 references and the error model of the tensor-core (3xTF32) 1x1 convolution.

Notation: t(x) is the fp32 value x with its 13 low mantissa bits cleared (the tf32 truncation).  Per product the
kernel forms
    t(a) t(w_hi) + t(a_lo) t(w_hi) + t(a) t(w_lo),    a_lo = a - t(a),  w_hi = t(w),  w_lo = w - t(w)
(the tensor core truncates the raw fp32 operands a, a_lo and w_lo to tf32 itself) and sums the 3K terms in fp32 in an
order the hardware chooses; then out = act3(act2(act1(sum + bias)) + residual) in fp32.

R1  float64 value of act3(act2(act1(A W^T + b)) + res)        -- the operation itself
R2  the same with every product replaced by the split above   -- what the kernel sums; every term is an 11-bit x 11-bit
                                                                 product, so each is exact in float64 (and in fp32)

Two kinds of fixture:
  exact dyadic fixtures  every term and every partial sum of R2 is a multiple of 2^-12 below 2^11 in magnitude, so it is
                         an fp32 number: whatever the order and rounding of the adds, the device must return R2 exactly;
  wide-range fixtures    checked against R1 with `bound` below.
"""
import numpy as np

ACT_NONE, ACT_RELU, ACT_RELU_N1_TO_1, ACT_RELU6 = 0, 1, 2, 3
U = 2.0 ** -10      # tf32 truncation: |x - t(x)| < U |x|
EPS = 2.0 ** -23    # one fp32 ulp relative to the magnitude: ulp(x) <= EPS |x|


def t(x):
    """x (fp32) with the 13 low mantissa bits cleared, as fp32."""
    x = np.ascontiguousarray(x, np.float32)
    return (x.view(np.uint32) & np.uint32(0xffffe000)).view(np.float32)


def tf32_round(x):
    """round to nearest tf32 (ties away): the fault `t` guards against (a tensor core that rounds its operand)."""
    x = np.ascontiguousarray(x, np.float32)
    return ((x.view(np.uint32) + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(np.float32)


def act(v, a):
    """the kernels' clamps, same comparisons (so a -0 passes through as it does there), in v's dtype"""
    z = lambda c: np.asarray(c, v.dtype)
    if a == ACT_RELU:
        return np.where(v < 0, z(0), v)
    if a == ACT_RELU6:
        y = np.where(v < 0, z(0), v)
        return np.where(y > 6, z(6), y)
    if a == ACT_RELU_N1_TO_1:
        y = np.where(v < -1, z(-1), v)
        return np.where(y > 1, z(1), y)
    assert a == ACT_NONE
    return v


def epilogue(total, b, res, act1, act2, act3):
    """act3(act2(act1(total + b)) + res), in total's dtype."""
    v = total + (b if b is not None else 0)
    v = act(act(v, act1), act2)
    return act(v + res, act3) if res is not None else v


def split_terms(A, W):
    """the three [M, N, K] term tensors of the 3xTF32 split, float64 (exact)."""
    A = np.asarray(A, np.float32); W = np.asarray(W, np.float32)
    a_hi = t(A); a_lo = (A - a_hi).astype(np.float32)
    w_hi = t(W); w_lo = (W - w_hi).astype(np.float32)
    a_hi, a_lo, w_hi, w_lo = (x.astype(np.float64) for x in (a_hi, t(a_lo), w_hi, t(w_lo)))
    return [a_hi[:, None, :] * w_hi[None], a_lo[:, None, :] * w_hi[None], a_hi[:, None, :] * w_lo[None]]


def r1(A, W, b=None, res=None, act1=0, act2=0, act3=0):
    total = np.asarray(A, np.float64) @ np.asarray(W, np.float64).T
    return epilogue(total, None if b is None else np.asarray(b, np.float64), None if res is None else np.asarray(res, np.float64),
                    act1, act2, act3)


def split_matmul(A, W, hi=t, drop=None):
    """sum over k of the split products, float64.  Exact for the dyadic fixtures.  Faults: drop = index of a term to
    leave out; hi = what the tensor core makes of the raw A operand (a_lo is always a - t(a), as the kernel computes it)."""
    A = np.asarray(A, np.float32); W = np.asarray(W, np.float32)
    a_hi = hi(A); a_lo = (A - t(A)).astype(np.float32)
    w_hi = t(W); w_lo = (W - w_hi).astype(np.float32)
    f = lambda x: x.astype(np.float64)
    terms = [f(a_hi) @ f(w_hi).T, f(t(a_lo)) @ f(w_hi).T, f(a_hi) @ f(t(w_lo)).T]
    return sum(x for i, x in enumerate(terms) if i != drop)


def r2(A, W, b=None, res=None, act1=0, act2=0, act3=0):
    return epilogue(split_matmul(A, W), None if b is None else np.asarray(b, np.float64),
                    None if res is None else np.asarray(res, np.float64), act1, act2, act3)


# ---- fp32 emulations of the kernel's sum (order and rounding of the adds are the hardware's business) -----------------
def _add_rtz(x, y):
    """fp32 x + y rounded toward zero (x, y fp32)."""
    # the float64 sum is exact while the exponents of x and y differ by less than 29; beyond that its own error (2^-53
    # relative) is far below the fp32 rounding emulated here
    s = x.astype(np.float64) + y.astype(np.float64)
    f = s.astype(np.float32)
    away = np.abs(f.astype(np.float64)) > np.abs(s)
    return np.where(away, np.nextafter(f, np.float32(0)), f).astype(np.float32)


def emulate(A, W, b=None, res=None, act1=0, act2=0, act3=0, order="forward"):
    """the kernel's arithmetic in fp32: the 3K split terms (fp32, exact) summed one by one in `order` ("forward", "reverse",
    "pairwise", or "rtz": forward with an adder that rounds toward zero), then the fp32 epilogue."""
    terms = np.concatenate([x.astype(np.float32) for x in split_terms(A, W)], axis=2)     # [M, N, 3K]
    if order == "reverse":
        terms = terms[:, :, ::-1]
    if order == "pairwise":
        while terms.shape[2] > 1:
            if terms.shape[2] % 2:
                terms = np.concatenate([terms, np.zeros(terms.shape[:2] + (1,), np.float32)], axis=2)
            terms = (terms[:, :, 0::2] + terms[:, :, 1::2]).astype(np.float32)
        acc = terms[:, :, 0]
    else:
        acc = np.zeros(terms.shape[:2], np.float32)
        for k in range(terms.shape[2]):
            acc = _add_rtz(acc, terms[:, :, k]) if order == "rtz" else (acc + terms[:, :, k]).astype(np.float32)
    if order == "rtz":
        v = _add_rtz(acc, np.broadcast_to(np.float32(0) if b is None else np.asarray(b, np.float32), acc.shape))
        v = act(act(v, act1), act2)
        return act(_add_rtz(v, np.asarray(res, np.float32)), act3) if res is not None else v
    return epilogue(acc, None if b is None else np.asarray(b, np.float32), None if res is None else np.asarray(res, np.float32),
                    act1, act2, act3).astype(np.float32)


ORDERS = ("forward", "reverse", "pairwise", "rtz")


def bound(A, W, b=None, res=None):
    """|kernel - R1| <= bound, elementwise.

    Split error per product (a = t(a) + a_lo, a_lo = t(a_lo) + a_ll, the same for w; |a_lo| < U|a|, |a_ll| < U|a_lo|):
        a w - [t(a) t(w) + t(a_lo) t(w) + t(a) t(w_lo)] = a_ll t(w) + t(a) w_ll + a_lo w_lo,   at most 3 U^2 |a| |w|.
    Accumulation: the kernel adds 3K exact terms, the bias and the residual: n = 3K + 2 fp32 additions.  Every partial
    sum is at most S = (1 + 2U) sum_k |a||w| + |b| + |res| in magnitude and an addition errs by at most one ulp of its
    result (round-to-nearest errs by half of one; one allows for an adder that truncates), so by at most EPS S; summed
    with the standard (1 - n EPS) correction, gamma_n = n EPS / (1 - n EPS).  The activations are clamps, 1-Lipschitz:
    they add nothing.
        bound = 3 U^2 sum_k |a||w| + gamma_n S
    """
    P = np.abs(np.asarray(A, np.float64)) @ np.abs(np.asarray(W, np.float64)).T
    K = np.asarray(A).shape[1]
    n = 3 * K + 2
    gamma = n * EPS / (1 - n * EPS)
    S = (1 + 2 * U) * P
    if b is not None:
        S = S + np.abs(np.asarray(b, np.float64))
    if res is not None:
        S = S + np.abs(np.asarray(res, np.float64))
    return 3 * U * U * P + gamma * S


# ---- fixtures ---------------------------------------------------------------------------------------------------------
def _fp32_exact(x):
    x = np.asarray(x, np.float64)
    return np.array_equal(x.astype(np.float32).astype(np.float64), x)


def _grid_exact(x):
    """multiple of 2^-12 and below 2^11: an fp32 number, and so is any sum of such values that stays below 2^11"""
    x = np.asarray(x, np.float64)
    return np.array_equal(np.round(x * 4096), x * 4096) and np.abs(x).max() < 2.0 ** 11


def _lo_grid(rng, shape, signed):
    """unsigned: i + j 2^-12, i in {0, 1}, j in {0..3}.  signed: +-(1 + j 2^-12), so that t(a) t(w) = +-1 stays on the
    grid when both operands carry low bits (and rows whose +-1 cancel keep the 2^-22 details visible in fp32)"""
    if signed:
        return ((1 + rng.integers(0, 4, shape) * 2.0 ** -12) * rng.choice([-1.0, 1.0], shape)).astype(np.float32)
    return (rng.integers(0, 2, shape) + rng.integers(0, 4, shape) * 2.0 ** -12).astype(np.float32)


def dyadic(kind, M, K, N, seed, bias=True, residual=False):
    """An exact dyadic fixture (A, W, b, res):
         "a_lo"   the low bits in A:  a = i + j 2^-12, w in {-1, 0, 1}              (a_lo t(w) != 0, t(a) w_lo == 0)
         "w_lo"   the mirror:         a in {-1, 0, 1}, w = i + j 2^-12              (t(a) w_lo != 0)
         "both"   both, signed, for small K: a_lo w_lo != 0 is what R2 drops, so R1 != R2 there
    The generator asserts what makes the device result order-independent: every split term and every partial sum (in
    any order, since each is bounded by the sum of the magnitudes) lies on the 2^-12 grid below 2^11."""
    rng = np.random.default_rng(seed)
    if kind == "a_lo":
        A = _lo_grid(rng, (M, K), False); W = rng.integers(-1, 2, (N, K)).astype(np.float32)
    elif kind == "w_lo":
        A = rng.integers(-1, 2, (M, K)).astype(np.float32); W = _lo_grid(rng, (N, K), False)
    else:
        assert kind == "both" and K <= 64
        A = _lo_grid(rng, (M, K), True); W = _lo_grid(rng, (N, K), True)
    b = (rng.integers(-16, 17, N) * 2.0 ** -4).astype(np.float32) if bias else None
    res = (rng.integers(-64, 65, (M, N)) * 2.0 ** -6).astype(np.float32) if residual else None
    # each operand part takes a handful of values: every product of two of them is on the grid
    a_hi, w_hi = t(A), t(W)
    a_lo, w_lo = t((A - a_hi).astype(np.float32)), t((W - w_hi).astype(np.float32))
    assert np.array_equal(a_lo, A - a_hi) and np.array_equal(w_lo, W - w_hi), "the low parts must be tf32 numbers"
    for x, y in ((a_hi, w_hi), (a_lo, w_hi), (a_hi, w_lo)):
        assert _grid_exact(np.multiply.outer(np.unique(x).astype(np.float64), np.unique(y).astype(np.float64)))
    f = lambda x: np.abs(x.astype(np.float64))
    mag = f(a_hi) @ f(w_hi).T + f(a_lo) @ f(w_hi).T + f(a_hi) @ f(w_lo).T
    mag = mag + (np.abs(b) if bias else 0) + (np.abs(res) if residual else 0)
    assert mag.max() < 2.0 ** 11, "partial sums could leave the exact range"
    for x in (b, res):
        assert x is None or _grid_exact(x)
    return A, W, b, res


def wide(kind, M, K, N, seed, bias=True, residual=False, decades=4):
    """A wide-range fixture: magnitudes log-uniform over `decades` decades, "mixed" signs, or "same" signs (what
    post-ReLU6 activations times positive weights look like)."""
    rng = np.random.default_rng(seed)
    mag = lambda shape: 10.0 ** rng.uniform(-decades / 2, decades / 2, shape)
    A = mag((M, K)); W = mag((N, K)) / np.sqrt(K)
    if kind == "mixed":
        A = A * rng.choice([-1.0, 1.0], (M, K)); W = W * rng.choice([-1.0, 1.0], (N, K))
    else:
        assert kind == "same"
    A, W = A.astype(np.float32), W.astype(np.float32)
    b = (rng.standard_normal(N) * 2).astype(np.float32) if bias else None
    res = (rng.standard_normal((M, N)) * 2).astype(np.float32) if residual else None
    return A, W, b, res


# ---- plausible faults of the kernel, as fp32 results -------------------------------------------------------------------
def mutants(A, W, b, res, act1, act2, act3):
    """name -> the fp32 output of a kernel with that fault (each computed exactly in float64, then rounded once)."""
    bb = None if b is None else np.asarray(b, np.float64)
    rr = None if res is None else np.asarray(res, np.float64)
    f = lambda total, **kw: epilogue(total, kw.get("b", bb), rr, act1, act2, act3).astype(np.float32)
    A32 = np.asarray(A, np.float32)
    shifted = np.roll(A32, -1, axis=0)                            # a_lo of the next row
    a_hi = t(A32).astype(np.float64); w_hi = t(W).astype(np.float64); w_lo = t((W - t(W)).astype(np.float32)).astype(np.float64)
    lo_next = t((shifted - t(shifted)).astype(np.float32)).astype(np.float64)
    out = {
        "drop a_hi*w_hi": f(split_matmul(A, W, drop=0)),
        "drop a_lo*w_hi": f(split_matmul(A, W, drop=1)),
        "drop a_hi*w_lo": f(split_matmul(A, W, drop=2)),
        "A rounded to tf32, not truncated": f(split_matmul(A, W, hi=tf32_round)),
        "a_lo of the next row": f(a_hi @ w_hi.T + lo_next @ w_hi.T + a_hi @ w_lo.T),
        "no bias": f(split_matmul(A, W), b=None),
    }
    if res is not None:
        v = act(act(split_matmul(A, W) + (bb if bb is not None else 0) + rr, act1), act2)
        out["residual before the activation"] = act(v, act3).astype(np.float32)
    return out

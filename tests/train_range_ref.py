"""TEST INFRASTRUCTURE: numpy model of the automatically scaled 3xF16 split of the training paths (csrc/autoscale.cuh,
csrc/tc_common.cuh: split_f16_keep_nonfinite) and the crafted inputs that probe it.  CPU-importable.

The rule, for a tensor x of fp32 values:
  e  = clamp(13 - ceil(log2 max|x|), -126, 126) over the FINITE elements, 0 when no finite element is non-zero;
  v  = fp32(x * 2^e)                     (a power of two: exact wherever v is a normal fp32)
  hi = fp16_rn(v), lo = fp16_rn(v - hi)  for a finite v (|v| <= 2^13, so nothing saturates);
  hi = v (+-inf, or NaN), lo = +0        for a non-finite v.
b2second.tc.pow2_scale is 2^e of the same rule.
"""
import numpy as np

FLT_MAX = float(np.finfo(np.float32).max)


def exponent(x):
    """e of the rule for the fp32 values x (anything np.asarray takes)"""
    a = np.abs(np.asarray(x, dtype=np.float32)).ravel()
    a = a[np.isfinite(a)]
    m = float(a.max()) if a.size else 0.0
    if m == 0.0:
        return 0
    f, ex = np.frexp(m)                    # m = f * 2^ex, f in [0.5, 1): ceil(log2 m) is ex - 1 for f = 0.5, else ex
    ceil_log2 = int(ex) - 1 if f == 0.5 else int(ex)
    return int(min(max(13 - ceil_log2, -126), 126))


def split(x, e):
    """(hi, lo) float16 arrays of the rule for the fp32 values x under the exponent e"""
    v = np.asarray(x, dtype=np.float32) * np.float32(2.0 ** e)
    with np.errstate(invalid="ignore", over="ignore"):
        hi = v.astype(np.float16)
        lo = np.where(np.isfinite(v), v - hi.astype(np.float32), np.float32(0.0)).astype(np.float16)
    return hi, lo


def _base(rng, shape, e):
    return (rng.standard_normal(shape) * 2.0 ** e).astype(np.float32)


def crafted_cases(shape=(6, 5), seed=0):
    """{name: fp32 array of `shape`}: the edges of the rule -- zeros and -0.0, a max of exactly 2^12, 2^13 and the next
    float above 2^13, FLT_MAX, the smallest normal and subnormal floats, a max below 2^-113 (the exponent clamp), and
    +inf, -inf and NaN at the first, middle and last element of values at gradient scale (2^-30)."""
    rng = np.random.default_rng(seed)
    n = int(np.prod(shape))
    out = {}
    z = np.zeros(shape, np.float32)
    out["all_zero"] = z.copy()
    t = z.copy().ravel()
    t[[1, n // 2]] = -0.0
    t[n - 1] = 0.0
    out["neg_zero"] = t.reshape(shape)
    t = _base(rng, shape, -30).ravel()
    t[3] = -0.0
    t[n // 3] = 0.0
    out["zeros_among_values"] = t.reshape(shape)
    for name, m in (("max_2^12", 2.0 ** 12), ("max_2^13", 2.0 ** 13),
                    ("max_above_2^13", float(np.nextafter(np.float32(2.0 ** 13), np.float32(np.inf)))),
                    ("flt_max", FLT_MAX), ("min_normal", 2.0 ** -126), ("min_subnormal", 2.0 ** -149),
                    ("below_clamp", 2.0 ** -115)):
        t = np.clip(_base(rng, shape, np.log2(m) - 3) if m > 2.0 ** -140 else np.zeros(shape, np.float32), -m, m)
        t = t.astype(np.float32).ravel()
        t[n // 2 + 1] = -m
        out[name] = t.reshape(shape)
    # a subnormal max with other subnormals below it
    t = (rng.integers(-40, 41, size=n) * 2.0 ** -149).astype(np.float32)
    t[0] = 2.0 ** -130
    out["subnormals"] = t.reshape(shape)
    for vname, v in (("+inf", np.inf), ("-inf", -np.inf), ("nan", np.nan)):
        for where, i in (("first", 0), ("middle", n // 2), ("last", n - 1)):
            t = _base(rng, shape, -30).ravel()
            t[i] = v
            out["%s_%s" % (vname, where)] = t.reshape(shape)
    t = np.full(shape, np.nan, np.float32).ravel()
    t[2] = np.inf
    out["no_finite"] = t.reshape(shape)
    return out


def same_bits(a, b):
    """float16 arrays equal bit for bit, NaN matched by isnan only"""
    a, b = np.asarray(a, np.float16), np.asarray(b, np.float16)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool((na == nb).all() and (a.view(np.uint16)[~na] == b.view(np.uint16)[~nb]).all())

"""TEST INFRASTRUCTURE: float64 references of the kernels that compute in plain fp32 -- the sparse convolution
(b2s_sparse_conv), its weight gradient (b2s_sparse_conv_wgrad), the PointPillars feature net (b2s_pfn / b2s_pfn_ex) and
the voxel mean (b2s_vfe_mean, b2s_voxelize's fused mean) -- with a rigorous per-element error bound of their fp32
arithmetic.  CPU-importable; the GPU tests call it on CUDA tensors.  u = 2^-24, gamma_n = n u / (1 - n u), and every
fp32 operation on a result r is taken to round it by at most u |r| + 2^-150 (the half-ulp of the subnormals: nothing
is flushed to zero).

Dot products.  An output y = s * sum(a * w) + shift formed by one sequential fmaf chain of n nonzero terms (n counted
exactly from the table) and an fmaf epilogue satisfies

    |y - y64| <= |s| * gamma_(n+1) * S1 + u * |pre| + (n + 1) * 2^-149,      S1 = sum |a * w| over those terms,

with y64 and pre = s * y64 + shift in float64 from the exact fp32 inputs.  The chain gives gamma_n * S1 (Higham, Accuracy
and Stability of Numerical Algorithms, 3.1); the epilogue rounds pre and multiplies the chain error by (1 + u), and
gamma_n * (1 + u) <= gamma_(n+1).  ReLU is 1-Lipschitz, so the bound of pre holds after it.  The weight gradient sums
one chain per 2048-row slab and then adds the m slab partials in order: the chains give gamma_nmax over the slab that is
longest for the element, the m - 1 additions gamma_(m-1) over the partials, together gamma_(nmax + m) * S1.

PFN.  Per real point slot the Linear input carries the rounding of its decoration, propagated explicitly:
    mean of the np points          gamma_np * mean|p| + u * |mean|
    pillar centre q * v + off      gamma_2 * (|q * v| + |off|)
    the offsets p - mean, p - c    (1 + u) * (error of mean or centre) + u * |offset|
    radius sqrt(x*x + y*y)         gamma_3 * r
each multiplied by |w| of its Linear column and summed (E); the chain of FIN terms adds gamma_FIN * (S1 + E) and the BN
fmaf u * |pre|.  ReLU and the max over slots are 1-Lipschitz, so the bound of the output is the largest slot bound; a
padded slot contributes relu(shift) exactly (upstream's masked zero rows: Linear 0, BN shift).

The worst-case bound is loose (about 1e-4 * S1 at n = 27 * 64), so it cannot see lost precision.  The aggregate check
    rms(max(0, |y - y64| - rest)) / rms(|s| * S1) <= RHO,       rest = the bound's u * |pre| and 2^-149 terms,
catches it.  RHO is the smallest power of two that the unmodified kernels meet with at least a 2x margin on every case of
tests/test_gpu_fp32_fp64.py.  Measured on an H100 80GB HBM3 at a 700 W power limit: the largest aggregate ratio of any
case is 4.73e-8 (the PFN, 5 features, T = 100, radius decoration), the largest of the sparse conv, its weight gradient
and the input gradient 4.46e-8, so RHO = 2^-23 = 1.19e-7 leaves a 2.5x margin (2^-24 would leave 1.26x).  The largest
per-element ratio |y - y64| / bound of any case is 0.81.  The emulated kernels of tests/test_fp32_ref.py reach 4.75e-8.

Simulated faults (computed in float64 from an actual result; the check must reject each):
    F1  thin:      one input channel of one tap dropped for the 64 rows of one k_sparse_conv tile (conv_f1); one 32-row
                   chunk of one slab dropped for every kernel offset (wgrad_f1)
    F2  local:     one neighbour of the last row dropped (conv_f2); one (row, offset) pair dropped (wgrad_f2)
    F4  precision: both operands rounded to a 10-bit mantissa, an accidental TF32 or fp16 step (conv_f4, wgrad_f4)
    PFN:           the mean over num - 1 points, the centre shifted by half a voxel in x, the padded-slot term dropped,
                   the padded-slot term applied when num == T (pfn_ref(..., fault=...))
"""
import collections

import numpy as np
import torch

U = 2.0 ** -24
ETA = 2.0 ** -149           # twice the underflow error of one rounding
RHO = 2.0 ** -23
SLAB, CHUNK, TILE = 2048, 32, 64    # b2s_sparse_conv_wgrad's slab and chunk, k_sparse_conv's rows per CTA

# y: the float64 value; bound: the per-element bound; unit: |s| * S1 (the aggregate's scale); rest: the bound's terms
# that are not relative to S1
Ref = collections.namedtuple("Ref", "y bound unit rest")


def gamma(n):
    n = torch.as_tensor(n, dtype=torch.float64)
    return n * U / (1.0 - n * U)


def round_mantissa(t, bits=10):
    """t rounded to `bits` explicit mantissa bits (float64 result; 10: the precision of fp16 and TF32)"""
    m, e = np.frexp(t.detach().cpu().double().numpy())
    m = np.round(m * 2.0 ** (bits + 1)) / 2.0 ** (bits + 1)
    return torch.from_numpy(np.ldexp(m, e)).to(t.device)


# ---- test data ----------------------------------------------------------------------------------------------------
# (kernel size, stride, padding, subm): SubM 3^3, 3^3 stride 2 (SECOND's downsampling), (3,1,1) stride (2,1,1)
# (SpMiddleFHD's last conv), 5^3 SubM (K = 125, past k_sparse_conv's K <= 27), 1x1x1
TABLES = {"subm": ((3, 3, 3), (1, 1, 1), (1, 1, 1), True), "strided": ((3, 3, 3), (2, 2, 2), (0, 1, 1), False),
          "k311": ((3, 1, 1), (2, 1, 1), (0, 0, 0), False), "subm5": ((5, 5, 5), (1, 1, 1), (2, 2, 2), True),
          "k1": ((1, 1, 1), (1, 1, 1), (0, 0, 0), True)}
SHAPE, BATCH = (9, 64, 56), 2


def surface_coords(rng, n):
    """about n distinct (b, z, y, x) voxels of a noisy surface in SHAPE x BATCH, sorted"""
    m = 4 * n + 64
    b, y, x = rng.integers(BATCH, size=m), rng.integers(SHAPE[1], size=m), rng.integers(SHAPE[2], size=m)
    z = np.clip(np.round(SHAPE[0] / 2 + 2 * np.sin(x / 5.0) + rng.normal(0, 0.9, size=m)), 0, SHAPE[0] - 1)
    idx = np.unique(np.stack([b, z, y, x], 1).astype(np.int32), axis=0)
    idx = idx[rng.permutation(idx.shape[0])[:n]]
    return idx[np.lexsort(idx.T[::-1])]


def table_rows(rng, table, n_out):
    """(n_in, nbr [n_out, K] int32) of `table` over a surface, cut to exactly n_out output rows"""
    ks, st, pd, subm = TABLES[table]
    n = max(n_out, 1)
    while True:
        idx = surface_coords(rng, n + 16)
        _, nbr = build_table(idx, SHAPE, ks, st, pd, subm)
        if nbr.shape[0] >= n_out:
            return idx.shape[0], nbr[:n_out]
        n *= 2


def pillars(rng, n, T, F, grid=(432, 496), vs=(0.16, 0.16), lo=(0.0, -39.68)):
    """n pillars of the PointPillars KITTI grid for b2s_pfn: (points [P, F] in shuffled order, slots [n, T] (-1 past
    num), num [n], coors [n, 4]).  Counts 1, T - 1, T and random; pillars at the four grid corners and at x ~ 69 m (the
    last column, where the centre offset cancels); x, the radius and the reflectance are positive."""
    num = rng.integers(1, T + 1, size=n)
    num[0::5], num[1::5], num[2::5] = 1, max(T - 1, 1), T
    gx, gy = rng.integers(grid[0], size=n), rng.integers(grid[1], size=n)
    corners = [(0, 0), (grid[0] - 1, 0), (0, grid[1] - 1), (grid[0] - 1, grid[1] - 1)]
    for i, (cx, cy) in enumerate(corners):
        gx[i], gy[i] = cx, cy
    gx[4:n:7] = grid[0] - 1
    coors = np.stack([np.zeros(n), np.zeros(n), gy, gx], 1).astype(np.int32)
    pts = []
    for i in range(n):
        p = rng.uniform(0, 1, (num[i], F))
        p[:, 0] = lo[0] + (gx[i] + rng.uniform(0.01, 0.99, num[i])) * vs[0]
        p[:, 1] = lo[1] + (gy[i] + rng.uniform(0.01, 0.99, num[i])) * vs[1]
        p[:, 2] = rng.uniform(-3, 1, num[i])
        pts.append(p)
    pts = np.concatenate(pts, 0).astype(np.float32)
    perm = rng.permutation(pts.shape[0])
    where = np.empty_like(perm)
    where[perm] = np.arange(perm.shape[0])
    slots = np.full((n, T), -1, np.int32)
    start = np.concatenate([[0], np.cumsum(num)[:-1]])
    for i in range(n):
        slots[i, :num[i]] = where[start[i]:start[i] + num[i]]
    return pts[perm], slots, num.astype(np.int32), coors


def pfn_layer(rng, F, radius, cout=64, n_below=8):
    """(w [cout, FIN], scale, shift) float32; the first n_below channels read only column 0 (x, or |xy|: positive) with
    scale -1 and shift > 0, so every real point falls below relu(shift) and the padded-slot rule alone decides them"""
    fin = F + (4 if radius else 5)
    w = (rng.standard_normal((cout, fin)) * 0.3).astype(np.float32)
    scale = (rng.uniform(0.5, 1.5, cout) * rng.choice([-1, 1], cout)).astype(np.float32)
    shift = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    w[:n_below] = 0
    w[:n_below, 0] = 1
    scale[:n_below] = -1
    shift[:n_below] = rng.uniform(0.2, 0.5, n_below)
    return w, scale, shift


# ---- tables -------------------------------------------------------------------------------------------------------
def _offsets(ksize):
    kz, ky, kx = ksize
    return np.stack(np.meshgrid(np.arange(kz), np.arange(ky), np.arange(kx), indexing="ij"), -1).reshape(-1, 3)


def build_table(idx, shape, ksize, stride=(1, 1, 1), padding=(0, 0, 0), subm=False):
    """index-level rulebook in numpy: idx [n, 4] int (b, z, y, x), shape (D, H, W) -> (out idx [n_out, 4] sorted,
    nbr [n_out, K] int32: the input row at out * stride - padding + offset k, offsets k row-major over ksize, -1: none).
    SubM: the outputs are the inputs and the kernel is centred."""
    idx = np.asarray(idx, np.int64)
    shape, ksize, stride = np.asarray(shape), np.asarray(ksize), np.asarray(stride)
    padding = ksize // 2 if subm else np.asarray(padding)
    offs = _offsets(ksize)
    if subm:
        out, oshape = idx, shape
    else:
        oshape = (shape + 2 * padding - ksize) // stride + 1
        cand = []
        for o in offs:
            q = idx[:, 1:] + padding - o
            ok = np.all((q % stride == 0) & (q >= 0) & (q // stride < oshape), 1)
            cand.append(np.concatenate([idx[ok, :1], q[ok] // stride], 1))
        out = np.unique(np.concatenate(cand, 0), axis=0) if cand else np.zeros((0, 4), np.int64)

    def key(b, p, sh):
        return ((b * sh[0] + p[:, 0]) * sh[1] + p[:, 1]) * sh[2] + p[:, 2]

    kin = key(idx[:, 0], idx[:, 1:], shape)
    order = np.argsort(kin)
    ks = kin[order]
    nbr = np.full((out.shape[0], offs.shape[0]), -1, np.int32)
    for k, o in enumerate(offs):
        if not len(ks):
            break
        p = out[:, 1:] * stride - padding + o
        kk = key(out[:, 0], p, shape)
        j = np.searchsorted(ks, kk).clip(0, len(ks) - 1)
        hit = np.all((p >= 0) & (p < shape), 1) & (ks[j] == kk)
        nbr[hit, k] = order[j[hit]]
    return out.astype(np.int32), nbr


def transpose_table(nbr, n_in):
    """nbrT [n_in, K]: nbrT[i, k] = o where nbr[o, k] = i, else -1 (the input side of a strided table)"""
    nbr = np.asarray(nbr)
    t = np.full((n_in, nbr.shape[1]), -1, np.int32)
    o, k = np.nonzero(nbr >= 0)
    t[nbr[o, k], k] = o
    return t


# ---- sparse convolution -------------------------------------------------------------------------------------------
def sparse_ref(x, w, nbr, scale=None, shift=None, relu=False):
    """y[o] = act(s * sum_k W[k]^T x[nbr[o, k]] + shift).  x [n_in, Cin] fp32, w [K, Cin, Cout], nbr [n_out, K]
    -> Ref with [n_out, Cout] float64 fields."""
    xd, wd = x.double(), w.double()
    n_out, K = nbr.shape
    cin, cout = wd.shape[1], wd.shape[2]
    y = torch.zeros(n_out, cout, dtype=torch.float64, device=xd.device)
    S1 = torch.zeros_like(y)
    nbr = nbr.to(xd.device).long()
    for k in range(K):
        ok = nbr[:, k] >= 0
        if bool(ok.any()):
            a = xd[nbr[ok, k]]
            y[ok] += a @ wd[k]
            S1[ok] += a.abs() @ wd[k].abs()
    n = ((nbr >= 0).sum(1, keepdim=True) * cin).double()
    s = torch.ones(cout, dtype=torch.float64, device=xd.device) if scale is None else scale.to(xd.device).double()
    pre = y * s + (0.0 if shift is None else shift.to(xd.device).double())
    s = s.abs().expand_as(y)
    rest = U * pre.abs() + (n + 1) * ETA
    return Ref(torch.relu(pre) if relu else pre, s * gamma(n + 1) * S1 + rest, s * S1, rest)


def _apply(got, delta, relu):
    out = got.to(delta.device, torch.float64) - delta
    return torch.relu(out) if relu else out


def conv_f1(got, x, w, nbr, scale=None, relu=False, tile=0, k=None, c=0):
    """F1: input channel c of tap k (default: the tap with the most neighbours in the tile) dropped for the rows of one
    64-row tile."""
    nbr = nbr.to(got.device).long()
    rows = slice(TILE * tile, min(nbr.shape[0], TILE * tile + TILE))
    t = nbr[rows]
    if k is None:
        k = int((t >= 0).sum(0).argmax())
    ok = t[:, k] >= 0
    delta = torch.zeros(got.shape, dtype=torch.float64, device=got.device)
    d = torch.zeros(t.shape[0], w.shape[2], dtype=torch.float64, device=got.device)
    d[ok] = x.double()[t[ok, k], c:c + 1].to(got.device) * w.double()[k, c].to(got.device)
    delta[rows] = d
    s = 1.0 if scale is None else scale.to(got.device).double()
    return _apply(got, delta * s, relu)


def conv_f2(got, x, w, nbr, scale=None, relu=False, row=None):
    """F2: one neighbour (the first present offset) of one row (default the last) dropped."""
    nbr = nbr.to(got.device).long()
    o = nbr.shape[0] - 1 if row is None else row
    k = int((nbr[o] >= 0).nonzero()[0])
    delta = torch.zeros(got.shape, dtype=torch.float64, device=got.device)
    delta[o] = x.double()[nbr[o, k]].to(got.device) @ w.double()[k].to(got.device)
    s = 1.0 if scale is None else scale.to(got.device).double()
    return _apply(got, delta * s, relu)


def conv_f4(got, ref, x, w, nbr, scale=None, shift=None, relu=False):
    """F4: the result of a kernel whose operands were rounded to a 10-bit mantissa"""
    bad = sparse_ref(round_mantissa(x), round_mantissa(w), nbr, scale, shift, relu).y
    return got.to(ref.y.device, torch.float64) + (bad - ref.y)


# ---- weight gradient ----------------------------------------------------------------------------------------------
def wgrad_ref(x, g, nbr):
    """dW[k] = sum_o x[nbr[o, k]]^T g[o] -> Ref with [K, Cin, Cout] fields (s = 1)"""
    xd, gd = x.double(), g.double()
    nbr = nbr.to(xd.device).long()
    n_out, K = nbr.shape
    y = torch.zeros(K, xd.shape[1], gd.shape[1], dtype=torch.float64, device=xd.device)
    S1 = torch.zeros_like(y)
    m = max(1, -(-n_out // SLAB))
    present = (nbr >= 0).double()
    per_slab = torch.stack([present[j * SLAB:(j + 1) * SLAB].sum(0) for j in range(m)]) if n_out else \
        torch.zeros(1, K, dtype=torch.float64, device=xd.device)
    nmax, ntot = per_slab.max(0).values, per_slab.sum(0)
    for k in range(K):
        ok = nbr[:, k] >= 0
        a, b = xd[nbr[ok, k]], gd[ok]
        y[k] = a.t() @ b
        S1[k] = a.abs().t() @ b.abs()
    rest = U * y.abs() + ((ntot + m) * ETA)[:, None, None]
    return Ref(y, gamma(nmax + m)[:, None, None] * S1 + rest, S1, rest)


def wgrad_f1(got, x, g, nbr, slab=0, chunk=0):
    """F1: rows of one 32-row chunk of one slab left out for every kernel offset"""
    nbr = nbr.to(got.device).long()
    r0 = slab * SLAB + chunk * CHUNK
    rows = slice(r0, min(nbr.shape[0], r0 + CHUNK))
    delta = torch.zeros(got.shape, dtype=torch.float64, device=got.device)
    xd, gd = x.double().to(got.device), g.double().to(got.device)
    for k in range(nbr.shape[1]):
        ok = nbr[rows, k] >= 0
        delta[k] = xd[nbr[rows][ok, k]].t() @ gd[rows][ok]
    return got.to(torch.float64) - delta


def wgrad_f2(got, x, g, nbr, row=None):
    """F2: one (row, offset) pair -- the last row's first neighbour -- left out"""
    nbr = nbr.to(got.device).long()
    o = nbr.shape[0] - 1 if row is None else row
    k = int((nbr[o] >= 0).nonzero()[0])
    delta = torch.zeros(got.shape, dtype=torch.float64, device=got.device)
    delta[k] = torch.outer(x.double()[nbr[o, k]], g.double()[o]).to(got.device)
    return got.to(torch.float64) - delta


def wgrad_f4(got, ref, x, g, nbr):
    bad = wgrad_ref(round_mantissa(x), round_mantissa(g), nbr).y
    return got.to(ref.y.device, torch.float64) + (bad - ref.y)


# ---- PointPillars feature net -------------------------------------------------------------------------------------
PFN_FAULTS = ("mean", "centre", "pad_drop", "pad_full")


def pfn_ref(points, slots, num, coors, w, scale, shift, vx, vy, xoff, yoff, radius=False, fault=None):
    """PillarFeatureNet (radius=False) / PillarFeatureNetRadius (True), one PFNLayer with BN folded into scale / shift.
    points [P, F] fp32, slots [n, T] (entries past num are not read), num [n], coors [n, 4] (b, z, y, x),
    w [Cout, FIN] -> Ref with [n, Cout] fields.  fault: one of PFN_FAULTS, simulated in float64."""
    dev = w.device
    n, T = slots.shape
    F = points.shape[1]
    num = num.to(dev).long()
    live = torch.arange(T, device=dev)[None, :] < num[:, None]                      # [n, T]
    sl = torch.where(live, slots.to(dev).long(), torch.zeros_like(slots.to(dev).long()))
    p = torch.where(live[..., None], points.to(dev).double()[sl], 0.0)             # [n, T, F], 0 past num
    fn = num.double()[:, None]
    cnt = (num - 1).clamp_min(1).double()[:, None] if fault == "mean" else fn
    keep = torch.arange(T, device=dev)[None, :] < (num - 1)[:, None] if fault == "mean" else live
    mean = (p[..., :3] * keep[..., None]).sum(1) / cnt                             # [n, 3]
    mabs = p[..., :3].abs().sum(1) / fn
    e_mean = gamma(num)[:, None] * mabs + U * mean.abs()
    q = coors.to(dev).double()
    cv = torch.stack([q[:, 3] * float(vx), q[:, 2] * float(vy)], 1)
    off = torch.tensor([float(xoff), float(yoff)], dtype=torch.float64, device=dev)
    centre = cv + off
    if fault == "centre":
        centre = centre + torch.tensor([float(vx) / 2, 0.0], dtype=torch.float64, device=dev)
    e_centre = gamma(2) * (cv.abs() + off.abs())
    if radius:
        r = torch.sqrt(p[..., 0] ** 2 + p[..., 1] ** 2)
        raw = torch.cat([r[..., None], p[..., 2:]], -1)
        e_raw = torch.cat([gamma(3) * r[..., None], torch.zeros_like(p[..., 2:])], -1)
    else:
        raw, e_raw = p, torch.zeros_like(p)
    d_mean = p[..., :3] - mean[:, None, :]
    d_centre = p[..., :2] - centre[:, None, :]
    inp = torch.cat([raw, d_mean, d_centre], -1)                                   # [n, T, FIN]
    err = torch.cat([e_raw, (1 + U) * e_mean[:, None, :] + U * d_mean.abs(),
                     (1 + U) * e_centre[:, None, :] + U * d_centre.abs()], -1)
    fin = inp.shape[-1]
    assert w.shape[1] == fin, (w.shape, fin)
    wd = w.double()
    acc = inp @ wd.t()                                                             # [n, T, Cout]
    S1 = inp.abs() @ wd.abs().t()
    E = err @ wd.abs().t()
    s, sh = scale.to(dev).double(), shift.to(dev).double()
    pre = acc * s + sh
    val = torch.relu(pre).masked_fill(~live[..., None], -float("inf"))
    pad = torch.relu(sh).expand(n, -1)
    padded = (num < T) if fault not in ("pad_drop", "pad_full") else (
        torch.zeros_like(num, dtype=torch.bool) if fault == "pad_drop" else num <= T)
    y = torch.maximum(val.max(1).values, torch.where(padded[:, None], pad, torch.full_like(pad, -float("inf"))))
    bound_t = s.abs() * (1 + U) * (gamma(fin) * (S1 + E) + E) + U * pre.abs() + (fin + 1) * ETA
    zero = torch.zeros_like(bound_t)
    bound = torch.where(live[..., None], bound_t, zero).max(1).values
    unit = torch.where(live[..., None], s.abs() * S1, zero).max(1).values
    rest = torch.where(live[..., None], U * pre.abs() + (fin + 1) * ETA, zero).max(1).values
    return Ref(y, bound, unit, rest)


def pfn_fault(got, ref, fault, *args, **kw):
    """the kernel result with one PFN fault applied: got + (faulty y64 - y64)"""
    bad = pfn_ref(*args, fault=fault, **kw).y
    return got.to(ref.y.device, torch.float64) + (bad - ref.y)


# ---- voxel mean ---------------------------------------------------------------------------------------------------
def vfe_ref(voxels, num, nf, radius=False, fault=None):
    """SimpleVoxel (radius False: the mean of the first nf features over the num points) and SimpleVoxelRadius
    ([|mean xy|, mean[2:nf]]).  voxels [n, T, F] -> Ref with [n, nf] / [n, nf - 1] fields.  fault "mean": the mean over
    num - 1 points."""
    v = voxels.double()[..., :nf]
    n, T = v.shape[:2]
    num = num.to(v.device).long()
    live = (torch.arange(T, device=v.device)[None, :] < num[:, None])[..., None]
    keep = (torch.arange(T, device=v.device)[None, :] < (num - 1)[:, None])[..., None] if fault == "mean" else live
    cnt = ((num - 1).clamp_min(1) if fault == "mean" else num).double()[:, None]
    mean = torch.where(keep, v, 0.0).sum(1) / cnt
    mabs = torch.where(live, v.abs(), 0.0).sum(1) / num.double()[:, None]
    e = gamma(num)[:, None] * mabs + U * mean.abs()
    if not radius:
        rest = U * mean.abs()
        return Ref(mean, e, mabs, rest)
    r = torch.sqrt(mean[:, 0] ** 2 + mean[:, 1] ** 2)
    er = (e[:, 0] + e[:, 1]) * (1 + gamma(3)) + gamma(3) * r
    y = torch.cat([r[:, None], mean[:, 2:]], 1)
    bound = torch.cat([er[:, None], e[:, 2:]], 1)
    unit = torch.cat([(mabs[:, 0] + mabs[:, 1])[:, None], mabs[:, 2:]], 1)
    return Ref(y, bound, unit, U * y.abs())


# ---- the check ----------------------------------------------------------------------------------------------------
def error_stats(got, ref):
    """-> {"ratio": max |y - y64| / bound, "rms": the aggregate ratio} of a kernel result `got` (ref.y's shape)"""
    err = (got.to(ref.y.device, torch.float64) - ref.y).abs()
    if err.numel() == 0:
        return {"ratio": 0.0, "rms": 0.0}
    ratio = torch.where(err == 0, torch.zeros_like(err), err / ref.bound)
    excess = (err - ref.rest).clamp_min(0.0)
    den = float(ref.unit.pow(2).mean().sqrt())
    num = float(excess.pow(2).mean().sqrt())
    rms = num / den if den > 0 else (0.0 if num == 0.0 else float("inf"))
    return {"ratio": float(ratio.max()), "rms": rms}


def assert_accurate(got, ref, what=""):
    st = error_stats(got, ref)
    assert st["ratio"] <= 1.0, "%s: |y - y64| reaches %.3g x the bound" % (what, st["ratio"])
    assert st["rms"] <= RHO, "%s: rms error %.3g x rms(|s| S1), above RHO = %.3g" % (what, st["rms"], RHO)
    return st


def assert_rejected(got, ref, what=""):
    st = error_stats(got, ref)
    assert not (st["ratio"] <= 1.0 and st["rms"] <= RHO), "%s: a simulated fault passes the check (%r)" % (what, st)
    return st

#!/usr/bin/env python
"""How many member-tiles of a dense grid query an fp32 absorption certificate could skip, predicted on the CPU.

The ensemble kernel blends in member order, num = fmaf(w_k, s_k, num) and den += w_k (DESIGN 4.1).  A member whose weight
is tiny but not zero leaves both sums bit for bit unchanged when, at every valid point of a tile,
  den_{k-1} + w_k == den_{k-1} in fp32                       (den half), and
  w_k * B_k < ulp(L) / 4,  L <= |num_{k-1}|,  B_k >= |s_k|   (num half: fmaf returns num_{k-1}).
Skipping such a member is exact.  This tool counts, for the seeded head of bench.py, the member-tiles that survive the
zero-weight skip and the ones the certificate would remove on top:
  * den half: the in-order fp32 partial sums of the weights (absorbed members do not change them);
  * B_k: a float64 interval bound of member k's output over the grid box (layer 0 with the latent folded, softplus with
    beta = 100, the latent-dependent layer-2 constant, the output layer), every pre-activation widened by a relative and an
    absolute slack, and at least 1 (quirk points blend 1.0);
  * L: what a kernel can know when it decides on member k.  Two rules:
    - per point (the kernel): at every valid point p with w_k(p) != +0, w_k(p) * B_k < ulp(L(p)) / 4 with
      L(p) = |num(p)| after the member two evaluated positions earlier minus w(p) * B of the member evaluated in between,
      rounded down (fp32 with directed rounding, as the kernel computes it); B_k finite; the first two evaluated members of
      a tile are never certified (keys absorbed_point, evaluated_point);
    - tile-wide (the kernel before per-point): the minimum of |num| over the tile after the member two evaluated positions
      earlier, minus max_w * B of the member evaluated in between (max_w rounded up to a power of two), paired with the
      tile's largest weight (keys absorbed, evaluated_absorb);
    - member by member (the kernel's dense grid queries): per point with L(p) = |num(p)| after member k - 1, no lag, and
      B_k of the point's 32^3-point sub-box of the grid (the box of its grid indices 32 c .. 32 c + 31 per axis); a (point,
      member) pair is evaluated when w != +0, the point is not a quirk row (it blends 1.0 without the network) and the
      certificate fails; member k's pairs run in ceil(n_k / 128) tiles (keys compact_pairs per member, compact_tiles;
      compact_pairs_box, compact_tiles_box with the whole-box B_k).
num and den come from the fp32 member outputs of the CPU reference (tests/ensemble_f64_common.py).

    python tools/absorbed_member_tiles.py [--latent 1] [--res 64] [--scale 1] [--plane-stride 1] [--quirk-period 0] [--compact]

replay() is the per-point rule over a batch of tiles in torch (any device): predict() runs it on its own decisions, and
tests/test_gpu_ensemble_absorb_replay.py on the decisions the kernel logged, with the kernel's weights, bounds and masks.
fold_consts() restates how the GPU folds the latent into the layer constants, so that member_bound can take the inputs the
kernel's bound has.

Every certified member is checked against the fp32 blend: the tool stops if one would change a bit of num or den.  It also
prints what better-informed inputs would certify: L without the lag (tile-wide and per point), with the tile's own max |s_k|
for B_k, and the members that change no bit at all (what no certificate can exceed).
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

# slack of the member-output bound against what the kernel computes (3-pass fp16 products with fp32 accumulation, softplus
# in log2 units with a polynomial lg2): every pre-activation interval grows by REL_SLACK * (|W| |h| + |b|) + ABS_SLACK
REL_SLACK = 2.0 ** -10
ABS_SLACK = 2.0 ** -10


def softplus64(x):
    """Softplus(beta=100, threshold=20) in float64, monotone."""
    bx = 100.0 * x
    return np.where(bx > 20.0, x, np.log1p(np.exp(np.minimum(bx, 20.0))) / 100.0)


def member_bound(P, m, z, anc, lo, hi, consts=None):
    """B >= |s_m(x)| for every x in the box [lo, hi] (3,), as the kernel computes s_m: float64 interval propagation in
    centre / radius form with REL_SLACK and ABS_SLACK per layer, at least 1.  inf when the bound is not finite.  consts: the
    per-layer constants (latent folded, fold_consts) in place of the float64 fold - the inputs member_bound_kernel has."""
    from ensemble_f64_common import SQRT2
    s = P.weight_set(m)
    layers = [(W[s].double().numpy(), b[s].double().numpy()) for W, b in P.layers]
    z = z.double().numpy()
    cond = np.concatenate([z[:P.G], z[P.G + m * P.L:P.G + (m + 1) * P.L]])
    a = anc[m] if m < P.n_loc else np.zeros(3)
    xl, xh = np.asarray(lo, np.float64) - a, np.asarray(hi, np.float64) - a
    if P.mirrored(m):
        xl, xh = xl.copy(), xh.copy()
        xl[0], xh[0] = -xh[0], -xl[0]
    xc, xr = (xl + xh) / 2, (xh - xl) / 2
    skip = P.n_layers // 2
    hc, hr = xc, xr
    with np.errstate(over='ignore', invalid='ignore'):
        for l, (W, b) in enumerate(layers):
            if l == 0:
                Wx, bias = W[:, :3], W[:, 3:] @ cond + b
            elif l == skip:
                n_h = hc.shape[0]
                Wx = W[:, :n_h + 3] / SQRT2
                bias = W[:, n_h + 3:] @ cond / SQRT2 + b
                hc, hr = np.concatenate([hc, xc]), np.concatenate([hr, xr])
            else:
                Wx, bias = W, b
            if consts is not None:
                bias = np.asarray(consts[l], np.float64)
            c = Wx @ hc + bias
            r = np.abs(Wx) @ hr + REL_SLACK * (np.abs(Wx) @ (np.abs(hc) + hr) + np.abs(bias)) + ABS_SLACK
            if l + 1 < len(layers):
                lo_, hi_ = softplus64(c - r), softplus64(c + r)
                hc, hr = (lo_ + hi_) / 2, (hi_ - lo_) / 2
            else:
                B = float(np.abs(c[0]) + r[0])
    return max(B, 1.0) if np.isfinite(B) else float('inf')


def pow2_above(x):
    """The smallest power of two strictly above x > 0 (float32 exponent field + 1), as the kernel stores a weight bound."""
    e = np.floor(np.log2(x.astype(np.float64)))
    return np.exp2(e + 1)


def ulp32(x):
    """ulp of positive normal float32 values x (float64 result)."""
    x = np.asarray(x, np.float32)
    return (np.nextafter(x, np.float32(np.inf)) - x).astype(np.float64)


def f32_up(x):
    """float64 -> the smallest float32 >= x."""
    x = np.asarray(x, np.float64)
    f = x.astype(np.float32)
    return np.where(f.astype(np.float64) < x, np.nextafter(f, np.float32(np.inf)), f)


def f32_down(x):
    """float64 -> the largest float32 <= x."""
    x = np.asarray(x, np.float64)
    f = x.astype(np.float32)
    return np.where(f.astype(np.float64) > x, np.nextafter(f, np.float32(-np.inf)), f)


def fmul_ru(a, b):
    """__fmul_ru of float32 operands: the product is exact in float64 (24 + 24 significant bits, no float64 underflow)."""
    with np.errstate(invalid='ignore', over='ignore'):
        return f32_up(np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64))


def fsub_rd(a, b):
    """__fsub_rd of float32 operands: the float64 difference plus its exact error (TwoSum) gives the float64 round-down,
    and rounding that down to float32 is the float32 round-down of the exact difference."""
    a = np.asarray(a, np.float32).astype(np.float64)
    b = -np.asarray(b, np.float32).astype(np.float64)
    with np.errstate(invalid='ignore', over='ignore'):
        s = a + b
        bb = s - a
        err = (a - (s - bb)) + (b - bb)
        s = np.where(np.isfinite(s) & (err < 0), np.nextafter(s, -np.inf), s)
    return f32_down(s)


def point_pass(w, B, pub, lag, valid):
    """The per-point rule of the kernel at each point (vectorised, float32 inputs): invalid points and w = +0 pass;
    otherwise L = pub - lag rounded down must be >= 2^-100 and w * B rounded up < 2^(e(L) - 25) = ulp(L) / 4 (2^103 for
    L = +inf).  pub = |num| two evaluated positions back, lag = w * B of the member in between rounded up, B = B_k as
    float32."""
    w = np.asarray(w, np.float32)
    L = fsub_rd(pub, lag)
    e = (L.view(np.uint32) >> 23).astype(np.int64) & 0xff
    thr = np.ldexp(1.0, e - 152)
    with np.errstate(invalid='ignore'):
        ok = (L >= np.float32(2.0 ** -100)) & (fmul_ru(w, B).astype(np.float64) < thr)
    return ~np.asarray(valid, bool) | (w == 0) | ok


def fmaf32(a, b, c):
    """fp32 fmaf(a, b, c), correctly rounded: a * b is exact in float64 and TwoSum gives the error e of s = a * b + c, which
    decides the one case where rounding s to float32 differs from rounding the exact sum (s halfway between two float32)."""
    a, b, c = (np.asarray(t, np.float32).astype(np.float64) for t in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    f = s.astype(np.float32)
    fd = f.astype(np.float64)
    up = np.nextafter(f, np.float32(np.inf))
    dn = np.nextafter(f, np.float32(-np.inf))
    f = np.where((s == (fd + up.astype(np.float64)) / 2) & (e > 0), up, f)
    return np.where((s == (fd + dn.astype(np.float64)) / 2) & (e < 0), dn, f)


def fold_consts(P32, z, m):
    """The per-layer constants of member m as the GPU folds the latent into them (csrc/simt.cu cvec_kernel, fp32): for
    layer 0 and the skip layer, fmaf(scale, sum_j W[n, K + j] u_j, b[n]) with the sum taken per lane of a warp (j = lane,
    lane + 32, ... by fmaf) and reduced by the xor butterfly; the other layers' biases.  float32 arrays, one per layer."""
    s_ = P32.weight_set(m)
    zz = z.float().numpy()
    u = np.concatenate([zz[:P32.G], zz[P32.G + m * P32.L:P32.G + (m + 1) * P32.L]]).astype(np.float32)
    C = u.shape[0]
    skip = P32.n_layers // 2
    out = []
    for l, (W, b) in enumerate(P32.layers):
        W, b = W[s_].float().numpy(), b[s_].float().numpy()
        if l not in (0, skip):
            out.append(b)
            continue
        Wc = W[:, W.shape[1] - C:]
        lanes = np.zeros((W.shape[0], 32), np.float32)
        for j0 in range(0, C, 32):
            n = min(32, C - j0)
            lanes[:, :n] = fmaf32(Wc[:, j0:j0 + n], u[None, j0:j0 + n], lanes[:, :n])
        for o in (16, 8, 4, 2, 1):
            lanes = lanes + lanes[:, np.arange(32) ^ o]
        scale = np.float32(1.0) if l == 0 else np.float32(1.0 / np.sqrt(2.0))
        out.append(fmaf32(lanes[:, 0], scale, b))
    return out


# ------------------------------------------------------------------------------------------------ replay of the per-point rule
# The producer's decisions, tile by tile, as torch tensors on any device (float64 arithmetic for the directed roundings).
def _t_f32_up(x):
    f = x.float()
    return torch_mod().where(f.double() < x, torch_mod().nextafter(f, f.new_tensor(float('inf'))), f)


def _t_f32_down(x):
    f = x.float()
    return torch_mod().where(f.double() > x, torch_mod().nextafter(f, f.new_tensor(float('-inf'))), f)


def torch_mod():
    import torch
    return torch


def t_fmul_ru(a, b):
    """__fmul_ru of float32 tensors (the product is exact in float64)."""
    return _t_f32_up(a.double() * b.double())


def t_fsub_rd(a, b):
    """__fsub_rd of float32 tensors (TwoSum in float64, then the float32 round-down), as fsub_rd."""
    torch = torch_mod()
    a, b = a.double(), -b.double()
    s = a + b
    bb = s - a
    err = (a - (s - bb)) + (b - bb)
    s = torch.where(torch.isfinite(s) & (err < 0), torch.nextafter(s, s.new_tensor(float('-inf'))), s)
    return _t_f32_down(s)


def t_point_pass(w, B, pub, lag, valid):
    """point_pass on float32 tensors: invalid points and w = +0 pass; else L = pub - lag (rounded down) >= 2^-100 and
    w * B (rounded up) < ulp(L) / 4 = 2^(e(L) - 25)."""
    torch = torch_mod()
    L = t_fsub_rd(pub, lag)
    e = (L.view(torch.int32) >> 23) & 0xff
    thr = torch.ldexp(torch.ones_like(L, dtype=torch.float64), (e - 152).double())
    ok = (L >= 2.0 ** -100) & (t_fmul_ru(w, B).double() < thr)
    return ~valid | (w == 0) | ok


# relative error of the kernel's blend weight against the replay's (expf: 2 ulp; the squared distance, its root and the
# quotient each round with 2^-24 relative and may contract differently; the exponent's absolute error is |ln w| times that)
W_REL = 2.0 ** -20


def replay(W, S, V, mask, amask, B32, follow=None, s_err=None):
    """The producer warpgroup's per-point decisions over a batch of tiles (DESIGN 4.1), replayed in torch.

    W, S: T x 128 x M float32 blend weights and member outputs (1.0 at quirk rows); V: T x 128 valid rows; mask: T x M the
    tile's members (pre-pass); amask: T x M its den-absorbed members; B32: M float32 bounds (+inf: never a candidate).
    follow: T x M members the kernel skipped; when given, they (not the replay's own verdicts) drive num, the two published
    |num| and the lag, so that every verdict is the rule applied to the state the kernel had.  s_err: T x 128 x M bound on
    |s_kernel - S| (default 0).  Returns dict of T x M bool: cand (a candidate: in both masks, finite B, two members of the
    tile evaluated before it), skip (the rule on the replay's state), sure_skip / sure_keep (the verdict under every w, s and
    num within the rounding differences between the replay and the kernel: w within W_REL (1 + |ln w|) relative, num within
    the accumulated sum of w |ds| + ulp(|num|) per member evaluated), and margin: T x M float64, the smallest
    (ulp(L) / 4 - w B) / (ulp(L) / 4) over the tile's deciding points (nan where no point decides)."""
    torch = torch_mod()
    T, R, M = W.shape
    dev = W.device
    f32 = torch.float32
    num = torch.zeros(T, R, dtype=f32, device=dev)
    dn = torch.zeros(T, R, dtype=torch.float64, device=dev)            # bound on |num_kernel - num|
    pp = [torch.zeros(T, R, dtype=f32, device=dev)] * 2
    pd = [torch.zeros(T, R, dtype=torch.float64, device=dev)] * 2
    lag = torch.zeros(T, R, dtype=f32, device=dev)
    lag_w = torch.zeros(T, R, dtype=torch.float64, device=dev)        # relative error bound of the lag's weight
    npos = torch.zeros(T, dtype=torch.int64, device=dev)
    out = {k: torch.zeros(T, M, dtype=torch.bool, device=dev) for k in ('cand', 'skip', 'sure_skip', 'sure_keep')}
    out['margin'] = torch.full((T, M), float('nan'), dtype=torch.float64, device=dev)
    inf = float('inf')
    for k in range(M):
        w, s = W[:, :, k], S[:, :, k]
        Bk = B32[k].reshape(1, 1).expand(T, R).float()
        ew = torch.where(w > 0, W_REL * (1.0 - torch.log(w.double().clamp_min(1e-45))), torch.zeros_like(dn))
        cand = mask[:, k] & amask[:, k] & bool(torch.isfinite(B32[k])) & (npos >= 2)
        ok = t_point_pass(w, Bk, pp[0], lag, V)
        w_hi, w_lo = _t_f32_up(w.double() * (1 + ew)), _t_f32_down(w.double() * (1 - ew))
        lag_hi, lag_lo = _t_f32_up(lag.double() * (1 + lag_w)), _t_f32_down(lag.double() * (1 - lag_w))
        pub_lo = _t_f32_down((pp[0].double() - pd[0]).clamp_min(0.0))
        pub_hi = _t_f32_up(pp[0].double() + pd[0])
        ok_pes = t_point_pass(w_hi, Bk, pub_lo, lag_hi, V)
        ok_opt = t_point_pass(w_lo, Bk, pub_hi, lag_lo, V)
        out['cand'][:, k] = cand
        out['skip'][:, k] = cand & ok.all(dim=1)
        out['sure_skip'][:, k] = cand & ok_pes.all(dim=1)
        out['sure_keep'][:, k] = ~cand | ~ok_opt.all(dim=1)
        L = t_fsub_rd(pp[0], lag)
        e = (L.view(torch.int32) >> 23) & 0xff
        thr = torch.ldexp(torch.ones_like(L, dtype=torch.float64), (e - 152).double())
        rel = (thr - t_fmul_ru(w, Bk).double()) / thr
        rel = torch.where(V & (w != 0) & (L >= 2.0 ** -100), rel, torch.full_like(rel, inf))
        mn = rel.min(dim=1).values
        out['margin'][:, k] = torch.where(cand & torch.isfinite(mn), mn, out['margin'][:, k])
        skipped = out['skip'][:, k] if follow is None else follow[:, k]
        ev = (mask[:, k] & ~skipped)[:, None]
        new = (w.double() * s.double() + num.double()).float()
        err = w.double() * (s_err[:, :, k].double() if s_err is not None else 0.0)
        dn_new = dn + err + (torch.nextafter(new.abs(), new.new_tensor(inf)) - new.abs()).double()
        num = torch.where(ev, new, num)
        dn = torch.where(ev, dn_new, dn)
        pp = [torch.where(ev, pp[1], pp[0]), torch.where(ev, num.abs(), pp[1])]
        pd = [torch.where(ev, pd[1], pd[0]), torch.where(ev, dn, pd[1])]
        lag = torch.where(ev, t_fmul_ru(w, Bk), lag)
        lag_w = torch.where(ev, ew, lag_w)
        npos += ev[:, 0].long()
    return out


def absorbable(den, w, num_lo, wmax_bound, B):
    """The certificate (vectorised): den + w == den in float32, and wmax_bound * B < ulp(num_lo) / 4 with num_lo a lower
    bound of |num| (float64), wmax_bound >= w and B >= |s|.  When it holds, fmaf(w, s, num) == num and den + w == den."""
    den, w = np.asarray(den, np.float32), np.asarray(w, np.float32)
    return ((den + w) == den) & num_half(np.asarray(num_lo, np.float64), np.float64(wmax_bound), B)


def grid_setup(latent_seed, scale=1.0):
    import torch
    from conftest import make_ensemble, sample_latent
    from ensemble_f64_common import Params, anchors
    dec = make_ensemble(0, scale=scale).eval()
    z = sample_latent(latent_seed).reshape(-1)
    P32, P64 = Params(dec, torch.float32), Params(dec, torch.float64)
    with torch.no_grad():
        anc32 = anchors(P32, z)
    return P32, P64, z, anc32


def predict(latent_seed=1, res=64, scale=1.0, mini=None, maxi=None, plane_stride=1, chunk_tiles=1024, quirk_period=0,
            tile='auto', planes=None):
    """dict of member-tile counts on the res^3 grid with the kernel's dense tiles (with plane_stride > 1: on the tiles of
    every plane_stride-th x-plane).  quirk_period > 0: the eval-mode query's quirk rows (grid index g % period == period - 1
    and the last point of the grid) blend 1.0 for every member, as in the kernel.  tile: as in zero_member_tiles.tile_layout
    for the whole grid.  planes = (x0, x1): only the tiles of x-planes x0 .. x1 - 1 of that layout; a block shape must not
    cross x0 or x1, so that the counts are those of the whole-grid query on these planes."""
    import torch
    from conftest import MAXI, MINI
    from ensemble_f64_common import members
    from zero_member_tiles import tile_layout, tile_points
    mini = MINI if mini is None else mini
    maxi = MAXI if maxi is None else maxi
    P32, P64, z, anc32 = grid_setup(latent_seed, scale)
    M = P32.M
    anc_np = anc32.numpy().astype(np.float32)
    axes = [np.linspace(mini[a], maxi[a], res).astype(np.float32) for a in range(3)]
    lo = np.array([axes[a].min() for a in range(3)], np.float64)
    hi = np.array([axes[a].max() for a in range(3)], np.float64)
    B = np.array([member_bound(P64, m, z, anc_np.astype(np.float64), lo, hi) for m in range(M)])
    count = res ** 3
    kind, block = tile_layout(res, 0, count, tile)
    ix, iy, iz, valid = tile_points(res, 0, count, kind, block)
    if planes is not None:
        x0, x1 = planes
        assert kind == 'blocked' and x0 % block[0] == 0 and x1 % block[0] == 0, 'planes must be whole blocks deep'
        keep = (ix[:, 0] >= x0) & (ix[:, 0] < x1)
        ix, iy, iz, valid = ix[keep], iy[keep], iz[keep], valid[keep]
    if plane_stride > 1:
        # a sample of the grid: the tiles of every plane_stride-th x-plane (a dense tile never crosses a plane)
        keep = ix[:, 0] % plane_stride == 0
        ix, iy, iz, valid = ix[keep], iy[keep], iz[keep], valid[keep]
    n_tiles = ix.shape[0]
    stats = {'tiles': int(n_tiles), 'member_tiles': int(n_tiles * M), 'zero': 0, 'den_absorbed': 0, 'absorbed': 0,
             'absorbed_no_lag': 0, 'absorbed_tile_max': 0, 'unchanged': 0, 'B': B,
             'absorbed_point': 0, 'absorbed_point_no_lag': 0, 'compact_pairs': np.zeros(M, np.int64),
             'compact_pairs_box': np.zeros(M, np.int64)}
    B32 = f32_up(B)                                     # the kernel's B_k (member_bound_kernel rounds up; inf stays inf)
    # B_k per 32^3-point sub-box (member by member): [member][sx][sy][sz]
    n_sub = (res + 31) // 32
    sub_lo = [[axes[a][32 * c:32 * c + 32].min() for c in range(n_sub)] for a in range(3)]
    sub_hi = [[axes[a][32 * c:32 * c + 32].max() for c in range(n_sub)] for a in range(3)]
    B32_sub = np.zeros((M, n_sub, n_sub, n_sub), np.float32)
    for m in range(M):
        for cx in range(n_sub):
            for cy in range(n_sub):
                for cz in range(n_sub):
                    lo_s = np.array([sub_lo[0][cx], sub_lo[1][cy], sub_lo[2][cz]], np.float64)
                    hi_s = np.array([sub_hi[0][cx], sub_hi[1][cy], sub_hi[2][cz]], np.float64)
                    B32_sub[m, cx, cy, cz] = f32_up(member_bound(P64, m, z, anc_np.astype(np.float64), lo_s, hi_s))
    gw = np.float32(np.exp(np.float32(-0.2) / np.float32(0.01)))
    for t0 in range(0, n_tiles, chunk_tiles):
        sl = slice(t0, min(n_tiles, t0 + chunk_tiles))
        X = np.stack([axes[0][ix[sl]], axes[1][iy[sl]], axes[2][iz[sl]]], axis=-1)       # T x 128 x 3
        V = valid[sl]
        T = X.shape[0]
        pts = torch.from_numpy(X.reshape(-1, 3))
        with torch.no_grad():
            S = members(P32, pts, z, anc32).numpy().reshape(T, 128, M)
        Q = np.zeros((T, 128), bool)
        if quirk_period > 0:
            g = (ix[sl] * res + iy[sl]) * res + iz[sl]
            Q = (g % quirk_period == quirk_period - 1) | (g == count - 1)
            S[Q] = 1.0
        with np.errstate(under='ignore'):
            d = anc_np[None, None] - X[:, :, None, :]                                       # T x 128 x 39 x 3
            d2 = np.float32(d[..., 2] * d[..., 2] + (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]))
            nrm = np.sqrt(d2) + np.float32(10e-6)
            Wt = np.exp(-(nrm * nrm) / np.float32(0.01)).astype(np.float32)
        Wt = np.concatenate([Wt, np.full((T, 128, 1), gw, np.float32)], axis=2)
        # skipped members leave num and den as they were, so the state is that of the full sequence
        num = np.zeros((T, 128), np.float32)
        den = np.zeros((T, 128), np.float32)
        pub = [np.full(T, -np.inf), np.full(T, -np.inf)]      # min |num| after the last two evaluated members (none: -inf)
        last_bound = np.zeros(T)                             # max_w * B of the last evaluated member
        inf32 = np.float32(np.inf)
        zero_all, den_all, unchanged_all = (np.zeros((T, M), bool) for _ in range(3))
        for k in range(M):
            w = Wt[:, :, k]
            zero = ~np.any(V & (w != 0), axis=1)
            den_abs = np.all(~V | ((den + w) == den), axis=1)
            wmax = np.where(V, w, 0).max(axis=1)
            wb = np.where(wmax > 0, pow2_above(np.maximum(wmax, np.float32(1e-45))), 0.0)
            mn_before = np.where(V, np.abs(num), inf32).min(axis=1).astype(np.float64)
            cert = den_abs & num_half(pub[0] - last_bound, wb, B[k]) & ~zero
            no_lag = den_abs & num_half(mn_before, wb, B[k]) & ~zero
            s = np.where(V, S[:, :, k], 0).astype(np.float64)
            # the same without lag, with the tile's own max |s_k| (at least 1) in place of B_k: what a per-tile bound could reach
            tile_b = np.maximum(np.abs(s).max(axis=1), 1.0)
            oracle = den_abs & num_half(mn_before, wb, tile_b) & ~zero
            new_num = (w.astype(np.float64) * s + num.astype(np.float64)).astype(np.float32)
            unchanged = den_abs & np.all(~V | (new_num == num), axis=1) & ~zero
            assert not np.any(cert & ~unchanged), 'the certificate passed a member that changes num'
            cand = den_abs & ~zero & np.isfinite(B32[k])
            no_lag_p = cand & np.all(point_pass(w, B32[k], np.abs(num), np.float32(0), V), axis=1)
            stats['absorbed_point_no_lag'] += int(no_lag_p.sum())
            # member by member: the exact state after member k - 1 at every point, quirk rows blended without the network
            need = V & (w != 0) & ~Q & ~(((den + w) == den) & point_pass(w, B32[k], np.abs(num), np.float32(0), V))
            stats['compact_pairs_box'][k] += int(need.sum())
            Bp = B32_sub[k][np.minimum(ix[sl], res - 1) >> 5, np.minimum(iy[sl], res - 1) >> 5, np.minimum(iz[sl], res - 1) >> 5]
            need = V & (w != 0) & ~Q & ~(((den + w) == den) & point_pass(w, Bp, np.abs(num), np.float32(0), V))
            stats['compact_pairs'][k] += int(need.sum())
            zero_all[:, k], den_all[:, k], unchanged_all[:, k] = zero, den_abs, unchanged
            stats['zero'] += int(zero.sum())
            stats['den_absorbed'] += int((den_abs & ~zero).sum())
            stats['absorbed'] += int(cert.sum())
            stats['absorbed_no_lag'] += int(no_lag.sum())
            stats['absorbed_tile_max'] += int(oracle.sum())
            stats['unchanged'] += int(unchanged.sum())
            ev = ~(zero | cert)
            num = new_num
            den = den + w
            mn = np.where(V, np.abs(num), inf32).min(axis=1).astype(np.float64)
            pub = [np.where(ev, pub[1], pub[0]), np.where(ev, mn, pub[1])]
            last_bound = np.where(ev, wb * B[k], last_bound)
        # the per-point rule (the kernel's): its own decisions drive the state
        r = replay(torch.from_numpy(Wt), torch.from_numpy(S), torch.from_numpy(V), torch.from_numpy(~zero_all),
                   torch.from_numpy(den_all), torch.from_numpy(B32.astype(np.float32)))
        cert_p = r['skip'].numpy()
        assert not np.any(cert_p & ~unchanged_all), 'the per-point rule passed a member that changes num'
        stats['absorbed_point'] += int(cert_p.sum())
    n = stats['member_tiles']
    stats['evaluated_now'] = n - stats['zero']
    stats['evaluated_absorb'] = stats['evaluated_now'] - stats['absorbed']
    stats['evaluated_point'] = stats['evaluated_now'] - stats['absorbed_point']
    stats['compact_tiles'] = int(((stats['compact_pairs'] + 127) // 128).sum())
    stats['compact_tiles_box'] = int(((stats['compact_pairs_box'] + 127) // 128).sum())
    return stats


def num_half(L, wmax_bound, B):
    """Per tile: wmax_bound * B < ulp(L) / 4 with L (float64) rounded down to float32; False where L is not a positive
    normal float32 or B is not finite."""
    ok = (L > np.finfo(np.float32).tiny) & np.isfinite(B)
    B = np.where(ok, B, 0.0)
    L = np.where(ok, L, 1.0)
    Lc = L.astype(np.float32)
    Lc = np.where(Lc.astype(np.float64) > L, np.nextafter(Lc, np.float32(0)), Lc)
    return ok & (wmax_bound * B < ulp32(Lc) / 4)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--latent', type=int, default=1)
    ap.add_argument('--res', type=int, default=64)
    ap.add_argument('--scale', type=float, default=1.0)
    ap.add_argument('--plane-stride', type=int, default=1, help='count the tiles of every n-th x-plane only (dense tiles)')
    ap.add_argument('--quirk-period', type=int, default=0, help='quirk period of the query (bench.py and ens_trace.py: 25000)')
    ap.add_argument('--tile', default='auto', help='auto or a block shape XxYxZ with X*Y*Z = 128 (zero_member_tiles.py)')
    ap.add_argument('--planes', type=int, nargs=2, metavar=('X0', 'X1'), default=None,
                    help='count the tiles of x-planes X0 .. X1-1 only (multiples of the block depth): compares layouts fairly')
    ap.add_argument('--compact', action='store_true', help='also print the member-by-member counts: pairs and compact tiles')
    args = ap.parse_args()
    r = predict(args.latent, args.res, args.scale, plane_stride=args.plane_stride, quirk_period=args.quirk_period,
                tile=args.tile, planes=args.planes)
    ev = r['evaluated_now']
    if args.plane_stride > 1:
        print('tiles of every %d-th x-plane' % args.plane_stride)
    if args.planes:
        print('tiles of x-planes %d .. %d' % (args.planes[0], args.planes[1] - 1))
    print('latent %d, %d^3 grid: %d tiles, %d member-tiles, %d evaluated with the zero-weight skip; den half holds on %d '
          '(%.1f %%), the tile-wide rule (the kernel before per-point) on %d (%.1f %%) -> %d evaluated'
          % (args.latent, args.res, r['tiles'], r['member_tiles'], ev, r['den_absorbed'], 100 * r['den_absorbed'] / ev,
             r['absorbed'], 100 * r['absorbed'] / ev, r['evaluated_absorb']))
    print('with L = min |num_{k-1}| (no lag): %d (%.1f %%); no lag and the tile max of |s_k| for B_k: %d (%.1f %%); '
          'members that change no bit of num and den: %d (%.1f %%)'
          % (r['absorbed_no_lag'], 100 * r['absorbed_no_lag'] / ev, r['absorbed_tile_max'],
             100 * r['absorbed_tile_max'] / ev, r['unchanged'], 100 * r['unchanged'] / ev))
    print('per point (the kernel): %d (%.1f %%) -> %d evaluated; per point without the lag: %d (%.1f %%)'
          % (r['absorbed_point'], 100 * r['absorbed_point'] / ev, r['evaluated_point'], r['absorbed_point_no_lag'],
             100 * r['absorbed_point_no_lag'] / ev))
    if args.compact:
        print('member by member (per point, no lag, quirk rows blended directly), whole-box B_k: %d (point, member) pairs '
              'evaluated in %d compact tiles (x%.3f fewer than per point)'
              % (r['compact_pairs_box'].sum(), r['compact_tiles_box'], r['evaluated_point'] / max(r['compact_tiles_box'], 1)))
        print('member by member, B_k per 32^3-point sub-box (the kernel): %d pairs in %d compact tiles (x%.3f fewer than '
              'per point)' % (r['compact_pairs'].sum(), r['compact_tiles'], r['evaluated_point'] / max(r['compact_tiles'], 1)))
        print('pairs per member: %s' % ' '.join(str(int(v)) for v in r['compact_pairs']))
    print('B_k: min %.3g, median %.3g, max %.3g' % (r['B'].min(), np.median(r['B']), r['B'].max()))


if __name__ == '__main__':
    main()

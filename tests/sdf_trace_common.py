"""Float64 restatement of the sphere tracer's contract (csrc/sdf_trace.cu, nphm_b200/evaluation/sdf_render.py): render.cu's pixel
rays, the box interval, and the march / bracket / refine / classify state machine, vectorised over rays in numpy."""
import numpy as np

LIVE, BRACKET, HIT, MISS, OUT_OF_STEPS, INVALID = range(6)


def pixel_rays(poses, K, rend_size):
    """World rays of every pixel of every view: (origin (V, H, W, 3), unit direction (V, H, W, 3), 1 / |d_eye| (V, H, W))."""
    H, W = rend_size
    K = np.asarray(K, np.float64)
    fx, fy, cx, cy = K[0][0], K[1][1], K[0][2], K[1][2]
    r, c = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')
    px, py = (c + 0.5 - cx) * (1.0 / fx), (cy - r - 0.5) * (1.0 / fy)
    d_eye = np.stack([px, py, -np.ones_like(px)], axis=-1)
    o, u, cos = [], [], []
    for Rt in poses:
        Rt = np.asarray(Rt, np.float64)
        d = d_eye @ Rt[:3, :3].T
        n = np.linalg.norm(d, axis=-1, keepdims=True)
        o.append(np.broadcast_to(Rt[:3, 3], d.shape))
        u.append(d / n)
        cos.append(1.0 / np.linalg.norm(d_eye, axis=-1))
    return np.stack(o), np.stack(u), np.stack(cos)


def box_interval(o, u, cos, mini, maxi, scale, znear, zfar):
    """(s_in, s_out) of rays (n, 3) inside {x : scale x in [mini, maxi]} at eye depth [znear, zfar]; a miss has s_in > s_out."""
    s_in, s_out = znear / cos, zfar / cos
    for a in range(3):
        b0, b1 = mini[a] / scale, maxi[a] / scale
        with np.errstate(divide='ignore', invalid='ignore'):
            t0, t1 = (b0 - o[:, a]) / u[:, a], (b1 - o[:, a]) / u[:, a]
        flat = u[:, a] == 0
        inside = (o[:, a] >= b0) & (o[:, a] <= b1)
        s_in = np.where(flat, s_in, np.maximum(s_in, np.minimum(t0, t1)))
        s_out = np.where(flat, np.where(inside, s_out, -1.0), np.minimum(s_out, np.maximum(t0, t1)))
    return s_in, s_out


def secant(lo, flo, hi, fhi):
    w = np.clip(flo / (flo - fhi), 0.1, 0.9)
    return lo + w * (hi - lo)


def march(field, o, u, s_in, s_out, scale=1.0, step_factor=0.6, hit_eps=5e-4, min_step=1e-4, max_steps=128, refine_steps=6,
          valid_fn=None):
    """The tracer's state machine on rays (n, 3): ``field(points (m, 3) scaled) -> f (m,)``, ``valid_fn`` the same for the posed
    search's flag (None: always valid).  Returns (status (n,), s (n,), steps (n,))."""
    n = len(s_in)
    status = np.where(s_in <= s_out, LIVE, MISS)
    s, lo, hi = s_in.copy(), s_in.copy(), s_in.copy()
    flo, fhi = np.full(n, -1.0), np.zeros(n)
    sgn = np.ones(n)                                          # the sign of f at the first sample: the march runs on sgn f
    steps = np.zeros(n, np.int64)

    def sample(idx):
        x = scale * (o[idx] + s[idx, None] * u[idx])
        return field(x), (np.ones(len(idx), bool) if valid_fn is None else valid_fn(x))

    for _ in range(max_steps):
        idx = np.nonzero(status == LIVE)[0]
        if len(idx) == 0:
            break
        f, ok = sample(idx)
        first = steps[idx] == 0
        sgn[idx[first]] = np.where(f[first] < 0, -1.0, 1.0)
        f = sgn[idx] * f
        steps[idx] += 1
        status[idx[~ok]] = INVALID
        idx, f = idx[ok], f[ok]
        br = (f < 0) & (flo[idx] > 0)
        b = idx[br]
        hi[b], fhi[b] = s[b], f[br]
        s[b] = secant(lo[b], flo[b], hi[b], fhi[b])
        status[b] = BRACKET
        hit = ~br & (f < hit_eps)
        status[idx[hit]] = HIT
        go = ~br & ~hit
        g, fg = idx[go], f[go]
        lo[g], flo[g] = s[g], fg
        s[g] = s[g] + step_factor * np.maximum(fg / scale, min_step)
        past = s[g] > s_out[g]
        status[g[past]] = MISS
        status[g[~past & (steps[g] >= max_steps)]] = OUT_OF_STEPS
    for _ in range(refine_steps):
        idx = np.nonzero(status == BRACKET)[0]
        if len(idx) == 0:
            break
        f, ok = sample(idx)
        f = sgn[idx] * f
        status[idx[~ok]] = INVALID
        idx, f = idx[ok], f[ok]
        neg = f < 0
        hi[idx[neg]], fhi[idx[neg]] = s[idx[neg]], f[neg]
        lo[idx[~neg]], flo[idx[~neg]] = s[idx[~neg]], f[~neg]
        s[idx] = secant(lo[idx], flo[idx], hi[idx], fhi[idx])
    status[status == BRACKET] = HIT
    return status, s, steps


def encode_normals(n):
    """render.cu's uint8 normal: normalise in float64, round to float32, round(clamp(0.5 n + 0.5, 0, 1) 255)."""
    n = np.asarray(n, np.float64)
    nf = (n / np.linalg.norm(n, axis=-1, keepdims=True)).astype(np.float32)
    return np.rint(np.clip(np.float32(0.5) * nf + np.float32(0.5), 0, 1).astype(np.float32) * np.float32(255)).astype(np.uint8)


def sphere(center, radius):
    c = np.asarray(center, np.float64)
    return lambda x: np.linalg.norm(x - c, axis=-1) - radius


def sphere_first_hit(o, u, center, radius, scale=1.0):
    """Closed-form first intersection (arc length) of rays with the sphere {x : |scale x - c| = radius}; NaN where they miss."""
    c = np.asarray(center, np.float64) / scale
    r = radius / scale
    oc = o - c
    b = (oc * u).sum(-1)
    disc = b * b - ((oc * oc).sum(-1) - r * r)
    with np.errstate(invalid='ignore'):
        t = -b - np.sqrt(disc)
    return np.where(disc >= 0, t, np.nan)

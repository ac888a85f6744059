"""ORACLE - test infrastructure only: an independent float64 ray caster for ``nphm_render_depth_normals`` (csrc/render.cu).

Möller–Trumbore per (triangle, pixel) pair over each triangle's screen bounding box (the whole image when a vertex lies in front
of the near plane, i.e. at eye depth < znear), vectorised over pairs with numpy.  Same camera convention as the kernel: the
world-to-eye matrix maps world points into a camera looking down -z with +y up, and pixel (r, c) samples the eye ray
``((c + 0.5 - cx)/fx, (cy - r - 0.5)/fy, -1)``; the hit's depth is its parameter along that ray (= -z_eye), kept for
``znear <= depth <= zfar``; the nearest hit wins, ties go to the lower triangle index.

Per pixel it returns the winner's depth and index, the unit fp64 face normal ``cross(v1 - v0, v2 - v0)``, the runner-up's depth
(to excuse near-ties) and the distance in pixels from the pixel centre to the nearest triangle boundary, over every triangle whose
bounding box holds the pixel (to excuse pixels whose coverage a last-bit rounding may decide).  Outside a triangle that distance
is bounded from below by the largest violated edge-line distance, which over-excuses a little near vertices.
"""
from __future__ import annotations

import numpy as np

_CHUNK = 1 << 22


def _boxes(pe, intr, H, W, znear):
    """Inclusive pixel boxes (r0, r1, c0, c1) of eye-space triangles pe (T, 3, 3); whole image when clipped by the near plane."""
    fx, fy, cx, cy = intr
    d = -pe[:, :, 2]
    clipped = (d < znear).any(axis=1)
    dd = np.where(clipped[:, None], 1.0, d)
    col = fx * pe[:, :, 0] / dd + cx - 0.5
    row = cy - fy * pe[:, :, 1] / dd - 0.5
    c0 = np.clip(np.floor(col.min(1)) - 1, 0, W - 1)
    c1 = np.clip(np.ceil(col.max(1)) + 1, 0, W - 1)
    r0 = np.clip(np.floor(row.min(1)) - 1, 0, H - 1)
    r1 = np.clip(np.ceil(row.max(1)) + 1, 0, H - 1)
    off = (col.max(1) < -1) | (col.min(1) > W) | (row.max(1) < -1) | (row.min(1) > H)
    r0 = np.where(clipped, 0, r0); r1 = np.where(clipped, H - 1, r1)
    c0 = np.where(clipped, 0, c0); c1 = np.where(clipped, W - 1, c1)
    empty = ~clipped & off
    return r0.astype(np.int64), r1.astype(np.int64), c0.astype(np.int64), c1.astype(np.int64), empty


def render_view(verts, faces, world_to_eye, intr, H, W, znear=0.1, zfar=2.0):
    """One view.  Returns a dict of (H, W) arrays: ``depth`` (0 = background), ``tri`` (-1), ``normal`` (H, W, 3; 0),
    ``second`` (runner-up depth, inf if none) and ``edge_px`` (inf where no box holds the pixel)."""
    v = np.asarray(verts, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    M = np.asarray(world_to_eye, np.float64).reshape(3, 4)
    fx, fy, cx, cy = [float(x) for x in intr]
    depth = np.zeros((H, W)); second = np.full((H, W), np.inf); tri = np.full((H, W), -1, np.int64)
    edge_px = np.full(H * W, np.inf)
    wn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    keep = np.flatnonzero(np.any(wn != 0, axis=1))                     # zero-area triangles cover nothing
    pe = (v[f[keep]] @ M[:, :3].T) + M[:, 3]                           # (T, 3, 3) eye space
    d = -pe[:, :, 2]
    alive = ~((d < znear).all(1) | (d > zfar).all(1))
    keep, pe = keep[alive], pe[alive]
    r0, r1, c0, c1, empty = _boxes(pe, (fx, fy, cx, cy), H, W, znear)
    keep, pe, r0, r1, c0, c1 = keep[~empty], pe[~empty], r0[~empty], r1[~empty], c0[~empty], c1[~empty]
    bw = c1 - c0 + 1
    counts = (r1 - r0 + 1) * bw
    hits_p, hits_d, hits_t = [], [], []
    start = 0
    while start < len(keep):
        stop = start + max(1, int(np.searchsorted(np.cumsum(counts[start:]), _CHUNK)))
        sl = slice(start, stop)
        cnt = counts[sl]
        ti = np.repeat(np.arange(start, stop), cnt)
        local = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        r = r0[ti] + local // bw[ti]
        c = c0[ti] + local % bw[ti]
        dx = (c + 0.5 - cx) / fx
        dy = (cy - r - 0.5) / fy
        D = np.stack([dx, dy, -np.ones_like(dx)], axis=1)
        P0, P1, P2 = pe[ti, 0], pe[ti, 1], pe[ti, 2]
        e1, e2 = P1 - P0, P2 - P0
        h = np.cross(D, e2)
        a = np.einsum('ij,ij->i', e1, h)
        ok = a != 0
        inv = np.where(ok, 1.0 / np.where(ok, a, 1.0), 0.0)
        s = -P0
        u = inv * np.einsum('ij,ij->i', s, h)
        q = np.cross(s, e1)
        w = inv * np.einsum('ij,ij->i', D, q)
        t = inv * np.einsum('ij,ij->i', e2, q)
        hit = ok & (u >= 0) & (w >= 0) & (u + w <= 1) & (t >= znear) & (t <= zfar)
        # signed pixel distance of the centre to the three edge lines (positive inside): boundary distance of the pair
        det = np.einsum('ij,ij->i', P0, np.cross(P1, P2))
        sd = []
        for A, B in ((P0, P1), (P1, P2), (P2, P0)):
            n = np.cross(A, B)
            val = np.einsum('ij,ij->i', n, D) * np.sign(det)
            sd.append(val / np.maximum(np.hypot(n[:, 0] / fx, n[:, 1] / fy), 1e-300))
        sd = np.stack(sd, axis=1)
        bd = np.where((sd >= 0).all(1), sd.min(1), np.where(sd < 0, -sd, 0).max(1))
        pix = r * W + c
        np.minimum.at(edge_px, pix, bd)
        hits_p.append(pix[hit]); hits_d.append(t[hit]); hits_t.append(keep[ti[hit]])
        start = stop
    if hits_p:
        p, dd, tt = np.concatenate(hits_p), np.concatenate(hits_d), np.concatenate(hits_t)
        order = np.lexsort((tt, dd, p))
        p, dd, tt = p[order], dd[order], tt[order]
        first = np.r_[True, p[1:] != p[:-1]]
        fi = np.flatnonzero(first)
        depth.reshape(-1)[p[fi]] = dd[fi]
        tri.reshape(-1)[p[fi]] = tt[fi]
        nxt = fi + 1
        has2 = (nxt < len(p)) & (p[np.minimum(nxt, len(p) - 1)] == p[fi])
        second.reshape(-1)[p[fi[has2]]] = dd[nxt[has2]]
    normal = np.zeros((H, W, 3))
    fg = tri >= 0
    n = wn[tri[fg]]
    normal[fg] = n / np.linalg.norm(n, axis=1, keepdims=True)
    return {'depth': depth, 'tri': tri, 'normal': normal, 'second': second, 'edge_px': edge_px.reshape(H, W)}


def render(verts, faces, world_to_eye, intrinsics, H, W, znear=0.1, zfar=2.0):
    """V views: world_to_eye (V, 3, 4), intrinsics (V, 4) -> dict of (V, H, W[, 3]) arrays."""
    views = [render_view(verts, faces, M, k, H, W, znear, zfar) for M, k in zip(world_to_eye, intrinsics)]
    return {key: np.stack([r[key] for r in views]) for key in views[0]}


def quantize_normals(normal):
    """The kernel's (and shaders/mesh.frag's) uint8 encoding of unit normals: round(clamp(0.5 n + 0.5, 0, 1) * 255) in fp32."""
    nf = np.asarray(normal).astype(np.float32)
    return np.rint(np.clip(np.float32(0.5) * nf + np.float32(0.5), 0, 1) * np.float32(255)).astype(np.uint8)

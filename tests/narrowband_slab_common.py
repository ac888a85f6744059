"""Numpy restatement of one x-slab of the narrow band (``nphm_band_slab_*`` in csrc/narrowband.cu, DESIGN §4.16), with the
interface of ``nphm_b200._native.NarrowBand``, so that the real host driver (``nphm_b200.utils.reconstruction``) runs on it
without a GPU.  "Gathering" a voxel yields its global flat index; the tests evaluate it by reading a dense volume, as oracle/band_oracle.py
does for the whole grid."""
import numpy as np
import torch

IDLE, WANTED, DONE = 0, 1, 2


def _side(v):
    return v >= 0


class OracleSlab:
    def __init__(self, res, block, l0, l1):
        self.res, self.block, self.l0, self.l1 = int(res), int(block), int(l0), int(l1)
        B, C = self.block, self.res - 1
        self.nb = -(-C // B)
        assert 0 <= l0 < l1 <= self.nb
        self.x0, self.x1 = l0 * B, min(l1 * B, C)
        self.ghost = l0 > 0
        self.first_plane = self.x0 - int(self.ghost)
        self.n_planes = self.x1 + 1 - self.first_plane
        self.plane_bytes = 5 * self.res * self.res
        self.device = torch.device('cpu')
        self.active_blocks = 0

    # -- geometry: global plane x -> local plane of the marks (from x0) and of the volume (from first_plane)
    def _own(self, vol):
        return vol.numpy()[int(self.ghost):]

    def _box(self, bx, by, bz):
        B, C = self.block, self.res - 1
        lo = [b * B for b in (bx, by, bz)]
        hi = [min(v + B, C) for v in lo]
        return lo, hi

    def _local_box(self, bx, by, bz):
        lo, hi = self._box(bx, by, bz)
        return (slice(lo[0] - self.x0, hi[0] - self.x0 + 1), slice(lo[1], hi[1] + 1), slice(lo[2], hi[2] + 1))

    def _blocks(self):
        for i in range(self.l1 - self.l0):
            for by in range(self.nb):
                for bz in range(self.nb):
                    yield i, self.l0 + i, by, bz

    def _compact(self):
        flat = self.marks.reshape(-1)
        self.list = np.nonzero(flat == WANTED)[0]
        flat[self.list] = DONE
        return len(self.list)

    def _mark(self):
        for i, bx, by, bz in self._blocks():
            if self.states[i, by, bz] == 1:
                box = self.marks[self._local_box(bx, by, bz)]
                box[box == IDLE] = WANTED
                self.states[i, by, bz] = 2
                self.active_blocks += 1
        return self._compact()

    # -- the steps
    def begin(self, quirk_period=0):
        r = self.res
        self.marks = np.zeros((self.x1 - self.x0 + 1, r, r), np.uint8)
        self.states = np.zeros((self.l1 - self.l0, self.nb, self.nb), np.uint8)
        self.active_blocks = 0
        if quirk_period:
            g = np.union1d(np.arange(quirk_period - 1, r ** 3, quirk_period), [r ** 3 - 1])
            g = g[(g >= self.x0 * r * r) & (g < (self.x1 + 1) * r * r)]
            self.marks.reshape(-1)[g - self.x0 * r * r] = WANTED
            B, C = self.block, r - 1
            for x, y, z in zip(*np.unravel_index(g, (r, r, r))):
                rng = [range(max(c - 1, 0) // B, min(c, C - 1) // B + 1) for c in (x, y, z)]
                for bx in rng[0]:
                    if self.l0 <= bx < self.l1:
                        for by in rng[1]:
                            for bz in rng[2]:
                                self.states[bx - self.l0, by, bz] = 1
        return self._compact()

    def corners(self):
        ci = np.minimum(np.arange(self.nb + 1) * self.block, self.res - 1)
        cx = ci[self.l0:self.l1 + 1] - self.x0
        sub = self.marks[np.ix_(cx, ci, ci)]
        self.marks[np.ix_(cx, ci, ci)] = np.where(sub == IDLE, WANTED, sub)
        return self._compact()

    def classify(self, tau, vol):
        v = self._own(vol)
        tau = np.float32(tau)
        for i, bx, by, bz in self._blocks():
            if self.states[i, by, bz]:
                continue
            lo, hi = self._box(bx, by, bz)
            c = np.array([v[x - self.x0, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])], np.float32)
            n_in = int(_side(c).sum())
            if np.any(~(np.abs(c) > tau)) or (n_in != 0 and n_in != 8):
                self.states[i, by, bz] = 1
        return self._mark()

    def grow(self, vol):
        v = self._own(vol)
        for i, bx, by, bz in self._blocks():
            if self.states[i, by, bz]:
                continue
            box = self._local_box(bx, by, bz)
            s0 = _side(v[box][0, 0, 0])
            if np.any((self.marks[box] == DONE) & (_side(v[box]) != s0)):
                self.states[i, by, bz] = 1
        return self._mark()

    def gather(self, n, mini, maxi):
        return torch.from_numpy(self.list[:n] + self.x0 * self.res * self.res)

    def scatter(self, values, vol):
        self._own(vol).reshape(-1)[self.list[:len(values)]] = values.numpy()

    def fill(self, vol):
        v = self._own(vol)
        B, r = self.block, self.res
        f = np.minimum(np.arange(r) // B, self.nb - 1) * B
        fx = f[self.x0:self.x1 + 1] - self.x0
        corner = v[np.ix_(fx, f, f)]
        v[...] = np.where(self.marks == DONE, v, corner)

    def block_states(self):
        return torch.from_numpy(self.states != 0)

    def volume(self):
        return torch.zeros(self.n_planes, self.res, self.res, dtype=torch.float32)

    def export(self, plane, vol):
        assert self.x0 <= plane <= self.x1
        p = plane - self.x0
        vals = np.ascontiguousarray(self._own(vol)[p], np.float32).view(np.uint8).reshape(-1)
        done = (self.marks[p] == DONE).astype(np.uint8).reshape(-1)
        return torch.from_numpy(np.concatenate([vals, done]))

    def import_(self, plane, buf, vol):
        r2 = self.res * self.res
        b = buf.numpy()
        vals = b[:4 * r2].view(np.float32).reshape(self.res, self.res)
        if plane == self.x0 - 1 and self.ghost:
            vol.numpy()[0] = vals
            return
        assert (plane == self.x0 and self.l0 > 0) or (plane == self.x1 and self.x1 < self.res - 1)
        done = b[4 * r2:].reshape(self.res, self.res).astype(bool)
        p = plane - self.x0
        take = done & (self.marks[p] != DONE)
        self.marks[p][take] = DONE
        self._own(vol)[p][take] = vals[take]


def oracle_slabs(res, block, world):
    from nphm_b200.utils.reconstruction import plan_block_slabs
    return [None if l1 <= l0 else OracleSlab(res, block, l0, l1) for l0, l1 in plan_block_slabs(res, block, world)]


def oracle_slab_mc(vol_full):
    """CPU stand-ins for marching_cubes_count / emit with the slab semantics of the CUDA kernels (negate = True): the oracle's
    sequential marching cubes on the planes up to the slab, keeping the part the slab's own cell layers add."""
    from oracle import nphm_oracle as O

    def count(vol, iso, negate, x_global0=0, ghost_lo=False):
        upto = x_global0 + vol.shape[0]
        assert np.array_equal(vol.numpy(), vol_full[x_global0:upto])       # the slab volume is the whole grid's, ghost included
        v_all, t_all = O.marching_cubes(vol_full[:upto], iso, negate)
        first_own = x_global0 + (1 if ghost_lo else 0)
        if first_own > 0:
            v_prev, t_prev = O.marching_cubes(vol_full[:first_own + 1], iso, negate)
        else:
            v_prev, t_prev = np.zeros((0, 3)), np.zeros((0, 3), np.uint64)
        return len(v_all) - len(v_prev), len(t_all) - len(t_prev), (v_all[len(v_prev):], t_all[len(t_prev):], len(v_prev)), None

    def emit(vol, params, ws, nv, nt, base):
        own_v, own_t, n_prev = params
        assert base == n_prev
        return torch.from_numpy(own_v.copy()), torch.from_numpy(own_t.astype(np.int64))

    return count, emit

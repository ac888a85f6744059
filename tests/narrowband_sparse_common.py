"""Numpy restatement of the block-sparse narrow band (``nphm_band_sparse_*`` in csrc/narrowband_sparse.cu, DESIGN §4.17) with the
interface of ``nphm_b200._native.SparseNarrowBand``, so that the real host driver (``nphm_b200.utils.reconstruction``) runs on it
without a GPU.  The storage is the kernels': per block a state and a brick slot, per block corner a value and a mark, a brick of
(B+1)^3 values and marks per allocated block, the planes a neighbour sent and the ghost plane; lists hold brick-local indices
(slot (B+1)^3 + local) or corner indices.  "Gathering" a voxel yields its global flat index, which the tests evaluate by reading
a dense volume, as narrowband_slab_common.py does."""
import numpy as np
import torch

IDLE, WANTED, DONE = 0, 1, 2
INACTIVE, ACTIVATED, MARKED, FORCED = 0, 1, 2, 3
NO_SLOT = -1


def _side(v):
    return v >= 0


class OracleSparseSlab:
    def __init__(self, res, block, l0, l1):
        self.res, self.block, self.l0, self.l1 = int(res), int(block), int(l0), int(l1)
        B, C = self.block, self.res - 1
        self.nb = self.blocks_per_axis = -(-C // B)
        assert 0 <= l0 < l1 <= self.nb
        self.x0, self.x1 = l0 * B, min(l1 * B, C)
        self.ghost = l0 > 0
        self.first_plane = self.x0 - int(self.ghost)
        self.n_planes = self.x1 + 1 - self.first_plane
        self.plane_bytes = 5 * self.res * self.res
        self.device = torch.device('cpu')
        self.E = B + 1
        self.V = self.E ** 3
        self.active_blocks = 0

    # -- geometry
    def _holders(self, x, lim0, lim1):
        B = self.block
        hi = min(x // B, self.nb - 1)
        lo = x // B - 1 if (x % B == 0 and x > 0) else hi
        return range(max(lo, lim0), min(hi, lim1) + 1)

    def _blocks_of(self, x, y, z):
        for bx in self._holders(x, self.l0, self.l1 - 1):
            for by in self._holders(y, 0, self.nb - 1):
                for bz in self._holders(z, 0, self.nb - 1):
                    yield bx - self.l0, by, bz

    def _local(self, b, x, y, z):
        B = self.block
        return ((x - (b[0] + self.l0) * B) * self.E + (y - b[1] * B)) * self.E + (z - b[2] * B)

    def _box(self, b):
        B, C = self.block, self.res - 1
        lo = [(b[0] + self.l0) * B, b[1] * B, b[2] * B]
        return lo, [min(v + B, C) for v in lo]

    def _corner(self, x, y, z):
        B, C = self.block, self.res - 1
        if all(v % B == 0 or v == C for v in (x, y, z)):
            c = [self.nb if v == C else v // B for v in (x, y, z)]
            return (c[0] - self.l0, c[1], c[2])
        return None

    def _fill_corner(self, x, y, z):
        B = self.block
        return (min(x // B, self.nb - 1) - self.l0, min(y // B, self.nb - 1), min(z // B, self.nb - 1))

    # -- storage
    def lookup(self, x, y, z, slot_limit=None):
        """(value, evaluated) of voxel (x, y, z) of planes [x0, x1]; not evaluated: the fill value."""
        lim = len(self.bricks) if slot_limit is None else slot_limit
        for b in self._blocks_of(x, y, z):
            s = self.slot[b]
            if 0 <= s < lim:
                e = self._local(b, x, y, z)
                if self.bmarks[s][e] == DONE:
                    return self.bvals[s][e], True
        c = self._corner(x, y, z)
        if c is not None and self.cmarks[c] == DONE:
            return self.cvals[c], True
        for j, p, has in ((0, self.x0, self.ghost), (1, self.x1, self.x1 < self.res - 1)):
            if has and x == p and self.pdone[j][y, z]:
                return self.pvals[j][y, z], True
        return self.cvals[self._fill_corner(x, y, z)], False

    def _store(self, x, y, z, v):
        for b in self._blocks_of(x, y, z):
            s = self.slot[b]
            if s != NO_SLOT:
                e = self._local(b, x, y, z)
                self.bvals[s][e] = v
                self.bmarks[s][e] = DONE
        c = self._corner(x, y, z)
        if c is not None:
            self.cvals[c] = v
            self.cmarks[c] = DONE

    def _owner(self, x, y, z):
        for b in self._blocks_of(x, y, z):
            if self.states[b] == FORCED:
                return self.slot[b], self._local(b, x, y, z)
        return None

    def _box_voxels(self, b):
        lo, hi = self._box(b)
        for x in range(lo[0], hi[0] + 1):
            for y in range(lo[1], hi[1] + 1):
                for z in range(lo[2], hi[2] + 1):
                    yield x, y, z

    def _allocate(self):
        old = len(self.bricks)
        new = [tuple(b) for b in np.argwhere(self.states == ACTIVATED)]          # block order: x, y, z
        for b in new:
            self.states[b] = FORCED
            self.slot[b] = len(self.bricks)
            self.sblock.append(b)
            self.bvals.append(np.zeros(self.V, np.float32))
            self.bmarks.append(np.zeros(self.V, np.uint8))
        for s in range(old, len(self.bricks)):
            b = self.sblock[s]
            for x, y, z in self._box_voxels(b):
                v, done = self.lookup(x, y, z, slot_limit=old)
                if done:
                    e = self._local(b, x, y, z)
                    self.bvals[s][e], self.bmarks[s][e] = v, DONE

    @property
    def bricks(self):
        return self.sblock

    def _list(self, kind):
        self.kind = kind
        if kind == 'corners':
            flat = self.cmarks.reshape(-1)
            self.list = np.nonzero(flat == WANTED)[0]
            flat[self.list] = DONE
        else:
            marks = np.concatenate(self.bmarks) if self.bmarks else np.zeros(0, np.uint8)
            self.list = np.nonzero(marks == WANTED)[0]
            for e in self.list:
                self.bmarks[e // self.V][e % self.V] = DONE
        return len(self.list)

    def _mark_and_list(self):
        self._allocate()
        for s, b in enumerate(self.sblock):
            if self.states[b] != FORCED:
                continue
            for x, y, z in self._box_voxels(b):
                e = self._local(b, x, y, z)
                if self.bmarks[s][e] != DONE and self._owner(x, y, z) == (s, e):
                    self.bmarks[s][e] = WANTED
        for b in self.sblock:
            if self.states[b] == FORCED:
                self.states[b] = MARKED
                self.active_blocks += 1
        return self._list('bricks')

    def _voxel(self, e):
        if self.kind == 'corners':
            n1 = self.nb + 1
            c = (e // (n1 * n1) + self.l0, (e // n1) % n1, e % n1)
            return tuple(min(v * self.block, self.res - 1) for v in c)
        b = self.sblock[e // self.V]
        lo, _ = self._box(b)
        loc = e % self.V
        return lo[0] + loc // (self.E * self.E), lo[1] + (loc // self.E) % self.E, lo[2] + loc % self.E

    def _push(self, x, y, z, v):
        for b in self._blocks_of(x, y, z):
            if self.states[b] == INACTIVE and _side(self.cvals[b]) != _side(v):
                self.states[b] = ACTIVATED

    # -- the steps
    def begin(self, quirk_period=0):
        r, nb = self.res, self.nb
        self.states = np.zeros((self.l1 - self.l0, nb, nb), np.uint8)
        self.slot = np.full((self.l1 - self.l0, nb, nb), NO_SLOT, np.int64)
        self.cmarks = np.zeros((self.l1 - self.l0 + 1, nb + 1, nb + 1), np.uint8)
        self.cvals = np.zeros((self.l1 - self.l0 + 1, nb + 1, nb + 1), np.float32)
        self.pvals = np.zeros((2, r, r), np.float32)
        self.pdone = np.zeros((2, r, r), bool)
        self.ghostv = np.zeros((r, r), np.float32)
        self.sblock, self.bvals, self.bmarks = [], [], []
        self.active_blocks = 0
        if quirk_period:
            g = np.union1d(np.arange(quirk_period - 1, r ** 3, quirk_period), [r ** 3 - 1])
            g = g[(g >= self.x0 * r * r) & (g < (self.x1 + 1) * r * r)]
            vox = list(zip(*np.unravel_index(g, (r, r, r))))
            for x, y, z in vox:
                for b in self._blocks_of(x, y, z):
                    self.states[b] = ACTIVATED
            self._allocate()
            for x, y, z in vox:
                s, e = self._owner(x, y, z)
                self.bmarks[s][e] = WANTED
        return self._list('bricks')

    def corners(self):
        self.cmarks[self.cmarks == IDLE] = WANTED
        return self._list('corners')

    def classify(self, tau, vol):
        assert vol is self
        tau = np.float32(tau)
        for b in zip(*np.nonzero(self.states == INACTIVE)):
            c = np.array([self.cvals[b[0] + dx, b[1] + dy, b[2] + dz] for dx in (0, 1) for dy in (0, 1) for dz in (0, 1)], np.float32)
            n_in = int(_side(c).sum())
            if np.any(~(np.abs(c) > tau)) or (n_in != 0 and n_in != 8):
                self.states[b] = ACTIVATED
        return self._mark_and_list()

    def grow(self, vol):
        assert vol is self
        for s, b in enumerate(self.sblock):
            lo, hi = self._box(b)
            for x, y, z in self._box_voxels(b):
                if x in (lo[0], hi[0]) or y in (lo[1], hi[1]) or z in (lo[2], hi[2]):
                    self._push(x, y, z, self.bvals[s][self._local(b, x, y, z)])
        for j, p, has in ((0, self.x0, self.ghost), (1, self.x1, self.x1 < self.res - 1)):
            if has:
                for y, z in zip(*np.nonzero(self.pdone[j])):
                    self._push(p, y, z, self.pvals[j][y, z])
        return self._mark_and_list()

    def gather(self, n, mini, maxi):
        r = self.res
        return torch.tensor([(x * r + y) * r + z for x, y, z in (self._voxel(e) for e in self.list[:n])], dtype=torch.int64)

    def scatter(self, values, vol):
        assert vol is self
        for e, v in zip(self.list, values.numpy()):
            self._store(*self._voxel(e), np.float32(v))

    def fill(self, vol):
        assert vol is self

    def block_states(self):
        return torch.from_numpy(self.states != 0)

    def volume(self):
        return self

    def planes(self, x_first, n_planes):
        out = np.empty((n_planes, self.res, self.res), np.float32)
        for i in range(n_planes):
            x = x_first + i
            if x < self.x0:
                out[i] = self.ghostv
                continue
            for y in range(self.res):
                for z in range(self.res):
                    out[i, y, z] = self.lookup(x, y, z)[0]
        return torch.from_numpy(out)

    def dense_volume(self):
        return self.planes(self.first_plane, self.n_planes)

    def export(self, plane, vol):
        assert vol is self and self.x0 <= plane <= self.x1
        r = self.res
        vals, done = np.empty((r, r), np.float32), np.empty((r, r), np.uint8)
        for y in range(r):
            for z in range(r):
                vals[y, z], d = self.lookup(plane, y, z)
                done[y, z] = d
        return torch.from_numpy(np.concatenate([vals.view(np.uint8).reshape(-1), done.reshape(-1)]))

    def import_(self, plane, buf, vol):
        assert vol is self
        r2 = self.res * self.res
        b = buf.numpy()
        vals = b[:4 * r2].view(np.float32).reshape(self.res, self.res)
        if plane == self.x0 - 1 and self.ghost:
            self.ghostv[...] = vals
            return
        assert (plane == self.x0 and self.ghost) or (plane == self.x1 and self.x1 < self.res - 1)
        j = 0 if plane == self.x0 else 1
        done = b[4 * r2:].reshape(self.res, self.res).astype(bool)
        for y, z in zip(*np.nonzero(done)):
            if not self.lookup(plane, y, z)[1]:
                self.pvals[j][y, z], self.pdone[j][y, z] = vals[y, z], True


def oracle_sparse_slabs(res, block, world):
    from nphm_b200.utils.reconstruction import plan_block_slabs
    return [None if l1 <= l0 else OracleSparseSlab(res, block, l0, l1) for l0, l1 in plan_block_slabs(res, block, world)]


def _mc_tables():
    """Edge, triangle and triangle-count tables of nphm_b200/csrc/mc_tables.h."""
    import os
    import re
    src = open(os.path.join(os.path.dirname(__file__), '..', 'nphm_b200', 'csrc', 'mc_tables.h')).read()

    def arr(name):
        body = src[src.index(name):]
        body = body[body.index('=') + 1:body.index('};')]
        return [int(v, 0) for v in re.findall(r'-?0x[0-9a-fA-F]+|-?\d+', body)]
    return np.array(arr('MC_EDGE_TABLE')), np.array(arr('MC_TRI_TABLE')).reshape(256, 16), np.array(arr('MC_NUM_TRIS'))


CORNER = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
EDGE_A = [0, 1, 2, 3, 4, 5, 6, 7, 0, 1, 2, 3]
EDGE_B = [1, 2, 3, 0, 5, 6, 7, 4, 4, 5, 6, 7]
EDGE_OF = {0: [[0, 4], [2, 6]], 1: [[3, 7], [1, 5]], 2: [[8, 11], [9, 10]]}
ORDER = [6, 5, 10, 0, 1, 2, 3, 4, 7, 8, 9, 11]
BEFORE = {e: sum(1 << f for f in ORDER[:ORDER.index(e)]) for e in range(12)}


def own_mask(gi, cj, ck):
    m = (1 << 6) | (1 << 5) | (1 << 10)
    if cj == 0 and ck == 0:
        m |= 1 << 0
    if ck == 0:
        m |= (1 << 2) | (1 << 1)
    if cj == 0:
        m |= (1 << 4) | (1 << 9)
    if gi == 0:
        m |= (1 << 7) | (1 << 11)
    if gi == 0 and ck == 0:
        m |= 1 << 3
    if gi == 0 and cj == 0:
        m |= 1 << 8
    return m


def brick_marching_cubes(store):
    """Restatement of nphm_band_sparse_mc_count / _emit on an OracleSparseSlab: (verts (n, 3) float64 in global index units, tris
    (m, 3) int64 ids relative to the slab's first vertex, negative for vertices of the ghost layer).  Segments are the cell rows of
    one active block; in sweep order they run (i, j, bz), and the vertex and triangle bases are exclusive scans of their counts."""
    edge, tri, ntri = _mc_tables()
    B, C, nb, x0 = store.block, store.res - 1, store.nb, store.x0
    pop = lambda v: bin(int(v)).count('1')                                  # noqa: E731
    flat = lambda b: (b[0] * nb + b[1]) * nb + b[2]                         # noqa: E731
    active = sorted((flat(b), b) for b in (tuple(int(c) for c in a) for a in np.argwhere(store.states == MARKED)))
    pos_of = {f: p for p, (f, _) in enumerate(active)}
    colcnt = np.zeros((store.l1 - store.l0) * nb, np.int64)
    for f, _ in active:
        colcnt[f // nb] += 1
    colstart = np.concatenate([[0], np.cumsum(colcnt)[:-1]])
    nseg = np.array([colcnt[(i // B - store.l0) * nb + j // B] for i in range(x0, store.x1) for j in range(C)], np.int64)
    rowbase = np.concatenate([[0], np.cumsum(nseg)[:-1]])

    def val(b, x, y, z):
        return store.bvals[store.slot[b]][store._local(b, x, y, z)]

    def cube_of(b, i, j, k):
        return sum(1 << c for c, (dx, dy, dz) in enumerate(CORNER) if _side(val(b, i + dx, j + dy, k + dz)))

    def seg_index(p, b, i, j):
        return rowbase[(i - x0) * C + j] + p - colstart[flat(b) // nb]

    segs = {}
    for p, (f, b) in enumerate(active):
        for i in range((b[0] + store.l0) * B, min((b[0] + store.l0) * B + B, C)):
            for j in range(b[1] * B, min(b[1] * B + B, C)):
                ks = range(b[2] * B, min(b[2] * B + B, C))
                cubes = [cube_of(b, i, j, k) for k in ks]
                segs[seg_index(p, b, i, j)] = (b, i, j, list(ks), cubes,
                                               sum(pop(edge[c] & own_mask(i, j, k)) for c, k in zip(cubes, ks)),
                                               sum(int(ntri[c]) for c in cubes))
    order = sorted(segs)
    vbase, tbase, nv, nt = {}, {}, 0, 0
    for s in order:
        vbase[s], tbase[s] = nv, nt
        nv, nt = nv + segs[s][5], nt + segs[s][6]
    # the ghost layer: cells X0 - 1 over the whole plane, from the ghost plane and plane X0
    gbase, ghost_v = {}, 0
    if store.ghost:
        px0 = store.planes(x0, 1).numpy()[0]
        gval = lambda dx, y, z: px0[y, z] if dx else store.ghostv[y, z]    # noqa: E731
        gcube = lambda j, k: sum(1 << c for c, (dx, dy, dz) in enumerate(CORNER) if _side(gval(dx, j + dy, k + dz)))  # noqa: E731
        for j in range(C):
            for k in range(C):
                gbase[(j, k)] = (ghost_v, gcube(j, k))
                ghost_v += pop(edge[gbase[(j, k)][1]] & own_mask(x0 - 1, j, k))

    def vertex_id(i, j, k, e, own):
        a, b = EDGE_A[e], EDGE_B[e]
        axis = 0 if CORNER[a][0] != CORNER[b][0] else (1 if CORNER[a][1] != CORNER[b][1] else 2)
        lo = a if CORNER[a][axis] == 0 else b
        ei, ej, ek = i + CORNER[lo][0], j + CORNER[lo][1], k + CORNER[lo][2]
        fi, fj, fk = ei, ej, ek
        if axis != 0:
            fi = ei - 1 if ei > 0 else ei
        if axis != 1:
            fj = ej - 1 if ej > 0 else 0
        if axis != 2:
            fk = ek - 1 if ek > 0 else 0
        d = [(ej - fj, ek - fk), (ei - fi, ek - fk), (ei - fi, ej - fj)][axis]
        eo = EDGE_OF[axis][d[0]][d[1]]
        if fi < x0:
            base, ocube = gbase[(fj, fk)]
            base -= ghost_v
        else:
            ob = (fi // B - store.l0, fj // B, fk // B)
            s = seg_index(pos_of[flat(ob)], ob, fi, fj)
            _, _, _, ks, cubes, _, _ = segs[s]
            n = fk - ks[0]
            base = vbase[s] + sum(pop(edge[c] & own_mask(fi, fj, kk)) for c, kk in zip(cubes[:n], ks[:n]))
            ocube = cubes[n]
        return base + pop(edge[ocube] & own_mask(fi, fj, fk) & BEFORE[eo])

    verts, tris = np.zeros((nv, 3)), np.zeros((nt, 3), np.int64)
    for s in order:
        b, i, j, ks, cubes, _, _ = segs[s]
        vrun, trun = vbase[s], tbase[s]
        for k, c in zip(ks, cubes):
            if c in (0, 255):
                continue
            created = int(edge[c]) & own_mask(i, j, k)
            for e in range(12):
                if created >> e & 1:
                    a, bb = EDGE_A[e], EDGE_B[e]
                    axis = 0 if CORNER[a][0] != CORNER[bb][0] else (1 if CORNER[a][1] != CORNER[bb][1] else 2)
                    fa = -float(val(b, i + CORNER[a][0], j + CORNER[a][1], k + CORNER[a][2]))
                    fb = -float(val(b, i + CORNER[bb][0], j + CORNER[bb][1], k + CORNER[bb][2]))
                    pos = [float(i + CORNER[a][0]), float(j + CORNER[a][1]), float(k + CORNER[a][2])]
                    qa = pos[axis]
                    qb = qa + float(CORNER[bb][axis] - CORNER[a][axis])
                    pos[axis] = (qb + qa) / 2.0 if fb == fa else (qb - qa) * (0.0 - fa) / (fb - fa) + qa
                    verts[vrun + pop(created & BEFORE[e])] = pos
            for q in range(3 * int(ntri[c])):
                tris[trun + q // 3, q % 3] = vertex_id(i, j, k, int(tri[c][q]), vrun)
            vrun += pop(created)
            trun += int(ntri[c])
    return verts, tris


def oracle_sparse_mc():
    """CPU stand-ins for ``_native.sparse_marching_cubes_count`` / ``emit`` through :func:`brick_marching_cubes`."""
    def count(store, iso, negate, x_global0=0, ghost_lo=False):
        assert x_global0 == store.first_plane and bool(ghost_lo) == store.ghost and negate and iso == 0.0
        v, t = brick_marching_cubes(store)
        return len(v), len(t), (v, t), None

    def emit(store, params, ws, nv, nt, base):
        v, t = params
        return torch.from_numpy(v), torch.from_numpy(t + base)

    return count, emit

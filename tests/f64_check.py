"""The float64 error criterion of the kernel tests (tests/test_gpu_chain_shapes.py, tests/test_gpu_ensemble_f64.py).

Per returned tensor, the same operation in fp32 PyTorch (TF32 off) is the yardstick of what fp32 arithmetic costs at this
shape, and

    err_native <= K * err_fp32 + FLOOR * max|ref64|

with both errors the maximum absolute difference from float64.  It is applied to the whole tensor and again, separately, to
parts of it (tiles, units, queries, members, scans), each with its own err_fp32 and max|ref64|: a wrong value confined to one
part is not hidden by larger values elsewhere.
"""
import math

import pytest

# a part is also allowed an error below the fp32 resolution of the whole tensor (the parts of a weight gradient behind rows
# whose softplus derivative is ~exp(-200) are ~1e-30 and come out as 0)
ULP = 2.0 ** -24

# Known defect of the layer chain: the backward scales the adjoint once, at the top of the chain (its largest magnitude to
# 2^10, mlp_chain.cu kGradExp), and stores every d_l below as an fp16 hi | lo pair.  Where the values of d_l stay below 2^-3
# after that scale, the lo part is subnormal and the weight and bias gradients built from them lose bits (measured: up to
# 1.5e-3 of max|ref| on lin0 of 4-8x2-1 at one row behind saturated softplus units).  Those checks, and only those, are told
# apart from the float64 adjoints: a check of layer l is in the range defect when d_l (over the part's output features) or any
# adjoint above it stays below LO_NORMAL after the device's scale.  If one of them fails and nothing else does, the test is
# reported as an expected failure; an error beyond KNOWN_MAX of the part's max|ref| fails it like any other violation.
LO_NORMAL = 2.0 ** -3
KNOWN_MAX = 1e-2


def _ratio(en, ef):
    return en / ef if ef > 0 else (0.0 if en == 0 else float('inf'))


class Check:
    """Collects err_native / err_fp32 of the tensors of one test; ``done()`` fails with every violation.  k, floor and
    floor_grad: the criterion's constants (floor_grad for weight and bias gradients); prefix: the tag of the printed lines."""

    def __init__(self, tag, k, floor, floor_grad=None, prefix='CHAIN'):
        self.tag = tag
        self.k, self.floor, self.floor_grad = k, floor, floor if floor_grad is None else floor_grad
        self.prefix = prefix
        self.bad = []
        self.known = []                  # violations inside the adjoint's fp16 subnormal range (see LO_NORMAL)
        self.n_known = 0
        self.worst = {}                  # what -> worst ratio over the tensor and its parts
        self.worst_rel = {}              # what -> worst err_native / max|ref64| of a part, relative to the part's own max
        self.need = {}                   # (what, 'tensor' | 'parts') -> the smallest floor that would have passed

    def _one(self, what, got, r64, r32, floor, scale=None, whole=0.0, known=False, need=None):
        en = float((got.double() - r64).abs().max()) if got.numel() else 0.0
        ef = float((r32.double() - r64).abs().max()) if got.numel() else 0.0
        sc = (float(r64.abs().max()) if r64.numel() else 0.0) if scale is None else scale
        bound = self.k * ef + floor * sc + ULP * whole
        if need is not None and sc > 0:
            self.need[need] = max(self.need.get(need, 0.0), (en - self.k * ef - ULP * whole) / sc)
        self.n_known += known
        if not en <= bound:
            msg = '%s: err_native %.3e > %.3e (err_fp32 %.3e, max|ref| %.3e)' % (what, en, bound, ef, sc)
            # inside the known range defect the error stays below a few fp16 ulps of the part; more is another bug
            (self.known if known and en <= KNOWN_MAX * sc + bound else self.bad).append(msg)
        return en, ef, sc

    def __call__(self, what, got, r64, r32, kind='rows', scale=None, known=(False, False), parts=(), floor=None,
                 part_floor=None):
        """kind: 'rows' (leading dims are rows: also the last 128-row tile), 'weight' (N x K: also the last 16 rows and the
        last 16 columns), 'bias' (also the last 16), 'cond' (B x D: also each query's row), 'scalar'.  scale: the magnitude
        the floor is relative to (default max|ref64|).  parts: more (name, index) pairs, each checked on got[index] with its
        own err_fp32 and max|ref64|.  floor: in place of the constructor's floor for this tensor; part_floor: for its parts
        (default: the same)."""
        assert got.shape == r64.shape, (what, tuple(got.shape), tuple(r64.shape))
        if floor is None:
            floor = self.floor_grad if kind in ('weight', 'bias') else self.floor
        part_floor = floor if part_floor is None else part_floor
        key = what.split(' ')[0] + ' ' + what.split(' ')[-1]
        en, ef, sc = self._one(what, got, r64, r32, floor, scale, known=known[0], need=(key, 'tensor'))
        checks = []
        if kind == 'rows':
            M = got.shape[0] * got.shape[1] if got.dim() >= 2 else got.shape[0]
            m0 = (M - 1) // 128 * 128
            flat = lambda t: t.reshape(M, -1)[m0:]
            checks.append(('last tile', flat(got), flat(r64), flat(r32), False))
        elif kind == 'weight':
            n0, k0 = (got.shape[0] - 1) // 16 * 16, (got.shape[1] - 1) // 16 * 16
            checks += [('last rows', got[n0:], r64[n0:], r32[n0:], known[1]),
                       ('last cols', got[:, k0:], r64[:, k0:], r32[:, k0:], known[0])]
        elif kind == 'bias':
            n0 = (got.shape[0] - 1) // 16 * 16
            checks.append(('last unit', got[n0:], r64[n0:], r32[n0:], known[1]))
        elif kind == 'cond':
            checks += [('query %d' % q, got[q], r64[q], r32[q], False) for q in range(got.shape[0])]
        checks += [(name, got[i], r64[i], r32[i], False) for name, i in parts]
        worst = _ratio(en, ef)
        rel = en / sc if sc > 0 else 0.0
        for name, g, a, b, kn in checks:
            if g.numel() == 0:
                continue
            pn, pf, _ = self._one('%s [%s]' % (what, name), g, a, b, part_floor,
                                  scale=sc if kind in ('weight', 'bias') else None, whole=sc, known=kn, need=(key, 'parts'))
            worst = max(worst, _ratio(pn, pf))
            rel = max(rel, pn / float(a.abs().max()) if float(a.abs().max()) > 0 else 0.0)
        self.worst[key] = max(self.worst.get(key, 0.0), worst)
        self.worst_rel[key] = max(self.worst_rel.get(key, 0.0), rel)
        print('%s %-16s %-44s err_native %.3e err_fp32 %.3e ratio %7.3f worst-part ratio %7.3f native/max|ref| %.2e'
              % (self.prefix, self.tag, what, en, ef, en / ef if ef > 0 else float('nan'), worst, en / sc if sc > 0 else 0.0))

    def grads(self, what, gw, gb, r64, r32, chains):
        """Weight and bias gradients of every layer; chains: [(adjoints d_l of the hidden layers, the device's scale of
        that adjoint chain)], whose range decides which checks fall under the known defect (adjoint_range)."""
        known = adjoint_range(chains, len(gw))
        for l, (a, b) in enumerate(zip(gw, gb)):
            self('%s lin%d.weight' % (what, l), a, r64[0][l], r32[0][l], 'weight', known=known[l])
            self('%s lin%d.bias' % (what, l), b, r64[1][l], r32[1][l], 'bias', known=known[l])

    def done(self):
        print('%s %-16s %d of the checks fall in the adjoint range defect, %d of them beyond the bound'
              % (self.prefix, self.tag, self.n_known, len(self.known)))
        for key, w in sorted(self.worst.items()):
            print('%s %-16s worst err_native / err_fp32 of %-36s %9.3f, err_native / own max|ref| %.2e, floor needed: '
                  'tensor %.2e, parts %.2e' % (self.prefix, self.tag, key, w, self.worst_rel[key],
                                               self.need.get((key, 'tensor'), 0.0), self.need.get((key, 'parts'), 0.0)))
        assert not self.bad, '%s: %d violations:\n%s' % (self.tag, len(self.bad), '\n'.join(self.bad[:40]))
        if self.known:
            pytest.xfail('%s: %d weight / bias gradient checks whose adjoint left its fp16 range exceed the bound (every other '
                         'check passed):\n%s' % (self.tag, len(self.known), '\n'.join(self.known[:20])))


def top_scale(*upstream):
    """The power of two the device scales an upstream gradient by: largest magnitude to [2^10, 2^11)."""
    m = max(float(g.abs().max()) for g in upstream)
    return 2.0 ** (10 - math.floor(math.log2(m))) if m > 0 else 1.0


def adjoint_range(chains, n_lin):
    """Per layer l: (whole layer in the range defect, its last 16-feature unit in it)."""
    known = [(False, False)] * n_lin
    below = False                          # an adjoint above this layer left the range: its error reaches every layer below
    for l in range(n_lin - 2, -1, -1):
        lay = unit = False
        for ds, scale in chains:
            d = ds[l].abs().reshape(-1, ds[l].shape[-1]) * scale
            n0 = (d.shape[1] - 1) // 16 * 16
            lay |= float(d.max()) < LO_NORMAL
            unit |= float(d[:, n0:].max()) < LO_NORMAL
        below |= lay
        known[l] = (below, below or unit)
    return known

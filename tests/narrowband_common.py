"""Decoders and analytic SDFs shared by the narrow-band tests and tools/bench_narrowband.py."""
import numpy as np
import torch

# NPM-size identity decoder (515 -> 1024 x 8 -> 1, seed 12): its xyz columns are scaled by NPM_XYZ_GAIN so that the SDF varies over
# the grid (|grad| up to ~0.3), and its output bias is raised by NPM_SURFACE_SHIFT, so that the zero level set splits the grid in two
NPM_XYZ_GAIN = 1000.0
NPM_SURFACE_SHIFT = 0.333


def make_npm_head(device):
    from nphm_b200.models.deepSDF import DeepSDF
    torch.manual_seed(12)
    dec = DeepSDF(lat_dim=512, hidden_dim=1024, nlayers=8, geometric_init=True)
    with torch.no_grad():
        dec.lin0.weight[:, :3].mul_(NPM_XYZ_GAIN)
        dec.lin8.bias.add_(NPM_SURFACE_SHIFT)
    return dec.to(device).eval(), torch.zeros(512, device=device)


def tilted_plate(p, h, gain=20.0, thickness=0.2, xp=np):
    """A plate thinner than the grid step h, tilted against the grid, with |grad| = gain: away from the few places where it
    passes next to a block corner it lies between coarse samples that are all far from 0, so the band has to grow along it."""
    n = np.array([1.0, 0.13, 0.07])
    nx, ny, nz = (float(c) for c in n / np.linalg.norm(n))
    d = nx * p[..., 0] + ny * p[..., 1] + nz * p[..., 2] - 0.031
    return gain * (xp.abs(d) - thickness * h)


SDFS = {
    'sphere': lambda X, Y, Z, h: np.sqrt(X ** 2 + Y ** 2 + Z ** 2) - 0.5,
    'torus': lambda X, Y, Z, h: np.sqrt((np.sqrt(X ** 2 + Y ** 2) - 0.5) ** 2 + Z ** 2) - 0.2,
    # two spheres whose gap is one block (4 grid steps)
    'two_spheres': lambda X, Y, Z, h: np.minimum(np.sqrt((X - 0.3 - 2 * h) ** 2 + Y ** 2 + Z ** 2) - 0.3,
                                                 np.sqrt((X + 0.3 + 2 * h) ** 2 + Y ** 2 + Z ** 2) - 0.3),
    'thin_plate': lambda X, Y, Z, h: tilted_plate(np.stack([X, Y, Z], -1), h),
}


def analytic_volume(name, res):
    """(res^3 float32 volume of SDFS[name] on [-1, 1]^3, grid step)."""
    ax = np.linspace(-1.0, 1.0, res)
    X, Y, Z = np.meshgrid(ax, ax, ax, indexing='ij')
    h = 2.0 / (res - 1)
    return SDFS[name](X, Y, Z, h).astype(np.float32), h

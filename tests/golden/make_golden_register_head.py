#!/usr/bin/env python
"""A small NPM DeepSDF whose zero-code head is the registration tests' asymmetric analytic head (tests/register_common.py):
a distance-like SDF for the register -> fit tests, where the seeded random decoders are not.  Trained on the CPU with a
fixed seed:   python tests/golden/make_golden_register_head.py   -> tests/golden/register_head.npz (the state dict)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import register_common as RC                       # noqa: E402
from conftest import MAXI, MINI                     # noqa: E402
from nphm_b200.models.deepSDF import DeepSDF       # noqa: E402

CONFIG = RC.HEAD_CONFIG


def main(steps=4000, batch=8192):
    torch.manual_seed(0)
    torch.set_num_threads(8)
    net = DeepSDF(**CONFIG)
    lo, hi = torch.tensor(MINI, dtype=torch.float64), torch.tensor(MAXI, dtype=torch.float64)
    surf, _ = RC.surface_points(RC.ASYMMETRIC, 20000, seed=11)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, steps, eta_min=2e-5)
    g = torch.Generator().manual_seed(1)
    for it in range(steps):
        # half uniform in the box, half within 0.03 of the surface
        u = lo + torch.rand(batch // 2, 3, generator=g, dtype=torch.float64) * (hi - lo)
        s = surf[torch.randint(0, surf.shape[0], (batch // 2,), generator=g)]
        s = s + 0.03 * torch.randn(s.shape, generator=g, dtype=torch.float64)
        x = torch.cat([u, s])
        y = RC.analytic_sdf(RC.ASYMMETRIC, x).float()
        near = (y.abs() < 0.05).float()
        pred, _ = net(x.float()[None], torch.zeros(1, x.shape[0], CONFIG['lat_dim']))
        err = (pred.reshape(-1) - y).abs()
        loss = (err * (1 + 9 * near)).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
        if it % 500 == 0 or it == steps - 1:
            print('step %d loss %.3g near-surface L1 %.3g' % (it, float(loss.detach()),
                                                              float((err.detach() * near).sum() / near.sum())))
    with torch.no_grad():
        pred, _ = net(surf.float()[None], torch.zeros(1, surf.shape[0], CONFIG['lat_dim']))
    print('|sdf| at the analytic surface: mean %.3g, max %.3g' % (float(pred.abs().mean()), float(pred.abs().max())))
    np.savez_compressed(os.path.join(HERE, 'register_head.npz'),
                        **{k: v.numpy() for k, v in net.state_dict().items()})


if __name__ == '__main__':
    main()

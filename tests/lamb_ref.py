"""Float64 restatement of the learner's clip + LAMB step (include/hrl_b200.h, hrl_clip_lamb_step), the reference the LAMB
tests compare the CUDA kernels and the learner against.

    c = min(1, max_norm / (|g| + 1e-6));  g' = c g
    m = m + (g' - m)(1 - b1);  v = b2 v + (1 - b2) g'^2
    u = (m / (1 - b1^t)) / (sqrt(v) / sqrt(1 - b2^t) + eps) + wd w
    r_i = |w_i| / |u_i| (1 when either is 0);  w <- w - lr lr_scale r_i u
"""
import numpy as np
import torch


def lamb_step(ws, gs, ms, vs, t, lr, lr_scale=1.0, max_norm=4.0, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5):
    """One step on lists of per-tensor arrays (any float dtype; computed in float64).  t: the step count after this step.
    Returns (w, m, v, ratios, grad_norm) with w, m, v lists of float64 arrays."""
    ws, gs, ms, vs = ([np.asarray(a, np.float64) for a in x] for x in (ws, gs, ms, vs))
    norm = float(np.sqrt(sum(float((g * g).sum()) for g in gs)))
    c = min(1.0, max_norm / (norm + 1e-6))
    b1, b2 = betas
    out_w, out_m, out_v, ratios = [], [], [], []
    for w, g, m, v in zip(ws, gs, ms, vs):
        g = c * g
        m = m + (g - m) * (1 - b1)
        v = b2 * v + (1 - b2) * g * g
        u = (m / (1 - b1 ** t)) / (np.sqrt(v) / np.sqrt(1 - b2 ** t) + eps) + weight_decay * w
        wn, un = float(np.sqrt((w * w).sum())), float(np.sqrt((u * u).sum()))
        r = wn / un if wn > 0 and un > 0 else 1.0
        out_w.append(w - lr * lr_scale * r * u)
        out_m.append(m)
        out_v.append(v)
        ratios.append(r)
    return out_w, out_m, out_v, ratios, norm


class Lamb64(torch.optim.Optimizer):
    """LAMB as a torch optimiser for oracle.torch_learner.CpuLearner (which clips the gradients before step()): the step is
    computed in float64 from the float32 weights and gradients, the moments are kept in float64, and the weights receive
    the float32 rounding of the result."""

    def __init__(self, params, lr, lr_scale=1.0, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5):
        super().__init__(params, dict(lr=lr, lr_scale=lr_scale, betas=betas, eps=eps, weight_decay=weight_decay))

    @torch.no_grad()
    def step(self):
        for group in self.param_groups:
            ps = group['params']
            for p in ps:
                st = self.state[p]
                if not st:
                    st['m'] = torch.zeros(p.shape, dtype=torch.float64)
                    st['v'] = torch.zeros(p.shape, dtype=torch.float64)
                    st['t'] = 0
                st['t'] += 1
            t = self.state[ps[0]]['t']
            w, m, v, _, _ = lamb_step([p.double().numpy() for p in ps],
                                      [p.grad.double().numpy() for p in ps],
                                      [self.state[p]['m'].numpy() for p in ps], [self.state[p]['v'].numpy() for p in ps],
                                      t, group['lr'], group['lr_scale'], max_norm=float('inf'), betas=group['betas'],
                                      eps=group['eps'], weight_decay=group['weight_decay'])
            for p, wi, mi, vi in zip(ps, w, m, v):
                st = self.state[p]
                st['m'], st['v'] = torch.from_numpy(mi), torch.from_numpy(vi)
                p.copy_(torch.from_numpy(wi).to(p.dtype))

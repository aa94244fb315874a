"""Float64 restatement of the learner's clip + Muon step (include/hrl_b200.h, hrl_clip_muon_step), the reference the Muon
tests compare the CUDA kernel and the learner against.

    c = min(1, max_norm / (|g| + 1e-6));  G = c g                                     (one global norm over every tensor)
    Muon-owned matrix W (r x k view), momentum M:
        M <- mu M + G;  N = G + mu M                                                  mu = 0.95
        X = N / (|N|_F + 1e-7), transposed when r > k
        5 times: A = X X^T;  B = b A + c A A;  X = a X + B X                          (a, b, c) = (3.4445, -4.7750, 2.0315)
        O = X (transposed back);  W <- W - lr (lr_scale 0.2 sqrt(max(r, k)) O + wd W)
    every other tensor: hrl_clip_adam_step's Adam (decay added to the gradient)

bf16=True rounds X (after the normalisation and after every iteration), A and B to bf16, nearest even, where the kernel
does; the products are still accumulated in float64.
"""
import numpy as np
import torch

MU = 0.95
NS = (3.4445, -4.7750, 2.0315)
STEPS = 5


def round_bf16(x):
    """float64 array -> the float64 values of its bf16 rounding (nearest even), through float32 as the kernel's fp32 values."""
    return torch.from_numpy(np.asarray(x, np.float64)).to(torch.float32).to(torch.bfloat16).double().numpy()


def orthogonalise(n, bf16=False):
    """The five Newton-Schulz iterations on the r x k matrix n; returns O (r x k, float64)."""
    a, b, c = NS
    n = np.asarray(n, np.float64)
    tall = n.shape[0] > n.shape[1]
    x = n.T if tall else n
    x = x / (np.sqrt((x * x).sum()) + 1e-7)
    rnd = round_bf16 if bf16 else (lambda v: v)
    x = rnd(x)
    for _ in range(STEPS):
        A = rnd(x @ x.T)
        B = rnd(b * A + c * (A @ A))
        x = rnd(a * x + B @ x)
    return x.T if tall else x


def ns_polynomial(s):
    """What the iterations do to a singular value s of the normalised input: p(p(p(p(p(s))))), p(x) = a x + b x^3 + c x^5."""
    a, b, c = NS
    s = np.asarray(s, np.float64)
    for _ in range(STEPS):
        s = a * s + b * s ** 3 + c * s ** 5
    return s


def matrix_view(shape):
    r = int(shape[0])
    return r, int(np.prod(shape)) // r


def muon_step(ws, gs, ms, vs, kinds, t, lr, lr_scale=1.0, max_norm=4.0, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5,
              bf16=False):
    """One step on lists of per-tensor arrays (any float dtype, shaped as the parameters; computed in float64).  kinds[i]:
    'matrix' (Muon-owned) or anything else (Adam).  t: the step count after this step.  Returns (w, m, v, o, grad_norm) with
    w, m, v lists of float64 arrays and o[i] the O of a Muon-owned tensor (r x k), else None."""
    ws, gs, ms, vs = ([np.asarray(a, np.float64) for a in x] for x in (ws, gs, ms, vs))
    norm = float(np.sqrt(sum(float((g * g).sum()) for g in gs)))
    c = min(1.0, max_norm / (norm + 1e-6))
    b1, b2 = betas
    out_w, out_m, out_v, out_o = [], [], [], []
    for w, g, m, v, kind in zip(ws, gs, ms, vs, kinds):
        g = c * g
        if kind == 'matrix':
            r, k = matrix_view(w.shape)
            m = MU * m + g
            o = orthogonalise((g + MU * m).reshape(r, k), bf16=bf16)
            out_w.append(w - lr * (lr_scale * 0.2 * np.sqrt(max(r, k)) * o.reshape(w.shape) + weight_decay * w))
            out_o.append(o)
        else:
            g = g + weight_decay * w
            m = m + (g - m) * (1 - b1)
            v = b2 * v + (1 - b2) * g * g
            out_w.append(w - lr / (1 - b1 ** t) * m / (np.sqrt(v) / np.sqrt(1 - b2 ** t) + eps))
            out_o.append(None)
        out_m.append(m)
        out_v.append(v)
    return out_w, out_m, out_v, out_o, norm


class Muon64(torch.optim.Optimizer):
    """Muon as a torch optimiser for oracle.torch_learner.CpuLearner (which clips the gradients before step()): the split
    comes from the library (ops.muon_plan on the parameters' shapes), the step is computed in float64 from the float32
    weights and gradients, the moments are kept in float64, and the weights receive the float32 rounding of the result."""

    def __init__(self, params, lr, lr_scale=1.0, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-5):
        super().__init__(params, dict(lr=lr, lr_scale=lr_scale, betas=betas, eps=eps, weight_decay=weight_decay))

    @torch.no_grad()
    def step(self):
        from handyrl_b200.ops import muon_plan
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
            kinds = muon_plan([tuple(p.shape) for p in ps])[0]
            w, m, v, _, _ = muon_step([p.double().numpy() for p in ps], [p.grad.double().numpy() for p in ps],
                                      [self.state[p]['m'].numpy() for p in ps], [self.state[p]['v'].numpy() for p in ps],
                                      kinds, t, group['lr'], group['lr_scale'], max_norm=float('inf'), betas=group['betas'],
                                      eps=group['eps'], weight_decay=group['weight_decay'])
            for p, wi, mi, vi in zip(ps, w, m, v):
                st = self.state[p]
                st['m'], st['v'] = torch.from_numpy(mi), torch.from_numpy(vi)
                p.copy_(torch.from_numpy(wi).to(p.dtype))

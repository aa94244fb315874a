"""float64 numpy reference of the learner diagnostics sums (include/hrl_b200.h, HRL_DIAG_*), built on the loss oracle's taps
(oracle.loss, pinned to the reference's goldens by test_oracle.py)."""
import numpy as np

from handyrl_b200._capi import DIAG_KEYS, NUM_DIAG


def diagnostics(batch, outs, args):
    """Returns (sums, n_near_one): sums = float64 array of NUM_DIAG in DIAG_KEYS order (optimiser entries 0), n_near_one = the
    number of counted policy samples whose float64 importance ratio lies within 1e-6 of 1 (their [rho > 1] is a coin flip in
    fp32, so a rho_clip comparison allows for them)."""
    from oracle import oracle
    g = lambda k: np.asarray(batch[k], dtype=np.float64)
    orc = oracle.loss(batch, outs, args, dtype=np.float64)
    bi = int(args.get('burn_in_steps', 0))
    B, T, P = g('turn_mask').shape[:3]
    Pa = np.asarray(batch['action_mask']).shape[2]
    q = np.zeros(P, dtype=int) if Pa == 1 else np.arange(P)          # the policy row of each column
    tm = g('turn_mask')[:, bi:, :, 0]
    om = g('observation_mask')[:, bi:, :, 0]
    em = g('episode_mask').reshape(B, T)[:, bi:, None]
    mu = g('selected_prob')[:, bi:, :, 0][:, :, q]
    logp = np.asarray(orc['logp'], np.float64)[:, bi:, :, 0][:, :, q]     # log pi(a) * episode_mask
    lr = logp - np.log(np.clip(mu, 1e-16, 1.0)) * em
    rho = np.exp(lr)
    adv = np.asarray(orc['advantage'], np.float64)[:, bi:, :, 0]
    s = dict.fromkeys(DIAG_KEYS, 0.0)
    s.update(n_pol=tm.sum(), rho=(tm * rho).sum(), rho_clip=(tm * (rho > 1)).sum(), logr=(tm * lr).sum(),
             logr2=(tm * lr * lr).sum(), adv=(tm * adv).sum(), adv2=(tm * adv * adv).sum())
    for head, tap, n, t, t2, e, e2 in (('value', 'target_value', 'n_val', 'tv', 'tv2', 'ev', 'ev2'),
                                        ('return', 'target_return', None, 'tr', 'tr2', 'er', 'er2')):
        if outs.get(head) is None:
            continue
        tgt = np.asarray(orc[tap], np.float64)[:, bi:, :, 0]
        err = tgt - np.asarray(outs[head], np.float64)[:, bi:, :, 0][:, :, q] * om
        if n:
            s[n] = om.sum()
        s[t], s[t2], s[e], s[e2] = (om * tgt).sum(), (om * tgt * tgt).sum(), (om * err).sum(), (om * err * err).sum()
    near = int(((tm != 0) & (np.abs(rho - 1) < 1e-6)).sum())
    return np.array([s[k] for k in DIAG_KEYS], dtype=np.float64), near


def compare(got, want, near, rtol=1e-5, atol=1e-5, err=''):
    """The kernel's sums against diagnostics(): counts exact, rho_clip exact up to the near-one samples, the rest rtol/atol."""
    got = np.asarray(got, np.float64)
    assert got.shape == (NUM_DIAG,)
    i = {k: n for n, k in enumerate(DIAG_KEYS)}
    assert got[i['n_pol']] == want[i['n_pol']] and got[i['n_val']] == want[i['n_val']], (err, got, want)
    d = got[i['rho_clip']] - want[i['rho_clip']]
    assert abs(d) <= near, (err, 'rho_clip', got[i['rho_clip']], want[i['rho_clip']], near)
    rest = [n for k, n in i.items() if k not in ('n_pol', 'n_val', 'rho_clip')]
    np.testing.assert_allclose(got[rest], want[rest], rtol=rtol, atol=atol, err_msg=err)

"""The fp64 model of the device L-BFGS step (tsb_newton_lbfgs_step) that test_newton_lbfgs uses: the per-sphere pair
ring, the two-loop recursion with a block-diagonal H0, the dense compact form of the same inverse-BFGS matrix, and the
whole step on an Fp64Problem with the device's rule.  Not a test module."""
import functools

import numpy as np

from _newton_model import (ACTIVE, ALPHAS, N_CONVERGED, STALLED, block_preconditioner, f32, reference_problem,
                           weight_ok)

# NEWTON_LBFGS_DEFAULTS
LBFGS_OPTS = dict(m=8, sigma=1e-4, eta=0.9, n_alpha=8, rel_floor=1e-6, gtol=0.0, curv_eps=1e-8)
# Steps the fp64 model needs on the small mixed pack (reference_problem) until every sphere is CONVERGED, with AMIPS off
# and on; test_newton_lbfgs pins them and the GPU run's budget on the mixed 64 x 4096 pack derives from them.
LBFGS_REF_STEPS = {False: 53, True: 48}
LBFGS_GPU_SLACK = 1.0          # the GPU budget is (1 + LBFGS_GPU_SLACK) times the model count: its spheres have 16x the tets


class History:
    """One sphere's ring of up to m pairs (s, y), oldest first, with the device's curvature test."""

    def __init__(self, m, curv_eps):
        self.m, self.curv_eps, self.pairs = m, curv_eps, []

    def push(self, s, y):
        """Keeps the pair (dropping the oldest from a full ring) when s.y > curv_eps |s| |y|; returns whether it did."""
        sy = float(s @ y)
        if not sy > self.curv_eps * np.sqrt(float(s @ s)) * np.sqrt(float(y @ y)):
            return False
        self.pairs.append((np.array(s, np.float64), np.array(y, np.float64)))
        del self.pairs[:-self.m]
        return True


def two_loop(b, pairs, H0):
    """H b for the L-BFGS inverse Hessian H of pairs (oldest first) over the dense H0, by the two-loop recursion."""
    q = np.array(b, np.float64)
    al = []
    for s, y in reversed(pairs):
        a = (s @ q) / (s @ y)
        al.append(a)
        q = q - a * y
    r = H0 @ q
    for (s, y), a in zip(pairs, reversed(al)):
        r = r + s * (a - (y @ r) / (s @ y))
    return r


def compact_inverse(pairs, H0):
    """The same inverse-BFGS matrix in compact form (Byrd, Nocedal and Schnabel 1994):
    H = H0 + [S, H0 Y] [[R^-T (D + Y^T H0 Y) R^-1, -R^-T], [-R^-1, 0]] [S, H0 Y]^T, R = triu(S^T Y), D = diag(S^T Y)."""
    if not pairs:
        return np.array(H0, np.float64)
    S = np.stack([s for s, _ in pairs], 1)
    Y = np.stack([y for _, y in pairs], 1)
    SY = S.T @ Y
    Ri = np.linalg.inv(np.triu(SY))
    k = len(pairs)
    W = np.block([[Ri.T @ (np.diag(np.diag(SY)) + Y.T @ H0 @ Y) @ Ri, -Ri.T], [-Ri, np.zeros((k, k))]])
    U = np.concatenate([S, H0 @ Y], 1)
    return H0 + U @ W @ U.T


def lbfgs_reference(P, x0, n_steps, o, y=None, w=None):
    """The device L-BFGS step in fp64: b = -grad Phi (zero on frozen spheres and where w_c is unusable), H0 = the
    kernel's block preconditioner on D + w_c I, the pair of the last step when the sphere moved (s = x - x_prev,
    y = b_prev - b, the curvature test), the two-loop, the fallback d = H0 b (history cleared) when b.d <= 0 on a sphere
    with pairs, the oracle's energy changes and inversion bound, the Armijo rule below eta alpha^, no step clearing the
    history and no step from an empty history stalling the sphere.  Returns the final x and per step and sphere a dict
    of what the rule saw and decided."""
    from test_hess_diag import hess_diag_blocks
    x = np.asarray(x0, np.float64).reshape(-1).copy()
    prox = y is not None
    y = np.asarray(y, np.float64).reshape(-1) if prox else None
    w = np.asarray(w, np.float64) if prox else np.zeros(P.S)
    alphas = ALPHAS[:o["n_alpha"]]
    sl = [slice(3 * P.vo[s], 3 * P.vo[s + 1]) for s in range(P.S)]
    hist_ = [History(o["m"], f32(o["curv_eps"])) for _ in range(P.S)]
    status = [ACTIVE] * P.S
    moved = [False] * P.S
    xp = bp = None
    hist = []
    for _ in range(n_steps):
        b = -P.grad(x)
        live = [status[s] == ACTIVE and weight_ok(w[s]) for s in range(P.S)]
        for s in range(P.S):
            if not live[s]:
                b[sl[s]] = 0.0
            elif w[s]:
                b[sl[s]] -= w[s] * (x[sl[s]] - y[sl[s]])
        D = hess_diag_blocks(P.orc, x, P.c1, P.c2, P.c3, P.order)
        d = np.zeros_like(x)
        out = []
        for s in range(P.S):
            h = dict(pair=-1, cleared=0, g=float(np.linalg.norm(b[sl[s]])))
            if live[s]:
                H0 = block_preconditioner(D[P.vo[s]:P.vo[s + 1]], float(np.float32(w[s])), o["rel_floor"])
                if moved[s]:
                    h["pair"] = int(hist_[s].push(x[sl[s]] - xp[sl[s]], bp[sl[s]] - b[sl[s]]))
                ds = two_loop(b[sl[s]], hist_[s].pairs, H0)
                if not b[sl[s]] @ ds > 0.0 and hist_[s].pairs:
                    hist_[s].pairs, h["cleared"] = [], 1
                    ds = H0 @ b[sl[s]]
                d[sl[s]] = ds
            h.update(bd=float(b[sl[s]] @ d[sl[s]]), dd=float(d[sl[s]] @ d[sl[s]]),
                     dx=float(d[sl[s]] @ (x[sl[s]] - y[sl[s]])) if w[s] > 0 else 0.0)
            out.append(h)
        xp, bp = x.copy(), b.copy()
        E0, inv0 = P.sphere_energy(x)
        dE = np.stack([P.sphere_energy(x + a * d)[0] - E0 for a in alphas], axis=1)
        ahat = P.inversion_bound(x, d)
        for s, h in enumerate(out):
            h.update(E0=E0[s], inv0=inv0[s], ahat=float(ahat[s]), alpha=0.0, k=-1, delta=0.0)
            if status[s] != ACTIVE:
                pass
            elif not weight_ok(w[s]):
                status[s] = STALLED
            elif h["g"] <= f32(o["gtol"]):
                status[s] = N_CONVERGED
            else:
                dphi = [dE[s, k] + (w[s] * (a * h["dx"] + 0.5 * a * a * h["dd"]) if w[s] > 0 else 0.0) for k, a in enumerate(alphas)]
                lim = f32(o["eta"]) * h["ahat"]
                if h["bd"] > 0.0:
                    h["k"] = next((k for k, a in enumerate(alphas) if a < lim and dphi[k] <= -f32(o["sigma"]) * a * h["bd"]), -1)
                if h["k"] >= 0:
                    h.update(alpha=alphas[h["k"]], delta=dphi[h["k"]])
                elif not hist_[s].pairs:
                    status[s] = STALLED
                else:
                    hist_[s].pairs, h["cleared"] = [], 1
            moved[s] = h["alpha"] > 0.0
            h.update(status=status[s], n_pairs=len(hist_[s].pairs))
            x[sl[s]] += h["alpha"] * d[sl[s]]
        hist.append(out)
    return x, hist


@functools.lru_cache(maxsize=None)
def lbfgs_reference_run(amips):
    """(P, x0, o, x, hist): the model on reference_problem(amips) with the default options and gtol = 1e-3 times the
    smallest starting |g_c|, LBFGS_REF_STEPS[amips] + 3 steps."""
    P, x0, _, o = reference_problem(amips, True)
    o = dict(LBFGS_OPTS, gtol=o["gtol"])
    x, hist = lbfgs_reference(P, x0, LBFGS_REF_STEPS[amips] + 3, o)
    return P, x0, o, x, hist

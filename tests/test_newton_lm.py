"""The damped (Levenberg-Marquardt) Newton step: tsb_pcg_set_blocks_ex / tsb_pcg_solve_ex (the shifted solve),
tsb_newton_* (the step), newton.DeviceNewton and SmoothnessBarrierEnergy.newton_step.

CPU: the batched PCG state machine of test_pcg_device extended with a per-component shift, against dense solves of
H + mu I (also for an indefinite H); the kernel's eigen-clamp-invert on D + mu I against newton.block_jacobi; the step's
decision rule as a numpy function with known answers; and an fp64 LM reference (dense per-sphere Hessians from the
matrix-form HVPs, the oracle's energies and inversion cubic) on a small mixed pack, which pins the algorithm and the step
counts the GPU runs are allowed.  GPU: the shifted solve's true residuals, one step against the public calls composed
with the numpy rule, convergence on the mixed 64 x 4096 pack, determinism and independence, handle variants and the
module route, and bookkeeping."""
import ctypes as C

import numpy as np
import pytest

from _helpers import GOLDEN
from test_pcg_device import (CHUNK, CONVERGED, NEGCURV, NEGCURV_FIRST, _shuffled_mesh, _spd,
                             batched_pcg_reference, jacobi_inverse_blocks, planes_of, sym6)
from tssplat_b200.mesh import connected_components, make_pack, perturb

ACTIVE, N_CONVERGED, STALLED = 0, 1, 2
ALPHAS = [2.0 ** -k for k in range(8)]
OPTS = dict(max_iter=20, rtol=1e-2, rel_floor=1e-6, tau=1e-3, mu_min=1e-12, mu_max=1e12, gtol=0.0, sigma=1e-4, eta=0.9,
            n_alpha=8)
COEF = (2e-4 / 3, 2e-4)
C3 = 1e-4
# steps the fp64 reference needs on its small mixed pack until every sphere is CONVERGED (test_lm_reference_*), and the
# allowance of the GPU runs on the 64 x 4096 mixed pack over that count
REF_STEPS = {False: 12, True: 20}
GPU_SLACK = 8
MAX_ROUNDING_FLIPS = 4        # tets one step may newly invert on a sphere through fp32 rounding (test_convergence_mixed_pack)


def f32(v):
    return float(np.float32(v))


# ---------------------------------------------------------------------------------------------------------------------
# the rule and the shifted solve in numpy


def batched_pcg_shifted(H_blocks, b, P, mu, max_iter, rtol):
    """batched_pcg_reference with a shift mu_c per component: the state machine on H_c + mu_c I (p.(Hp + mu p) in the
    curvature and r -= alpha (Hp + mu p) in the update are the operator H_c + mu_c I applied to p)."""
    return batched_pcg_reference([Hc + m * np.eye(len(Hc)) for Hc, m in zip(H_blocks, mu)], b, P, max_iter, rtol)


def new_state(S):
    return [dict(mu=None, nu=None, status=ACTIVE) for _ in range(S)]


def init_mu(st, maxD, o):
    """mu_c = tau * max (D_v)_ii on a sphere's first step, clamped to [mu_min, mu_max]; returns the fp32 shifts."""
    for s, m in zip(st, maxD):
        if s["mu"] is None:
            s["mu"] = min(f32(o["mu_max"]), max(f32(o["mu_min"]), f32(o["tau"]) * float(m)))
            s["nu"] = 2.0
    return np.array([s["mu"] for s in st], np.float32)


def decide(s, g, bd, dHd, mu_f, dd, dE, ahat, o, alphas=ALPHAS):
    """The decision of tsb_newton_step for one sphere (newton_decide_kernel, operation for operation in fp64): updates
    the state s (mu, nu, status) and returns (alpha, k, delta, rho).  bd and dHd are the solve's fp32 records, mu_f the
    fp32 shift the solve used, dE[k] = E(x + alpha_k d) - E(x) and ahat the inversion-free step over (0, 1], fp32."""
    if s["status"] != ACTIVE:
        return 0.0, -1, 0.0, 0.0
    if g <= f32(o["gtol"]):
        s["status"] = N_CONVERGED
        return 0.0, -1, 0.0, 0.0
    lim = f32(o["eta"]) * float(ahat)
    ks = -1
    if bd > 0.0:
        for k in range(o["n_alpha"]):
            a = alphas[k]
            if a < lim and float(dE[k]) <= -f32(o["sigma"]) * a * bd:
                ks = k
                break
    pred = bd - 0.5 * (dHd - float(mu_f) * dd)
    rho = -float(dE[0]) / pred if pred > 0.0 else 1.0
    if ks == 0:
        t = 2.0 * rho - 1.0
        s["mu"] = max(f32(o["mu_min"]), s["mu"] * max(1.0 / 3.0, 1.0 - t * t * t))
        s["nu"] = 2.0
    else:
        s["mu"] = min(f32(o["mu_max"]), s["mu"] * s["nu"])
        s["nu"] *= 2.0
    if ks < 0 and s["mu"] == f32(o["mu_max"]):
        s["status"] = STALLED
    return (alphas[ks], ks, float(dE[ks]), rho) if ks >= 0 else (0.0, -1, 0.0, rho)


# ---------------------------------------------------------------------------------------------------------------------
# CPU


def test_shifted_batched_pcg_against_dense_solves():
    rng = np.random.default_rng(11)
    m = 15
    Q = np.linalg.qr(rng.normal(size=(m, m)))[0]
    indef = (Q * np.r_[-2.0, -0.5, rng.uniform(0.5, 20, m - 2)]) @ Q.T          # two negative eigenvalues
    H = [_spd(rng, m), indef, _spd(rng, m, 1e-3, 1.0), indef]
    b = [rng.normal(size=m) for _ in H]
    b[3] = Q @ np.r_[1.0, 1.0, rng.normal(size=m - 2)]
    mu = [0.5, 2.5, 0.0, 2.5]                                                    # 2.5 > 2 = -lambda_min(indef)
    P = [np.diag(1.0 / np.maximum(np.diag(Hc) + m_, 1e-3)) for Hc, m_ in zip(H, mu)]
    res = batched_pcg_shifted(H, b, P, mu, 200, 1e-10)
    for c, r in enumerate(res):
        assert r["status"] == CONVERGED, (c, r["status"])
        A = H[c] + mu[c] * np.eye(m)
        assert np.allclose(r["d"], np.linalg.solve(A, b[c]), rtol=1e-7, atol=1e-9 * np.abs(r["d"]).max())
        assert abs(r["d_H_d"] - r["d"] @ A @ r["d"]) <= 1e-8 * abs(r["d_H_d"])        # d_H_d is d^T (H + mu I) d
    # unshifted, the indefinite components stop at negative curvature
    plain = batched_pcg_reference([H[1], H[3]], [b[1], b[3]], [None, None], 200, 1e-10)
    assert all(r["status"] in (NEGCURV, NEGCURV_FIRST) for r in plain)
    # a shift of 0 is the unshifted state machine, bitwise
    z = batched_pcg_shifted(H[:1], b[:1], [None], [0.0], 50, 1e-10)[0]
    u = batched_pcg_reference(H[:1], b[:1], [None], 50, 1e-10)[0]
    assert np.array_equal(z["d"], u["d"]) and z["n_hvp"] == u["n_hvp"]


def test_shifted_blocks_against_block_jacobi():
    """The kernel's eigen-clamp-invert on D + mu I (pcg_blocks_shift_kernel adds mu to the diagonal in fp64 before the
    Jacobi sweeps) against newton.block_jacobi of the shifted planes, within test_pcg_device's 8-ulp bound; a shift large
    enough turns every indefinite block SPD, so no block is clamped or zeroed."""
    import torch
    from tssplat_b200.newton import block_jacobi
    rng = np.random.default_rng(3)
    Q = np.linalg.qr(rng.normal(size=(300, 3, 3)))[0]
    lam = np.concatenate([rng.uniform(0.1, 10, size=(100, 3)), rng.uniform(-5, 5, size=(100, 3)),
                          np.c_[np.zeros((100, 2)), rng.uniform(0.1, 5, size=100)]])
    D = np.einsum("nij,nj,nkj->nik", Q, lam, Q)
    D = (0.5 * (D + D.transpose(0, 2, 1))).astype(np.float32).astype(np.float64)
    for mu in (1e-3, 0.7, 6.0):
        Dm = D + np.float64(np.float32(mu)) * np.eye(3)
        ref = sym6(block_jacobi(torch.from_numpy(planes_of(Dm)), rel_floor=1e-6).numpy())
        got = jacobi_inverse_blocks(Dm, np.float64(np.float32(1e-6))).astype(np.float32).astype(np.float64)
        scale = np.abs(ref).max(axis=1, keepdims=True)
        assert (np.abs(got - ref) <= 8 * 2.0 ** -24 * scale + 1e-300).all()
        if mu == 6.0:
            assert np.allclose(sym6(np.linalg.inv(Dm)), got, rtol=1e-5, atol=1e-6 * scale)


def _rule(s, **kw):
    a = dict(g=1.0, bd=1.0, dHd=1.5, mu_f=1.0, dd=1.0, dE=[-0.5] + [-0.3 * 2.0 ** -k for k in range(1, 8)], ahat=np.inf,
             o=dict(OPTS))
    a.update(kw)
    return decide(s, **a)


def test_decision_rule_known_answers():
    # rho = 1: pred = bd - (dHd - mu dd) / 2 = 1 - 0.25 = 0.75, dE(1) = -0.75: the full step, mu / 3, nu = 2
    s = dict(mu=3.0, nu=8.0, status=ACTIVE)
    assert _rule(s, dE=[-0.75] + [-0.1] * 7) == (1.0, 0, -0.75, 1.0)
    assert s == dict(mu=1.0, nu=2.0, status=ACTIVE)
    # rho > 1: the factor is clamped at 1/3 (1 - (2 rho - 1)^3 < 1/3)
    s = dict(mu=3.0, nu=2.0, status=ACTIVE)
    a, k, _, rho = _rule(s, dE=[-1.5] + [-0.1] * 7)
    assert (a, k) == (1.0, 0) and rho == 2.0 and s["mu"] == 1.0
    # 0 < rho < 1/2: the factor is 1 - (2 rho - 1)^3 > 1
    s = dict(mu=1.0, nu=2.0, status=ACTIVE)
    _, k, _, rho = _rule(s, dE=[-0.15] + [-0.1] * 7)
    assert k == 0 and abs(rho - 0.2) < 1e-15 and abs(s["mu"] - (1.0 - (2 * rho - 1) ** 3)) < 1e-15
    # rho < 0: the full step raises the energy; a shorter one is taken, mu * nu, nu doubles
    s = dict(mu=1.0, nu=4.0, status=ACTIVE)
    a, k, d, rho = _rule(s, dE=[0.2, -0.2] + [-0.01] * 6)
    assert (a, k, d) == (0.5, 1, -0.2) and rho < 0 and s == dict(mu=4.0, nu=8.0, status=ACTIVE)
    # the full step lies past eta * ahat: backtrack to the largest inversion-free Armijo step
    s = dict(mu=1.0, nu=2.0, status=ACTIVE)
    a, k, _, _ = _rule(s, ahat=np.float32(0.3))                 # 0.9 * 0.3 = 0.27: 1/4 is the first below
    assert (a, k) == (0.25, 2) and s["mu"] == 2.0
    s = dict(mu=1.0, nu=2.0, status=ACTIVE)
    assert _rule(s, ahat=np.float32(0.25))[:2] == (0.125, 3)  # 1/4 = 0.25 is not < 0.225
    # no step is acceptable: alpha = 0, k = -1
    s = dict(mu=1.0, nu=2.0, status=ACTIVE)
    assert _rule(s, dE=[1.0] * 8)[:3] == (0.0, -1, 0.0) and s == dict(mu=2.0, nu=4.0, status=ACTIVE)
    # Armijo's sufficient decrease: dE = -sigma alpha bd exactly passes, a hair above does not
    s = dict(mu=1.0, nu=2.0, status=ACTIVE)
    sig = f32(1e-4)
    assert _rule(s, dE=[-sig * 1.0] + [0.0] * 7)[1] == 0
    s = dict(mu=1.0, nu=2.0, status=ACTIVE)
    assert _rule(s, dE=[np.nextafter(-sig, 0.0)] + [0.0] * 7)[1] == -1
    # mu clamped at mu_min ...
    s = dict(mu=2e-12, nu=2.0, status=ACTIVE)
    _rule(s, dE=[-0.75] + [-0.1] * 7)
    assert s["mu"] == f32(1e-12)
    # ... and at mu_max, which with no step is STALLED (frozen)
    s = dict(mu=0.6e12, nu=2.0, status=ACTIVE)
    assert _rule(s, dE=[1.0] * 8)[1] == -1 and s["mu"] == f32(1e12) and s["status"] == STALLED
    assert _rule(s, dE=[-0.75] + [-0.1] * 7)[:2] == (0.0, -1) and s["status"] == STALLED        # stays frozen
    # mu_max reached while a shorter step was taken: not stalled
    s = dict(mu=0.6e12, nu=2.0, status=ACTIVE)
    assert _rule(s, dE=[1.0, -0.3] + [-0.1] * 6)[1] == 1 and s["mu"] == f32(1e12) and s["status"] == ACTIVE
    # g <= gtol: CONVERGED and frozen, mu untouched, and it stays frozen
    s = dict(mu=1.0, nu=2.0, status=ACTIVE)
    o = dict(OPTS, gtol=1e-3)
    assert _rule(s, g=f32(1e-3), o=o) == (0.0, -1, 0.0, 0.0) and s == dict(mu=1.0, nu=2.0, status=N_CONVERGED)
    assert _rule(s, g=1.0, o=o) == (0.0, -1, 0.0, 0.0) and s["status"] == N_CONVERGED
    # b.d <= 0: no step, even with an energy decrease
    for bd in (0.0, -1.0):
        s = dict(mu=1.0, nu=2.0, status=ACTIVE)
        assert _rule(s, bd=bd, dE=[-5.0] * 8)[:2] == (0.0, -1) and s["mu"] == 2.0
    # pred <= 0: rho = 1
    s = dict(mu=3.0, nu=2.0, status=ACTIVE)
    assert _rule(s, bd=1.0, dHd=10.0, dd=0.0)[3] == 1.0 and s["mu"] == 1.0
    # n_alpha limits the table
    s = dict(mu=1.0, nu=2.0, status=ACTIVE)
    assert _rule(s, ahat=np.float32(0.3), o=dict(OPTS, n_alpha=2))[:2] == (0.0, -1)


# ---------------------------------------------------------------------------------------------------------------------
# fp64 LM reference


class Fp64Problem:
    """Per-sphere fp64 energy, gradient, dense Hessian blocks, line search and inversion bound of a pack, from
    ReferenceEnergyOracle and the matrix-form HVPs of test_hvp / test_hvp_amips."""

    def __init__(self, pk, c1, c2, c3, order=2):
        from oracle.tet_energy_oracle import ReferenceEnergyOracle
        self.pk, self.orc = pk, ReferenceEnergyOracle(pk.verts, pk.tets)
        self.c1, self.c2, self.c3, self.order = c1, c2, c3, order
        self.vo, self.S = pk.vert_offsets, pk.num_spheres
        self.tsid = np.searchsorted(self.vo, pk.tets[:, 0], side="right") - 1

    def sphere_energy(self, x):
        from oracle.tet_energy_oracle import _det3
        x = np.asarray(x, np.float64).reshape(-1)
        Mx = self.orc.M @ x
        F = (self.orc.G @ x).reshape(-1, 3, 3)
        J = _det3(F)
        bar = np.maximum(-J, 0) ** self.order
        ok = J > 0
        tr = (F * F).sum(axis=(1, 2))
        psi = np.where(ok, tr / (3.0 * np.where(ok, J, 1.0) ** (2.0 / 3.0)) - 1.0, 0.0)
        sm = 0.5 * (x * Mx).reshape(-1, 3).sum(1)
        E = np.array([self.c1 * sm[self.vo[s]:self.vo[s + 1]].sum() for s in range(self.S)])
        E += np.bincount(self.tsid, self.c2 * bar + self.c3 * psi, minlength=self.S)
        return E, np.bincount(self.tsid, J < 0, minlength=self.S).astype(int)

    def grad(self, x):
        g = self.orc.backward(1.0, x, self.c1, self.c2, self.order)
        if self.c3:
            g = g + self.orc.amips_backward(1.0, x, self.c3)
        return g.reshape(-1)

    def hess_blocks(self, x):
        """Dense H_c per sphere: spheres share no vertices, so one HVP along the sum of every sphere's j-th unit vector
        gives column j of every block."""
        from test_hvp import hvp
        from test_hvp_amips import amips_hvp_terms
        m3 = 3 * np.diff(self.vo)
        H = [np.zeros((k, k)) for k in m3]
        for j in range(int(m3.max())):
            e = np.zeros(3 * len(self.pk.verts))
            for s in range(self.S):
                if j < m3[s]:
                    e[3 * self.vo[s] + j] = 1.0
            col = hvp(self.orc, x, e, self.c1, self.c2, self.order).reshape(-1)
            if self.c3:
                col = col + self.c3 * amips_hvp_terms(self.orc, x, e)[0]
            for s in range(self.S):
                if j < m3[s]:
                    H[s][:, j] = col[3 * self.vo[s]:3 * self.vo[s + 1]]
        return H

    def inversion_bound(self, x, d):
        from test_line_search import cubic_coeffs, first_root
        r = first_root(cubic_coeffs(self.orc, x, d), 1.0)
        out = np.full(self.S, np.inf)
        np.minimum.at(out, self.tsid, r)
        return out


def lm_reference(P, x0, n_steps, o, record=None):
    """tsb_newton_step's algorithm in fp64: -grad, diagonal blocks, mu init, the shifted PCG state machine with the
    kernel's block preconditioner, the line search from the oracle's energies and cubic, the rule, the step."""
    x = np.asarray(x0, np.float64).reshape(-1).copy()
    st = new_state(P.S)
    hist = []
    for _ in range(n_steps):
        b = -P.grad(x)
        H = P.hess_blocks(x)
        for s in range(P.S):
            if st[s]["status"] != ACTIVE:
                b[3 * P.vo[s]:3 * P.vo[s + 1]] = 0.0
        D = [np.stack([Hc[3 * i:3 * i + 3, 3 * i:3 * i + 3] for i in range(len(Hc) // 3)]) for Hc in H]
        mu_f = init_mu(st, [Dc[:, [0, 1, 2], [0, 1, 2]].max() for Dc in D], o)
        Pc = []
        for Dc, m in zip(D, mu_f):
            inv = jacobi_inverse_blocks(Dc + float(m) * np.eye(3), o["rel_floor"])
            B = np.zeros((3 * len(Dc), 3 * len(Dc)))
            for i, q in enumerate(inv):
                B[3 * i:3 * i + 3, 3 * i:3 * i + 3] = [[q[0], q[5], q[4]], [q[5], q[1], q[3]], [q[4], q[3], q[2]]]
            Pc.append(B)
        bs = [b[3 * P.vo[s]:3 * P.vo[s + 1]] for s in range(P.S)]
        sol = batched_pcg_shifted(H, bs, Pc, [float(m) for m in mu_f], o["max_iter"], o["rtol"])
        d = np.concatenate([r["d"] for r in sol])
        E0, inv0 = P.sphere_energy(x)
        dE = np.stack([P.sphere_energy(x + a * d)[0] - E0 for a in ALPHAS[:o["n_alpha"]]], axis=1)
        ahat = P.inversion_bound(x, d)
        step = []
        for s, r in enumerate(sol):
            g = float(np.linalg.norm(bs[s]))
            out = decide(st[s], g, r["b_dot_d"], r["d_H_d"], mu_f[s], float(sol[s]["d"] @ sol[s]["d"]), dE[s], ahat[s], o)
            step.append(dict(zip(("alpha", "k", "delta", "rho"), out), g=g, mu=st[s]["mu"], status=st[s]["status"],
                             pcg=r["status"], E0=E0[s], inv0=inv0[s], bd=r["b_dot_d"], dHd=r["d_H_d"], mu_f=float(mu_f[s]),
                             dd=float(sol[s]["d"] @ sol[s]["d"])))
        for s in range(P.S):
            x[3 * P.vo[s]:3 * P.vo[s + 1]] += step[s]["alpha"] * sol[s]["d"]
        hist.append(step)
    E, inv = P.sphere_energy(x)
    return x, hist, E, inv


_REF = {}


def _ref_run(amips):
    if amips not in _REF:
        pk = make_pack(3, 256, seed=4)
        x = perturb(pk, sigma_rel=0.02, seed=1).astype(np.float64)
        rough = perturb(pk, sigma_rel=0.35, seed=3)
        x[pk.vert_offsets[0]:pk.vert_offsets[1]] = rough[pk.vert_offsets[0]:pk.vert_offsets[1]]
        P = Fp64Problem(pk, *COEF, C3 if amips else 0.0)
        g0 = [np.linalg.norm(P.grad(x)[3 * P.vo[s]:3 * P.vo[s + 1]]) for s in range(P.S)]
        o = dict(OPTS, gtol=1e-3 * min(g0))                # |g_c| down by 1e3 for the sphere that starts lowest
        _REF[amips] = (P, x, o, lm_reference(P, x, REF_STEPS[amips] + 3, o))
    return _REF[amips]


@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_lm_reference_mixed_pack(amips):
    P, x0, o, (x, hist, E, inv) = _ref_run(amips)
    assert hist[0][0]["inv0"] > 0 and all(h["inv0"] == 0 for h in hist[0][1:])      # sphere 0 starts with inverted tets
    from oracle.tet_energy_oracle import _det3
    J0 = _det3((P.orc.G @ x0.reshape(-1)).reshape(-1, 3, 3))
    J = _det3((P.orc.G @ x).reshape(-1, 3, 3))
    assert not ((J0 > 0) & (J <= 0)).any()                                         # no tet with J > 0 inverts
    for t, step in enumerate(hist):
        nxt = hist[t + 1] if t + 1 < len(hist) else None
        for s, r in enumerate(step):
            E1 = nxt[s]["E0"] if nxt else E[s]
            assert E1 <= r["E0"] + 1e-12 * abs(r["E0"]), (t, s)                     # energy never increases
            assert abs((E1 - r["E0"]) - r["delta"]) <= 1e-9 * abs(r["E0"])          # the line search's change is the step's
            if nxt:
                assert nxt[s]["inv0"] <= r["inv0"]
    conv = [next((t for t, step in enumerate(hist) if step[s]["status"] == N_CONVERGED), None) for s in range(P.S)]
    print(f"amips={amips}: converged at steps {conv}, mu {[h['mu'] for h in hist[-1]]}, "
          f"k {[[h['k'] for h in step] for step in hist]}")
    assert all(c is not None and c <= REF_STEPS[amips] for c in conv), conv


def test_lm_reference_full_step_rho_is_one():
    """AMIPS off and no inverted tet: the energy is c1/2 x^T M x, quadratic, so a first step that takes the full step
    has rho = 1 to rounding, whatever mu is."""
    P, x0, o, (x, hist, E, inv) = _ref_run(False)
    quiet = [h for h in hist[0][1:]]
    assert all(h["inv0"] == 0 and h["k"] == 0 for h in quiet)
    for h in quiet:
        # the solve's records here are fp64 (the kernel's are fp32), so rho is exact up to the CG recurrence's rounding
        assert abs(h["rho"] - 1.0) <= 1e-9, h["rho"]
        assert h["mu_f"] > 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU


def _torch():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch


@pytest.fixture(scope="module")
def ext():
    _torch()
    from tssplat_b200 import tet_spheres_ext
    return tet_spheres_ext


def _handle(ext, V, T, **kw):
    return ext.TetSpheres(np.ascontiguousarray(V, np.float32).reshape(-1), np.ascontiguousarray(T, np.int32).reshape(-1), **kw)


def _cuda(a):
    return _torch().from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


_PACKS = {}


def _pack(name):
    """(pack, x): "big" = 64 x 4096 near rest (0.02 h); "mixed" = the same pack with every fourth sphere at 0.35 h;
    "small" = make_pack(3, 512) with sphere 0 at 0.35 h."""
    if name not in _PACKS:
        pk = make_pack(3, 512, seed=4) if name == "small" else make_pack(64, 4096, seed=0, unique=8)
        x = perturb(pk, sigma_rel=0.02, seed=1)
        if name != "big":
            rough = perturb(pk, sigma_rel=0.35, seed=3)
            for s in range(0, pk.num_spheres, 4):
                x[pk.vert_offsets[s]:pk.vert_offsets[s + 1]] = rough[pk.vert_offsets[s]:pk.vert_offsets[s + 1]]
        _PACKS[name] = (pk, x)
    return _PACKS[name]


def _labels(V, T):
    """(sphere id per vertex, 0 on orphans; orphan mask; S)."""
    lab = connected_components(len(V), T)
    used = np.zeros(len(V), bool)
    used[np.unique(T)] = True
    return np.where(used, np.searchsorted(np.unique(lab[used]), lab), 0), ~used, len(np.unique(lab[used]))


def _seg_sum(torch, v, sid, S):
    return torch.zeros(S, dtype=torch.float64, device=v.device).index_add_(0, sid, v)


def _sphere_max_diag(torch, planes, sid, orph, S):
    m = planes[0].max(dim=1).values.masked_fill(orph, -np.inf)
    return torch.full((S,), -np.inf, dtype=torch.float32, device=m.device).scatter_reduce_(0, sid, m, "amax")


@pytest.mark.gpu
@pytest.mark.parametrize("mesh", ["big", "a_veg", "shuffled"])
def test_damped_solve_true_residual_and_blocks(ext, mesh):
    """(H + mu_c I) d = b to rtol on every CONVERGED sphere, from tsb_hvp_ex plus mu d; the shifted blocks against
    block_jacobi of D + mu I; shift = None is bitwise the unshifted calls."""
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DevicePCG, block_jacobi
    if mesh == "big":
        pk, x_np = _pack("big")
        V, T, kw = pk.verts, pk.tets, {}
    elif mesh == "a_veg":
        d = np.load(GOLDEN + "/a_veg_mesh.npz")
        V, T = d["verts"].astype(np.float32), d["tets"].astype(np.int32)
        h = np.linalg.norm(V[T[:, 1]] - V[T[:, 0]], axis=1).mean()
        x_np, kw = (V + np.random.default_rng(6).normal(scale=0.02 * h, size=V.shape)).astype(np.float32), dict(force_global=True)
    else:
        V, T, x_np = _shuffled_mesh()
        kw = {}
    sp = _handle(ext, V, T, enable_amips=True, deterministic=True, **kw)
    sid_np, orph_np, S = _labels(V, T)
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    x = _cuda(x_np)
    c1, c2 = COEF
    _, g = sp.energy_grad(x, c1, c2, 2, c3=C3)
    b = -g
    planes = sp.hess_diag(x, c1, c2, 2, c3=C3)
    mx = _sphere_max_diag(torch, planes, sid, orph, S)
    mu = (mx * torch.tensor([1e-3, 1e-2, 1e-1], device="cuda").repeat(S)[:S]).contiguous()     # a different shift per sphere
    ws = DevicePCG(sp)
    inv = ws.set_blocks(planes, want_inverse=True, shift=mu).double().cpu().numpy()
    P = planes.double().cpu().clone()
    mu_v = torch.where(orph, 0.0, mu[sid].double()).cpu()
    P[0] += mu_v[:, None]
    ref = sym6(block_jacobi(P, rel_floor=1e-6).numpy())
    scale = np.abs(ref).max(axis=1, keepdims=True)
    assert (np.abs(inv - ref) <= 8 * 2.0 ** -24 * scale).all()
    assert not inv[orph_np].any()
    rtol = 1e-3
    res = ws.solve(x, b, c1, c2, 2, c3=C3, max_iter=2000, rtol=rtol, check_every=25, shift=mu)
    conv = res.status == CONVERGED
    assert conv.any()
    d = res.d
    r = b - sp.hvp(x, d, c1, c2, 2, c3=C3)[0] - mu[sid][:, None] * d
    true_res = _seg_sum(torch, (r.double() ** 2).sum(1).masked_fill(orph, 0), sid, S).sqrt() / \
        _seg_sum(torch, (b.double() ** 2).sum(1).masked_fill(orph, 0), sid, S).sqrt()
    assert (true_res[conv] <= 1.2 * rtol).all(), float(true_res[conv].max())
    dHd = _seg_sum(torch, (d.double() * (b - r).double()).sum(1), sid, S)          # d^T (H + mu I) d
    assert torch.allclose(res.d_H_d.double()[conv], dHd[conv], rtol=2e-2)
    assert not d[orph].any()
    # shift = None: the unshifted calls, bitwise
    ws.set_blocks(planes)
    a = ws.solve(x, b, c1, c2, 2, c3=C3, max_iter=30, rtol=rtol)
    d0 = torch.empty_like(d)
    rec = torch.zeros((S, 8), dtype=torch.int32, device="cuda")
    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=C3)
    opt = _capi.tsb_pcg_options_t(max_iter=30, rtol=rtol, check_every=0)
    st = torch.cuda.current_stream().cuda_stream
    inv0 = torch.empty((len(V), 6), device="cuda")
    assert _capi.lib.tsb_pcg_set_blocks(ws._s, planes.data_ptr(), 1e-6, inv0.data_ptr(), st) == 0
    assert _capi.lib.tsb_pcg_solve(ws._s, x.data_ptr(), b.data_ptr(), C.byref(terms), C.byref(opt), d0.data_ptr(),
                                   rec.data_ptr(), None, st) == 0
    assert torch.equal(a.d, d0) and torch.equal(a.status, rec[:, 4]) and torch.equal(a.n_hvp, rec[:, 3])
    assert torch.equal(ws.set_blocks(planes, want_inverse=True), inv0)


@pytest.mark.gpu
def test_shift_converges_where_unshifted_stops_at_negative_curvature(ext):
    """The mixed 64 x 4096 pack with AMIPS on and c1 = 2e-4 / 64: the quiet spheres' Hessian is indefinite, so the
    unshifted solve stops at negative curvature; shifted by the damping of a first Newton step they converge."""
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _pack("mixed")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    x = _cuda(x_np)
    c1, c2 = 2e-4 / 64, 2e-4
    _, g = sp.energy_grad(x, c1, c2, 2, c3=C3)
    planes = sp.hess_diag(x, c1, c2, 2, c3=C3)
    ws = DevicePCG(sp)
    ws.set_blocks(planes)
    quiet = torch.arange(pk.num_spheres, device="cuda") % 4 != 0
    plain = ws.solve(x, -g, c1, c2, 2, c3=C3, max_iter=600, rtol=1e-3, check_every=25)
    neg = torch.isin(plain.status[quiet], torch.tensor([NEGCURV, NEGCURV_FIRST], device="cuda"))
    assert int(neg.sum()) >= 0.9 * int(quiet.sum()), plain.status
    sid = torch.from_numpy(np.repeat(np.arange(pk.num_spheres), np.diff(pk.vert_offsets))).cuda()
    mu = (1e-2 * _sphere_max_diag(torch, planes, sid, torch.zeros_like(sid, dtype=torch.bool), pk.num_spheres)).contiguous()
    ws.set_blocks(planes, shift=mu)
    damped = ws.solve(x, -g, c1, c2, 2, c3=C3, max_iter=600, rtol=1e-3, check_every=25, shift=mu)
    print(f"unshifted products (quiet) {float(plain.n_hvp[quiet].float().mean()):.1f}; damped {float(damped.n_hvp[quiet].float().mean()):.1f}")
    assert (damped.status[quiet] == CONVERGED).all(), damped.status
    assert (plain.status[quiet][neg] != CONVERGED).all()


def _compose_step(torch, sp, ws, x, st, c1, c2, c3, o, sid, orph, S):
    """One tsb_newton_step from the public calls and the numpy rule; st is the per-sphere state, updated.  Returns the
    new x and per sphere (alpha, k, status, mu)."""
    _, b = sp.energy_grad(x, c1, c2, 2, -1.0, c3=c3)
    frozen = torch.tensor([s["status"] != ACTIVE for s in st], device="cuda")
    b = torch.where(frozen[sid][:, None] & ~orph[:, None], torch.zeros_like(b), b)
    planes = sp.hess_diag(x, c1, c2, 2, c3=c3)
    shift = torch.from_numpy(init_mu(st, _sphere_max_diag(torch, planes, sid, orph, S).cpu().numpy(), o)).cuda()
    ws.set_blocks(planes, rel_floor=o["rel_floor"], shift=shift)
    res = ws.solve(x, b, c1, c2, 2, c3=c3, max_iter=o["max_iter"], rtol=o["rtol"], shift=shift)
    ls = sp.line_search(x, res.d, ALPHAS[:o["n_alpha"]], c1, c2, 2, c3=c3, per_sphere=True)
    keep = ~orph
    gn = _seg_sum(torch, (b.double() ** 2).sum(1)[keep], sid[keep], S).sqrt().cpu().numpy()
    dd = _seg_sum(torch, (res.d.double() ** 2).sum(1)[keep], sid[keep], S).cpu().numpy()
    bd, dHd, sd, ss = (t.cpu().numpy() for t in (res.b_dot_d, res.d_H_d, ls.sphere_delta[:, :, 0], ls.sphere_max_step))
    out = [decide(st[c], float(gn[c]), float(bd[c]), float(dHd[c]), shift[c].item(), float(dd[c]), sd[c], ss[c], o)
           for c in range(S)]
    a = torch.tensor([r[0] for r in out], dtype=torch.float32, device="cuda")
    return ws.axpy(x, a, res.d), out


@pytest.mark.gpu
@pytest.mark.parametrize("c3", [0.0, C3], ids=["amips-off", "amips-on"])
def test_step_equals_its_composition(ext, c3):
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    sid_np, orph_np, S = _labels(pk.verts, pk.tets)
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    o = dict(OPTS, gtol=0.05)
    x1, x2 = _cuda(x_np), _cuda(x_np)
    st = new_state(S)
    n_conv = 0
    for t in range(6):
        r = nw.step(x1, c1, c2, 2, c3=c3, **o)
        x2, out = _compose_step(torch, sp, nw.pcg, x2, st, c1, c2, c3, o, sid, orph, S)
        assert torch.equal(x1, x2), t
        assert r.k.cpu().tolist() == [q[1] for q in out] and r.alpha.cpu().tolist() == [q[0] for q in out]
        assert r.status.cpu().tolist() == [s["status"] for s in st]
        assert np.allclose(r.mu.cpu().numpy(), [s["mu"] for s in st], rtol=1e-12, atol=0)
        n_conv = int((r.status == N_CONVERGED).sum())
    assert n_conv >= 1                                   # the rule's CONVERGED branch was exercised


def _stats(E, x, it):
    st = E.sphere_stats(x, it)
    c1, c2 = E.coeff_scheduler(it)
    return (c1 * st.smooth + c2 * st.barrier + E.amips_coeff * st.amips), st.n_inverted


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_convergence_mixed_pack(ext, amips):
    """The mixed 64 x 4096 pack through SmoothnessBarrierEnergy.newton_step: every step's per-sphere energy change is
    <= 0 and a fresh sphere_stats launch agrees with the start plus the summed deltas (with AMIPS on, on the quiet spheres:
    a rough sphere un-inverts tets to J just above 0, where psi ~ J^(-2/3) makes an fp32 re-evaluation of the energy
    meaningless); the inverted-tet count never grows
    on the quiet spheres; every quiet sphere ends CONVERGED within the fp64 reference's step count plus GPU_SLACK.  On the
    rough spheres the inversion bound holds for the line search's own cubic: a tet whose J sits a few roundings above 0
    can still come out inverted once x + alpha d is rounded to fp32 (a handful of tets out of ~12 000 over the run, while
    the rough spheres' inverted count falls by hundreds), so there the total must fall and no step may add more than
    MAX_ROUNDING_FLIPS."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    pk, x_np = _pack("mixed")
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000,
                                                        amips_coeff=C3 if amips else 0.0, deterministic=True))
    x = torch.nn.Parameter(_cuda(x_np))
    it = 0
    e_start, inv_start = _stats(E, x, it)
    g0 = E.newton_step(x.detach().clone(), it, max_iter=1).grad_norm        # |g_c| at the start (x untouched)
    E.device_newton.reset()
    quiet = torch.arange(pk.num_spheres, device="cuda") % 4 != 0
    gtol = 1e-3 * float(g0[quiet].min())
    acc = torch.zeros(pk.num_spheres, dtype=torch.float64, device="cuda")
    inv_prev = inv_start
    n = REF_STEPS[amips] + GPU_SLACK
    for t in range(n):
        r = E.newton_step(x, it, gtol=gtol)
        assert (r.delta <= 0).all(), t
        acc += r.delta.double()
        e, inv = _stats(E, x, it)
        # the line search's deltas are cancellation-free fp32 sums; sphere_stats sums fp32 per-tet energies
        tol = 1e-4 * e_start.abs()
        err = (e - e_start - acc).abs()
        checked = quiet if amips else torch.ones_like(quiet)
        assert (err[checked] <= tol[checked]).all(), (t, float((err / tol)[checked].max()))
        assert (inv[quiet] <= inv_prev[quiet]).all(), t
        up = (inv - inv_prev).clamp(min=0)
        assert int(up.max()) <= MAX_ROUNDING_FLIPS, (t, up)
        if up.any():
            print(f"step {t}: {int(up.sum())} tet(s) newly inverted by fp32 rounding on the rough spheres")
        inv_prev = inv
    assert int(inv[~quiet].sum()) < int(inv_start[~quiet].sum())
    st = r.status
    print(f"amips={amips}: status {st.cpu().tolist()}, gtol {gtol:.3e}, mu range {float(r.mu.min()):.3e}..{float(r.mu.max()):.3e}, "
          f"inverted {inv_start[~quiet].sum().item()} -> {inv[~quiet].sum().item()}")
    assert (st[quiet] == N_CONVERGED).all(), st


def _run_steps(torch, nw, x, n, c1, c2, c3, **o):
    """n steps; every record field of every step as raw bits in one int32 tensor."""
    recs = [nw.step(x, c1, c2, 2, c3=c3, **o) for _ in range(n)]
    return torch.cat([torch.cat([f.reshape(-1).contiguous().view(torch.int32) for f in r]) for r in recs])


@pytest.mark.gpu
def test_determinism_graphs_and_independence(ext):
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("mixed")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    o = dict(max_iter=10)

    def run(x0):
        nw.reset()
        x = x0.clone()
        out = _run_steps(torch, nw, x, 10, c1, c2, C3, **o)
        torch.cuda.synchronize()
        return x, out

    x0 = _cuda(x_np)
    xa, ra = run(x0)
    xb, rb = run(x0)
    assert torch.equal(xa, xb) and torch.equal(ra, rb)
    other = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(other):
        xc, rc = run(x0)
    assert torch.equal(xa, xc) and torch.equal(ra, rc)
    # the 10 steps captured in one CUDA graph, replayed twice
    xg = x0.clone()
    nw.reset()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):                         # warm-up outside the capture (allocator)
        _run_steps(torch, nw, x0.clone(), 1, c1, c2, C3, **o)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        nw.reset()
        rg = _run_steps(torch, nw, xg, 10, c1, c2, C3, **o)
    for _ in range(2):
        xg.copy_(x0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(xg, xa) and torch.equal(rg, ra)
    # another start for sphere 5 only: every other sphere's trajectory bitwise unchanged
    vo = pk.vert_offsets
    x1 = x0.clone()
    x1[vo[5]:vo[6]] += 0.01 * torch.randn_like(x1[vo[5]:vo[6]])
    nw.reset()
    xs = x1.clone()
    recs = [nw.step(xs, c1, c2, 2, c3=C3, **o) for _ in range(10)]
    nw.reset()
    xr = x0.clone()
    refs = [nw.step(xr, c1, c2, 2, c3=C3, **o) for _ in range(10)]
    keep = torch.ones(len(x0), dtype=torch.bool, device="cuda")
    keep[vo[5]:vo[6]] = False
    others = torch.arange(pk.num_spheres, device="cuda") != 5
    assert torch.equal(xs[keep], xr[keep]) and not torch.equal(xs[~keep], xr[~keep])
    for p, q in zip(recs, refs):
        for f in p._fields:
            assert torch.equal(getattr(p, f)[others], getattr(q, f)[others]), f


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(warps_per_cta=8), dict(warps_per_cta=16), dict(force_global=True)], ids=["w8", "w16", "global"])
def test_handle_variants_and_orphans(ext, kw):
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    V, T, x_np = _shuffled_mesh()
    sp = _handle(ext, V, T, deterministic=True, **kw)
    assert sp.info["mode_global"] == int(bool(kw.get("force_global")))
    _, orph_np, S = _labels(V, T)
    orph = torch.from_numpy(orph_np).cuda()
    x = _cuda(x_np)
    x0 = x.clone()
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    for _ in range(8):
        r = nw.step(x, c1, c2, 2)
        assert torch.equal(x[orph], x0[orph])
        assert (r.delta <= 0).all() and not torch.isnan(x).any()
    st = sp.energy_grad_spheres(x, c1, c2, 2, want_grad=False)[2]
    st0 = sp.energy_grad_spheres(x0, c1, c2, 2, want_grad=False)[2]
    assert (c1 * st.smooth + c2 * st.barrier < c1 * st0.smooth + c2 * st0.barrier).all()


@pytest.mark.gpu
def test_module_and_ext_routes(ext):
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    pk, x_np = _pack("small")
    flags = dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000, deterministic=True)
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    x = torch.nn.Parameter(_cuda(x_np))
    it = 5
    c1, c2 = E.coeff_scheduler(it)
    r = E.newton_step(x, it, max_iter=15)
    assert E.device_newton.pcg is E.device_pcg and (r.alpha > 0).any() and not torch.equal(x.detach(), _cuda(x_np))
    # the same step through tet_spheres_ext on a second module's handle
    from tssplat_b200.newton import DeviceNewton
    E2 = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    nw = DeviceNewton(E2.tet_sp)
    y = _cuda(x_np)
    r2 = ext.newton_step(y, nw, c1, c2, E2.order_at(it), max_iter=15)
    assert torch.equal(y, x.detach()) and torch.equal(r2.mu, r.mu)
    # minimize: check_every reads the active count and stops at 0 (quiet start: every sphere converges)
    nw.reset()
    y = _cuda(perturb(pk, sigma_rel=0.02, seed=1))
    n, last = nw.minimize(y, 200, c1, c2, 2, check_every=5, gtol=1e-2 * float(r.grad_norm.max()))
    assert n < 200 and n % 5 == 0 and int((last.status == ACTIVE).sum()) == 0


@pytest.mark.gpu
def test_bookkeeping(ext):
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DeviceNewton, DevicePCG
    pk, x_np = _pack("small")
    a = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    b_ = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    info0 = dict(a.info)
    ws = DevicePCG(a)
    pcg_bytes = ws.device_bytes
    nw = DeviceNewton(a, ws)
    info = _capi.tsb_info_t()
    _capi.check(_capi.lib.tsb_get_info(a._h, C.byref(info)), a._h)
    assert {k: getattr(info, k) for k, _ in _capi.tsb_info_t._fields_} == info0
    assert int(_capi.lib.tsb_pcg_device_bytes(ws._s)) == pcg_bytes
    n, S = a.n, a.info["n_components"]
    chunks = int(sum(-(-int(m) // CHUNK) for m in np.diff(pk.vert_offsets)))
    assert nw.device_bytes == 48 * n + 24 * chunks + 172 * S + 176
    # chaining: after a step on the stream, the handle's other calls give what a fresh handle gives
    x = _cuda(x_np)
    c1, c2 = COEF
    y = x.clone()
    nw.step(y, c1, c2, 2, c3=C3)
    outs = []
    for h in (a, b_):
        e, g = h.energy_grad(y, c1, c2, 2, c3=C3)
        outs.append((e.clone(), g, h.hvp(y, x, c1, c2, 2, c3=C3)[0], h.hess_diag(y, c1, c2, 2, c3=C3)))
    torch.cuda.synchronize()
    for p, q in zip(*outs):
        assert torch.equal(p, q)
    # argument errors: nothing launched
    E = _capi.TSB_E_INVALID
    st = torch.cuda.current_stream().cuda_stream
    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=0.0)
    z = x.clone()
    for bad in (dict(max_iter=0), dict(rtol=-1.0), dict(rel_floor=float("nan")), dict(tau=0.0), dict(tau=float("inf")),
                dict(mu_min=0.0), dict(mu_min=2.0, mu_max=1.0), dict(mu_max=float("inf")), dict(gtol=-1.0),
                dict(sigma=0.0), dict(sigma=1.0), dict(eta=0.0), dict(eta=1.5), dict(n_alpha=0), dict(n_alpha=9)):
        o = nw.options(**bad)
        assert _capi.lib.tsb_newton_step(nw._nw, z.data_ptr(), C.byref(terms), C.byref(o), None, st) == E, bad
    o = nw.options()
    o.reserved[2] = 1
    assert _capi.lib.tsb_newton_step(nw._nw, z.data_ptr(), C.byref(terms), C.byref(o), None, st) == E
    o = nw.options()
    assert _capi.lib.tsb_newton_step(nw._nw, None, C.byref(terms), C.byref(o), None, st) == E
    assert _capi.lib.tsb_newton_step(nw._nw, z.data_ptr(), None, C.byref(o), None, st) == E
    assert _capi.lib.tsb_newton_step(nw._nw, z.data_ptr(), C.byref(terms), None, None, st) == E
    assert _capi.lib.tsb_newton_step(None, z.data_ptr(), C.byref(terms), C.byref(o), None, st) == E
    bad_order = _capi.tsb_terms_t(c1=c1, c2=c2, order=3, c3=0.0)
    assert _capi.lib.tsb_newton_step(nw._nw, z.data_ptr(), C.byref(bad_order), C.byref(o), None, st) == E
    torch.cuda.synchronize()
    assert torch.equal(z, x)
    plain = _handle(ext, pk.verts, pk.tets)
    pn = DeviceNewton(plain)
    with pytest.raises(RuntimeError, match="enable_amips"):
        pn.step(z, c1, c2, 2, c3=0.5)
    with pytest.raises(TypeError):
        pn.step(z, c1, c2, 2, bogus=1)
    with pytest.raises(RuntimeError, match="another handle"):
        DeviceNewton(plain, ws)
    out = C.c_void_p()
    assert _capi.lib.tsb_newton_create(None, C.byref(out)) == E and _capi.lib.tsb_newton_create(ws._s, None) == E
    # minimize with check_every > 0 is refused while capturing; the capture survives and nothing was recorded
    graph = torch.cuda.CUDAGraph()
    w = x.clone()
    with torch.cuda.graph(graph):
        w.add_(1.0)
        with pytest.raises(RuntimeError, match="captured"):
            nw.minimize(w, 3, c1, c2, 2, check_every=1)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(w, x + 1.0)

"""The damped (Levenberg-Marquardt) Newton step: tsb_pcg_set_blocks_ex / tsb_pcg_solve_ex (the shifted solve),
tsb_newton_* (the step), newton.DeviceNewton and SmoothnessBarrierEnergy.newton_step.

CPU: the batched PCG state machine of _newton_model extended with a per-component shift, against dense solves of
H + mu I (also for an indefinite H); the kernel's eigen-clamp-invert on D + mu I against newton.block_jacobi; the step's
decision rule with known answers; the fp64 reference's full steps on the quiet spheres.  GPU: the shifted solve's true
residuals, the module route, and bookkeeping.  What the damped step shares with the other Newton steps (the fp64
reference's step counts, the step against its composition, convergence, determinism, handle variants) runs through
the shared checks of _newton_checks."""
import ctypes as C

import numpy as np
import pytest

from _helpers import GOLDEN
from _newton_checks import (check_composition, check_convergence, check_determinism, check_handle_variants,
                            check_reference)
from _newton_model import (ACTIVE, C3, CHUNK, COEF, CONVERGED, N_CONVERGED, NEGCURV, NEGCURV_FIRST, OPTS, STALLED,  # noqa: F401
                           _cuda, _handle, _labels, _pack, _seg_sum, _shuffled_mesh, _spd, _sphere_max_diag, _torch,
                           batched_pcg_reference, decide_damped, ext, f32, jacobi_inverse_blocks, planes_of, reference_run,
                           sym6)
from tssplat_b200.mesh import perturb


# ---------------------------------------------------------------------------------------------------------------------
# the shifted solve in numpy


def batched_pcg_shifted(H_blocks, b, P, mu, max_iter, rtol):
    """batched_pcg_reference with a shift mu_c per component: the state machine on H_c + mu_c I (p.(Hp + mu p) in the
    curvature and r -= alpha (Hp + mu p) in the update are the operator H_c + mu_c I applied to p)."""
    return batched_pcg_reference([Hc + m * np.eye(len(Hc)) for Hc, m in zip(H_blocks, mu)], b, P, max_iter, rtol)


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
    return decide_damped(s, **a)


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


def test_lm_reference_full_step_rho_is_one():
    """AMIPS off and no inverted tet: the energy is c1/2 x^T M x, quadratic, so a first step that takes the full step
    has rho = 1 to rounding, whatever mu is."""
    hist = reference_run("lm", "amips-off")[7]
    quiet = [h for h in hist[0][1:]]
    assert all(h["inv0"] == 0 and h["k"] == 0 for h in quiet)
    for h in quiet:
        # the solve's records here are fp64 (the kernel's are fp32), so rho is exact up to the CG recurrence's rounding
        assert abs(h["rho"] - 1.0) <= 1e-9, h["rho"]
        assert h["mu_f"] > 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU


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


# ---------------------------------------------------------------------------------------------------------------------
# the checks every Newton step shares (_newton_checks)


@pytest.mark.parametrize("variant", ["amips-off", "amips-on"])
def test_lm_reference_mixed_pack(variant):
    check_reference("lm", variant)


@pytest.mark.gpu
@pytest.mark.parametrize("c3", [0.0, C3], ids=["amips-off", "amips-on"])
def test_step_equals_its_composition(ext, c3):
    check_composition(ext, "lm", c3, prox=False)


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_convergence_mixed_pack(ext, amips):
    check_convergence(ext, "lm", amips)


@pytest.mark.gpu
def test_determinism_graphs_and_independence(ext):
    check_determinism(ext, "lm")


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["w8", "w16", "global"])
def test_handle_variants_and_orphans(ext, variant):
    check_handle_variants(ext, "lm", variant)

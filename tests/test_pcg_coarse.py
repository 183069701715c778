"""The affine coarse space of the per-sphere solve (tsb_pcg_enable_coarse, tsb_pcg_set_coarse, tsb_pcg_coarse_matrix and
the two-level tsb_pcg_apply_precond): the closed-form coarse matrix against Z^T H Z in fp64, the host tables, the fp64
two-level PCG model, and on the device the coarse matrix and the preconditioner against fp64, the no-op case, bitwise
repeatability of solves and Newton steps, the products it saves, memory and the argument rules."""
import numpy as np
import pytest

from _coarse_model import (coarse_matrices, coarse_tables, fspace_closed_form, pinv_floor, shift_term, sphere_basis,
                           two_level_pcg)
from _newton_model import (COEF, GPU_SLACK, PROX_REF_STEPS, PSD_REF_STEPS, REF_STEPS, Fp64Problem, _cuda, _handle, _labels,
                           _pack, _torch, _weights, block_preconditioner, dense_sphere_hessians, ext)
from tssplat_b200.mesh import make_pack, perturb

U = 2.0 ** -24
C3 = 1e-4


def _small(rough):
    pk = make_pack(2, 512, seed=4)
    return pk, perturb(pk, sigma_rel=0.35 if rough else 0.02, seed=1)


# ---- CPU ----

@pytest.mark.parametrize("amips,project,rough", [(False, False, False), (True, False, False), (True, True, False),
                                                 (False, False, True), (True, False, True), (False, True, True)])
def test_closed_form_is_ZtHZ(amips, project, rough):
    """E_c = sum_t c2 H_b + c3 H_a equals Z^T H Z of the dense sphere Hessian to 1e-10 of |Z|^T |H| |Z|; c1 does not
    enter it, and H annihilates translations up to the c1 M term's rounding."""
    from oracle.tet_energy_oracle import ReferenceEnergyOracle
    pk, x = _small(rough)
    orc = ReferenceEnergyOracle(pk.verts, pk.tets)
    c1, c2 = COEF
    c3 = C3 if amips else 0.0
    E, _ = coarse_matrices(orc, pk, x, c2, c3, 2, project)
    H = dense_sphere_hessians(orc, pk, x, c1, c2, c3, 2, project)
    M = dense_sphere_hessians(orc, pk, x, 1.0, 0.0, 0.0, 2, False)
    for s in range(pk.num_spheres):
        Z, _ = sphere_basis(pk, s, round32=False)
        ref = Z.T @ H[s] @ Z
        scale = (np.abs(Z).T @ np.abs(H[s]) @ np.abs(Z)).max()
        assert np.abs(E[s] - ref).max() <= 1e-10 * scale, s
        assert np.abs(Z.T @ M[s] @ Z).max() <= 1e-10 * np.abs(M[s]).max() * np.abs(Z).max() ** 2
        T = np.tile(np.eye(3), (len(Z) // 3, 1))
        assert np.abs(H[s] @ T - c1 * M[s] @ T).max() <= 1e-10 * max(np.abs(H[s]).max(), 1e-300)


@pytest.mark.parametrize("order", [2, 4])
def test_device_closed_form_matches_psi_hessians(order):
    """The corner-form coefficients the device's tet pass uses give the F-space Hessians of the oracle."""
    from test_hess_diag import psi_hessians
    pk, x = _small(True)
    from oracle.tet_energy_oracle import ReferenceEnergyOracle
    orc = ReferenceEnergyOracle(pk.verts, pk.tets)
    F = (orc.G @ x.astype(np.float64).reshape(-1)).reshape(-1, 3, 3)
    for amips in (False, True):
        got = fspace_closed_form(F, order, amips)
        ref = psi_hessians(F, amips=True) if amips else psi_hessians(F, order=order)
        assert np.abs(got - ref).max() <= 1e-9 * np.abs(ref).max()


def test_tables():
    """Every tet exactly once, grouped by component and ascending inside it, chunks of <= 256 tets of one component,
    contiguous and in component order; Y the rest offsets from the component mean; S = Y^T Y."""
    pk = make_pack(3, 700, seed=2)
    T = coarse_tables(pk.verts, pk.tets)
    ne, S = len(pk.tets), T["S"]
    assert sorted(T["tet"].tolist()) == list(range(ne))
    lab = T["comp_label"][pk.tets[T["tet"], 0]]
    assert (np.diff(lab) >= 0).all()
    ch = T["tchunk"].reshape(-1, 3)
    assert (ch[:, 2] - ch[:, 1] <= 256).all() and (ch[:, 2] > ch[:, 1]).all()
    assert ch[0, 1] == 0 and ch[-1, 2] == ne and (ch[1:, 1] == ch[:-1, 2]).all()
    for k, (c, b, e) in enumerate(ch):
        assert (lab[b:e] == c).all()
        assert T["comp_tchunk"][c] <= k < T["comp_tchunk"][c + 1]
    for c in range(S):
        t = T["tet"][lab == c]
        assert (np.diff(t) > 0).all()
    np.testing.assert_array_equal(T["tets"].reshape(-1, 4), pk.tets[T["tet"]])
    Y = T["Y"].reshape(-1, 3).astype(np.float64)
    for c in range(S):
        e0, e1 = T["comp_off"][c], T["comp_off"][c + 1]
        X = pk.verts[T["vert"][e0:e1]].astype(np.float64)
        np.testing.assert_allclose(Y[e0:e1], X - X.mean(0), atol=1e-7)
        np.testing.assert_allclose(T["Smat"][6 * c:6 * c + 6], [*(Y[e0:e1] ** 2).sum(0), Y[e0:e1, 1] @ Y[e0:e1, 2],
                                                                 Y[e0:e1, 0] @ Y[e0:e1, 2], Y[e0:e1, 0] @ Y[e0:e1, 1]], rtol=1e-12)


# The fp64 model table the coarse space was specified from: one 4096-tet sphere of make_pack(1, seed=0), c1 = 2e-4 / 64, c2 = 2e-4, c3 = 1e-4 when on,
# order 2, b = -grad E, block Jacobi with rel_floor 1e-6, E+ with eigenvalues <= 1e-8 lambda_max dropped; products to
# rtol = 1e-3 (False: stopped at negative curvature).  (sigma_rel, AMIPS, model, LM tau or None) -> (Jacobi, coarse).
# Its row at tau = 1e-2 clamps E's eigenvalues instead of dropping them and is not a model of this preconditioner.
MODEL_TABLE = {
    (0.02, False, "exact", None): ((37, True), (37, True)),
    (0.02, False, "exact", 1e-3): ((34, True), (33, True)),
    (0.02, True, "exact", 1e-3): ((42, True), (28, True)),
    (0.02, True, "exact", None): ((162, False), (114, False)),
    (0.02, True, "psd", None): ((116, True), (39, True)),
    (0.35, False, "psd", None): ((171, True), (115, True)),
    (0.35, True, "psd", None): ((176, True), (193, True)),
    (0.35, True, "exact", 1e-3): ((18, True), (18, True)),
}


def _model_run(pk, x, amips, model, tau, H, P):
    c2, c3 = 2e-4, (C3 if amips else 0.0)
    b = -P.grad(x).reshape(-1)
    E, _ = coarse_matrices(P.orc, pk, x, c2, c3, 2, model == "psd")
    m = len(H) // 3
    D = np.stack([H[3 * i:3 * i + 3, 3 * i:3 * i + 3] for i in range(m)])
    mu = 0.0 if tau is None else tau * np.einsum("tii->ti", D).max()
    A = H + mu * np.eye(len(H))
    Pinv = block_preconditioner(D, mu, 1e-6)
    Z, Y = sphere_basis(pk, 0, round32=False)
    Einv = pinv_floor(E[0] + shift_term(Y, mu), 1e-8)
    return (two_level_pcg(A, b, Pinv, Z, np.zeros((9, 9)), 400, 1e-3), two_level_pcg(A, b, Pinv, Z, Einv, 400, 1e-3),
            Pinv, Z, Einv, A)


def test_model_reproduces_table():
    """The fp64 two-level PCG model reproduces MODEL_TABLE row by row (DESIGN.md section 5, "Affine coarse space", lists
    this model's own counts): the same stop (converged or negative curvature) and the same product counts to within max(1, 8 %).  The counts
    are exact on the 0.02 h rows except the AMIPS LM row (29 here, 28 in the table); the 0.35 h PSD solves (cond ~ 1e8 as
    J -> 0+) move by several products under 1e-7 perturbations of the basis (108 with Y rounded to fp32, 116 with fp64
    Y, against the table's 115; 182 against 193 with AMIPS on).  The preconditioner is SPD on the unshifted, indefinite H with AMIPS on."""
    pk = make_pack(1, 4096, seed=0)
    cache = {}
    for (sig, amips, model, tau), ref in MODEL_TABLE.items():
        key = (sig, amips, model)
        if key not in cache:
            x = perturb(pk, sigma_rel=sig, seed=1)
            P = Fp64Problem(pk, 2e-4 / 64, 2e-4, C3 if amips else 0.0)
            cache[key] = (x, P, P.hess_blocks(x, project=model == "psd")[0])
        x, P, H = cache[key]
        kj, kc, Pinv, Z, Einv, A = _model_run(pk, x, amips, model, tau, H, P)
        print(f"{(sig, amips, model, tau)}: Jacobi {kj}, coarse {kc}, table {ref}")
        for got, want in zip((kj, kc), ref):
            assert got[1] == want[1] and abs(got[0] - want[0]) <= max(1, 0.08 * want[0]), (sig, amips, model, tau, got, want)
        if (sig, amips, model, tau) == (0.02, True, "exact", None):
            assert np.linalg.eigvalsh(A).min() < 0
            Mp = Pinv + Z @ Einv @ Z.T
            assert np.linalg.eigvalsh(0.5 * (Mp + Mp.T)).min() > 0


# ---- GPU ----

def _setup(ext, hessian="exact", amips=True, name="small", precond="jacobi", deterministic=True):
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _pack(name)
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=amips, deterministic=deterministic)
    return torch, pk, sp, DevicePCG(sp, hessian=hessian, precond=precond, coarse="affine"), x_np


@pytest.mark.gpu
@pytest.mark.parametrize("hessian", ["exact", "psd"])
@pytest.mark.parametrize("amips", [False, True])
def test_coarse_matrix_against_fp64(ext, hessian, amips):
    """Every entry of coarse_matrix() is within kappa u A of the fp64 E_c on the same fp32 x, A the entry's magnitude sum
    over the sphere's tets; tets whose activity fp32 rounding can flip (|J| < 1e-5 |F|^3) are left out of both.  kappa =
    64 exact, 2048 PSD (the fp32 operator of the projection); the worst measured value is printed."""
    from oracle.tet_energy_oracle import ReferenceEnergyOracle
    torch, pk, sp, pcg, x = _setup(ext, hessian, amips)
    c1, c2 = COEF
    c3 = C3 if amips else 0.0
    x32 = x.astype(np.float32)
    orc = ReferenceEnergyOracle(pk.verts, pk.tets)
    F = (orc.G @ x32.astype(np.float64).reshape(-1)).reshape(-1, 3, 3)
    J = np.linalg.det(F)
    near = np.abs(J) < 1e-5 * np.linalg.norm(F, axis=(1, 2)) ** 3
    pcg.set_coarse(_cuda(x32), c1, c2, 2, c3=c3)
    got = pcg.coarse_matrix().cpu().numpy()
    E, A = coarse_matrices(orc, pk, x32, c2, c3, 2, hessian == "psd")
    if near.any():       # the flip-prone tets' own contributions, with either activity, bound the difference
        from _newton_model import tet_hessians
        Hb, Ha = tet_hessians(orc, x32, 2, c3, hessian == "psd")
        sid = np.searchsorted(pk.vert_offsets, orc.tets[:, 0], side="right") - 1
        np.add.at(A, sid[near], 1e6 * np.abs(c2 * Hb + c3 * Ha)[near])
    kappa = 64 if hessian == "exact" else 2048
    worst = (np.abs(got - E) / (U * A + 1e-300)).max()
    print(f"{hessian} amips={amips}: worst |E - E64| / (u A) = {worst:.3g} (kappa {kappa})")
    assert worst <= kappa
    assert np.abs(E).max() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [None, 1e-3])
def test_apply_precond_against_fp64(ext, shift):
    """z = P r + Z E+ Z^T r per sphere against fp64 from the device's own inverse blocks and coarse matrix, to 1e-4 of
    |z| (E+ in fp64 from the same E + shift S; the fp32 rounding of Y, P r and the sum)."""
    torch, pk, sp, pcg, x = _setup(ext)
    c1, c2 = COEF
    xc = _cuda(x)
    S = pcg.n_spheres
    pcg.set_coarse(xc, c1, c2, 2, c3=C3)
    sh = None if shift is None else torch.full((S,), shift, dtype=torch.float32, device="cuda")
    inv = pcg.set_blocks(sp.hess_diag(xc, c1, c2, 2, c3=C3), want_inverse=True, shift=sh).double().cpu().numpy()
    E = pcg.coarse_matrix().cpu().numpy()
    _, g = sp.energy_grad(xc, c1, c2, 2, -1.0, c3=C3)
    r = g.reshape(-1, 3).contiguous()
    z = pcg.apply_precond(r).double().cpu().numpy()
    rn = r.double().cpu().numpy()
    for s in range(S):
        v0, v1 = pk.vert_offsets[s], pk.vert_offsets[s + 1]
        Z, Y = sphere_basis(pk, s)
        Einv = pinv_floor(E[s] + shift_term(Y, 0.0 if shift is None else float(np.float32(shift))), 1e-8)
        rs = rn[v0:v1].reshape(-1)
        Pr = np.einsum("vij,vj->vi", np.stack([[[q[0], q[5], q[4]], [q[5], q[1], q[3]], [q[4], q[3], q[2]]] for q in inv[v0:v1]]),
                       rn[v0:v1]).reshape(-1)
        ref = Pr + Z @ (Einv @ (Z.T @ rs))
        assert np.linalg.norm(z[v0:v1].reshape(-1) - ref) <= 1e-4 * np.linalg.norm(ref), s


@pytest.mark.gpu
def test_no_op_on_benign_pack(ext):
    """AMIPS off, 0.02 h: no active tet, so E = 0 and, unshifted, E+ = 0: d and the records are those of block Jacobi."""
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    pk = make_pack(3, 512, seed=4)
    x = _cuda(perturb(pk, sigma_rel=0.02, seed=1))
    sp = _handle(ext, pk.verts, pk.tets, deterministic=True)
    c1, c2 = COEF
    pc, pj = DevicePCG(sp, coarse="affine"), DevicePCG(sp)
    pc.set_coarse(x, c1, c2, 2)
    assert not pc.coarse_matrix().any()
    planes = sp.hess_diag(x, c1, c2, 2)
    pc.set_blocks(planes)
    pj.set_blocks(planes)
    _, g = sp.energy_grad(x, c1, c2, 2, -1.0)
    b = g.reshape(-1, 3).contiguous()
    rc, rj = pc.solve(x, b, c1, c2, 2, max_iter=30), pj.solve(x, b, c1, c2, 2, max_iter=30)
    for k in rc._fields:
        if k != "iters_run":
            assert torch.equal(getattr(rc, k), getattr(rj, k)), k


def _step(nw, method, x, c3, anchor=None, weight=None):
    c1, c2 = COEF
    if method in ("lm", "psd"):
        return nw.step(x, c1, c2, 2, c3=c3)
    if method == "prox":
        return nw.step(x, c1, c2, 2, c3=c3, anchor=anchor, weight=weight)
    return (nw.tr_step if method == "tr" else nw.trls_step)(x, c1, c2, 2, c3=c3)


@pytest.mark.gpu
def test_solve_repeatable_and_independent(ext):
    """On a deterministic handle the coarse solve's d and records are bitwise repeatable across calls, streams and a CUDA
    graph replay, and changing one sphere's b leaves every other sphere's d and record bitwise unchanged."""
    torch, pk, sp, pcg, x_np = _setup(ext)
    c1, c2 = COEF
    x = _cuda(x_np)
    S = pcg.n_spheres
    mu = torch.full((S,), 1e-4, dtype=torch.float32, device="cuda")
    pcg.set_coarse(x, c1, c2, 2, c3=C3)
    pcg.set_blocks(sp.hess_diag(x, c1, c2, 2, c3=C3), shift=mu)
    _, g = sp.energy_grad(x, c1, c2, 2, -1.0, c3=C3)
    b = g.reshape(-1, 3).contiguous()
    solve = lambda bb: pcg.solve(x, bb, c1, c2, 2, c3=C3, max_iter=30, rtol=1e-3, shift=mu)
    fields = [k for k in ("d", "status", "n_hvp", "rel_residual", "b_dot_d", "d_H_d")]
    r0 = solve(b)
    same = lambda r, q: all(torch.equal(getattr(r, k), getattr(q, k)) for k in fields)
    assert same(r0, solve(b))
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        r1 = solve(b)
    torch.cuda.current_stream().wait_stream(st)
    torch.cuda.synchronize()
    assert same(r0, r1)
    sid, orph, _ = _labels(pk.verts, pk.tets)
    b2 = b.clone()
    b2[torch.from_numpy((sid == 1) & ~orph).cuda()] *= -2.0
    r2 = solve(b2)
    others = torch.from_numpy(sid != 1).cuda()
    keep = torch.arange(S, device="cuda") != 1
    assert torch.equal(r2.d[others], r0.d[others]) and not torch.equal(r2.d, r0.d)
    for k in fields[1:]:
        assert torch.equal(getattr(r2, k)[keep], getattr(r0, k)[keep]), k
    # a CUDA graph of set_coarse, set_blocks and the solve replays bitwise
    planes = torch.empty((2, sp.n, 3), dtype=torch.float32, device="cuda")
    planes.copy_(sp.hess_diag(x, c1, c2, 2, c3=C3))
    torch.cuda.synchronize()
    g_ = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g_):
        pcg.set_coarse(x, c1, c2, 2, c3=C3)
        pcg.set_blocks(planes, shift=mu)
        rg = solve(b)
    rg.d.zero_()
    g_.replay()
    torch.cuda.synchronize()
    assert same(r0, rg)


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["lm", "psd"])
def test_step_forms_coarse_matrix_at_its_point(ext, method):
    """A Newton step forms E_c at its own x with its own terms: the coarse matrix it leaves is bitwise the one set_coarse
    forms at that x."""
    torch, pk, sp, _, x_np = _setup(ext, "psd" if method == "psd" else "exact")
    from tssplat_b200.newton import DeviceNewton
    nw = DeviceNewton(sp, hessian="psd" if method == "psd" else "exact", coarse="affine")
    x0 = _cuda(x_np)
    x = x0.clone()
    _step(nw, method, x, C3)
    E_step = nw.pcg.coarse_matrix()
    assert not torch.equal(x, x0)
    nw.pcg.set_coarse(x0, *COEF, 2, c3=C3)
    assert torch.equal(E_step, nw.pcg.coarse_matrix()) and E_step.abs().max() > 0


@pytest.mark.gpu
def test_newton_direction_through_flags(ext):
    """FLAGS.newton_coarse = "affine": SmoothnessBarrierEnergy's solver workspace has the coarse space, and
    newton_direction is bitwise set_coarse, set_blocks and solve on it."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    pk, x_np = _pack("small")
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000,
                                                        amips_coeff=C3, deterministic=True, newton_coarse="affine"))
    x = _cuda(x_np)
    r = E.newton_direction(x, 0, max_iter=30)
    pcg = E.device_pcg
    assert pcg.coarse == "affine"
    c1, c2 = E.coeff_scheduler(0)
    pcg.set_coarse(x, c1, c2, 2, c3=C3)
    pcg.set_blocks(E.tet_sp.hess_diag(x, c1, c2, 2, c3=C3))
    _, g = E.tet_sp.energy_grad(x, c1, c2, 2, -1.0, c3=C3)
    q = pcg.solve(x, g.reshape(x.shape), c1, c2, 2, c3=C3, max_iter=30)
    assert torch.equal(r.d, q.d) and torch.equal(r.n_hvp, q.n_hvp)


@pytest.mark.gpu
@pytest.mark.parametrize("method,amips", [("lm", False), ("lm", True), ("prox", True), ("psd", True), ("sgs", False)])
def test_convergence_mixed_pack(ext, method, amips):
    """The mixed 64 x 4096 pack through SmoothnessBarrierEnergy with FLAGS.newton_coarse = "affine": no step raises a
    sphere's objective, and every quiet sphere ends CONVERGED (gtol = 1e-3 min |g_c| over them) within the step budgets
    of the existing tests: REF_STEPS + GPU_SLACK (LM), max PROX_REF_STEPS + GPU_SLACK (proximal, weights 1e-4 .. 1 times
    the sphere's largest Hessian diagonal entry), PSD_REF_STEPS["plain"] + GPU_SLACK (projected), 30 (SGS)."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    pk, x_np = _pack("mixed")
    flags = dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000, amips_coeff=C3 if amips else 0.0,
                 deterministic=True, newton_coarse="affine")
    if method == "psd":
        flags["newton_hessian"] = "psd"
    if method == "sgs":
        flags["newton_precond"] = "sgs"
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    x = torch.nn.Parameter(_cuda(x_np))
    it, S = 0, pk.num_spheres
    g0 = E.newton_step(x.detach().clone(), it, max_iter=1).grad_norm
    E.device_newton.reset()
    assert E.device_newton.coarse == "affine"
    quiet = torch.arange(S, device="cuda") % 4 != 0
    gtol = 1e-3 * float(g0[quiet].min())
    n = {"lm": REF_STEPS[amips] + GPU_SLACK, "prox": max(PROX_REF_STEPS.values()) + GPU_SLACK,
         "psd": PSD_REF_STEPS["plain"] + GPU_SLACK, "sgs": 30}[method]
    if method == "prox":
        y = x.detach().clone()
        sid = torch.from_numpy(np.repeat(np.arange(S), np.diff(pk.vert_offsets))).cuda()
        w = _weights(torch, E.hess_diag(x, it), sid, torch.zeros_like(sid, dtype=torch.bool), S, [1e-4, 1e-3, 1e-2, 1e-1, 1.0])
    for t in range(n):
        r = E.prox_step(x, y, it, w, restart=(t == 0), gtol=gtol) if method == "prox" else E.newton_step(x, it, gtol=gtol)
        assert (r.delta <= 0).all(), t
        if (r.status[quiet] == 1).all():
            break
    print(f"{method} amips={amips}: quiet spheres CONVERGED after {t + 1} steps (budget {n})")
    assert (r.status[quiet] == 1).all(), (t, r.status.tolist())


@pytest.mark.gpu
def test_trust_region_steps_refused(ext):
    """The trust-region steps refuse a coarse workspace (TSB_E_INVALID before any launch): x is left as it was."""
    torch, pk, sp, _, x_np = _setup(ext)
    from tssplat_b200.newton import DeviceNewton
    nw = DeviceNewton(sp, coarse="affine")
    x = _cuda(x_np)
    x0 = x.clone()
    for method in ("tr", "trls"):
        with pytest.raises(RuntimeError, match="coarse"):
            _step(nw, method, x, C3)
    torch.cuda.synchronize()
    assert torch.equal(x, x0)


@pytest.mark.gpu
@pytest.mark.parametrize("method,precond", [("lm", "jacobi"), ("prox", "jacobi"), ("psd", "jacobi"), ("lm", "sgs")])
def test_steps_repeatable_and_independent(ext, method, precond):
    """Three Newton steps from the same x give bitwise the same x across calls and on another stream; changing one
    sphere's start leaves every other sphere's x bitwise unchanged."""
    torch, pk, sp, _, x_np = _setup(ext, "psd" if method == "psd" else "exact", precond=precond)
    from tssplat_b200.newton import DeviceNewton
    anchor = _cuda(x_np) if method == "prox" else None
    weight = torch.full((len(pk.vert_offsets) - 1,), 1e-3, dtype=torch.float32, device="cuda") if method == "prox" else None

    def run(x0, stream=None):
        nw = DeviceNewton(sp, hessian="psd" if method == "psd" else "exact", precond=precond, coarse="affine")
        x = x0.clone()
        with torch.cuda.stream(stream or torch.cuda.current_stream()):
            for _ in range(3):
                _step(nw, method, x, C3, anchor, weight)
        torch.cuda.synchronize()
        return x

    x0 = _cuda(x_np)
    a = run(x0)
    assert torch.equal(a, run(x0))
    assert torch.equal(a, run(x0, torch.cuda.Stream()))
    assert not torch.equal(a, x0)
    sid, orph, S = _labels(pk.verts, pk.tets)
    x1 = x0.clone()
    m0 = torch.from_numpy((sid == 0) & ~orph).cuda()
    x1[m0] += 1e-3
    b = run(x1)
    rest = torch.from_numpy(sid != 0).cuda()
    assert torch.equal(a[rest], b[rest])


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["lm", "prox", "psd"])
def test_graph_of_steps_replays(ext, method):
    """A Newton step on a coarse workspace is capturable after the first call and replays bitwise."""
    torch, pk, sp, _, x_np = _setup(ext, "psd" if method == "psd" else "exact")
    from tssplat_b200.newton import DeviceNewton
    nw = DeviceNewton(sp, hessian="psd" if method == "psd" else "exact", coarse="affine")
    x = _cuda(x_np)
    anchor = x.clone() if method == "prox" else None
    weight = torch.full((nw.n_spheres,), 1e-3, dtype=torch.float32, device="cuda") if method == "prox" else None
    _step(nw, method, x, C3, anchor, weight)
    x0 = x.clone()
    nw.reset()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _step(nw, method, x, C3, anchor, weight)
    torch.cuda.current_stream().wait_stream(s)
    ref = x.clone()
    g = torch.cuda.CUDAGraph()
    x.copy_(x0)
    nw.reset()
    with torch.cuda.graph(g):
        _step(nw, method, x, C3, anchor, weight)
    x.copy_(x0)
    nw.reset()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(x, ref)


# Mean-product ratio coarse / Jacobi of the fp64 model on the quiet spheres 1, 2, 3, 5, 6, 7 of the mixed 64 x 4096 pack
# (COEF, c3 = 1e-4, to rtol 1e-3): LM (tau = 1e-3) 190 / 223 = 0.852, PSD 238 / 1088 = 0.219.  The GPU margins allow 6 %
# (LM) and 35 % (PSD) over them for fp32 rounding and the other 42 quiet spheres; test_model_ratio_on_mixed_pack checks
# the model's ratio on those six spheres against the same margins.
PRODUCT_MARGINS = {"exact": 0.91, "psd": 0.3}


def _mixed_model_products(s, project, tau):
    from types import SimpleNamespace
    pk, x = _pack("mixed")
    v0, v1 = pk.vert_offsets[s], pk.vert_offsets[s + 1]
    m = (pk.tets[:, 0] >= v0) & (pk.tets[:, 0] < v1)
    sub = SimpleNamespace(verts=pk.verts[v0:v1], tets=pk.tets[m] - v0, vert_offsets=np.array([0, v1 - v0]), num_spheres=1)
    xs = x[v0:v1]
    P = Fp64Problem(sub, COEF[0], COEF[1], C3)
    H = P.hess_blocks(xs, project=project)[0]
    b = -P.grad(xs).reshape(-1)
    E, _ = coarse_matrices(P.orc, sub, xs, COEF[1], C3, 2, project)
    D = np.stack([H[3 * i:3 * i + 3, 3 * i:3 * i + 3] for i in range(len(H) // 3)])
    mu = 0.0 if tau is None else tau * np.einsum("tii->ti", D).max()
    A = H + mu * np.eye(len(H))
    Pinv = block_preconditioner(D, mu, 1e-6)
    Z, Y = sphere_basis(sub, 0)
    Einv = pinv_floor(E[0] + shift_term(Y, mu), 1e-8)
    return (two_level_pcg(A, b, Pinv, Z, np.zeros((9, 9)), 400, 1e-3)[0], two_level_pcg(A, b, Pinv, Z, Einv, 400, 1e-3)[0])


def test_model_ratio_on_mixed_pack():
    """The fp64 model's product ratio on the quiet spheres 1, 2, 3, 5, 6, 7 of the mixed pack sits under PRODUCT_MARGINS by
    the slack the GPU test allows (per sphere, LM 33-39 -> 30-33, PSD 171-199 -> 37-42)."""
    for hessian, tau in (("exact", 1e-3), ("psd", None)):
        k = np.array([_mixed_model_products(s, hessian == "psd", tau) for s in (1, 2, 3, 5, 6, 7)], float)
        ratio = k[:, 1].sum() / k[:, 0].sum()
        print(f"{hessian}: model products {k.tolist()}, ratio {ratio:.3f}")
        assert ratio * (1.06 if hessian == "exact" else 1.35) <= PRODUCT_MARGINS[hessian] + 1e-9


@pytest.mark.gpu
@pytest.mark.parametrize("hessian,tau", [("exact", 1e-3), ("psd", None)])
def test_products_fall_on_mixed_pack(ext, hessian, tau):
    """Mixed 64 x 4096 pack, AMIPS on: mean products to rtol 1e-3 over the quiet spheres (every fourth sphere is the 0.35 h
    one) with the coarse space are at most PRODUCT_MARGINS of block Jacobi's (set from the fp64 model on this pack, see
    there; measured on an H100: LM 32.3 / 37.4 = 0.864, PSD 40.3 / 179.2 = 0.225); the measured ratio is printed."""
    margin = PRODUCT_MARGINS[hessian]
    torch, pk, sp, pc, x_np = _setup(ext, hessian, name="mixed")
    from tssplat_b200.newton import DevicePCG
    pj = DevicePCG(sp, hessian=hessian)
    c1, c2 = COEF
    x = _cuda(x_np)
    S = pc.n_spheres
    planes = sp.hess_diag(x, c1, c2, 2, c3=C3)
    sid, orph, _ = _labels(pk.verts, pk.tets)
    dmax = torch.zeros(S, dtype=torch.float32, device="cuda").index_reduce_(
        0, torch.from_numpy(sid).cuda(), planes[0].max(1).values, "amax", include_self=False)
    mu = None if tau is None else (tau * dmax).contiguous()     # the LM step's first shift tau max (D_v)_ii per sphere
    _, g = sp.energy_grad(x, c1, c2, 2, -1.0, c3=C3)
    b = g.reshape(-1, 3).contiguous()
    pc.set_coarse(x, c1, c2, 2, c3=C3)
    pc.set_blocks(planes, shift=mu)
    pj.set_blocks(planes, shift=mu)
    rc = pc.solve(x, b, c1, c2, 2, c3=C3, max_iter=400, rtol=1e-3, shift=mu)
    rj = pj.solve(x, b, c1, c2, 2, c3=C3, max_iter=400, rtol=1e-3, shift=mu)
    quiet = torch.tensor([s % 4 != 0 for s in range(S)], device="cuda")
    kc, kj = rc.n_hvp[quiet].double().mean().item(), rj.n_hvp[quiet].double().mean().item()
    print(f"{hessian}: mean products over quiet spheres coarse {kc:.1f}, Jacobi {kj:.1f}, ratio {kc / kj:.3f}")
    assert kc <= margin * kj


@pytest.mark.gpu
def test_memory_and_refusals(ext):
    torch, pk, sp, pc, x_np = _setup(ext)
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DevicePCG
    pj = DevicePCG(sp)
    T = coarse_tables(pk.verts, pk.tets)
    rows, S, ne = len(T["vert"]), T["S"], len(pk.tets)
    chunks = sum(-(-(T["comp_off"][c + 1] - T["comp_off"][c]) // 256) for c in range(S))
    tch = len(T["tchunk"]) // 3
    assert pc.device_bytes - pj.device_bytes == 12 * rows + 72 * chunks + 372 * tch + 700 * S + 56 * ne + 4
    assert DevicePCG(sp).device_bytes == pj.device_bytes
    lib = _capi.lib
    V, E = sp.vertices, sp.elements
    assert lib.tsb_pcg_enable_coarse(pc._s, V.ctypes.data, E.ctypes.data, int(sp.nele), 1e-8) != 0     # twice
    bad = [(V.ctypes.data, E.ctypes.data, int(sp.nele) - 1, 1e-8), (V.ctypes.data, E.ctypes.data, int(sp.nele), -1.0),
           (V.ctypes.data, E.ctypes.data, int(sp.nele), float("nan")), (None, E.ctypes.data, int(sp.nele), 1e-8)]
    E2 = E.copy()
    E2[0] = E2.reshape(-1)[-1]          # a tet across two spheres
    bad.append((V.ctypes.data, E2.ctypes.data, int(sp.nele), 1e-8))
    for args in bad:
        p = DevicePCG(sp)
        n0 = p.device_bytes
        assert lib.tsb_pcg_enable_coarse(p._s, *args) == _capi.TSB_E_INVALID, args
        assert p.device_bytes == n0
    with pytest.raises(RuntimeError):
        pj.set_coarse(_cuda(x_np), *COEF, 2)
    with pytest.raises(RuntimeError):
        pj.coarse_matrix()
    with pytest.raises(ValueError):
        DevicePCG(sp, coarse="quadratic")

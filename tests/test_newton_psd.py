"""Projected Newton: tsb_pcg_enable_psd, tsb_pcg_hvp_psd and the PSD mode of the solve and the Newton steps, where every
tet's barrier or AMIPS Hessian is replaced by its positive semidefinite projection in deformation-gradient space.

CPU: an fp64 numpy restatement of the closed-form projection (signed SVD, scaling block, pair eigenvalues, the product
rule in the rotated frame) against numpy.linalg.eigh of the 9 x 9 F-space Hessian assembled from the matrix-form dP[dF]
of test_hess_diag, on random, rotated, degenerate, near-rest and inverted F; known answers; the dense per-sphere projected
Hessian of the small mixed pack is PSD where the exact one is not.  GPU: tsb_pcg_hvp_psd against the fp64 projected
oracle on handle variants; agreement with tsb_hvp_ex where every active tet is already PSD; per-sphere curvature;
bitwise repeatability and independence; the PSD solve and Newton steps, and the steps within the fp64 projected
reference's count; argument errors and memory; the module route.  The projected reference itself and the steps against
their composition run through the shared checks of _newton_checks."""
import ctypes as C

import numpy as np
import pytest

from _newton_checks import check_composition, check_reference
from _newton_model import (C3, COEF, GPU_SLACK, PSD_MUST, PSD_REF_STEPS, _cases, _cuda, _handle, _pack, _psd_pack,  # noqa: F401
                           _records, _rot, _small_mixed, _torch, dense_sphere_hessians, ext, reference_problem,
                           reference_run, tet_hessians)
from test_hess_diag import psi_hessians
from tssplat_b200.mesh import make_pack

REL = 1e-4          # GPU projected product against the fp64 oracle, relative L2 per sphere


# ---------------------------------------------------------------------------------------------------------------------
# fp64 closed form in numpy


def signed_svd(F):
    """F = U diag(s) V^T with U, V proper rotations, |s_3| smallest and sign s_3 = sign det F."""
    U, s, Vt = np.linalg.svd(F)
    s = s.copy()
    if np.linalg.det(U) < 0:
        U[:, 2] *= -1
        s[2] *= -1
    if np.linalg.det(Vt) < 0:
        Vt[2] *= -1
        s[2] *= -1
    return U, s, Vt.T


PAIRS = ((0, 1, 2), (0, 2, 1), (1, 2, 0))


def closed_form(F, order=None):
    """(U, s, V, A, lam_s[3], lam_a[3]) of the barrier (order given, det F < 0) or AMIPS (order None, det F > 0)."""
    U, s, V = signed_svd(F)
    J = s[0] * s[1] * s[2]
    if order is not None:
        m = -J
        d1, d2 = -order * m ** (order - 1), order * (order - 1) * m ** (order - 2)
        g = np.array([s[1] * s[2], s[0] * s[2], s[0] * s[1]])
        A = d2 * np.outer(g, g) + d1 * np.array([[0, s[2], s[1]], [s[2], 0, s[0]], [s[1], s[0], 0]])
        ls = np.array([-d1 * s[k] for _, _, k in PAIRS])
        la = -ls
    else:
        j23 = np.cbrt(J) ** 2
        al, ga = 2.0 / (3.0 * j23), 2.0 * (s @ s) / (9.0 * j23)
        A = np.array([[-al / 3 + 5 / 3 * ga / s[i] ** 2 if i == j else
                       -2 / 3 * al * (s[i] / s[j] + s[j] / s[i]) + 2 / 3 * ga / (s[i] * s[j]) for j in range(3)] for i in range(3)])
        r = np.array([ga / (s[i] * s[j]) for i, j, _ in PAIRS])
        ls, la = al + r, al - r
    return U, s, V, A, ls, la


def projected_apply(F, dF, order=None):
    """P(H)[dF] = U D' V^T with Dh = U^T dF V, diag D' = A+ diag Dh, and per pair s, a = (Dh_ij +- Dh_ji) / 2,
    D'_ij = ls+ s + la+ a, D'_ji = ls+ s - la+ a (the kernel's rule)."""
    U, s, V, A, ls, la = closed_form(F, order)
    w, Q = np.linalg.eigh(A)
    Ap = (Q * np.maximum(w, 0)) @ Q.T
    Dh = U.T @ dF @ V
    Dp = np.diag(Ap @ np.diag(Dh))
    for P, (i, j, _) in enumerate(PAIRS):
        sy, an = 0.5 * (Dh[i, j] + Dh[j, i]), 0.5 * (Dh[i, j] - Dh[j, i])
        Dp[i, j] = max(ls[P], 0) * sy + max(la[P], 0) * an
        Dp[j, i] = max(ls[P], 0) * sy - max(la[P], 0) * an
    return U @ Dp @ V.T


def analytic_eigs(F, order=None):
    _, _, _, A, ls, la = closed_form(F, order)
    return np.sort(np.concatenate([np.linalg.eigvalsh(A), ls, la]))


def closed_form_matrix(F, order=None):
    """The 9 x 9 (row-major vec F) matrix of projected_apply."""
    cols = []
    for q in range(9):
        dF = np.zeros((3, 3))
        dF[q // 3, q % 3] = 1.0
        cols.append(projected_apply(F, dF, order).reshape(9))
    return np.stack(cols, 1)


def eigh_projection(H):
    w, Q = np.linalg.eigh(0.5 * (H + H.T))
    return (Q * np.maximum(w, 0)) @ Q.T, w


@pytest.mark.parametrize("term", ["barrier2", "barrier4", "amips"])
def test_closed_form_against_eigh(term):
    rng = np.random.default_rng(7)
    order = {"barrier2": 2, "barrier4": 4, "amips": None}[term]
    seen = 0
    for name, F in _cases(rng):
        if order is None and name == "s3 -> 0-":
            # J -> 0 is a barrier case: an AMIPS tet there has curvature ~ 1 / s_3^2 (here 1e16 against 1e3), beyond
            # what eigh of the assembled matrix resolves to 1e-10
            seen += 1
            continue
        J = np.linalg.det(F)
        if (order is None) != (J > 0):          # barrier on inverted F, AMIPS on the others: flip one column's sign
            F = F @ np.diag([1.0, 1.0, -1.0])
        H = psi_hessians(F[None], order=order, amips=order is None)[0]
        Pe, w = eigh_projection(H)
        scale = max(np.abs(w).max(), 1e-300)
        ev = analytic_eigs(F, order)
        assert np.allclose(ev, np.sort(w), rtol=0, atol=1e-10 * scale), (name, ev, np.sort(w))
        Pc = closed_form_matrix(F, order)
        assert np.abs(Pc - Pe).max() <= 1e-10 * scale, (name, np.abs(Pc - Pe).max() / scale)
        assert np.linalg.eigvalsh(0.5 * (Pc + Pc.T)).min() >= -1e-12 * scale, name
        seen += 1
    assert seen == len(_cases(np.random.default_rng(7)))


def test_known_answers():
    rng = np.random.default_rng(3)
    # AMIPS at a rotation: the Hessian is already PSD, spectrum {0 x 4, 4/3 x 5}
    for F in (np.eye(3), _rot(rng)):
        H = psi_hessians(F[None], amips=True)[0]
        assert np.allclose(analytic_eigs(F), [0, 0, 0, 0] + [4 / 3] * 5, atol=1e-12)
        assert np.allclose(closed_form_matrix(F), H, atol=1e-12)
    # barrier: each pair keeps exactly one of +-phi' s_k
    for order in (2, 4):
        F = _rot(rng) @ np.diag([1.2, 0.8, -0.3]) @ _rot(rng).T
        _, s, _, _, ls, la = closed_form(F, order)
        m = -np.prod(s)
        d1 = -order * m ** (order - 1)
        for P, (_, _, k) in enumerate(PAIRS):
            assert np.isclose(abs(ls[P]), abs(d1 * s[k])) and ((ls[P] > 0) != (la[P] > 0))


@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_dense_projected_hessian_is_psd_on_the_small_mixed_pack(amips):
    from oracle.tet_energy_oracle import ReferenceEnergyOracle
    pk, x = _small_mixed()
    orc = ReferenceEnergyOracle(pk.verts, pk.tets)
    c1, c2 = COEF
    c3 = C3 if amips else 0.0
    Hp = dense_sphere_hessians(orc, pk, x, c1, c2, c3, 2, True)
    He = dense_sphere_hessians(orc, pk, x, c1, c2, c3, 2, False)
    for s, (P, E) in enumerate(zip(Hp, He)):
        wp, we = np.linalg.eigvalsh(P), np.linalg.eigvalsh(E)
        assert wp.min() >= -1e-12 * wp.max(), (s, wp.min(), wp.max())
        print(f"sphere {s}: projected min {wp.min():.3e}, exact min {we.min():.3e}, max {we.max():.3e}")
    assert np.linalg.eigvalsh(He[0]).min() < -1e-6 * np.linalg.eigvalsh(He[0]).max()      # the rough sphere is not


# ---------------------------------------------------------------------------------------------------------------------
# GPU


def projected_hvp_oracle(orc, x, v, c1, c2, c3, order):
    """fp64 c1 M v + G^T (c2 P(H_b) + c3 P(H_a)) G v and the unweighted curvatures (vMv, vHb+v, vHa+v)."""
    x, v = np.asarray(x, np.float64).reshape(-1), np.asarray(v, np.float64).reshape(-1)
    Hb, Ha = tet_hessians(orc, x, order, c3, True)
    dF = (orc.G @ v).reshape(-1, 9)
    yb, ya = np.einsum("tij,tj->ti", Hb, dF), np.einsum("tij,tj->ti", Ha, dF)
    Mv = orc.M @ v
    hv = c1 * Mv + orc.G.T @ (c2 * yb + c3 * ya).reshape(-1)
    mag = np.abs(c1) * np.abs(orc.M) @ np.abs(v) + np.abs(orc.G.T) @ np.abs(c2 * yb + c3 * ya).reshape(-1)
    return hv, mag, (float(v @ Mv), float((dF * yb).sum()), float((dF * ya).sum()))


def _sphere_rel(pk, got, ref, mag, spheres):
    out = []
    for s in spheres:
        sl = slice(3 * pk.vert_offsets[s], 3 * pk.vert_offsets[s + 1])
        out.append(np.linalg.norm(got[sl] - ref[sl]) / np.linalg.norm(mag[sl]))
    return np.array(out)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mixed8", "mixed64"])
@pytest.mark.parametrize("kw", [dict(), dict(deterministic=True), dict(force_global=True)], ids=["default", "det", "global"])
def test_hvp_psd_against_fp64_oracle(ext, name, kw):
    torch = _torch()
    from oracle.tet_energy_oracle import ReferenceEnergyOracle, _det3
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _psd_pack(name)
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, **kw)
    ws = DevicePCG(sp, hessian="psd")
    sub = pk.slice_spheres(0, 8)                    # the oracle on the first eight spheres (two of them rough)
    orc = ReferenceEnergyOracle(sub.verts, sub.tets)
    n_sub = sub.n
    xs = x_np[:n_sub].astype(np.float64)
    J = _det3((orc.G @ xs.reshape(-1)).reshape(-1, 3, 3))
    assert np.abs(J).min() > 1e-7 * np.abs(J).max()          # no tet within fp32 rounding of J = 0
    rng = np.random.default_rng(5)
    v_np = rng.standard_normal((pk.n, 3)).astype(np.float32)
    x, v = _cuda(x_np), _cuda(v_np)
    c1, c2 = COEF
    worst = 0.0
    for order in (2, 4):
        for c3 in (0.0, C3):
            hv, curv = ws.hvp_psd(x, v, c1, c2, order, c3=c3)
            ref, mag, (vmv, vhb, vha) = projected_hvp_oracle(orc, xs, v_np[:n_sub], c1, c2, c3, order)
            got = hv.double().cpu().numpy().reshape(-1)[:3 * n_sub]
            rel = _sphere_rel(sub, got, ref, mag, range(8))
            worst = max(worst, rel.max())
            assert (rel <= REL).all(), (order, c3, rel)
            if name == "mixed8":                     # the record covers the whole pack = the oracle's
                cv = curv.double().cpu().numpy()
                assert abs(cv[1] - vmv) <= 1e-4 * abs(vmv) and abs(cv[2] - vhb) <= 1e-4 * abs(vhb) + 1e-30
                assert abs(cv[3] - vha) <= 1e-4 * abs(vha) + 1e-30
                assert abs(cv[0] - (c1 * vmv + c2 * vhb + c3 * vha)) <= 1e-4 * (c1 * abs(vmv) + c2 * abs(vhb) + c3 * abs(vha))
    print(f"{name} {kw}: worst per-sphere relative error {worst:.2e}")


@pytest.mark.gpu
def test_hvp_psd_equals_exact_where_every_tet_is_psd(ext):
    """At a similarity map of the rest shape (scaled by 1.3, rotated, shifted) no tet is inverted and every tet's AMIPS
    Hessian is PSD (its twist eigenvalues are 0; checked in the oracle), so the projected and exact products agree to
    REL, AMIPS off and on.  (A generic near-rest perturbation already makes some AMIPS twist eigenvalues negative.)"""
    torch = _torch()
    from oracle.tet_energy_oracle import ReferenceEnergyOracle
    from tssplat_b200.newton import DevicePCG
    pk = make_pack(8, 1024, seed=2)
    R = np.linalg.qr(np.random.default_rng(2).standard_normal((3, 3)))[0]
    R = R if np.linalg.det(R) > 0 else -R
    x_np = (1.3 * pk.verts @ R.T + np.array([0.1, -0.2, 0.3])).astype(np.float32)
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    ws = DevicePCG(sp, hessian="psd")
    orc = ReferenceEnergyOracle(pk.verts, pk.tets)
    rng = np.random.default_rng(6)
    v_np = rng.standard_normal((pk.n, 3)).astype(np.float32)
    x, v = _cuda(x_np), _cuda(v_np)
    c1, c2 = COEF
    for c3 in (0.0, C3):
        Hb, Ha = tet_hessians(orc, x_np, 2, c3, False)
        for H in (Hb, Ha):
            # PSD up to the fp32 rounding of x (the twist eigenvalues are 0 at an exact similarity)
            assert np.linalg.eigvalsh(0.5 * (H + H.transpose(0, 2, 1))).min() >= -1e-5 * max(np.abs(H).max(), 1e-300)
        hv, _ = ws.hvp_psd(x, v, c1, c2, 2, c3=c3)
        he, _ = sp.hvp(x, v, c1, c2, 2, c3=c3)
        _, mag, _ = projected_hvp_oracle(orc, x_np, v_np, c1, c2, c3, 2)
        rel = _sphere_rel(pk, hv.double().cpu().numpy().reshape(-1), he.double().cpu().numpy().reshape(-1), mag, range(8))
        assert (rel <= REL).all(), (c3, rel)


@pytest.mark.gpu
def test_sphere_curvature_nonnegative_on_the_rough_pack(ext):
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _psd_pack("mixed64")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    ws = DevicePCG(sp, hessian="psd")
    x = _cuda(x_np)
    c1, c2 = COEF
    rng = np.random.default_rng(9)
    vo = pk.vert_offsets
    for s in (0, 1, 4, 5):
        for order, c3 in ((2, 0.0), (4, C3)):
            v = torch.zeros((pk.n, 3), device="cuda")
            v[vo[s]:vo[s + 1]] = torch.from_numpy(rng.standard_normal((vo[s + 1] - vo[s], 3)).astype(np.float32)).cuda()
            _, curv = ws.hvp_psd(x, v, c1, c2, order, c3=c3)
            cv = curv.double().cpu().numpy()
            tol = 1e-6 * np.abs(cv[1:]).sum()
            assert cv[1] > 0 and cv[2] >= -tol and cv[3] >= -tol, (s, order, cv)
            assert cv[0] >= 0, (s, order, cv)


@pytest.mark.gpu
def test_hvp_psd_bitwise_repeatable_and_independent(ext):
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _psd_pack("mixed64")
    spd = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    spn = _handle(ext, pk.verts, pk.tets, enable_amips=True)
    wd, wn = DevicePCG(spd, hessian="psd"), DevicePCG(spn, hessian="psd")
    x = _cuda(x_np)
    v = torch.randn((pk.n, 3), device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    c1, c2 = COEF
    for order, c3 in ((2, 0.0), (4, C3)):
        a, ca = wd.hvp_psd(x, v, c1, c2, order, c3=c3)
        b, cb = wd.hvp_psd(x, v, c1, c2, order, c3=c3)
        d, cd = wn.hvp_psd(x, v, c1, c2, order, c3=c3)
        assert torch.equal(a, b) and torch.equal(ca, cb)
        assert torch.equal(a, d) and torch.equal(ca, cd), "default and deterministic handles differ"
        other = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(other):
            e, ce = wn.hvp_psd(x, v, c1, c2, order, c3=c3)
        torch.cuda.synchronize()
        assert torch.equal(a, e) and torch.equal(ca, ce)
        # graph replay, with new data copied into the captured buffers
        xg, vg = x.clone(), v.clone()
        s = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            wd.hvp_psd(xg, vg, c1, c2, order, c3=c3)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            hg, cg = wd.hvp_psd(xg, vg, c1, c2, order, c3=c3)
        vg.copy_(2 * v)
        g.replay()
        torch.cuda.synchronize()
        a2, c2b = wd.hvp_psd(x, 2 * v, c1, c2, order, c3=c3)
        assert torch.equal(hg, a2) and torch.equal(cg, c2b)
        # another sphere's x or v changed: this sphere's rows bitwise unchanged
        vo = pk.vert_offsets
        x2, v2 = x.clone(), v.clone()
        x2[vo[5]:vo[6]] += 0.01 * torch.randn_like(x2[vo[5]:vo[6]])
        v2[vo[7]:vo[8]] *= 3.0
        f, _ = wd.hvp_psd(x2, v2, c1, c2, order, c3=c3)
        keep = torch.ones(pk.n, dtype=torch.bool, device="cuda")
        keep[vo[5]:vo[6]] = False
        keep[vo[7]:vo[8]] = False
        assert torch.equal(f[keep], a[keep]) and not torch.equal(f[~keep], a[~keep])


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_psd_solve_never_stops_at_negative_curvature(ext, amips):
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _psd_pack("mixed64")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    c1, c2 = COEF
    c3 = C3 if amips else 0.0
    x = _cuda(x_np)
    _, g = sp.energy_grad(x, c1, c2, 2, -1.0, c3=c3)
    out = {}
    for mode in ("exact", "psd"):
        ws = DevicePCG(sp, hessian=mode)
        ws.set_blocks(sp.hess_diag(x, c1, c2, 2, c3=c3))
        r = ws.solve(x, g, c1, c2, 2, c3=c3, max_iter=200, rtol=1e-3)
        out[mode] = r
        st = r.status.cpu().numpy()
        print(f"{mode} amips={amips}: status counts {np.bincount(st, minlength=5).tolist()}, products mean "
              f"{r.n_hvp.double().mean().item():.1f} max {r.n_hvp.max().item()}")
    st = out["psd"].status.cpu().numpy()
    assert not np.isin(st, [2, 3]).any(), st
    assert (out["psd"].d_H_d >= 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_psd_newton_steps(ext, amips):
    """PSD-mode Newton steps on the mixed 64 x 4096 pack: the energy never rises, no inverted tet is added on the quiet
    spheres, the quiet spheres converge to the exact mode's gtol, and 5 captured steps replay bitwise; the proximal
    step runs in the same mode."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton, DevicePCG
    pk, x_np = _psd_pack("mixed64")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    nw = DeviceNewton(sp, hessian="psd")
    assert nw.hessian == "psd" and nw.pcg.hessian == "psd"
    with pytest.raises(RuntimeError, match="hessian"):
        DeviceNewton(sp, pcg=DevicePCG(sp), hessian="psd")
    c1, c2 = COEF
    c3 = C3 if amips else 0.0
    x = _cuda(x_np)
    S = pk.num_spheres
    quiet = np.arange(S) % 4 != 0
    g0 = sp.energy_grad_spheres(x, c1, c2, 2, c3=c3)[0]
    _, g = sp.energy_grad(x, c1, c2, 2, -1.0, c3=c3)
    sid = torch.from_numpy(np.repeat(np.arange(S), np.diff(pk.vert_offsets))).cuda()
    gn = torch.zeros(S, dtype=torch.float64, device="cuda").index_add_(0, sid, (g.double() ** 2).sum(1)).sqrt().cpu().numpy()
    gtol = 1e-3 * float(gn[quiet].min())
    first = None
    for t in range(28):
        r = nw.step(x, c1, c2, 2, c3=c3, gtol=gtol)
        first = r if first is None else first
        assert (r.delta <= 0).all(), t
    st = r.status.cpu().numpy()
    print(f"psd amips={amips}: status {st.tolist()}, first pcg status {np.bincount(first.pcg_status.cpu().numpy(), minlength=5)}")
    assert (st[quiet] == 1).all(), st
    assert not np.isin(first.pcg_status.cpu().numpy(), [2, 3]).any()
    # bitwise: two runs and a graph of 5 steps
    xa, xb, xg = _cuda(x_np), _cuda(x_np), _cuda(x_np)
    nw.reset()
    ra = _records(torch, [nw.step(xa, c1, c2, 2, c3=c3, max_iter=10) for _ in range(5)])
    nw.reset()
    rb = _records(torch, [nw.step(xb, c1, c2, 2, c3=c3, max_iter=10) for _ in range(5)])
    assert torch.equal(xa, xb) and torch.equal(ra, rb)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        nw.step(_cuda(x_np), c1, c2, 2, c3=c3, max_iter=10)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        nw.reset()
        rg = _records(torch, [nw.step(xg, c1, c2, 2, c3=c3, max_iter=10) for _ in range(5)])
    for _ in range(2):
        xg.copy_(_cuda(x_np))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(xg, xa) and torch.equal(rg, ra)
    # the proximal step in PSD mode
    nw.reset()
    y = _cuda(x_np)
    xp = _cuda(x_np)
    rp = nw.step(xp, c1, c2, 2, c3=c3, anchor=y, weight=1e-3, max_iter=10)
    assert (rp.delta <= 0).all() and (rp.alpha > 0).any()


@pytest.mark.gpu
def test_psd_argument_errors_and_device_bytes(ext):
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DevicePCG, DeviceNewton
    pk, x_np = _pack("small")
    L, E, EM = _capi.lib, _capi.TSB_E_INVALID, _capi.TSB_E_MESH
    sp = _handle(ext, pk.verts, pk.tets, deterministic=True)
    info_bytes = sp.info["device_bytes"]
    ws = DevicePCG(sp)
    b0 = ws.device_bytes
    V = np.ascontiguousarray(pk.verts, np.float32).reshape(-1)
    T = np.ascontiguousarray(pk.tets, np.int32).reshape(-1)
    x = _cuda(x_np)
    st = torch.cuda.current_stream().cuda_stream
    terms = _capi.tsb_terms_t(c1=COEF[0], c2=COEF[1], order=2, c3=0.0)
    hv = torch.zeros_like(x)
    assert L.tsb_pcg_hvp_psd(ws._s, x.data_ptr(), x.data_ptr(), C.byref(terms), hv.data_ptr(), None, st) == E
    assert L.tsb_pcg_enable_psd(ws._s, V.ctypes.data, T.ctypes.data, pk.nele - 1) == E
    Tb = T.copy()
    Tb[5] = pk.n
    assert L.tsb_pcg_enable_psd(ws._s, V.ctypes.data, Tb.ctypes.data, pk.nele) == EM
    Tb = T.copy()
    vo = pk.vert_offsets
    Tb[1] = vo[1]                                        # tet 0 of sphere 0 reaches into sphere 1
    assert L.tsb_pcg_enable_psd(ws._s, V.ctypes.data, Tb.ctypes.data, pk.nele) == EM
    assert ws.device_bytes == b0 and int(L.tsb_pcg_device_bytes(ws._s)) == b0
    assert L.tsb_pcg_enable_psd(ws._s, V.ctypes.data, T.ctypes.data, pk.nele) == 0
    n, ne = pk.n, pk.nele
    assert int(L.tsb_pcg_device_bytes(ws._s)) == b0 + 237 * ne + 4 * (n + 1) + 16 * (-(-ne // 256)) + 16
    assert L.tsb_pcg_enable_psd(ws._s, V.ctypes.data, T.ctypes.data, pk.nele) == E      # twice
    info = _capi.tsb_info_t()
    L.tsb_get_info(sp._h, C.byref(info))
    assert info.device_bytes == info_bytes
    # capture: refused before anything is created, and the capture survives
    graph = torch.cuda.CUDAGraph()
    g = x.clone()
    with torch.cuda.graph(graph):
        g.add_(1.0)
        with pytest.raises(RuntimeError, match="capture"):
            DevicePCG(sp, hessian="psd")
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g, x + 1.0)
    hv.fill_(7.0)
    for bad in (dict(c1=-1.0), dict(c2=-1.0), dict(c3=-1.0), dict(c1=float("nan")), dict(order=3), dict(c3=0.5)):
        t = _capi.tsb_terms_t(**{**dict(c1=COEF[0], c2=COEF[1], order=2, c3=0.0), **bad})
        assert L.tsb_pcg_hvp_psd(ws._s, x.data_ptr(), x.data_ptr(), C.byref(t), hv.data_ptr(), None, st) == E, bad
    for args in ((None, x.data_ptr(), C.byref(terms), hv.data_ptr()), (x.data_ptr(), None, C.byref(terms), hv.data_ptr()),
                 (x.data_ptr(), x.data_ptr(), None, hv.data_ptr()), (x.data_ptr(), x.data_ptr(), C.byref(terms), None)):
        assert L.tsb_pcg_hvp_psd(ws._s, *args, None, st) == E
    for alias in ((x.data_ptr(), hv.data_ptr()), (hv.data_ptr(), x.data_ptr())):   # hv_out is v or x
        assert L.tsb_pcg_hvp_psd(ws._s, alias[0], alias[1], C.byref(terms), hv.data_ptr(), None, st) == E
    torch.cuda.synchronize()
    assert (hv == 7.0).all()
    # a negative coefficient in the PSD solve and Newton step
    o = _capi.tsb_pcg_options_t(max_iter=5, rtol=1e-3, check_every=0)
    neg = _capi.tsb_terms_t(c1=COEF[0], c2=-1.0, order=2, c3=0.0)
    d = torch.zeros_like(x)
    assert L.tsb_pcg_solve_ex(ws._s, x.data_ptr(), x.data_ptr(), C.byref(neg), C.byref(o), None, d.data_ptr(), None, None, st) == E
    nw = DeviceNewton(sp, hessian="psd")
    with pytest.raises(RuntimeError, match="c1, c2 and c3 >= 0"):
        nw.step(x, COEF[0], -1.0, 2)
    with pytest.raises(RuntimeError, match="hvp_psd needs"):
        DevicePCG(sp).hvp_psd(x, x, *COEF, 2)
    with pytest.raises(ValueError):
        DevicePCG(sp, hessian="projected")


@pytest.mark.gpu
def test_module_route(ext):
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    pk, x_np = _pack("small")
    flags = dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000, deterministic=True, amips_coeff=C3)
    E0 = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    Ep = SmoothnessBarrierEnergy(pk.verts, pk.tets, dict(flags, newton_hessian="psd"))
    Ee = SmoothnessBarrierEnergy(pk.verts, pk.tets, dict(flags, newton_hessian="exact"))
    it = 5
    xs = [torch.nn.Parameter(_cuda(x_np)) for _ in range(3)]
    rs = [E.newton_step(x, it, max_iter=15) for E, x in zip((E0, Ep, Ee), xs)]
    assert E0.device_pcg.hessian == "exact" and Ep.device_pcg.hessian == "psd" and Ep.device_newton.pcg is Ep.device_pcg
    assert torch.equal(xs[0], xs[2]) and torch.equal(rs[0].mu, rs[2].mu)            # unchanged without the flag
    assert not torch.equal(xs[0], xs[1]) and (rs[1].alpha > 0).any()
    d = Ep.newton_direction(xs[1].detach(), it, max_iter=20)
    assert not np.isin(d.status.cpu().numpy(), [2, 3]).any()
    y = xs[1].detach().clone()
    r = Ep.prox_step(xs[1], y, it, 1e-2, n_steps=2)
    assert (r.delta <= 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["plain", "small"])
def test_psd_steps_converge_within_the_reference_count(ext, kind):
    """On the projected reference's own pack, the spheres of PSD_MUST (with w = 0 all three, the rough one included) are
    CONVERGED within PSD_REF_STEPS + GPU_SLACK PSD-mode steps, no step raises Phi, and with the small weight the rough
    sphere's Phi falls at every step.  With the small weight the converged spheres' GPU fixed point is the fp64
    exact-mode fixed point (the proximal fp64 reference) within the stationarity bound, using the oracle's gradient at
    the GPU point."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    P, x0, w, o = reference_problem(scale="small")
    sp = _handle(ext, P.pk.verts, P.pk.tets, enable_amips=True, deterministic=True)
    w = np.zeros_like(w) if kind == "plain" else w
    nw = DeviceNewton(sp, hessian="psd")
    x = _cuda(x0.reshape(-1, 3))
    y = x.clone()
    wt = torch.tensor(w, dtype=torch.float32, device="cuda")
    must = list(PSD_MUST[kind])
    steps = None
    for t in range(PSD_REF_STEPS[kind] + GPU_SLACK + 1):
        r = nw.step(x, P.c1, P.c2, 2, anchor=y if kind != "plain" else None, weight=wt if kind != "plain" else None,
                    max_iter=o["max_iter"], rtol=o["rtol"], gtol=o["gtol"])
        assert (r.delta <= 0).all(), t
        if kind == "small":
            assert float(r.delta[0]) < 0, t                      # the rough sphere keeps descending
        if steps is None and (r.status[must] == 1).all():
            steps = t
            if kind == "plain":
                break
    print(f"{kind}: spheres {must} CONVERGED at GPU step {steps}, reference {PSD_REF_STEPS[kind]}, status {r.status.tolist()}")
    assert steps is not None and steps <= PSD_REF_STEPS[kind] + GPU_SLACK, r.status
    if kind == "small":
        xe = reference_run("prox", "small")[6]
        xg = x.double().cpu().numpy().reshape(-1)
        yf = x0.reshape(-1)
        wv = np.repeat(w, np.diff(P.vo) * 3)
        gx, ge = P.grad(xg) + wv * (xg - yf), P.grad(xe) + wv * (xe - yf)
        for s in must:
            sl = slice(3 * P.vo[s], 3 * P.vo[s + 1])
            bound = (np.linalg.norm(gx[sl]) + np.linalg.norm(ge[sl])) / w[s]
            assert np.linalg.norm(xg[sl] - xe[sl]) <= bound, (s, np.linalg.norm(xg[sl] - xe[sl]), bound)


# ---------------------------------------------------------------------------------------------------------------------
# the checks every Newton step shares (_newton_checks)


@pytest.mark.parametrize("kind", ["plain", "small"])
def test_psd_reference_mixed_pack(kind):
    check_reference("psd", kind)


@pytest.mark.gpu
@pytest.mark.parametrize("c3", [0.0, C3], ids=["amips-off", "amips-on"])
def test_psd_steps_equal_their_composition(ext, c3):
    for prox in (False, True):
        check_composition(ext, "psd", c3, prox)

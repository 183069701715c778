"""The symmetric Gauss-Seidel preconditioner on the device (tsb_pcg_enable_sgs, tsb_pcg_set_matrix, tsb_pcg_apply_precond):
the sweep against its fp64 model built from the device's own matrix, blocks and colours; bitwise repeatability; the
solve and every Newton step on an SGS workspace; and the argument rules."""
import numpy as np
import pytest

from _newton_model import (BOUNDARY, COEF, CONVERGED, NEGCURV, NEGCURV_BOUNDARY, NEGCURV_FIRST, OPTS, STEPS, TR_OPTS,
                           TRLS_OPTS, _cuda, _handle, _labels, _pack, _seg_sum, _torch, _weights, compose, ext, new_state)
from _sgs_model import block, sgs_apply, sgs_running_bound
from tssplat_b200.mesh import perturb

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
C3 = 1e-4


def _setup(ext, hessian="exact", amips=True, deterministic=True, name="small"):
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _pack(name)
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=amips, deterministic=deterministic)
    pcg = DevicePCG(sp, hessian=hessian, precond="sgs")
    return torch, pk, sp, pcg, _cuda(x_np)


def _b(sp, x, c1, c2, c3):
    _, g = sp.energy_grad(x, c1, c2, 2, -1.0, c3=c3)
    return g.reshape(-1, 3).contiguous()


@pytest.mark.parametrize("hessian", ["exact", "psd"])
@pytest.mark.parametrize("shift", [None, 1e-3])
def test_apply_matches_fp64_model(ext, hessian, shift):
    """z = M^-1 r per sphere against sgs_apply in fp64 on the device's own A (DeviceHessian.assemble gives the bits
    set_matrix stores), inverse blocks and colours.  Bound per entry: sgs_running_bound, a first-order bound of the fp32
    sweep that charges every fp32 operation of a row one unit roundoff of the magnitude it forms, and propagates earlier
    rows' errors through |Dinv| |A| like the values.  Measured errors sit well inside it; the test also checks that the
    error is not trivially zero everywhere and the bound not vacuous (under 1e-2 of |z| on most entries of the
    quiet spheres)."""
    torch, pk, sp, pcg, x = _setup(ext, hessian)
    c1, c2 = COEF
    c3 = C3
    planes = pcg.set_matrix(x, c1, c2, 2, c3=c3)
    S = pcg.n_spheres
    sh = None if shift is None else torch.full((S,), shift, dtype=torch.float32, device="cuda")
    inv = pcg.set_blocks(planes, want_inverse=True, shift=sh).double().cpu().numpy()
    vals = pcg.hessian_ws.assemble(x, c1, c2, 2, c3=c3)
    r = _b(sp, x, c1, c2, c3)
    z = pcg.apply_precond(r).double().cpu().numpy().reshape(-1)
    colors = pcg.colors.cpu().numpy()
    rn = r.double().cpu().numpy().reshape(-1)
    tight = 0
    for c in range(S):
        verts = pcg.hessian_ws.sphere_vertices(c)
        A = pcg.hessian_ws.sphere(vals, c).toarray().astype(np.float64)
        Dinv = np.stack([block(q) for q in inv[verts]])
        idx = (3 * verts[:, None] + np.arange(3)).reshape(-1)
        ref = sgs_apply(A, Dinv, colors[verts], rn[idx])
        zbar, err = sgs_running_bound(A, Dinv, colors[verts], rn[idx])
        got = z[idx]
        assert (np.abs(got - ref) <= err * U * (1 + 1e-6) + 1e-30).all(), c
        assert np.abs(got - ref).max() > 0 or c > 0
        tight += int((err * U <= 1e-2 * np.abs(ref) + 1e-30).mean() > 0.5)
    assert tight >= S - 1       # the rough sphere's z cancels more, so its bound is looser


def test_apply_repeatable_independent_and_captured(ext):
    torch, pk, sp, pcg, x = _setup(ext)
    c1, c2 = COEF
    pcg.set_blocks(pcg.set_matrix(x, c1, c2, 2, c3=C3))
    r = _b(sp, x, c1, c2, C3)
    z0 = pcg.apply_precond(r).clone()
    assert torch.equal(z0, pcg.apply_precond(r))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        z1 = pcg.apply_precond(r)
    s.synchronize()
    assert torch.equal(z0, z1)
    # a sphere's z does not depend on another sphere's r
    sid, orph, S = _labels(pk.verts, pk.tets)
    r2 = r.clone()
    other = torch.from_numpy((sid != 0) & ~orph).cuda()
    r2[other] *= -3.0
    z2 = pcg.apply_precond(r2)
    mine = torch.from_numpy((sid == 0) & ~orph).cuda()
    assert torch.equal(z2[mine], z0[mine]) and not torch.equal(z2[other], z0[other])
    # a CUDA graph of set_matrix, set_blocks and apply replays bitwise
    out_planes = torch.empty((2, sp.n, 3), dtype=torch.float32, device="cuda")
    zo = torch.zeros_like(r)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pcg.set_blocks(pcg.set_matrix(x, c1, c2, 2, c3=C3, out=out_planes))
        pcg.apply_precond(r, out=zo)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pcg.set_blocks(pcg.set_matrix(x, c1, c2, 2, c3=C3, out=out_planes))
        pcg.apply_precond(r, out=zo)
    zo.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(zo, z0)


@pytest.mark.parametrize("hessian", ["exact", "psd"])
def test_solve_reaches_rtol(ext, hessian):
    """The LM-shifted solve in SGS mode converges on every sphere; the true residual |b - (A + mu I) d| from an fp64
    product with the assembled matrix is within 4 rtol |b| (the recurrence's residual meets rtol), and b.d and d_H_d
    agree with fp64 to 1e-3."""
    torch, pk, sp, pcg, x = _setup(ext, hessian)
    c1, c2 = COEF
    S = pcg.n_spheres
    planes = pcg.set_matrix(x, c1, c2, 2, c3=C3)
    mu = torch.full((S,), float(planes[0].max()) * 1e-2, dtype=torch.float32, device="cuda")
    pcg.set_blocks(planes, shift=mu)
    b = _b(sp, x, c1, c2, C3)
    res = pcg.solve(x, b, c1, c2, 2, c3=C3, max_iter=200, rtol=1e-3, shift=mu)
    assert (res.status == CONVERGED).all()
    vals = pcg.hessian_ws.assemble(x, c1, c2, 2, c3=C3)
    bn, dn = b.double().cpu().numpy().reshape(-1), res.d.double().cpu().numpy().reshape(-1)
    m = float(mu[0])
    for c in range(S):
        verts = pcg.hessian_ws.sphere_vertices(c)
        idx = (3 * verts[:, None] + np.arange(3)).reshape(-1)
        A = pcg.hessian_ws.sphere(vals, c).toarray().astype(np.float64) + m * np.eye(len(idx))
        rr = bn[idx] - A @ dn[idx]
        assert np.linalg.norm(rr) <= 4e-3 * np.linalg.norm(bn[idx]), c
        assert abs(float(res.b_dot_d[c]) - bn[idx] @ dn[idx]) <= 1e-3 * abs(bn[idx] @ dn[idx])
        assert abs(float(res.d_H_d[c]) - dn[idx] @ A @ dn[idx]) <= 1e-3 * abs(dn[idx] @ A @ dn[idx])
    # fewer products than block Jacobi on the same workspace shape
    from tssplat_b200.newton import DevicePCG
    pj = DevicePCG(sp, hessian=hessian)
    pj.set_blocks(sp.hess_diag(x, c1, c2, 2, c3=C3) if hessian == "exact" else planes, shift=mu)
    rj = pj.solve(x, b, c1, c2, 2, c3=C3, max_iter=200, rtol=1e-3, shift=mu)
    print(f"{hessian}: products SGS {res.n_hvp.tolist()}, Jacobi {rj.n_hvp.tolist()}")
    assert int(res.n_hvp.sum()) < int(rj.n_hvp.sum())


def test_radius_inf_is_the_plain_solve(ext):
    torch, pk, sp, pcg, x = _setup(ext)
    c1, c2 = COEF
    pcg.set_blocks(pcg.set_matrix(x, c1, c2, 2, c3=C3))
    b = _b(sp, x, c1, c2, C3)
    a = pcg.solve(x, b, c1, c2, 2, c3=C3, max_iter=30, rtol=1e-4)
    t = pcg.solve(x, b, c1, c2, 2, c3=C3, max_iter=30, rtol=1e-4, radius=float("inf"))
    assert torch.equal(a.d, t.d)
    for f in ("status", "n_hvp", "rel_residual", "b_dot_d", "d_H_d"):
        assert torch.equal(getattr(a, f), getattr(t, f)), f
    # the unshifted solve on the mixed pack: the rough sphere stops at negative curvature, the quiet ones do not
    assert int(a.status[0]) in (NEGCURV, NEGCURV_FIRST)
    assert not np.isin(a.status[1:].cpu().numpy(), (NEGCURV, NEGCURV_FIRST)).any()
    # a small radius: every sphere ends on the boundary
    r = pcg.solve(x, b, c1, c2, 2, c3=C3, max_iter=30, rtol=1e-4, radius=1e-6)
    assert set(r.status.tolist()) <= {BOUNDARY, NEGCURV_BOUNDARY}


class _SgsHandle:
    """The handle as compose() sees it, with the diagonal planes of the SGS workspace's matrix in place of hess_diag."""

    def __init__(self, sp, pcg):
        self.sp, self.pcg = sp, pcg

    def __getattr__(self, k):
        return getattr(self.sp, k)

    def hess_diag(self, x, c1, c2, order, c3=0.0):
        return self.pcg.set_matrix(x, c1, c2, order, c3=c3)


@pytest.mark.parametrize("method,prox", [("lm", False), ("lm", True), ("psd", False)])
def test_damped_steps_match_composition(ext, method, prox):
    """Six damped steps on an SGS workspace against the public calls (set_matrix in place of hess_diag) and the numpy
    rule: bitwise the same x, the same alpha, k and status, mu to fp64 rounding."""
    from tssplat_b200.newton import DeviceNewton
    step = STEPS[method]
    torch, pk, sp, pcg, x1 = _setup(ext, "psd" if step.projected else "exact")
    nw = DeviceNewton(sp, pcg, precond="sgs")
    sid_np, orph_np, S = _labels(pk.verts, pk.tets)
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    c1, c2 = COEF
    o = dict(OPTS, gtol=0.05)
    y = w = None
    if prox:
        y = _cuda(perturb(pk, sigma_rel=0.01, seed=5))
        w = _weights(torch, sp.hess_diag(x1, c1, c2, 2, c3=C3), sid, orph, S, [1e-3, 1e-1, 1.0])
    x2 = x1.clone()
    st = new_state(S)
    wrap = _SgsHandle(sp, pcg)
    for t in range(6):
        r = nw._step("lm", x1, c1, c2, 2, C3, y, w, o)
        x2, out = compose(torch, wrap, pcg, x2, st, c1, c2, C3, o, step, sid, orph, S, y=y, w=w)
        assert torch.equal(x1, x2), t
        assert r.alpha.cpu().tolist() == [q["alpha"] for q in out], t
        assert r.k.cpu().tolist() == [q["k"] for q in out], t
        assert r.status.cpu().tolist() == [s["status"] for s in st], t
        assert np.allclose(r.mu.cpu().numpy(), [s["mu"] for s in st], rtol=1e-12, atol=0), t


@pytest.mark.parametrize("method", ["tr", "trls"])
@pytest.mark.parametrize("prox", [False, True])
def test_tr_steps_on_sgs(ext, method, prox):
    """Trust-region steps on an SGS workspace.  The first step starts from a radius small enough that every solve ends on
    its boundary, so its |d|_M is that radius, radius_init sqrt(b^T M^-1 b), with b^T M^-1 b from apply_precond (to
    1e-4: the recurrences and the sweep round differently).  Then x moves only on spheres that took a step, and every
    step taken lowers the objective."""
    from tssplat_b200.newton import DeviceNewton
    torch, pk, sp, pcg, x = _setup(ext)
    nw = DeviceNewton(sp, pcg, precond="sgs")
    sid_np, orph_np, S = _labels(pk.verts, pk.tets)
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    c1, c2 = COEF
    o = dict(TRLS_OPTS if method == "trls" else TR_OPTS, gtol=0.05, radius_init=1e-3)
    y = w = None
    if prox:
        y = x.clone()
        w = _weights(torch, sp.hess_diag(x, c1, c2, 2, c3=C3), sid, orph, S, [1e-3, 1e-1, 1.0])
    b = _b(sp, x, c1, c2, C3)
    keep = ~orph
    if prox:    # the trust-region step solves with the shift w_c: its blocks are D + w_c I
        pcg.set_blocks(pcg.set_matrix(x, c1, c2, 2, c3=C3), shift=w)
    else:
        pcg.set_blocks(pcg.set_matrix(x, c1, c2, 2, c3=C3))
    Mb = pcg.apply_precond(b)
    bMb = _seg_sum(torch, (b.double() * Mb.double()).sum(1)[keep], sid[keep], S).cpu().numpy()
    took_any = 0
    for t in range(6):
        x0 = x.clone()
        r = nw._step(method, x, c1, c2, 2, C3, y, w, o)
        if t == 0:
            assert set(r.pcg_status.tolist()) <= {BOUNDARY, NEGCURV_BOUNDARY}
            assert np.allclose(r.d_norm.cpu().numpy(), o["radius_init"] * np.sqrt(bMb), rtol=1e-4, atol=0)
        a = r.alpha.cpu().numpy()
        still = torch.from_numpy(np.isin(sid_np, np.flatnonzero(a == 0)) | orph_np).cuda()
        assert not (x - x0).abs().sum(1)[still].any(), t
        assert (r.delta.cpu().numpy()[a > 0] < 0).all(), t
        took_any += int((a > 0).sum())
    assert took_any > 0


def test_convergence_mixed_pack(ext):
    """The LM step on the mixed 64 x 4096 pack (AMIPS off) with an SGS workspace: every quiet sphere converges within 30
    steps, and on the first step no more quiet spheres' solves stop at max_iter than with block Jacobi."""
    from tssplat_b200.newton import DeviceNewton
    torch, pk, sp, pcg, x = _setup(ext, amips=False, deterministic=False, name="mixed")
    nw = DeviceNewton(sp, pcg, precond="sgs")
    c1, c2 = COEF
    quiet = np.array([s % 4 != 0 for s in range(pcg.n_spheres)])
    g0 = _b(sp, x, c1, c2, 0.0)
    sid, orph, S = _labels(pk.verts, pk.tets)
    gn = _seg_sum(torch, (g0.double() ** 2).sum(1)[torch.from_numpy(~orph).cuda()],
                  torch.from_numpy(sid[~orph]).cuda(), S).sqrt().cpu().numpy()
    o = dict(OPTS, gtol=float(1e-3 * gn.min()))
    from tssplat_b200.newton import DeviceNewton as DN
    rj = DN(sp)._step("lm", x.clone(), c1, c2, 2, 0.0, None, None, o)
    trunc_j = int((rj.pcg_status.cpu().numpy()[quiet] == 0).sum())
    first = None
    for t in range(30):
        r = nw._step("lm", x, c1, c2, 2, 0.0, None, None, o)
        if first is None:
            first = r.pcg_status.cpu().numpy()
        if (r.status.cpu().numpy()[quiet] == 1).all():
            break
    assert (r.status.cpu().numpy()[quiet] == 1).all(), t
    trunc_s = int((first[quiet] == 0).sum())
    print(f"quiet spheres converged after {t + 1} steps, {pcg.n_colors} colours; quiet spheres at max_iter on the first "
          f"step: SGS {trunc_s}, Jacobi {trunc_j}")
    assert trunc_s <= trunc_j


def test_graph_of_steps_replays(ext):
    from tssplat_b200.newton import DeviceNewton
    torch, pk, sp, pcg, x = _setup(ext)
    nw = DeviceNewton(sp, pcg, precond="sgs")
    c1, c2 = COEF
    o = dict(OPTS, gtol=0.05)
    xs = x.clone()
    nw._step("lm", xs, c1, c2, 2, C3, None, None, o)        # first call outside the capture
    nw.reset()
    xa = x.clone()
    for _ in range(3):
        nw._step("lm", xa, c1, c2, 2, C3, None, None, o)
    nw.reset()
    xg = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for _ in range(3):
            nw._step("lm", xg, c1, c2, 2, C3, None, None, o)
    torch.cuda.synchronize()
    xg.copy_(x)
    nw.reset()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(xg, xa)


def test_bad_arguments(ext):
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.hessian import DeviceHessian
    from tssplat_b200.newton import DevicePCG, DeviceNewton
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True)
    pj = DevicePCG(sp)
    x, r = _cuda(x_np), _cuda(x_np)
    with pytest.raises(RuntimeError, match="precond"):
        pj.apply_precond(r)
    with pytest.raises(RuntimeError, match="precond"):
        pj.set_matrix(x, *COEF, 2)
    lib = _capi.lib
    assert lib.tsb_pcg_apply_precond(pj._s, r.data_ptr(), torch.empty_like(r).data_ptr(), None) != 0
    assert "tsb_pcg_enable_sgs" in pj._error(pj._s)
    assert lib.tsb_pcg_set_matrix(pj._s, x.data_ptr(), None, None, None) != 0
    # a Hessian workspace of another solver workspace
    other = DevicePCG(sp)
    hs = DeviceHessian(other)
    assert lib.tsb_pcg_enable_sgs(pj._s, hs._hs) != 0 and "another solver workspace" in pj._error(pj._s)
    # twice
    hs2 = DeviceHessian(pj)
    assert lib.tsb_pcg_enable_sgs(pj._s, hs2._hs) == 0
    assert lib.tsb_pcg_enable_sgs(pj._s, hs2._hs) != 0 and "already enabled" in pj._error(pj._s)
    # capture of the first enable
    p3 = DevicePCG(sp)
    hs3 = DeviceHessian(p3)
    with pytest.raises(RuntimeError, match="capture"):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            r.add_(0.0)
            DevicePCG(sp, precond="sgs")
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        DevicePCG(sp, precond="ilu")
    with pytest.raises(RuntimeError, match="precond"):
        DeviceNewton(sp, other, precond="sgs")
    # a component over the shared-memory limit: a 28^3 grid of points, every cube cut into six tets, is one component of
    # 21952 vertices (the limit is about 19 k on an H100)
    V, T = _grid_mesh(28)
    spb = _handle(ext, V, T)
    with pytest.raises(RuntimeError, match="component 0 has 21952 vertices"):
        DevicePCG(spb, precond="sgs")


def _grid_mesh(k):
    """k^3 grid points, each cube cut into the six tets around its main diagonal (Kuhn)."""
    g = np.stack(np.meshgrid(*[np.arange(k)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float32) / k
    idx = lambda i, j, l: (i * k + j) * k + l
    c = np.stack(np.meshgrid(*[np.arange(k - 1)] * 3, indexing="ij"), -1).reshape(-1, 3)
    tets = []
    for perm in ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)):
        p = c.copy()
        path = [idx(*p.T)]
        for ax in perm:
            p = p.copy()
            p[:, ax] += 1
            path.append(idx(*p.T))
        tets.append(np.stack(path, 1))
    return g, np.concatenate(tets).astype(np.int32)

"""Line search along a direction (tsb_line_search, TetSpheres.line_search, SmoothnessBarrierEnergy.line_search).

CPU: an fp64 check (line_terms) built on ReferenceEnergyOracle -- each term's change E_t(x + alpha d) - E_t(x) and the
first root of det F(x + alpha d) from the cubic's exact coefficients -- tested against the closed form of the smoothness
change and a dense scan of J(alpha); known answers; and an fp32 re-enactment of the kernel's root finder on random and
adversarial cubics.  GPU: the kernel against the fp64 check per term, alpha and sphere, repeatability, chaining, handle
info, argument checks and an Armijo step end to end."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sps
from scipy.sparse.csgraph import connected_components

from _helpers import PLAN_SHAPE_MESHES, min_abs_J
from oracle.tet_energy_oracle import ReferenceEnergyOracle, _cof3, _det3
from tssplat_b200.mesh import make_pack, perturb

REL = 1e-5
ALPHAS8 = [2.0 ** -k for k in range(8)]          # 1, 1/2, ..., 1/128
ALPHAS1 = [0.3]
C3 = 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# fp64 check


def cubic_coeffs(orc, x, d):
    """(J0, J1, J2, J3) per tet with det F(x + a d) = J0 + J1 a + J2 a^2 + J3 a^3: F = G x, dF = G d,
    J1 = cof(F) : dF, J2 = F : cof(dF), J3 = det dF."""
    F = (orc.G @ np.asarray(x, np.float64).reshape(-1)).reshape(-1, 3, 3)
    dF = (orc.G @ np.asarray(d, np.float64).reshape(-1)).reshape(-1, 3, 3)
    return _det3(F), (_cof3(F) * dF).sum(axis=(1, 2)), (F * _cof3(dF)).sum(axis=(1, 2)), _det3(dF)


def first_root(c, amax, iters=200):
    """fp64 first root in (0, amax] of the cubics c = (J0, J1, J2, J3) with J0 > 0 (+inf: none, or J0 <= 0): the
    critical points split [0, amax] into monotone pieces; the first piece whose end has J <= 0 is bisected."""
    J0, J1, J2, J3 = (np.asarray(a, np.float64) for a in c)
    ev = lambda a: J0 + a * (J1 + a * (J2 + a * J3))
    n = len(J0)
    A, B = 3 * J3, 2 * J2
    D = B * B - 4 * A * J1
    with np.errstate(divide="ignore", invalid="ignore"):
        sq = np.sqrt(np.maximum(D, 0))
        q = -0.5 * (B + np.copysign(sq, B))
        ra = np.where(A != 0, q / np.where(A != 0, A, 1), np.where(J2 != 0, -J1 / np.where(J2 != 0, 2 * J2, 1), 0))
        rb = np.where((A != 0) & (q != 0), J1 / np.where(q != 0, q, 1), ra)
    ok2 = (A != 0) & (D > 0) | (A == 0) & (J2 != 0)
    q1 = np.where(ok2, np.minimum(ra, rb), 0.0)
    q2 = np.where(ok2, np.maximum(ra, rb), 0.0)
    lo, hi = np.zeros(n), np.full(n, -1.0)
    for e in (np.where((q1 > 0) & (q1 < amax), q1, 0.0), np.where((q2 > 0) & (q2 < amax), q2, 0.0), np.full(n, amax)):
        act = (hi < 0) & (e > lo)
        Je = ev(e)
        hi = np.where(act & (Je <= 0), e, hi)
        lo = np.where(act & (Je > 0), e, lo)
    br = (hi >= 0) & (J0 > 0) & (amax > 0)
    a, b = lo.copy(), np.where(br, hi, lo)
    for _ in range(iters):
        m = 0.5 * (a + b)
        pos = ev(m) > 0
        a, b = np.where(pos, m, a), np.where(pos, b, m)
    return np.where(br, a, np.inf)


def _terms_at(orc, y, order_list=(2, 4)):
    """Per-tet barrier (both orders) and AMIPS values and J at y, per-vertex M y."""
    F = (orc.G @ y).reshape(-1, 3, 3)
    J = _det3(F)
    m = np.maximum(-J, 0)
    ok = J > 0
    tr = (F * F).sum(axis=(1, 2))
    psi = np.where(ok, tr / (3.0 * np.where(ok, J, 1.0) ** (2.0 / 3.0)) - 1.0, 0.0)
    return {2: m * m, 4: m ** 4}, psi, J


def line_terms(orc, x, d, alphas, order, c3):
    """fp64 per-tet and per-vertex pieces of the line search at x along d: a namespace with
    smooth0/smooth [K] per vertex rows (u_i.(M u)_i / 2 at x, and its change), barrier0 / amips0 per tet at x, the
    per-tet changes db [K, T], da [K, T], the energies at x + alpha d, the first root per tet and alpha*."""
    x = np.asarray(x, np.float64).reshape(-1)
    d = np.asarray(d, np.float64).reshape(-1)
    u = x - orc_rest(orc)
    Mu, Md = orc.M @ u, orc.M @ d
    b0, a0, J0 = _terms_at(orc, x)
    out = SimpleNamespace(alphas=np.asarray(alphas, np.float64), b0=b0[order], a0=a0 if c3 else np.zeros_like(a0),
                          s0=0.5 * (u * Mu).reshape(-1, 3).sum(1), ds=[], db=[], da=[], b1=[], a1=[], s1=[], Jal=[])
    for a in out.alphas:
        y = x + a * d
        b1, a1, Ja = _terms_at(orc, y)
        uy = u + a * d
        s1 = 0.5 * (uy * (orc.M @ uy)).reshape(-1, 3).sum(1)
        out.ds.append((a * u * Md + 0.5 * a * a * d * Md).reshape(-1, 3).sum(1))   # per vertex row: closed form
        out.db.append(b1[order] - out.b0)
        out.da.append((a1 - a0) if c3 else np.zeros_like(a1))
        out.b1.append(b1[order]); out.a1.append(a1 if c3 else np.zeros_like(a1)); out.s1.append(s1); out.Jal.append(Ja)
    for k in ("ds", "db", "da", "b1", "a1", "s1", "Jal"):
        setattr(out, k, np.array(getattr(out, k)))
    out.cub = cubic_coeffs(orc, x, d)
    # rounding allowance of the barrier: an fp32 J(alpha) carries an absolute error of a few ulps of the magnitude of
    # det's products, (|F| + alpha |dF|)^3, which is a large relative error for a tet just past J = 0; p m^(p-1) times
    # 8 ulps of that magnitude, per tet
    F = (orc.G @ x).reshape(-1, 3, 3)
    dF = (orc.G @ d).reshape(-1, 3, 3)
    out.nF, out.ndF = np.sqrt((F * F).sum(axis=(1, 2))), np.sqrt((dF * dF).sum(axis=(1, 2)))
    out.berr = np.array([order * np.maximum(-Ja, 0) ** (order - 1) * 2.0 ** -21 * (out.nF + a * out.ndF) ** 3
                         for a, Ja in zip(out.alphas, out.Jal)])
    out.roots = first_root(out.cub, float(out.alphas.max()))
    out.step = float(out.roots.min()) if len(out.roots) else np.inf
    return out


_REST = {}


def orc_rest(orc):
    return _REST[id(orc)]


def make_oracle(V, T):
    orc = ReferenceEnergyOracle(V, T)
    _REST[id(orc)] = np.asarray(V, np.float32).astype(np.float64).reshape(-1)
    return orc


def components(V, T):
    """Component label per vertex (-1: orphan) and per tet, in the order of the components' lowest vertex ids."""
    n = len(V)
    T = np.asarray(T, np.int64).reshape(-1, 4)
    r = np.repeat(T[:, 0], 3)
    c = T[:, 1:].reshape(-1)
    A = sps.coo_matrix((np.ones(len(r)), (r, c)), shape=(n, n))
    _, lab = connected_components(A, directed=False)
    used = np.zeros(n, bool)
    used[T.reshape(-1)] = True
    first = {}
    for v in range(n):
        if used[v] and lab[v] not in first:
            first[lab[v]] = len(first)
    vl = np.array([first[lab[v]] if used[v] else -1 for v in range(n)])
    return vl, vl[T[:, 0]], len(first)


# ---------------------------------------------------------------------------------------------------------------------
# CPU


@pytest.fixture(scope="module")
def small():
    pk = make_pack(3, 512, seed=4)
    orc = make_oracle(pk.verts, pk.tets)
    h = np.linalg.norm(pk.verts[pk.tets[:, 1]] - pk.verts[pk.tets[:, 0]], axis=1).mean()
    rng = np.random.default_rng(5)
    return SimpleNamespace(pk=pk, orc=orc, h=h, x=perturb(pk, sigma_rel=0.02, seed=1).astype(np.float64),
                           d=rng.normal(scale=0.1 * h, size=pk.verts.shape))


def test_smoothness_change_is_closed_form(small):
    """The per-row closed form alpha u^T M d + 1/2 alpha^2 d^T M d equals the difference of two oracle energies."""
    orc, x, d = small.orc, small.x, small.d
    lt = line_terms(orc, x, d, ALPHAS8, 2, C3)
    for k, a in enumerate(ALPHAS8):
        e0, _ = orc.energy_terms(x - orc_rest(orc).reshape(-1, 3), 2)
        e1, _ = orc.energy_terms(x + a * d - orc_rest(orc).reshape(-1, 3), 2)
        assert lt.ds[k].sum() == pytest.approx(e1 - e0, rel=1e-9, abs=1e-12 * e0)
        assert lt.s1[k].sum() - lt.s0.sum() == pytest.approx(lt.ds[k].sum(), rel=1e-9, abs=1e-12 * e0)


def test_cubic_coefficients_and_first_root_against_dense_scan(small):
    orc, x, d = small.orc, small.x, 3.0 * small.d
    J0, J1, J2, J3 = cubic_coeffs(orc, x, d)
    for a in (0.0, 0.37, 1.0, 2.5):
        F = (orc.G @ (x + a * d).reshape(-1)).reshape(-1, 3, 3)
        assert np.allclose(J0 + a * (J1 + a * (J2 + a * J3)), _det3(F), rtol=1e-10, atol=1e-12)
    amax = 1.0
    roots = first_root((J0, J1, J2, J3), amax)
    grid = np.linspace(0, amax, 20001)
    vals = J0[None] + grid[:, None] * (J1[None] + grid[:, None] * (J2[None] + grid[:, None] * J3[None]))
    neg = vals <= 0
    has = neg.any(axis=0) & (J0 > 0)
    scan = np.where(has, grid[np.argmax(neg, axis=0)], np.inf)
    assert has.sum() > 20 and np.isfinite(roots).sum() >= has.sum()
    # every scanned crossing is found, at or before the scan's first nonpositive grid point and within one grid step
    assert np.all(roots[has] <= scan[has]) and np.all(roots[has] >= scan[has] - grid[1] - 1e-12)
    # a root the scan missed lies in a dip narrower than the grid: J at the root is 0 and J > 0 on the grid before it
    miss = np.isfinite(roots) & ~has
    assert np.all(np.abs(J0[miss] + roots[miss] * (J1[miss] + roots[miss] * (J2[miss] + roots[miss] * J3[miss]))) <= 1e-9)


def _rot(axis, ang):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def known_answer_cases(X):
    """(name, x, d, checks) of the known answers on rest positions X."""
    A = np.array([[0.3, -0.1, 0.2], [0.05, -0.2, 0.1], [0.0, 0.4, 0.1]])
    R = _rot([1.0, 2.0, 0.5], 0.7)
    return [("zero", X, np.zeros_like(X)),
            ("affine", X + 0.01, X @ A.T + np.array([0.5, -1.0, 2.0])),
            ("squash", X, X @ (np.diag([1.0, 1.0, -2.0]) - np.eye(3)).T),
            ("collapse", X, -X),
            ("rotation", X, X @ (R - np.eye(3)).T)]


def sbound(orc, x, d, a):
    """Rounding scale of the smoothness change alpha u^T M d + 1/2 alpha^2 d^T M d: the same forms on |u|, |M|, |d|."""
    u = np.abs(np.asarray(x, np.float64).reshape(-1) - orc_rest(orc))
    dd = np.abs(np.asarray(d, np.float64).reshape(-1))
    Ma = abs(orc.M)
    return a * float(u @ (Ma @ dd)) + 0.5 * a * a * float(dd @ (Ma @ dd))


def test_known_answers_fp64(small):
    orc = small.orc
    X = orc_rest(orc).reshape(-1, 3)
    T = orc.nele
    al = [0.25, 0.5, 1.0, 1.5]
    for name, x, d in known_answer_cases(X):
        lt = line_terms(orc, x, d, al, 2, 1.0)
        if name == "zero":
            assert not lt.ds.any() and not lt.db.any() and not lt.da.any() and lt.step == np.inf
        else:                       # linear maps of X: the smoothness does not change
            for k, a in enumerate(al):
                assert abs(lt.ds[k].sum()) <= 1e-12 * sbound(orc, x, d, a), name
        if name == "squash":        # J(alpha) = 1 - 3 alpha on every tet
            assert lt.step == pytest.approx(1 / 3, rel=1e-12)
            assert lt.db[2].sum() == pytest.approx(T * 2.0 ** 2, rel=1e-9)
        if name == "collapse":      # J = (1 - alpha)^3: triple root at 1; a similarity for alpha < 1
            assert lt.step == pytest.approx(1.0, abs=1e-5)
            assert np.abs(lt.da[:2]).max() <= 1e-9
        if name == "rotation":
            assert np.abs(lt.da[2]).max() <= 1e-9 and lt.step == np.inf


# ---- fp32 re-enactment of the kernel's root finder -------------------------------------------------------------------


def kernel_root_fp32(c, amax):
    """The kernel's root finder in fp32, vectorised: critical points, monotone pieces with the double-root tolerance, 32
    halvings of the bit range.  (numpy has no fused multiply-add: each FMA rounds twice here.)"""
    f = np.float32
    J, J1, J2, J3 = (np.asarray(a, f) for a in c)
    amax = f(amax)
    n = len(J)

    def ev(a):
        return J + a * (J1 + a * (J2 + a * J3))

    with np.errstate(all="ignore"):
        A, B = f(3) * J3, f(2) * J2
        D = B * B - f(4) * A * J1
        qq = f(-0.5) * (B + np.copysign(np.sqrt(np.maximum(D, f(0))), B))
        ra = qq / np.where(A != 0, A, f(1))
        rb = np.where(qq != 0, J1 / np.where(qq != 0, qq, f(1)), ra)
        lin = -J1 / np.where(J2 != 0, f(2) * J2, f(1))
    cub = (J3 != 0) & (D > 0)
    q1 = np.where(cub, np.minimum(ra, rb), np.where((J3 == 0) & (J2 != 0), lin, f(0))).astype(f)
    q2 = np.where(cub, np.maximum(ra, rb), f(0)).astype(f)
    q1 = np.where((q1 > 0) & (q1 < amax), q1, f(0)).astype(f)
    q2 = np.where((q2 > 0) & (q2 < amax), q2, f(0)).astype(f)
    lo, hi = np.zeros(n, f), np.full(n, f(-1))
    go = (J > 0) & (amax > 0)
    for i, e in enumerate((q1, q2, np.full(n, amax, f))):
        act = go & (hi < 0) & (e > lo)
        Je = ev(e)
        tol = (f(4.8e-7) * (np.abs(J) + e * (np.abs(J1) + e * (np.abs(J2) + e * np.abs(J3))))).astype(f) if i < 2 else f(0)
        hit = act & (Je <= tol)
        hi = np.where(hit, e, hi)
        lo = np.where(hit & (Je > 0) | act & ~hit, e, lo)
    br = hi >= 0
    a = np.where(br, lo, f(0)).view(np.uint32)
    b = np.where(br, hi, f(0)).view(np.uint32)
    for _ in range(32):
        m = a + ((b - a) >> 1)
        pos = ev(m.view(f)) > 0
        a, b = np.where(pos, m, a), np.where(pos, b, m)
    return np.where(br, a.view(f), f(np.inf)).astype(np.float64)


def _adversarial():
    """(J0, J1, J2, J3, amax) rows: a double root, a quadratic, a linear, two roots in range, a root at amax, J0 a few
    ulps above 0, a triple root, and a dip that returns above 0 before amax."""
    r = []
    r.append((1.0, -1.0, -1.0, 1.0, 2.0))            # (1 - a)^2 (1 + a): double root at 1
    r.append((0.25, -1.0, 1.0, 0.0, 2.0))            # (a - 1/2)^2: quadratic double root
    r.append((1.0, -2.0, 0.0, 0.0, 2.0))             # linear: 1/2
    r.append((0.18, -0.72, 0.1, 1.0, 1.0))           # (a - 0.3)(a - 0.6)(a + 1): first root 0.3
    r.append((1.0, -0.5, 0.0, 0.0, 2.0))             # linear root exactly at amax = 2
    r.append((3e-45, -1.0, 0.0, 0.0, 1.0))           # J0 a denormal above 0
    r.append((1e-7, -1.0, 0.5, 0.0, 1.0))            # J0 a few ulps of 1 above 0
    r.append((1.0, -3.0, 3.0, -1.0, 2.0))            # (1 - a)^3
    r.append((0.1, -1.0, 2.0, 0.0, 1.0))             # 2 (a - 0.25)^2 - 0.025: dips below, back above before amax
    r.append((1.0, 0.0, -1.0, 0.0, 0.5))             # root 1 beyond amax: none
    return np.array(r)


def test_root_finder_fp32_reenactment():
    rng = np.random.default_rng(7)
    n = 100_000
    J0 = np.abs(rng.normal(size=n)) + 1e-3
    c = [J0, rng.normal(size=n) * 2, rng.normal(size=n) * 2, rng.normal(size=n)]
    c = [np.asarray(a, np.float32).astype(np.float64) for a in c]      # the same (fp32) coefficients for both
    amax = 1.5
    ref = first_root(c, amax)
    got = kernel_root_fp32(c, amax)
    fin = np.isfinite(ref)
    assert fin.sum() > 10_000
    assert np.all(np.isfinite(got[fin])), "the fp32 finder missed a first root"
    # simple roots: |J'(alpha*)| well away from 0
    J0, J1, J2, J3 = c
    a = ref[fin]
    slope = np.abs(J1[fin] + a * (2 * J2[fin] + 3 * a * J3[fin]))
    scale = np.abs(J0[fin]) + a * (np.abs(J1[fin]) + a * (np.abs(J2[fin]) + a * np.abs(J3[fin])))
    simple = slope * np.maximum(a, 1e-30) > 1e-3 * scale
    assert simple.mean() > 0.95
    rel = np.abs(got[fin][simple] - a[simple]) / a[simple]
    assert rel.max() <= 1e-4, rel.max()
    # no root found where fp64 has none, except within rounding of a tangency
    extra = ~fin & np.isfinite(got)
    assert extra.sum() <= 1e-4 * n
    # the fp32 cubic is > 0 at the returned value
    g = got[np.isfinite(got)].astype(np.float32)
    cc = [np.asarray(x, np.float32)[np.isfinite(got)] for x in c]
    assert np.all(cc[0] + g * (cc[1] + g * (cc[2] + g * cc[3])) > 0)


@pytest.mark.parametrize("i", range(len(_adversarial())))
def test_root_finder_adversarial(i):
    row = _adversarial()[i]
    c = [np.array([v]) for v in row[:4]]
    amax = row[4]
    ref = first_root(c, amax)[0]
    got = kernel_root_fp32([a.astype(np.float32).astype(np.float64) for a in c], amax)[0]
    expect = {0: 1.0, 1: 0.5, 2: 0.5, 3: 0.3, 4: 2.0, 6: 1e-7, 7: 1.0, 8: 0.25 - np.sqrt(0.0125), 9: np.inf}
    if i in expect:
        e = expect[i]
        if np.isinf(e):
            assert np.isinf(got) and np.isinf(ref)
        else:
            tol = 1e-2 if i in (0, 1, 7) else 1e-5        # multiple roots: fp32 eps^(1/2), eps^(1/3)
            assert abs(got - e) <= tol * e and np.isfinite(ref), (i, got, ref, e)
            assert got <= e * (1 + 1e-6) or i in (0, 1, 7)
    else:       # denormal J0: a root at (about) 3e-45
        assert np.isfinite(got) and got < 1e-40


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


_MESHES = {}


def _mesh(name):
    """(V, T, oracle, {case: x}, d) with a benign (sigma 0.02 h) and an inverted (sigma 0.35 h) input; the plan-shape
    meshes take test_hvp_amips's benign, mirrored and stretched inputs instead."""
    if name not in _MESHES:
        from test_hvp import _mesh as hvp_mesh
        V, T, _, _, _ = hvp_mesh(name)
        V = np.asarray(V, np.float32)
        T64 = np.asarray(T, np.int64).reshape(-1, 4)
        h = np.linalg.norm(V[T64[:, 1]] - V[T64[:, 0]], axis=1).mean()
        rng = np.random.default_rng(21)
        used = np.unique(T64)
        xs = {}
        if name in PLAN_SHAPE_MESHES:         # the inputs of the products' suites: benign, mirrored, stretched
            from test_hvp_amips import _mesh as amips_mesh
            ins = amips_mesh(name)[3]
            xs = {"benign": ins["benign_o2"][0], "inverted": ins["inverted_o2"][0], "stretched": ins["stretched_o2"][0]}
        for case, s in (("benign", 0.02), ("inverted", 0.35)):
            x = V.copy()
            x[used] += rng.normal(scale=s * h, size=(len(used), 3)).astype(np.float32)
            xs.setdefault(case, x)
        assert min_abs_J(V, T, xs["benign"]) > 1e-3
        d = np.zeros_like(V)
        d[used] = rng.normal(scale=0.1 * h, size=(len(used), 3)).astype(np.float32)
        _MESHES[name] = (V, T, make_oracle(V, T), xs, d)
    return _MESHES[name]


_LT = {}


def _lt(name, case, alphas, order, c3):
    key = (name, case, tuple(alphas), order, c3)
    if key not in _LT:
        V, T, orc, xs, d = _mesh(name)
        _LT[key] = line_terms(orc, xs[case].astype(np.float64), d.astype(np.float64), alphas, order, c3)
    return _LT[key]


def _run(sp, x, d, alphas, order, c3, c1=2e-3, c2=0.8, per_sphere=True):
    torch = _torch()
    r = sp.line_search(torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda(),
                       torch.from_numpy(np.ascontiguousarray(d, np.float32)).cuda(), alphas, c1, c2, order, c3=c3,
                       per_sphere=per_sphere)
    torch.cuda.synchronize()
    return r


def _amips_comparable(lt, k):
    """alpha_k is below half the first root, and no tet has |J(alpha_k)| within 1e-5 of its scale (its AMIPS
    activity would be decided by rounding)."""
    a = lt.alphas[k]
    if not a < 0.5 * lt.step:
        return False
    J0, J1, J2, J3 = lt.cub
    scale = np.abs(J0) + a * (np.abs(J1) + a * (np.abs(J2) + a * np.abs(J3)))
    return not np.any(np.abs(lt.Jal[k]) <= 1e-5 * scale)


def step_window(lt, tm):
    """Where the kernel's smallest root over the tets tm may lie: each tet's fp64 root within 1e-4 of itself plus the
    conditioning of its fp32 J (8 ulps of the cubic's terms over |J'| at the root; a tet whose J(x) is near 0 has a
    root near 0 that fp32 knows only to that accuracy).  (+inf, +inf) when no tet has a root."""
    r = lt.roots[tm]
    fin = np.isfinite(r)
    # a tet whose fp64 J(x) is within rounding of 0 may count as uninverted in fp32, with a root near 0
    amb = np.any((lt.cub[0][tm] <= 0) & (np.abs(lt.cub[0][tm]) <= 2.0 ** -20 * lt.nF[tm] ** 3))
    if not fin.any():
        return (0.0 if amb else np.inf), np.inf
    J0, J1, J2, J3 = (c[tm][fin] for c in lt.cub)
    a = r[fin]
    scale = (lt.nF[tm][fin] + a * lt.ndF[tm][fin]) ** 3
    slope = np.abs(J1 + a * (2 * J2 + 3 * a * J3))
    err = 1e-4 * a + 2.0 ** -20 * scale / np.maximum(slope, 1e-300)
    return (0.0 if amb else float((a - err).min())), float((a + err).min())


def _check(sp, name, case, alphas, order, c3, vlab=None, tlab=None, S=None):
    V, T, orc, xs, d = _mesh(name)
    c1, c2 = 2e-3, 0.8
    lt = _lt(name, case, alphas, order, c3)
    r = _run(sp, xs[case], d, alphas, order, c3, c1, c2)
    delta = r.delta.cpu().numpy().astype(np.float64)
    step = float(r.max_step)
    key = (name, case, len(alphas), order, c3)
    compared_a = 0
    for k in range(len(alphas)):
        ds, db, da = lt.ds[k].sum(), lt.db[k].sum(), lt.da[k].sum()
        assert abs(delta[k, 1] - ds) <= REL * (lt.s0.sum() + lt.s1[k].sum()) + 1e-12, (key, k, delta[k], ds)
        assert abs(delta[k, 2] - db) <= REL * (lt.b0.sum() + lt.b1[k].sum()) + lt.berr[k].sum() + 1e-12, (key, k, delta[k], db)
        if c3 == 0:
            assert delta[k, 3] == 0.0
        elif _amips_comparable(lt, k):
            compared_a += 1
            assert abs(delta[k, 3] - da) <= REL * (lt.a0.sum() + lt.a1[k].sum()) + 1e-12, (key, k, delta[k], da)
        tot = c1 * delta[k, 1] + c2 * delta[k, 2] + c3 * delta[k, 3]
        assert abs(delta[k, 0] - tot) <= 1e-6 * (abs(c1 * delta[k, 1]) + abs(c2 * delta[k, 2]) + abs(c3 * delta[k, 3])) + 1e-30
    lo, hi = step_window(lt, np.ones(len(lt.roots), bool))
    assert lo <= step <= hi, (key, step, lt.step)
    # a step of 0.99 min(step, amax) inverts no tet that x had uninverted (fp64)
    a = 0.99 * min(step, max(alphas))
    J0, J1, J2, J3 = lt.cub
    Ja = J0 + a * (J1 + a * (J2 + a * J3))
    resolved = J0 > 2.0 ** -14 * (np.abs(J0) + a * (np.abs(J1) + a * (np.abs(J2) + a * np.abs(J3))))   # fp32 knows J(x) > 0
    assert not np.any(resolved & (Ja <= 0)), key
    # per sphere
    sd = r.sphere_delta.cpu().numpy().astype(np.float64)
    ss = r.sphere_max_step
    assert float(ss.min()) == step and (step == np.inf or bool((ss == r.max_step).any()))
    scale = np.abs(sd).sum(axis=0)
    assert np.all(np.abs(sd.sum(axis=0) - delta) <= 1e-6 * scale + 1e-30), key
    if vlab is not None:
        for c in range(S):
            vm, tm = vlab == c, tlab == c
            for k in range(len(alphas)):
                es = lt.s0[vm].sum() + lt.s1[k][vm].sum()
                assert abs(sd[c, k, 1] - lt.ds[k][vm].sum()) <= REL * es + 1e-12, (key, c, k)
                eb = REL * (lt.b0[tm].sum() + lt.b1[k][tm].sum()) + lt.berr[k][tm].sum()
                assert abs(sd[c, k, 2] - lt.db[k][tm].sum()) <= eb + 1e-12, (key, c, k)
            lo, hi = step_window(lt, tm)
            assert lo <= float(ss[c]) <= hi, (key, c, float(ss[c]), lo, hi)
    return compared_a


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(warps_per_cta=8), dict(deterministic=True), dict(warps_per_cta=8, deterministic=True)],
                         ids=["w16", "w8", "w16-det", "w8-det"])
def test_line_search_staged_pack(ext, kw):
    V, T, *_ = _mesh("pack64x4096")
    sp = _handle(ext, V, T, enable_amips=True, **kw)
    assert sp.info["mode_global"] == 0
    vlab, tlab, S = components(V, T)
    n = 0
    for case in ("benign", "inverted"):
        for order in (2, 4):
            for c3 in (0.0, C3):
                for alphas in (ALPHAS1, ALPHAS8):
                    per = (case == "benign" and order == 2 and alphas is ALPHAS8 and not kw)
                    n += _check(sp, "pack64x4096", case, alphas, order, c3, *((vlab, tlab, S) if per else ()))
    assert n > 0


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(force_global=True), dict(force_global=True, warps_per_cta=8, deterministic=True)],
                         ids=["global", "global-w8-det"])
def test_line_search_a_veg_global(ext, kw):
    V, T, *_ = _mesh("a_veg")
    sp = _handle(ext, V, T, enable_amips=True, **kw)
    assert sp.info["mode_global"] == 1
    vlab, tlab, S = components(V, T)
    for case in ("benign", "inverted"):
        for order, c3 in ((2, C3), (4, 0.0)):
            _check(sp, "a_veg", case, ALPHAS8, order, c3, vlab, tlab, S)
    _check(sp, "a_veg", "benign", ALPHAS1, 2, C3)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(force_global=True), dict(warps_per_cta=8, ring_slots=3, deterministic=True)],
                         ids=["staged", "global", "w8-ring3-det"])
def test_line_search_shuffled_ids_with_orphans(ext, kw):
    V, T, *_ = _mesh("shuffled")
    sp = _handle(ext, V, T, enable_amips=True, **kw)
    vlab, tlab, S = components(V, T)
    assert (vlab < 0).sum() == 500
    for case in ("benign", "inverted"):
        for order, c3 in ((2, C3), (4, 0.0)):
            _check(sp, "shuffled", case, ALPHAS8, order, c3, vlab, tlab, S)


@pytest.mark.gpu
def test_per_sphere_matches_sphere_records(ext):
    """On the 64-sphere pack the per-sphere changes agree with differences of two energy_grad_spheres records at x and
    at fp32(x + alpha d) (that rounding of x + alpha d perturbs u by ~1e-7 |x|: hence the looser bound)."""
    torch = _torch()
    V, T, orc, xs, d = _mesh("pack64x4096")
    sp = _handle(ext, V, T, enable_amips=True)
    x = xs["benign"]
    r = _run(sp, x, d, ALPHAS8, 2, C3)
    sd = r.sphere_delta.cpu().numpy().astype(np.float64)
    xt = torch.from_numpy(x).cuda()
    _, _, s0 = sp.energy_grad_spheres(xt, 2e-3, 0.8, 2, want_grad=False, c3=C3)
    lt = _lt("pack64x4096", "benign", ALPHAS8, 2, C3)
    _, tlab, S = components(V, T)
    berr = np.array([[lt.berr[k][tlab == c].sum() for c in range(S)] for k in range(len(ALPHAS8))])
    for k, a in enumerate(ALPHAS8):
        y = torch.from_numpy((x.astype(np.float64) + a * d.astype(np.float64)).astype(np.float32)).cuda()
        _, _, s1 = sp.energy_grad_spheres(y, 2e-3, 0.8, 2, want_grad=False, c3=C3)
        for j, f in ((1, "smooth"), (2, "barrier"), (3, "amips")):
            if f == "amips" and not a < 0.5 * float(r.max_step):
                continue            # past half the first root a tet's AMIPS activity may change: compared below it
            e0, e1 = getattr(s0, f).cpu().numpy(), getattr(s1, f).cpu().numpy()
            tol = 1e-4 * (e0 + e1) + (2 * berr[k] if f == "barrier" else 0.0) + 1e-9
            assert np.all(np.abs(sd[:, k, j] - (e1 - e0)) <= tol), (k, f)


@pytest.mark.gpu
def test_known_answers_gpu(ext):
    V, T, orc, *_ = _mesh("pack64x4096")
    sp = _handle(ext, V, T, enable_amips=True)
    X = V.astype(np.float64)
    Tn = len(np.asarray(T).reshape(-1, 4))
    al = [0.25, 0.5, 1.0, 1.5]
    for name, x, d in known_answer_cases(X):
        x32, d32 = x.astype(np.float32), d.astype(np.float32)
        r = _run(sp, x32, d32, al, 2, 1.0)
        dl, step = r.delta.cpu().numpy().astype(np.float64), float(r.max_step)
        if name == "zero":
            assert not dl.any() and step == np.inf
            continue
        for k, a in enumerate(al):
            assert abs(dl[k, 1]) <= 1e-5 * sbound(orc, x32, d32, a), (name, k, dl[k])
        if name == "squash":
            assert step == pytest.approx(1 / 3, rel=1e-4)
            assert dl[2, 2] == pytest.approx(Tn * 4.0, rel=1e-5)
        if name == "collapse":
            assert abs(step - 1.0) <= 1e-2
            assert np.abs(dl[:2, 3]).max() <= 1e-6 * Tn
        if name == "rotation":
            assert abs(dl[2, 3]) <= 1e-6 * Tn


@pytest.mark.gpu
def test_bitwise_repeatable_streams_graphs_and_handles(ext):
    torch = _torch()
    _capi = _lib()
    V, T, _, xs, d = _mesh("pack64x4096")
    a = _handle(ext, V, T, enable_amips=True)
    b = _handle(ext, V, T, enable_amips=True, deterministic=True)
    x, dt = torch.from_numpy(xs["inverted"]).cuda(), torch.from_numpy(d).cuda()
    S = a.info["n_components"]
    ref = a.line_search(x, dt, ALPHAS8, 2e-3, 0.8, 4, c3=C3, per_sphere=True)
    for h in (a, a, b):
        r = h.line_search(x, dt, ALPHAS8, 2e-3, 0.8, 4, c3=C3, per_sphere=True)
        for u, v in zip(ref, r):
            assert torch.equal(u, v)
    s = torch.cuda.Stream()
    al = torch.tensor(ALPHAS8, device="cuda")
    outs = [torch.empty((8, 4), device="cuda"), torch.empty((), device="cuda"), torch.empty((S, 8, 4), device="cuda"),
            torch.empty((S,), device="cuda")]
    terms = _capi.tsb_terms_t(c1=2e-3, c2=0.8, order=4, c3=C3)
    call = lambda: _capi.lib.tsb_line_search(b._h, x.data_ptr(), dt.data_ptr(), C.byref(terms), al.data_ptr(), 8,
                                             *[o.data_ptr() for o in outs], s.cuda_stream)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        assert call() == 0
    s.synchronize()
    for u, v in zip(ref, outs):
        assert torch.equal(u, v)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        assert call() == 0
    other = [0.3 * v for v in ALPHAS8]
    ref2 = a.line_search(x, dt, other, 2e-3, 0.8, 4, c3=C3, per_sphere=True)
    torch.cuda.synchronize()
    for vals, want in ((other, ref2), (ALPHAS8, ref), (other, ref2)):
        al.copy_(torch.tensor(vals))
        for o in outs:
            o.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        for u, v in zip(want, outs):
            assert torch.equal(u, v)


@pytest.mark.gpu
@pytest.mark.parametrize("det,case,c3", [(False, "benign", 0.0), (True, "inverted", C3)], ids=["default", "det"])
def test_energy_grad_after_line_search(ext, det, case, c3):
    """energy_grad -> line_search -> energy_grad (and hvp) on one stream: the second results are bitwise the first.  A
    default handle adds AMIPS and inverted tets with atomics, so it runs benign x without AMIPS."""
    torch = _torch()
    V, T, _, xs, d = _mesh("pack64x4096")
    sp = _handle(ext, V, T, enable_amips=True, deterministic=det)
    x, dt = torch.from_numpy(xs[case]).cuda(), torch.from_numpy(d).cuda()
    e1, g1 = sp.energy_grad(x, 2e-3, 0.8, 2, c3=c3)
    e1 = e1.clone()
    sp.line_search(x, dt, ALPHAS8, 2e-3, 0.8, 2, c3=C3, per_sphere=True)
    e2, g2 = sp.energy_grad(x, 2e-3, 0.8, 2, c3=c3)
    sp.line_search(x, dt, ALPHAS1, 2e-3, 0.8, 4)
    hv1, _ = sp.hvp(x, dt, 2e-3, 0.8, 2, c3=c3)
    sp.line_search(x, dt, ALPHAS1, 2e-3, 0.8, 4)
    hv2, _ = sp.hvp(x, dt, 2e-3, 0.8, 2, c3=c3)
    torch.cuda.synchronize()
    assert torch.equal(e1, e2) and torch.equal(g1, g2) and torch.equal(hv1, hv2)


def _lib():
    from tssplat_b200 import _capi
    return _capi


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["plain", "amips"])
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
@pytest.mark.parametrize("nw", [16, 8], ids=["w16", "w8"])
def test_handle_info_unchanged_by_line_search(ext, amips, det, nw):
    """The line search adds instantiations, never plan data, shared memory, grid or device memory (its records reuse
    the per-sphere statistics' scratch): device_bytes changes by 0 bytes."""
    torch = _torch()
    from test_hvp_amips import _INFO_PINS
    V, T, _, xs, d = _mesh("pack64x4096")
    sp = _handle(ext, V, T, enable_amips=amips, deterministic=det, warps_per_cta=nw)
    before = dict(sp.info)
    sp.line_search(torch.from_numpy(xs["benign"]).cuda(), torch.from_numpy(d).cuda(), ALPHAS8, 2e-3, 0.8, 2,
                   c3=C3 if amips else 0.0, per_sphere=True)
    torch.cuda.synchronize()
    from tssplat_b200 import _capi
    info = _capi.tsb_info_t()
    assert _capi.lib.tsb_get_info(sp._h, C.byref(info)) == 0
    after = {k: getattr(info, k) for k, _ in _capi.tsb_info_t._fields_}
    assert after == before
    if torch.cuda.get_device_properties(0).multi_processor_count == 132:
        assert (after["grid"], after["smem_bytes"], after["device_bytes"]) == _INFO_PINS[(amips, det, nw)]


@pytest.mark.gpu
def test_line_search_bad_arguments(ext):
    torch = _torch()
    _capi = _lib()
    V, T, _, xs, d = _mesh("shuffled")
    plain, am = _handle(ext, V, T), _handle(ext, V, T, enable_amips=True)
    x, dt = torch.from_numpy(xs["benign"]).cuda(), torch.from_numpy(d).cuda()
    al = torch.tensor(ALPHAS8, device="cuda")
    S = am.info["n_components"]
    outs = [torch.full((8, 4), 7.0, device="cuda"), torch.full((), 7.0, device="cuda"),
            torch.full((S, 8, 4), 7.0, device="cuda"), torch.full((S,), 7.0, device="cuda")]
    st = torch.cuda.current_stream().cuda_stream
    E = _capi.TSB_E_INVALID
    f = _capi.lib.tsb_line_search
    P = [o.data_ptr() for o in outs]
    t = lambda order=2, c3=0.5: C.byref(_capi.tsb_terms_t(c1=1.0, c2=1.0, order=order, c3=c3))
    assert f(plain._h, x.data_ptr(), dt.data_ptr(), t(), al.data_ptr(), 8, *P, st) == E      # c3 without enable_amips
    assert "enable_amips" in _capi.last_error(plain._h)
    for n_alpha in (0, -1, 9):
        assert f(am._h, x.data_ptr(), dt.data_ptr(), t(), al.data_ptr(), n_alpha, *P, st) == E
    assert f(am._h, None, dt.data_ptr(), t(), al.data_ptr(), 8, *P, st) == E
    assert f(am._h, x.data_ptr(), None, t(), al.data_ptr(), 8, *P, st) == E
    assert f(am._h, x.data_ptr(), dt.data_ptr(), None, al.data_ptr(), 8, *P, st) == E
    assert f(am._h, x.data_ptr(), dt.data_ptr(), t(), None, 8, *P, st) == E
    assert f(am._h, x.data_ptr(), dt.data_ptr(), t(), al.data_ptr(), 8, None, *P[1:], st) == E
    assert f(am._h, x.data_ptr(), dt.data_ptr(), t(order=3), al.data_ptr(), 8, *P, st) == E
    assert f(None, x.data_ptr(), dt.data_ptr(), t(), al.data_ptr(), 8, *P, st) == E
    torch.cuda.synchronize()
    for o in outs:
        assert bool((o == 7.0).all())
    with pytest.raises(RuntimeError, match="enable_amips"):
        plain.line_search(x, dt, ALPHAS8, 1.0, 1.0, 2, c3=0.5)
    # optional outputs may be NULL; the module-level form
    assert f(am._h, x.data_ptr(), dt.data_ptr(), t(), al.data_ptr(), 8, P[0], None, None, None, st) == 0
    r = ext.line_search(dt, x, am, ALPHAS8, 1.0, 1.0, 2, c3=0.5)
    torch.cuda.synchronize()
    assert torch.equal(r.delta, outs[0]) and r.sphere_delta is None and r.sphere_max_step is None


@pytest.mark.gpu
def test_armijo_step_end_to_end(ext):
    """d = -g; the largest of eta * step * 2^-k (eta = 0.9) that meets Armijo by delta decreases the fp64 energy by at
    least the Armijo amount and inverts no tet."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    V, T, orc, xs, _ = _mesh("pack64x4096")
    flags = dict(smooth_eng_coeff=2e-3, barrier_coeff=0.8, increase_order_iter=100, amips_coeff=C3)
    E = SmoothnessBarrierEnergy(V, np.asarray(T).reshape(-1, 4), flags)
    it = 10
    c1, c2 = E.coeff_scheduler(it)
    x = torch.from_numpy(xs["benign"]).cuda()
    _, g = E.tet_sp.energy_grad(x, c1, c2, E.order_at(it), c3=C3)
    dvec = -g.reshape(x.shape)
    h = float(np.linalg.norm(V[T.reshape(-1, 4)[:, 1]] - V[T.reshape(-1, 4)[:, 0]], axis=1).mean())
    t0 = 0.5 * h / float(g.abs().max())
    r0 = E.line_search(x, dvec, it, [t0])
    a_hat = min(float(r0.max_step), t0)
    eta, cA = 0.9, 1e-4
    trials = [eta * a_hat * 2.0 ** -k for k in range(8)]
    r = E.line_search(x, dvec, it, trials)
    gd = -float((g.double() ** 2).sum())
    dl = r.delta.cpu().numpy().astype(np.float64)
    ok = [k for k in range(8) if dl[k, 0] <= cA * trials[k] * gd]
    assert ok, dl[:, 0]
    a = trials[ok[0]]
    x64 = xs["benign"].astype(np.float64)
    y64 = x64 + a * dvec.cpu().numpy().astype(np.float64)
    rest = orc_rest(orc).reshape(-1, 3)

    def energy(z):
        sm, _ = orc.energy_terms(z - rest, E.order_at(it))
        _, bar = orc.energy_terms(z, E.order_at(it))
        am, *_ = orc.amips_terms(z)
        return c1 * sm + c2 * bar + C3 * am

    e0, e1 = energy(x64), energy(y64)
    assert e1 - e0 <= cA * a * gd + 1e-5 * abs(e0), (e1 - e0, cA * a * gd)
    J0 = _det3((orc.G @ x64.reshape(-1)).reshape(-1, 3, 3))
    J1 = _det3((orc.G @ y64.reshape(-1)).reshape(-1, 3, 3))
    assert not np.any((J0 > 0) & (J1 <= 0))

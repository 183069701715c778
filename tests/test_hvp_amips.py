"""Hessian-vector products with the AMIPS term (tsb_hvp_ex, TetSpheres.hvp(c3=...), SmoothnessBarrierEnergy with
FLAGS.amips_coeff).

CPU: an fp64 matrix-form AMIPS hvp on the oracle's G and _cof3 (defined here) against central differences of
ReferenceEnergyOracle.amips_backward, its symmetry and curvature, known answers at rest, an fp32 re-enactment of the
kernel's branch that calibrates the GPU tolerance, and mutations the tolerance rejects.  GPU: the kernel against the
fp64 check per term and combined, tsb_hvp_ex(c3 = 0) against tsb_hvp, bitwise repeatability, chaining with
tsb_energy_grad_ex, handle info, argument checks and autograd."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from _helpers import PLAN_SHAPE_MESHES, check_handle_plan_shape, min_abs_J, mirror_components, plan_shape_cases
from oracle.tet_energy_oracle import ReferenceEnergyOracle, _cof3, _det3, rest_inverse
from test_hvp import _cof_pair, _mesh as _hvp_mesh, check_spheres_and_pole_row, hvp_terms, row_scales
from tssplat_b200.mesh import make_pack, perturb

REL = 1e-5                  # smoothness and barrier terms, as tests/test_hvp.py
REL_A = 2e-5                # the AMIPS term, as the AMIPS gradient tests
GH = 0.7                    # gradH of the GPU runs
TERMS3 = [(0.0, 0.0, 1.0), (2e-3, 0.8, 0.5)]
STRETCH = np.diag([1.4, 0.75, 1.0])      # anisotropic: F far from a similarity


# ---------------------------------------------------------------------------------------------------------------------
# fp64 AMIPS Hessian-vector product, in matrix form.  psi(F) = I1 / (3 J^(2/3)) - 1 for J = det F > 0, 0 otherwise;
# P = dpsi/dF = a (F - beta C) with a = 2 / (3 J^(2/3)), beta = I1 / (3 J), C = cof F.  Along dF = G v:
#     dJ = C : dF,  da = -2/3 a dJ / J,  dbeta = 2 (F : dF) / (3 J) - I1 dJ / (3 J^2),
#     dC = cof_pair(F, dF) + cof_pair(dF, F),  dP = da (F - beta C) + a (dF - dbeta C - beta dC),
#     H_a v = G^T dP,  v^T H_a v = sum_t dF_t : dP_t.


def amips_hvp_terms(orc, x, v, drop=None):
    """(sum_t H_a,t v [3n], per-tet v^T H_a,t v) at x along v.  drop: "dC" or "dbeta" leaves that term out (the
    mutation tests)."""
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    v = np.asarray(v, dtype=np.float64).reshape(-1)
    F = (orc.G @ x).reshape(-1, 3, 3)
    dF = (orc.G @ v).reshape(-1, 3, 3)
    J = _det3(F)
    ok = J > 0
    Js = np.where(ok, J, 1.0)
    C = _cof3(F)
    tr = (F * F).sum(axis=(1, 2))
    dJ = np.einsum("tij,tij->t", C, dF)
    a = 2.0 / (3.0 * Js ** (2.0 / 3.0))
    da = -2.0 / 3.0 * a * dJ / Js
    beta = tr / (3.0 * Js)
    dbeta = 2.0 * np.einsum("tij,tij->t", F, dF) / (3.0 * Js) - tr * dJ / (3.0 * Js ** 2)
    dC = _cof_pair(F, dF) + _cof_pair(dF, F)
    if drop == "dC":
        dC = np.zeros_like(dC)
    if drop == "dbeta":
        dbeta = np.zeros_like(dbeta)
    e = lambda s: s[:, None, None]
    dP = e(da) * (F - e(beta) * C) + e(a) * (dF - e(dbeta) * C - e(beta) * dC)
    dP[~ok] = 0
    return orc.G.T @ dP.reshape(-1), np.einsum("tij,tij->t", dF, dP)


def _rel(a, b):
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300)


def _stretched(V, sigma_scale, seed):
    """V stretched by STRETCH about its centroid, plus N(0, sigma_scale^2) noise: every tet's F far from a similarity."""
    V = np.asarray(V, np.float64)
    c = V.mean(axis=0)
    x = (V - c) @ STRETCH.T + c + np.random.default_rng(seed).normal(scale=sigma_scale, size=V.shape)
    return x.astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# CPU


@pytest.fixture(scope="module")
def small():
    pk = make_pack(3, 512, seed=4)
    orc = ReferenceEnergyOracle(pk.verts, pk.tets)
    h = np.linalg.norm(pk.verts[pk.tets[:, 1]] - pk.verts[pk.tets[:, 0]], axis=1).mean()
    xs = {"benign": perturb(pk, sigma_rel=0.02, seed=1).astype(np.float64),
          "stretched": _stretched(pk.verts, 0.02 * h, 3).astype(np.float64),
          "inverted": mirror_components(perturb(pk, sigma_rel=0.02, seed=2), pk.tets).astype(np.float64)}
    for x in xs.values():
        assert min_abs_J(pk.verts, pk.tets, x) > 1e-2      # away from J = 0: psi and the barrier are smooth around x
    rng = np.random.default_rng(5)
    return SimpleNamespace(pk=pk, orc=orc, x=xs, v=rng.normal(size=pk.verts.shape), w=rng.normal(size=pk.verts.shape))


def _fd(orc, x, v, c1, c2, c3, order, eps=1e-6):
    g = lambda y: (orc.backward(1.0, y, c1, c2, order) if (c1 or c2) else 0.0) + orc.amips_backward(1.0, y, c3)
    return (g(x + eps * v) - g(x - eps * v)) / (2 * eps)


def _full_hvp(orc, x, v, c1, c2, c3, order):
    Mv, Hbv, _, _ = hvp_terms(orc, x, v, order)
    Hav, _ = amips_hvp_terms(orc, x, v)
    return (c1 * Mv + c2 * Hbv + c3 * Hav).reshape(-1, 3)


@pytest.mark.parametrize("terms", [(0.0, 0.0, 1.0), (1e-3, 1.0, 0.5)], ids=["amips", "combined"])
@pytest.mark.parametrize("case", ["benign", "stretched", "inverted"])
def test_amips_hvp_matches_central_differences(small, case, terms):
    c1, c2, c3 = terms
    x, v, orc = small.x[case], small.v, small.orc
    hv = _full_hvp(orc, x, v, c1, c2, c3, 2)
    assert _rel(hv, _fd(orc, x, v, c1, c2, c3, 2)) <= 1e-6
    Hav, q = amips_hvp_terms(orc, x, v)
    assert np.count_nonzero(q) > 0 and np.linalg.norm(Hav) > 0


@pytest.mark.parametrize("case", ["benign", "stretched", "inverted"])
def test_amips_hvp_symmetric_and_curvature(small, case):
    x, v, w, orc = small.x[case], small.v.reshape(-1), small.w.reshape(-1), small.orc
    Hav, q = amips_hvp_terms(orc, x, v)
    Haw, _ = amips_hvp_terms(orc, x, w)
    a, b = np.dot(w, Hav), np.dot(v, Haw)
    assert abs(a - b) <= 1e-10 * max(abs(a), abs(b))
    assert q.sum() == pytest.approx(np.dot(v, Hav), rel=1e-10)
    if case == "inverted":                   # inverted tets (J < 0) have no AMIPS term
        F = (orc.G @ x.reshape(-1)).reshape(-1, 3, 3)
        assert (_det3(F) < 0).any() and not q[_det3(F) < 0].any()


def test_amips_hvp_known_answers_at_rest(small):
    """At x = X every F = I.  psi is invariant under rotation and uniform scaling, so H_a v = 0 for v = W X with W skew
    and for v = s X, and the second-order expansion of psi at I gives v^T H_a v = 4/3 sum_t |dev sym dF_t|^2."""
    orc = small.orc
    X = small.pk.verts.astype(np.float32).astype(np.float64)
    H0, q0 = amips_hvp_terms(orc, X, small.v)
    scale = np.abs(H0).max()
    W = np.array([[0.0, -0.4, 1.1], [0.4, 0.0, -0.3], [-1.1, 0.3, 0.0]])
    for va in (X @ W.T, 0.8 * X, X @ W.T - 0.3 * X + np.array([1.0, 2.0, -0.5])):
        Hv, q = amips_hvp_terms(orc, X, va)
        assert np.abs(Hv).max() <= 1e-10 * scale and np.abs(q).max() <= 1e-10 * np.abs(q0).max()
    for v in (small.v, small.w):
        dF = (orc.G @ v.reshape(-1)).reshape(-1, 3, 3)
        S = 0.5 * (dF + dF.transpose(0, 2, 1))
        dev = S - (np.trace(S, axis1=1, axis2=2) / 3.0)[:, None, None] * np.eye(3)
        expect = 4.0 / 3.0 * (dev * dev).sum(axis=(1, 2))
        _, q = amips_hvp_terms(orc, X, v)
        assert np.allclose(q, expect, rtol=1e-9, atol=1e-12 * expect.max())


def _fp32_reenactment(orc_T, V, x, v):
    """The kernel's AMIPS branch in fp32 per tet (same operations, same order; B = fp32 Dm^-1, J = e1.(e2 x e3) / det Dm
    with fp32 1/det Dm), the corners summed into fp32 rows in tet order (as the atomics or the deterministic gather
    do, in another order): sum_t H_a,t v as [n, 3]."""
    f32 = np.float32
    T = np.asarray(orc_T, np.int64)
    B = rest_inverse(V, T).astype(f32)
    Xd = np.asarray(V, np.float32).astype(np.float64)[T]
    Dm = np.transpose(Xd[:, 1:] - Xd[:, :1], (0, 2, 1))
    idet = (1.0 / np.linalg.det(Dm)).astype(f32)
    P = np.asarray(x, f32)[T]
    Q = np.asarray(v, f32)[T]
    e = [P[:, k] - P[:, 0] for k in (1, 2, 3)]
    f = [Q[:, k] - Q[:, 0] for k in (1, 2, 3)]
    J = (e[0] * np.cross(e[1], e[2])).sum(axis=1, dtype=f32) * idet
    ok = J > 0
    Fm = np.zeros((len(T), 3, 3), f32)
    dF = np.zeros((len(T), 3, 3), f32)
    for c in range(3):
        for r in range(3):
            Fm[:, r, c] = e[0][:, r] * B[:, 0, c] + e[1][:, r] * B[:, 1, c] + e[2][:, r] * B[:, 2, c]
            dF[:, r, c] = f[0][:, r] * B[:, 0, c] + f[1][:, r] * B[:, 1, c] + f[2][:, r] * B[:, 2, c]

    def cofp(A, Bm, r, c):
        r1, r2, c1, c2 = (r + 1) % 3, (r + 2) % 3, (c + 1) % 3, (c + 2) % 3
        return A[:, r1, c1] * Bm[:, r2, c2] - A[:, r1, c2] * Bm[:, r2, c1]

    tr = np.zeros(len(T), f32)
    fdf = np.zeros(len(T), f32)
    dJ = np.zeros(len(T), f32)
    for r in range(3):
        for c in range(3):
            tr = tr + Fm[:, r, c] * Fm[:, r, c]
            fdf = fdf + Fm[:, r, c] * dF[:, r, c]
            dJ = dJ + cofp(Fm, Fm, r, c) * dF[:, r, c]
    Js = np.where(ok, J, f32(1))
    cb = np.cbrt(Js).astype(f32)
    j23 = cb * cb
    iJ = f32(1) / Js
    a = f32(2) / (f32(3) * j23)
    bq = tr * f32(1 / 3) * iJ
    da = -f32(2 / 3) * a * dJ * iJ
    dbq = (f32(2) * fdf - tr * dJ * iJ) * f32(1 / 3) * iJ
    dP = np.zeros_like(Fm)
    for r in range(3):
        for c in range(3):
            Cc = cofp(Fm, Fm, r, c)
            dC = cofp(Fm, dF, r, c) + cofp(dF, Fm, r, c)
            dP[:, r, c] = da * (Fm[:, r, c] - bq * Cc) + a * (dF[:, r, c] - dbq * Cc - bq * dC)
    out = np.zeros((len(V), 3), f32)
    g0 = np.zeros((len(T), 3), f32)
    for k in range(3):
        g = dP[:, :, 0] * B[:, k, 0, None] + dP[:, :, 1] * B[:, k, 1, None] + dP[:, :, 2] * B[:, k, 2, None]
        g[~ok] = 0
        np.add.at(out, T[:, k + 1], g)
        g0 -= g
    np.add.at(out, T[:, 0], g0)
    return out.astype(np.float64)


def test_fp32_reenactment_within_tolerance(small):
    """The tolerance of the GPU checks holds for an fp32 re-enactment of the kernel's branch with room to spare, and
    dropping the dC or the dbeta term of the product is rejected by it by orders of magnitude."""
    pk, orc, v = small.pk, small.orc, small.v
    ratios = {}
    for case, x in small.x.items():
        ref, _ = amips_hvp_terms(orc, x, v)
        ours = _fp32_reenactment(pk.tets, pk.verts, x.astype(np.float32), v.astype(np.float32))
        ratios[case] = _rel(ours, ref.reshape(-1, 3)) / REL_A
        for drop in ("dC", "dbeta"):
            bad, _ = amips_hvp_terms(orc, x, v, drop=drop)
            assert _rel(bad, ref) > 100 * REL_A, (case, drop)
    print("fp32 re-enactment, AMIPS hvp error / tolerance:", {k: f"{r:.3g}" for k, r in ratios.items()})
    assert max(ratios.values()) < 0.5, ratios


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
    """(rest, tets, oracle, inputs {case: (x, order)}, direction): the meshes of tests/test_hvp.py, without its input
    with tets near J = 0, plus an anisotropically stretched input."""
    if name not in _MESHES:
        V, T, orc, inputs, v = _hvp_mesh(name)
        inputs = {k: xo for k, xo in inputs.items() if "035" not in k}
        T64 = np.asarray(T, np.int64)
        h = np.linalg.norm(V[T64[:, 1]] - V[T64[:, 0]], axis=1).mean()
        inputs["stretched_o2"] = (_stretched(V, 0.005 * h, 11), 2)     # h: the mean edge of all spheres, small ones too
        for key, (x, _) in inputs.items():
            assert min_abs_J(V, T, x) > 0.05, (name, key)       # psi's Hessian grows like 1/J^2: keep J well away from 0
        _MESHES[name] = (V, T, orc, inputs, v)
    return _MESHES[name]


def _hvp_ex(sp, x, v, c1, c2, c3, order, gradH=GH):
    torch = _torch()
    hv, curv = sp.hvp(torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda(),
                      torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda(), c1, c2, order, gradH=gradH,
                      want_curv=True, c3=c3)
    return hv.cpu().numpy().astype(np.float64), curv.cpu().numpy().astype(np.float64)


def _check_against_fp64(sp, mesh, key_prefix, orphans=None):
    V, T, orc, inputs, v = _mesh(mesh)
    vv = v.astype(np.float64)
    active = 0
    for case, (x, order) in inputs.items():
        x64 = x.astype(np.float64)
        Mv, Hbv, vMv, q = hvp_terms(orc, x64, vv, order)
        Hav, qa = amips_hvp_terms(orc, x64, vv)
        active += np.count_nonzero(qa)          # 0 for a wholly mirrored mesh: then the AMIPS product must be exactly 0
        for c1, c2, c3 in TERMS3:
            key = (key_prefix, case, c1, c2, c3)
            hv, curv = _hvp_ex(sp, x, v, c1, c2, c3, order)
            parts = (c1 * Mv, c2 * Hbv, c3 * Hav)
            ref = GH * sum(parts).reshape(-1, 3)
            bound = GH * (REL * np.linalg.norm(parts[0]) + REL * np.linalg.norm(parts[1]) + REL_A * np.linalg.norm(parts[2]))
            assert np.linalg.norm(hv - ref) <= bound, (key, np.linalg.norm(hv - ref) / bound)
            if orphans is not None:
                assert not hv[orphans].any(), key
            if mesh in PLAN_SHAPE_MESHES:
                sc = row_scales(mesh, case, x, order)
                prts = [(GH * REL, parts[0].reshape(-1, 3)), (GH * REL, parts[1].reshape(-1, 3)), (GH * REL_A, parts[2].reshape(-1, 3))]
                A = GH * (c1 * sc[0] + c2 * sc[1] + c3 * sc[2])
                for name, w in check_spheres_and_pole_row(mesh, key, hv - ref, prts, A).items():
                    WORST[(mesh, name)] = max(WORST.get((mesh, name), 0.0), w)
            total = c1 * vMv + c2 * q.sum() + c3 * qa.sum()
            scale = REL * (c1 * abs(vMv) + c2 * np.abs(q).sum()) + REL_A * c3 * np.abs(qa).sum()
            assert abs(curv[0] - total) <= scale, (key, curv, total)
            assert abs(curv[1] - vMv) <= REL * abs(vMv), (key, curv[1], vMv)
            assert abs(curv[2] - q.sum()) <= REL * max(np.abs(q).sum(), 1e-300), (key, curv[2], q.sum())
            assert abs(curv[3] - qa.sum()) <= REL_A * np.abs(qa).sum(), (key, curv[3], qa.sum())
    assert active > 0


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(warps_per_cta=8), dict(deterministic=True),
                                dict(warps_per_cta=8, deterministic=True)],
                         ids=["w16", "w8", "w16-det", "w8-det"])
def test_amips_hvp_staged_pack(ext, kw):
    V, T, *_ = _mesh("pack64x4096")
    sp = _handle(ext, V, T, enable_amips=True, **kw)
    assert sp.info["mode_global"] == 0
    _check_against_fp64(sp, "pack64x4096", str(kw))


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(force_global=True), dict(force_global=True, warps_per_cta=8, deterministic=True)],
                         ids=["global", "global-w8-det"])
def test_amips_hvp_a_veg_global(ext, kw):
    V, T, *_ = _mesh("a_veg")
    sp = _handle(ext, V, T, enable_amips=True, **kw)
    assert sp.info["mode_global"] == 1
    _check_against_fp64(sp, "a_veg", str(kw))


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(force_global=True), dict(warps_per_cta=8, ring_slots=3, deterministic=True)],
                         ids=["staged", "global", "w8-ring3-det"])
def test_amips_hvp_shuffled_ids_with_orphans(ext, kw):
    V, T, *_ = _mesh("shuffled")
    sp = _handle(ext, V, T, enable_amips=True, **kw)
    orphans = np.ones(len(V), bool)
    orphans[np.unique(T)] = False
    assert orphans.sum() == 500
    _check_against_fp64(sp, "shuffled", str(kw), orphans=orphans)


@pytest.mark.gpu
@pytest.mark.parametrize("mesh,kw", plan_shape_cases())
def test_amips_hvp_plan_shapes(ext, mesh, kw):
    """The AMIPS products on the plans only these meshes produce (assert_plan_shape)."""
    V, T, *_ = _mesh(mesh)
    sp = _handle(ext, V, T, enable_amips=True, **kw)
    check_handle_plan_shape(mesh, sp, kw, enable_amips=True)
    _check_against_fp64(sp, mesh, str(kw))


WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nAMIPS hvp on the plan-shape meshes: worst |err_s| / bound per sphere, |err_0| / (u A_0) on the pole row:")
        for k, v in sorted(WORST.items()):
            print(f"  {k}: {v:.3g}")


def _lib():
    from tssplat_b200 import _capi
    return _capi


def _call_ex(sp, x, v, c1, c2, c3, order, hv, curv, stream, gradH=GH):
    _capi = _lib()
    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=order, c3=c3)
    return _capi.lib.tsb_hvp_ex(sp._h, x.data_ptr(), v.data_ptr(), C.byref(terms), gradH, None, hv.data_ptr(),
                                curv.data_ptr() if curv is not None else None, stream)


@pytest.mark.gpu
@pytest.mark.parametrize("det,case", [(False, "benign_o2"), (True, "inverted_o2")], ids=["default", "det"])
def test_hvp_ex_c3_zero_is_tsb_hvp(ext, det, case):
    """tsb_hvp_ex with c3 = 0 runs tsb_hvp's launch: hv and curv[0..2] bitwise, curv[3] = 0; tsb_hvp on an AMIPS handle
    is bitwise tsb_hvp on a handle without it (the plans are the same).  A default handle adds inverted tets with
    atomics, so it is compared on an input without them."""
    torch = _torch()
    _capi = _lib()
    V, T, _, inputs, v = _mesh("pack64x4096")
    x_np, order = inputs[case]
    x, vt = torch.from_numpy(x_np).cuda(), torch.from_numpy(v).cuda()
    am, plain = _handle(ext, V, T, enable_amips=True, deterministic=det), _handle(ext, V, T, deterministic=det)
    st = torch.cuda.current_stream().cuda_stream
    c1, c2 = 2e-3, 0.8
    hv0, cv0 = torch.empty_like(x), torch.full((3,), float("nan"), device="cuda")
    hv1, cv1 = torch.empty_like(x), torch.full((4,), float("nan"), device="cuda")
    hv2, cv2 = torch.empty_like(x), torch.full((3,), float("nan"), device="cuda")
    assert _capi.lib.tsb_hvp(am._h, x.data_ptr(), vt.data_ptr(), c1, c2, order, GH, None, hv0.data_ptr(), cv0.data_ptr(), st) == 0
    assert _call_ex(am, x, vt, c1, c2, 0.0, order, hv1, cv1, st) == 0
    assert _capi.lib.tsb_hvp(plain._h, x.data_ptr(), vt.data_ptr(), c1, c2, order, GH, None, hv2.data_ptr(), cv2.data_ptr(), st) == 0
    torch.cuda.synchronize()
    assert torch.equal(hv0, hv1) and torch.equal(cv0, cv1[:3]) and float(cv1[3]) == 0.0
    assert torch.equal(hv0, hv2) and torch.equal(cv0, cv2)
    # the Python form: c3 = 0 keeps the 3-entry curvature
    hv3, cv3 = am.hvp(x, vt, c1, c2, order, gradH=GH, want_curv=True, c3=0.0)
    assert cv3.numel() == 3 and torch.equal(hv3, hv0) and torch.equal(cv3, cv0)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(force_global=True, warps_per_cta=8)], ids=["staged", "global-w8"])
def test_amips_hvp_deterministic_bitwise(ext, kw):
    torch = _torch()
    V, T, _, inputs, v = _mesh("pack64x4096")
    x_np, order = inputs["inverted_o2"]
    det = _handle(ext, V, T, enable_amips=True, deterministic=True, **kw)
    x, vt = torch.from_numpy(x_np).cuda(), torch.from_numpy(v).cuda()
    c1, c2, c3 = 2e-3, 0.8, 0.5
    hv0, cv0 = det.hvp(x, vt, c1, c2, order, gradH=GH, want_curv=True, c3=c3)
    assert cv0.numel() == 4 and float(cv0[3]) != 0.0
    for _ in range(3):
        hv1, cv1 = det.hvp(x, vt, c1, c2, order, gradH=GH, want_curv=True, c3=c3)
        assert torch.equal(hv0, hv1) and torch.equal(cv0, cv1)
    s = torch.cuda.Stream()
    hv_g, cv_g = torch.empty_like(hv0), torch.empty_like(cv0)
    with torch.cuda.stream(s):
        assert _call_ex(det, x, vt, c1, c2, c3, order, hv_g, cv_g, s.cuda_stream) == 0
    s.synchronize()
    assert torch.equal(hv0, hv_g) and torch.equal(cv0, cv_g)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        assert _call_ex(det, x, vt, c1, c2, c3, order, hv_g, cv_g, s.cuda_stream) == 0
    for _ in range(3):
        hv_g.fill_(float("nan"))
        cv_g.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(hv0, hv_g) and torch.equal(cv0, cv_g)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(force_global=True), dict(deterministic=True),
                                dict(deterministic=True, force_global=True, warps_per_cta=8)],
                         ids=["staged", "global", "det", "det-global-w8"])
def test_energy_grad_ex_after_hvp_ex(ext, kw):
    """tsb_energy_grad_ex(c3), tsb_hvp_ex(c3), tsb_energy_grad_ex(c3) on one stream give what a handle that never ran
    tsb_hvp_ex gives: bitwise on a deterministic handle; on a default handle the energies bitwise and the gradient
    within fp32 summation noise (every J > 0 tet adds its AMIPS gradient with atomics)."""
    torch = _torch()
    V, T, _, inputs, v = _mesh("pack64x4096")
    x_np, order = inputs["inverted_o2"]
    x = torch.from_numpy(x_np).cuda()
    x2 = torch.from_numpy((x_np * np.float32(1.001)).astype(np.float32)).cuda()
    vt = torch.from_numpy(v).cuda()
    a, b = _handle(ext, V, T, enable_amips=True, **kw), _handle(ext, V, T, enable_amips=True, **kw)
    c1, c2, c3 = 2e-3, 0.8, 0.5
    ea1, ga1 = a.energy_grad(x, c1, c2, order, c3=c3)
    ea1 = ea1.clone()
    a.hvp(x, vt, c1, c2, order, want_curv=True, c3=c3)
    ea2, ga2 = a.energy_grad(x2, c1, c2, order, c3=c3)
    eb1, gb1 = b.energy_grad(x, c1, c2, order, c3=c3)
    eb1 = eb1.clone()
    eb2, gb2 = b.energy_grad(x2, c1, c2, order, c3=c3)
    torch.cuda.synchronize()
    assert torch.equal(ea1, eb1) and torch.equal(ea2, eb2)
    if kw.get("deterministic"):
        assert torch.equal(ga1, gb1) and torch.equal(ga2, gb2)
    else:
        for ga, gb in ((ga1, gb1), (ga2, gb2)):
            assert float((ga - gb).norm()) <= 1e-6 * float(gb.norm())


# info of the 64 x 4096 pack's handles on an H100 80GB HBM3 (132 SMs), the values these handles reported before
# tsb_hvp_ex was added: the AMIPS product adds instantiations, never plan data, shared memory or grid
_INFO_PINS = {
    # (enable_amips, deterministic, warps_per_cta): (grid, smem_bytes, device_bytes)
    (False, False, 16): (132, 205184, 19306920), (False, False, 8): (132, 130304, 18708648),
    (False, True, 16): (132, 205184, 36752816), (False, True, 8): (132, 130304, 36150448),
    (True, False, 16): (132, 205184, 32094632), (True, False, 8): (132, 130304, 31492264),
    (True, True, 16): (132, 205184, 49532336), (True, True, 8): (132, 130304, 48929968),
}


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["plain", "amips"])
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
@pytest.mark.parametrize("nw", [16, 8], ids=["w16", "w8"])
def test_handle_info_unchanged(ext, amips, det, nw):
    torch = _torch()
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the pinned values are those of a 132-SM H100")
    V, T, *_ = _mesh("pack64x4096")
    sp = _handle(ext, V, T, enable_amips=amips, deterministic=det, warps_per_cta=nw)
    got = (sp.info["grid"], sp.info["smem_bytes"], sp.info["device_bytes"])
    assert got == _INFO_PINS[(amips, det, nw)], got


@pytest.mark.gpu
def test_hvp_ex_bad_arguments(ext):
    torch = _torch()
    _capi = _lib()
    V, T, _, inputs, v = _mesh("shuffled")
    plain, am = _handle(ext, V, T), _handle(ext, V, T, enable_amips=True)
    x = torch.from_numpy(inputs["benign_o2"][0]).cuda()
    vt = torch.from_numpy(v).cuda()
    hv = torch.empty_like(x)
    st = torch.cuda.current_stream().cuda_stream
    E = _capi.TSB_E_INVALID
    assert _call_ex(plain, x, vt, 1.0, 1.0, 0.5, 2, hv, None, st) == E                 # c3 != 0 without enable_amips
    assert "enable_amips" in _capi.last_error(plain._h)
    with pytest.raises(RuntimeError, match="enable_amips"):
        plain.hvp(x, vt, 1.0, 1.0, 2, c3=0.5)
    call = _capi.lib.tsb_hvp_ex
    assert call(am._h, x.data_ptr(), vt.data_ptr(), None, 1.0, None, hv.data_ptr(), None, st) == E   # null terms
    assert _call_ex(am, x, vt, 1.0, 1.0, 0.5, 3, hv, None, st) == E                    # order 3
    terms = _capi.tsb_terms_t(c1=1.0, c2=1.0, order=2, c3=0.5)
    assert call(am._h, None, vt.data_ptr(), C.byref(terms), 1.0, None, hv.data_ptr(), None, st) == E
    assert call(am._h, x.data_ptr(), None, C.byref(terms), 1.0, None, hv.data_ptr(), None, st) == E
    assert call(am._h, x.data_ptr(), vt.data_ptr(), C.byref(terms), 1.0, None, None, None, st) == E
    assert call(None, x.data_ptr(), vt.data_ptr(), C.byref(terms), 1.0, None, hv.data_ptr(), None, st) == E
    # still usable, the module-level form and a CUDA gradH
    hv1 = ext.hvp(vt, x, am, 1.0, 1.0, 2, c3=0.5)
    hv2, _ = am.hvp(x, vt, 1.0, 1.0, 2, gradH=torch.tensor(2.0, device="cuda"), c3=0.5)
    torch.cuda.synchronize()
    assert float((2 * hv1 - hv2).norm()) <= 1e-6 * float(hv2.norm())


def _energy(V, T, amips_coeff, twice=None, deterministic=True):
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    flags = dict(smooth_eng_coeff=2e-3, barrier_coeff=0.8, increase_order_iter=100, deterministic=deterministic)
    if amips_coeff is not None:
        flags["amips_coeff"] = amips_coeff
    if twice is not None:
        flags["twice_differentiable"] = twice
    return SmoothnessBarrierEnergy(V, T.reshape(-1, 4), flags)


@pytest.mark.gpu
@pytest.mark.parametrize("twice", [False, True], ids=["once", "twice"])
def test_module_amips_energy_and_gradient(ext, twice):
    torch = _torch()
    V, T, _, inputs, _ = _mesh("shuffled")
    E_mod = _energy(V, T, 0.5, twice)
    c1, c2 = E_mod.coeff_scheduler(10)
    x = torch.from_numpy(inputs["inverted_o2"][0]).cuda().requires_grad_(True)
    E = E_mod(x, 10, c1, c2)
    assert "SmoothnessBarrierAmipsFunc" in type(E.grad_fn).__name__
    e_ref, g_ref = E_mod.tet_sp.energy_grad(x.detach(), c1, c2, 2, c3=0.5)
    assert e_ref.numel() == 4 and float(e_ref[3]) > 0
    assert torch.equal(E.detach(), e_ref[0])
    E.backward(torch.tensor(1.5, device="cuda"))
    torch.cuda.synchronize()
    assert torch.equal(x.grad, (1.5 * g_ref).reshape(x.shape))       # deterministic handle: the same gradient, scaled
    stats = E_mod.sphere_stats(x, 10)
    assert float(stats.amips.sum()) == pytest.approx(float(e_ref[3]), rel=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("it", [10, 500], ids=["order2", "order4"])
def test_module_amips_twice_differentiable(ext, it):
    torch = _torch()
    V, T, orc, inputs, v = _mesh("shuffled")
    c3 = 0.5
    E_mod = _energy(V, T, c3, True)
    c1, c2 = E_mod.coeff_scheduler(it)
    order = E_mod.order_at(it)
    x_np = inputs["inverted_o2"][0]
    x = torch.from_numpy(x_np).cuda().requires_grad_(True)
    w = torch.from_numpy(v).cuda()
    ref = torch.from_numpy(_full_hvp(orc, x_np.astype(np.float64), v.astype(np.float64), c1, c2, c3, order)).cuda()
    tol = 2e-5 * float(ref.norm())
    assert float((E_mod.hvp(x, w, it).double() - ref).norm()) <= tol
    E = E_mod(x, it, c1, c2)
    (g,) = torch.autograd.grad(E, x, create_graph=True)
    (hw,) = torch.autograd.grad((g * w).sum(), x)
    assert float((hw.double() - ref).norm()) <= tol
    _, vh = torch.autograd.functional.vhp(lambda xx: E_mod(xx, it, c1, c2), x.detach(), w)
    assert float((vh.double() - ref).norm()) <= tol
    E = E_mod(x, it, c1, c2)
    (g,) = torch.autograd.grad(E, x, create_graph=True)
    (h,) = torch.autograd.grad((g * w).sum(), x, create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(h.sum(), x)


@pytest.mark.gpu
@pytest.mark.parametrize("coeff", [None, 0.0], ids=["absent", "zero"])
def test_module_without_amips_unchanged(ext, coeff, monkeypatch):
    """amips_coeff absent or 0: a handle without enable_amips, the route and outputs of the module without the flag."""
    torch = _torch()
    from tssplat_b200 import energies
    V, T, _, inputs, v = _mesh("shuffled")

    def boom(*a, **k):
        raise AssertionError("the AMIPS route ran without amips_coeff")

    monkeypatch.setattr(energies.SmoothnessBarrierAmipsFunc, "apply", boom)
    E_mod = _energy(V, T, coeff, deterministic=False)
    E_ref = _energy(V, T, None, deterministic=False)
    assert E_mod.amips_coeff == 0.0
    x_np = inputs["benign_o2"][0]
    xs = [torch.from_numpy(x_np).cuda().requires_grad_(True) for _ in range(2)]
    Es = [m(xx, 10, 2e-3, 0.8) for m, xx in ((E_mod, xs[0]), (E_ref, xs[1]))]
    assert type(Es[0].grad_fn).__name__ == type(Es[1].grad_fn).__name__
    for E in Es:
        E.backward()
    assert torch.equal(Es[0].detach(), Es[1].detach()) and torch.equal(xs[0].grad, xs[1].grad)
    w = torch.from_numpy(v).cuda()
    assert torch.equal(E_mod.hvp(xs[0], w, 10), E_ref.hvp(xs[1], w, 10))
    # the handle has no AMIPS term: c3 != 0 is rejected
    with pytest.raises(RuntimeError, match="enable_amips"):
        E_mod.tet_sp.energy_grad(xs[0].detach(), 2e-3, 0.8, 2, c3=0.5)


def test_module_default_has_no_amips():
    """A module assembled without __init__ (bench.py's autograd arm does) has amips_coeff 0: the route it always had."""
    import torch
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    eng = SmoothnessBarrierEnergy.__new__(SmoothnessBarrierEnergy)
    torch.nn.Module.__init__(eng)
    assert eng.amips_coeff == 0.0

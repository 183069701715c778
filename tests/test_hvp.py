"""Hessian-vector products of the smoothness and barrier energy (tsb_hvp, TetSpheres.hvp, the twice-differentiable
autograd route of SmoothnessBarrierEnergy).

CPU: an fp64 matrix-form hvp on the oracle's operators (defined here) against central differences of its own gradient, its symmetry, its curvature,
and two known answers.  GPU: the kernel against the oracle per term and combined, curv_out, bitwise repeatability on a
deterministic handle, a tsb_energy_grad after a tsb_hvp on one stream, argument checks, and autograd."""
import ctypes as C
import os
from types import SimpleNamespace

import numpy as np
import pytest

from _helpers import (CELL_FORMAT, GOLDEN, PLAN_SHAPE_MESHES, build_host_plan, check_handle_plan_shape, min_abs_J,
                      mirror_components, plan_shape_cases, plan_shape_mesh, walk_streams)
from oracle.tet_energy_oracle import ReferenceEnergyOracle, _cof3, _det3
from tssplat_b200.mesh import make_pack, perturb

REL = 1e-5                  # kernel vs the fp64 oracle
GH = 0.7                    # gradH of the GPU runs
TERMS = [(1.0, 0.0), (0.0, 1.0), (2e-3, 0.8)]
U = 2.0 ** -24              # fp32 unit roundoff
# plan-shape meshes: per sphere |err_s| <= max(REL |ref_s|, KAPPA_SPHERE u |A_s|) (A: the row magnitudes |c1 M| |v| +
# |c2 H_b| |v| + |c3 H_a| |v|), and on the pole's row 0 (988 streamed entries, 1972 tets) |err_0| <= KAPPA_ROW u A_0
# per coordinate (test_pole_row_kappa: an fp32 re-enactment of the row stays within KAPPA_ROW / 4)
KAPPA_SPHERE = 64
KAPPA_ROW = 16


# ---------------------------------------------------------------------------------------------------------------------
# fp64 Hessian-vector products on top of ReferenceEnergyOracle's operators, in matrix form (the kernel evaluates the
# same quantities in cross-product form on the tet's edges, so the two stay independent).
# H(x) = c1 M + c2 sum_t H_t(x), phi(J) = max(-J, 0)^p.  Per tet with J < 0:
#     F = G x,  dF = G v,  dJ = cof(F) : dF,
#     H_t v = G^T (phi''(J) dJ cof(F) + phi'(J) d cof(F)[dF]),   phi' = -p (-J)^(p-1),  phi'' = p (p-1) (-J)^(p-2)


def _cof_pair(A, B):
    """The symmetric bilinear form behind the cofactor: _cof3(F) = _cof_pair(F, F), entry by entry with every 2x2-minor
    product a*b written A_a*B_b."""
    C = np.empty_like(A)
    C[:, 0, 0] = A[:, 1, 1] * B[:, 2, 2] - A[:, 1, 2] * B[:, 2, 1]
    C[:, 0, 1] = A[:, 1, 2] * B[:, 2, 0] - A[:, 1, 0] * B[:, 2, 2]
    C[:, 0, 2] = A[:, 1, 0] * B[:, 2, 1] - A[:, 1, 1] * B[:, 2, 0]
    C[:, 1, 0] = A[:, 0, 2] * B[:, 2, 1] - A[:, 0, 1] * B[:, 2, 2]
    C[:, 1, 1] = A[:, 0, 0] * B[:, 2, 2] - A[:, 0, 2] * B[:, 2, 0]
    C[:, 1, 2] = A[:, 0, 1] * B[:, 2, 0] - A[:, 0, 0] * B[:, 2, 1]
    C[:, 2, 0] = A[:, 0, 1] * B[:, 1, 2] - A[:, 0, 2] * B[:, 1, 1]
    C[:, 2, 1] = A[:, 0, 2] * B[:, 1, 0] - A[:, 0, 0] * B[:, 1, 2]
    C[:, 2, 2] = A[:, 0, 0] * B[:, 1, 1] - A[:, 0, 1] * B[:, 1, 0]
    return C


def hvp_terms(orc, x, v, order):
    """(M v, sum_t H_t v, v^T M v, per-tet v^T H_t v) at x along v; H_t is 0 for tets with J >= 0."""
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    v = np.asarray(v, dtype=np.float64).reshape(-1)
    Mv = orc.M @ v
    F = (orc.G @ x).reshape(-1, 3, 3)
    dF = (orc.G @ v).reshape(-1, 3, 3)
    J = _det3(F)
    inv = J < 0
    m = np.where(inv, -J, 0)
    if order == 2:
        d1, d2 = -2.0 * m, np.full_like(m, 2.0)
    elif order == 4:
        d1, d2 = -4.0 * m ** 3, 12.0 * m ** 2
    else:
        raise ValueError("order must be 2 or 4")
    C = _cof3(F)
    dJ = np.einsum("tij,tij->t", C, dF)
    dC = _cof_pair(F, dF) + _cof_pair(dF, F)          # directional derivative of cof at F along dF
    P = (d2 * dJ)[:, None, None] * C + d1[:, None, None] * dC
    P[~inv] = 0
    Hbv = orc.G.T @ P.reshape(-1)
    q = np.einsum("tij,tij->t", P, dF)                # v^T H_t v = dF : P_t
    return Mv, Hbv, float(np.dot(v, Mv)), q


def hvp(orc, x, v, c1, c2, order):
    """H(x) v of c1 * smooth + c2 * barrier, [n, 3]."""
    Mv, Hbv, _, _ = hvp_terms(orc, x, v, order)
    return (c1 * Mv + c2 * Hbv).reshape(-1, 3)


def curvature(orc, x, v, c1, c2, order):
    """v^T H(x) v as [c1 vMv + c2 vHbv, vMv, vHbv] (what tsb_hvp writes to curv_out)."""
    _, _, vMv, q = hvp_terms(orc, x, v, order)
    vHbv = float(q.sum())
    return np.array([c1 * vMv + c2 * vHbv, vMv, vHbv])


def _rel(a, b):
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300)


def _inverted(pack, sigma=0.02, seed=0):
    """Perturbed, then every second sphere mirrored (its tets at J near -1): inverted tets with J far from 0, where the
    barrier's Hessian is smooth and fp32 and fp64 agree on the active set."""
    return mirror_components(perturb(pack, sigma_rel=sigma, seed=seed), pack.tets)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle


@pytest.fixture(scope="module")
def small():
    pk = make_pack(3, 512, seed=4)
    orc = ReferenceEnergyOracle(pk.verts, pk.tets)
    xb = perturb(pk, sigma_rel=0.02, seed=1).astype(np.float64)
    xi = _inverted(pk, seed=2).astype(np.float64)
    for x in (xb, xi):
        assert min_abs_J(pk.verts, pk.tets, x) > 1e-2       # away from J = 0: the barrier is smooth around x
    rng = np.random.default_rng(5)
    return SimpleNamespace(pk=pk, orc=orc, x={"benign": xb, "inverted": xi}, v=rng.normal(size=xb.shape),
                           w=rng.normal(size=xb.shape))


@pytest.mark.parametrize("order", [2, 4])
@pytest.mark.parametrize("case", ["benign", "inverted"])
def test_oracle_hvp_matches_central_differences(small, case, order):
    x, v, orc = small.x[case], small.v, small.orc
    c1, c2 = 1e-3, 1.0
    eps = 1e-6
    fd = (orc.backward(1.0, x + eps * v, c1, c2, order) - orc.backward(1.0, x - eps * v, c1, c2, order)) / (2 * eps)
    hv = hvp(orc, x, v, c1, c2, order)
    assert _rel(hv, fd) <= 1e-6
    if case == "inverted":      # the barrier term is a real part of the product
        _, Hbv, _, q = hvp_terms(orc, x, v, order)
        assert np.linalg.norm(Hbv) > 1e-3 * np.linalg.norm(hv) and np.count_nonzero(q) > 0


@pytest.mark.parametrize("order", [2, 4])
@pytest.mark.parametrize("case", ["benign", "inverted"])
def test_oracle_hvp_symmetric_and_curvature(small, case, order):
    x, v, w, orc = small.x[case], small.v, small.w, small.orc
    c1, c2 = 1e-3, 1.0
    hv, hw = hvp(orc, x, v, c1, c2, order).reshape(-1), hvp(orc, x, w, c1, c2, order).reshape(-1)
    a, b = np.dot(w.reshape(-1), hv), np.dot(v.reshape(-1), hw)
    assert abs(a - b) <= 1e-10 * max(abs(a), abs(b))
    curv = curvature(orc, x, v, c1, c2, order)
    assert curv[0] == pytest.approx(np.dot(v.reshape(-1), hv), rel=1e-12)
    Mv, Hbv, vMv, q = hvp_terms(orc, x, v, order)
    assert curv[1] == pytest.approx(np.dot(v.reshape(-1), Mv), rel=1e-12) and curv[1] == vMv
    assert curv[2] == pytest.approx(np.dot(v.reshape(-1), Hbv), rel=1e-10, abs=1e-300)


def test_oracle_known_answers(small):
    orc, x, v = small.orc, small.x["benign"], small.v
    for order in (2, 4):
        Mv, Hbv, _, q = hvp_terms(orc, x, v, order)
        assert not Hbv.any() and not q.any()                 # no inverted tet: H v = c1 M v
        assert np.array_equal(hvp(orc, x, v, 0.3, 5.0, order).reshape(-1), 0.3 * Mv)
    # affine v (v = A X + b): M v = 0, and with no inverted tet H v = 0
    X = small.pk.verts.astype(np.float32).astype(np.float64)
    A = np.array([[0.3, -1.2, 0.5], [2.0, 0.1, -0.7], [0.4, 0.9, 1.5]])
    va = X @ A.T + np.array([0.2, -3.0, 1.0])
    hv = hvp(orc, x, va, 1.0, 1.0, 2)
    scale = abs(orc.M).sum(axis=1).max() * np.abs(va).max()
    assert np.abs(hv).max() <= 1e-12 * scale


def _pole_row_fp32(v, c1, tet_rows, seed):
    """Row 0 of c1 M v + the tet products on the pole, re-enacted in fp32: the smoothness row pass over the GLOBAL plan's
    row block in lane order (each lane a sequence of fp32 fused multiply-adds w (v_j - v_0), then the pairwise lane
    reduction), plus the tets' fp64 contributions rounded to fp32 and added in a random order (the atomics' order)."""
    V, T = plan_shape_mesh("pole")
    plan = build_host_plan(V, T, force_global=1)
    CELL, IB, _ = CELL_FORMAT[True]
    st, f32 = plan["stream"], np.float32
    v32 = np.asarray(v, f32)
    blocks = [(p, hdr) for p, hdr in walk_streams(plan)[0] if (hdr & 0xFFFFFF == 0).any()]
    assert len(blocks) == 1
    p, hdr = blocks[0]
    len4, L = int((hdr[0] >> 24) & 63), 1 << int(hdr[0] >> 30)
    lanes = np.arange(L) + np.flatnonzero((hdr & 0xFFFFFF) == 0)[0]
    acc = np.zeros((L, 3), f32)
    for q in range(len4):
        j = st[p + q * CELL:p + q * CELL + 128 * IB].view(np.uint32).reshape(32, 4)[lanes].astype(np.int64)
        w = st[p + q * CELL + 128 * IB:p + q * CELL + 128 * IB + 512].view(f32).reshape(32, 4)[lanes]
        for c in range(4):
            d = (v32[j[:, c]] - v32[0]).astype(f32)
            acc = (w[:, c, None].astype(np.float64) * d + acc).astype(f32)
    while len(acc) > 1:
        acc = (acc[:len(acc) // 2] + acc[len(acc) // 2:]).astype(f32)
    out = (f32(c1) * acc[0]).astype(f32)
    for t in np.random.default_rng(seed).permutation(len(tet_rows)):
        out = (out + tet_rows[t].astype(f32)).astype(f32)
    return out.astype(np.float64)


def test_pole_row_kappa():
    """KAPPA_ROW holds with a factor 4 to spare for the fp32 re-enactment of the pole's row 0 (_pole_row_fp32) on every
    input and term combination of the GPU checks, with and without AMIPS."""
    from test_hess_diag import tet_hessians
    from test_hvp_amips import _mesh as amips_mesh
    V, T, orc, inputs, v = amips_mesh("pole")
    T64 = np.asarray(T, np.int64)
    vv = v.astype(np.float64)
    assert (T64[:, 0] == 0).all()                              # every tet has the pole as corner 0
    worst = 0.0
    for case, (x, order) in inputs.items():
        sc = row_scales("pole", case, x, order)
        for c1, c2, c3 in ((1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (2e-3, 0.8, 0.0), (0.0, 0.0, 1.0), (2e-3, 0.8, 0.5)):
            Ht, _ = tet_hessians(V, T64, x, c2, c3, order)
            tet_rows = np.einsum("tab,tb->ta", Ht[:, :3], vv[T64].reshape(-1, 12))
            Mv = (orc.M @ vv.reshape(-1)).reshape(-1, 3)
            ref = c1 * Mv[0] + tet_rows.sum(axis=0)
            A = c1 * sc[0][0] + c2 * sc[1][0] + c3 * sc[2][0]
            for seed in range(3):
                err = np.abs(_pole_row_fp32(v, c1, tet_rows, seed) - ref)
                assert (err[A == 0] == 0).all()                # e.g. the barrier alone with no inverted tet
                worst = max(worst, (err[A > 0] / (U * A[A > 0])).max(initial=0.0))
    print(f"pole row 0, fp32 re-enactment: max |err_0| / (u A_0) = {worst:.3g} (KAPPA_ROW {KAPPA_ROW})")
    assert worst <= KAPPA_ROW / 4


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
    """(rest, tets, oracle, inputs {case: (x, order)}, direction) of a test mesh, built once."""
    if name not in _MESHES:
        if name == "pack64x4096":
            pk = make_pack(64, 4096, seed=0, unique=8)
            V, T = pk.verts, pk.tets
            inputs = {"benign_o2": (perturb(pk, sigma_rel=0.02, seed=1), 2), "inverted_o2": (_inverted(pk, seed=2), 2),
                      "inverted035_o4": (perturb(pk, sigma_rel=0.35, seed=3), 4)}
        elif name == "a_veg":
            d = np.load(os.path.join(GOLDEN, "a_veg_mesh.npz"))
            V, T = d["verts"].astype(np.float32), d["tets"].astype(np.int32)
            rng = np.random.default_rng(6)
            h = np.linalg.norm(V[T[:, 1]] - V[T[:, 0]], axis=1).mean()
            xb = (V + rng.normal(scale=0.02 * h, size=V.shape)).astype(np.float32)
            xi = xb.copy()
            xi[:, 2] = 2 * xi[:, 2].mean() - xi[:, 2]              # the whole mesh mirrored: every tet inverted
            inputs = {"benign_o2": (xb, 2), "inverted_o2": (xi, 2), "inverted_o4": (xi, 4)}
        elif name == "shuffled":
            # a 3 x 1024 pack under a random vertex relabelling into a larger id space: orphan vertices everywhere,
            # non-contiguous components
            pk = make_pack(3, 1024, seed=1)
            rng = np.random.default_rng(8)
            n = len(pk.verts) + 500
            ids = rng.permutation(n)[:len(pk.verts)]
            V = rng.normal(size=(n, 3)).astype(np.float32)
            V[ids] = pk.verts
            T = ids[pk.tets].astype(np.int32)
            xb = V.copy()
            xb[ids] = perturb(pk, sigma_rel=0.02, seed=1)
            xi = V.copy()
            xi[ids] = _inverted(pk, seed=2)
            inputs = {"benign_o2": (xb, 2), "inverted_o2": (xi, 2), "inverted_o4": (xi, 4)}
        elif name in PLAN_SHAPE_MESHES:
            V, T = plan_shape_mesh(name)
            T64 = T.astype(np.int64)
            P = V[T64].astype(np.float64)              # h: the tets' shortest edge (the pole's are 1 long, 0.1 wide)
            h = np.min([np.linalg.norm(P[:, a] - P[:, b], axis=1) for a in range(4) for b in range(a)], axis=0).mean()
            used = np.unique(T64)
            xb = V.copy()
            xb[used] += np.random.default_rng(6).normal(scale=0.02 * h, size=(len(used), 3)).astype(np.float32)
            xi = mirror_components(xb, T)
            inputs = {"benign_o2": (xb, 2), "inverted_o2": (xi, 2), "inverted_o4": (xi, 4)}
        else:
            raise KeyError(name)
        for key, (x, order) in inputs.items():
            if "035" not in key:
                assert min_abs_J(V, T, x) > 1e-3, (name, key)
        orc = ReferenceEnergyOracle(V, T)
        v = np.random.default_rng(9).normal(size=(len(V), 3)).astype(np.float32)
        _MESHES[name] = (V, T, orc, inputs, v)
    return _MESHES[name]


_SCALES = {}


def row_scales(mesh, case, x, order):
    """[3, n, 3]: |M| |v|, sum_t |H_b,t| |v| and sum_t |H_a,t| |v| at input `case` (x, order) of a plan-shape mesh, the
    terms of the row magnitude A of the per-sphere and pole-row bounds."""
    if (mesh, case) not in _SCALES:
        from test_hess_diag import tet_hessians
        V, T, orc, _, v = _mesh(mesh)
        av = np.abs(v.astype(np.float64))
        out = [(abs(orc.M) @ av.reshape(-1)).reshape(-1, 3)]
        for c2, c3 in ((1.0, 0.0), (0.0, 1.0)):
            At = tet_hessians(V, T, x, c2, c3, order)[1]
            y = np.einsum("tab,tb->ta", At, av[T].reshape(-1, 12)).reshape(-1, 4, 3)
            s = np.zeros_like(av)
            np.add.at(s, np.asarray(T, np.int64), y)
            out.append(s)
        _SCALES[(mesh, case)] = np.stack(out)
    return _SCALES[(mesh, case)]


def check_spheres_and_pole_row(mesh, key, err, parts, A):
    """Per sphere |err_s| <= max(sum_k rel_k |part_k,s|, KAPPA_SPHERE u |A_s|) for parts = [(rel_k, part_k [n, 3])] (the
    suite's own whole-mesh bound, taken per sphere), and on the pole |err_0| <= KAPPA_ROW u A_0.  Returns the worst ratio
    of each."""
    from tssplat_b200.mesh import connected_components
    V, T, *_ = _mesh(mesh)
    lab = connected_components(len(V), np.asarray(T).reshape(-1, 4))
    nrm = lambda a: np.sqrt(np.bincount(lab, weights=(a * a).sum(axis=1)))
    bound = np.maximum(sum(rel * nrm(p) for rel, p in parts), KAPPA_SPHERE * U * nrm(A))
    e = nrm(err)
    assert (e <= bound).all(), (key, int(np.argmax(e / bound)), (e / bound).max())
    worst = {"sphere": (e / np.maximum(bound, 1e-300)).max()}
    if mesh == "pole":
        a0, e0 = A[0], np.abs(err[0])
        assert (e0[a0 == 0] == 0).all(), (key, e0)          # e.g. the barrier alone with no inverted tet
        r = e0[a0 > 0] / (U * a0[a0 > 0])
        assert (r <= KAPPA_ROW).all(), (key, r)
        worst["row 0"] = r.max(initial=0.0)
    return worst


WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nhvp on the plan-shape meshes: worst |err_s| / bound per sphere, |err_0| / (u A_0) on the pole row:")
        for k, v in sorted(WORST.items()):
            print(f"  {k}: {v:.3g}")


def _hvp(sp, x, v, c1, c2, order, gradH=GH):
    torch = _torch()
    hv, curv = sp.hvp(torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda(),
                      torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda(), c1, c2, order, gradH=gradH, want_curv=True)
    return hv.cpu().numpy().astype(np.float64), curv.cpu().numpy().astype(np.float64)


def _check_against_oracle(sp, mesh, key_prefix, orphans=None):
    V, T, orc, inputs, v = _mesh(mesh)
    vv = v.astype(np.float64)
    for case, (x, order) in inputs.items():
        x64 = x.astype(np.float64)
        Mv, Hbv, vMv, q = hvp_terms(orc, x64, vv, order)
        for c1, c2 in TERMS:
            key = (key_prefix, case, c1, c2)
            hv, curv = _hvp(sp, x, v, c1, c2, order)
            ref = GH * (c1 * Mv + c2 * Hbv).reshape(-1, 3)
            if np.linalg.norm(ref) == 0:
                assert not hv.any(), key                      # barrier alone, no inverted tet: exactly 0
            else:
                assert _rel(hv, ref) <= REL, (key, _rel(hv, ref))
            if orphans is not None:
                assert not hv[orphans].any(), key
            if mesh in PLAN_SHAPE_MESHES:
                sc = row_scales(mesh, case, x, order)
                parts = [(REL, ref)]
                for name, w in check_spheres_and_pole_row(mesh, key, hv - ref, parts, GH * (c1 * sc[0] + c2 * sc[1])).items():
                    WORST[(mesh, name)] = max(WORST.get((mesh, name), 0.0), w)
            scale = c1 * abs(vMv) + c2 * np.abs(q).sum()
            assert abs(curv[0] - (c1 * vMv + c2 * q.sum())) <= REL * scale, (key, curv, vMv, q.sum())
            assert abs(curv[1] - vMv) <= REL * abs(vMv), (key, curv[1], vMv)
            assert abs(curv[2] - q.sum()) <= REL * max(np.abs(q).sum(), 1e-300), (key, curv[2], q.sum())
            if "inverted" in case:
                assert np.count_nonzero(q) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(warps_per_cta=8), dict(deterministic=True),
                                dict(warps_per_cta=8, deterministic=True)],
                         ids=["w16", "w8", "w16-det", "w8-det"])
def test_hvp_staged_pack(ext, kw):
    V, T, *_ = _mesh("pack64x4096")
    sp = _handle(ext, V, T, **kw)
    assert sp.info["mode_global"] == 0
    _check_against_oracle(sp, "pack64x4096", str(kw))


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(force_global=True), dict(force_global=True, warps_per_cta=8, deterministic=True)],
                         ids=["global", "global-w8-det"])
def test_hvp_a_veg_global(ext, kw):
    V, T, *_ = _mesh("a_veg")
    sp = _handle(ext, V, T, **kw)
    assert sp.info["mode_global"] == 1
    _check_against_oracle(sp, "a_veg", str(kw))


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(force_global=True), dict(warps_per_cta=8, ring_slots=3, deterministic=True)],
                         ids=["staged", "global", "w8-ring3-det"])
def test_hvp_shuffled_ids_with_orphans(ext, kw):
    V, T, *_ = _mesh("shuffled")
    sp = _handle(ext, V, T, **kw)
    orphans = np.ones(len(V), bool)
    orphans[np.unique(T)] = False
    assert orphans.sum() == 500
    _check_against_oracle(sp, "shuffled", str(kw), orphans=orphans)


@pytest.mark.gpu
@pytest.mark.parametrize("mesh,kw", plan_shape_cases())
def test_hvp_plan_shapes(ext, mesh, kw):
    """The products on the plans only these meshes produce (assert_plan_shape): the pole's ring-wrapping row block, whole-
    area staging, GLOBAL by size, segment headers past the shared-memory table."""
    V, T, *_ = _mesh(mesh)
    sp = _handle(ext, V, T, **kw)
    check_handle_plan_shape(mesh, sp, kw)
    _check_against_oracle(sp, mesh, str(kw))


def _inverted_touched(T, x):
    """Vertices of the tets with J < 0 at x (with a margin: tets near J = 0 count)."""
    P = np.asarray(x, np.float64)[T]
    e = P[:, 1:] - P[:, :1]
    det = np.einsum("ij,ij->i", e[:, 0], np.cross(e[:, 1], e[:, 2]))
    touched = np.zeros(int(T.max()) + 1, bool)
    touched[T[det < 1e-3 * np.abs(det).max()].reshape(-1)] = True
    return touched


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(force_global=True, warps_per_cta=8)], ids=["staged", "global-w8"])
def test_hvp_deterministic_bitwise(ext, kw):
    torch = _torch()
    V, T, _, inputs, v = _mesh("pack64x4096")
    x_np, order = inputs["inverted_o2"]
    det = _handle(ext, V, T, deterministic=True, **kw)
    plain = _handle(ext, V, T, **kw)
    x = torch.from_numpy(x_np).cuda()
    vt = torch.from_numpy(v).cuda()
    c1, c2 = 2e-3, 0.8
    hv0, cv0 = det.hvp(x, vt, c1, c2, order, gradH=GH, want_curv=True)
    for _ in range(3):
        hv1, cv1 = det.hvp(x, vt, c1, c2, order, gradH=GH, want_curv=True)
        assert torch.equal(hv0, hv1) and torch.equal(cv0, cv1)
    s = torch.cuda.Stream()                                   # another stream, and graph replays
    hv_g = torch.empty_like(hv0)
    cv_g = torch.empty_like(cv0)
    from tssplat_b200 import _capi
    with torch.cuda.stream(s):
        assert _capi.lib.tsb_hvp(det._h, x.data_ptr(), vt.data_ptr(), c1, c2, order, GH, None, hv_g.data_ptr(),
                                 cv_g.data_ptr(), s.cuda_stream) == 0
    s.synchronize()
    assert torch.equal(hv0, hv_g) and torch.equal(cv0, cv_g)
    g = torch.cuda.CUDAGraph()
    hv_g.fill_(float("nan"))
    with torch.cuda.graph(g, stream=s):
        assert _capi.lib.tsb_hvp(det._h, x.data_ptr(), vt.data_ptr(), c1, c2, order, GH, None, hv_g.data_ptr(),
                                 cv_g.data_ptr(), s.cuda_stream) == 0
    for _ in range(3):
        hv_g.fill_(float("nan"))
        cv_g.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(hv0, hv_g) and torch.equal(cv0, cv_g)
    # rows no inverted tet touches: bitwise those of a default handle
    hv_p, _ = plain.hvp(x, vt, c1, c2, order, gradH=GH)
    free = torch.from_numpy(~_inverted_touched(T, x_np)).cuda()
    assert int(free.sum()) > 0 and int((~free).sum()) > 0
    assert torch.equal(hv0[free], hv_p[free])


@pytest.mark.gpu
@pytest.mark.parametrize("kw,case", [(dict(), "benign_o2"), (dict(force_global=True), "benign_o2"),
                                     (dict(warps_per_cta=8), "benign_o2"), (dict(deterministic=True), "inverted_o2"),
                                     (dict(deterministic=True, force_global=True, warps_per_cta=8), "inverted_o2")],
                         ids=["staged", "global", "w8", "det", "det-global-w8"])
def test_energy_grad_after_hvp_unchanged(ext, kw, case):
    """tsb_energy_grad, tsb_hvp, tsb_energy_grad on one stream: both gradient launches give bitwise what a handle that
    never ran tsb_hvp gives (the hvp launch leaves the done counters, energy sentinels and deterministic flags armed)."""
    torch = _torch()
    V, T, _, inputs, v = _mesh("pack64x4096")
    x_np, order = inputs[case]
    x = torch.from_numpy(x_np).cuda()
    x2 = torch.from_numpy((x_np * np.float32(1.001)).astype(np.float32)).cuda()
    vt = torch.from_numpy(v).cuda()
    a, b = _handle(ext, V, T, **kw), _handle(ext, V, T, **kw)
    c1, c2 = 2e-3, 0.8
    ea1, ga1 = a.energy_grad(x, c1, c2, order)
    ea1 = ea1.clone()
    a.hvp(x, vt, c1, c2, order, want_curv=True)
    ea2, ga2 = a.energy_grad(x2, c1, c2, order)
    eb1, gb1 = b.energy_grad(x, c1, c2, order)
    eb1 = eb1.clone()
    eb2, gb2 = b.energy_grad(x2, c1, c2, order)
    torch.cuda.synchronize()
    assert torch.equal(ea1, eb1) and torch.equal(ga1, gb1)
    assert torch.equal(ea2, eb2) and torch.equal(ga2, gb2)


@pytest.mark.gpu
def test_hvp_bad_arguments(ext):
    torch = _torch()
    from tssplat_b200 import _capi
    V, T, _, inputs, v = _mesh("shuffled")
    sp = _handle(ext, V, T)
    x = torch.from_numpy(inputs["benign_o2"][0]).cuda()
    vt = torch.from_numpy(v).cuda()
    hv = torch.empty_like(x)
    st = torch.cuda.current_stream().cuda_stream
    call = _capi.lib.tsb_hvp
    assert call(sp._h, x.data_ptr(), vt.data_ptr(), 1.0, 1.0, 3, 1.0, None, hv.data_ptr(), None, st) == _capi.TSB_E_INVALID
    assert call(sp._h, x.data_ptr(), None, 1.0, 1.0, 2, 1.0, None, hv.data_ptr(), None, st) == _capi.TSB_E_INVALID
    assert call(sp._h, x.data_ptr(), vt.data_ptr(), 1.0, 1.0, 2, 1.0, None, None, None, st) == _capi.TSB_E_INVALID
    assert call(sp._h, None, vt.data_ptr(), 1.0, 1.0, 2, 1.0, None, hv.data_ptr(), None, st) == _capi.TSB_E_INVALID
    assert call(None, x.data_ptr(), vt.data_ptr(), 1.0, 1.0, 2, 1.0, None, hv.data_ptr(), None, st) == _capi.TSB_E_INVALID
    with pytest.raises(RuntimeError):
        sp.hvp(x, vt[:-1], 1.0, 1.0, 2)
    with pytest.raises(RuntimeError):
        sp.hvp(x, vt.double(), 1.0, 1.0, 2)
    # the module-level form, and a CUDA gradH
    hv1 = ext.hvp(vt, x, sp, 1.0, 1.0, 2)
    hv2, _ = sp.hvp(x, vt, 1.0, 1.0, 2, gradH=torch.tensor(2.0, device="cuda"))
    assert torch.equal(2 * hv1, hv2)


def _energy(ext_unused, V, T, twice, deterministic=True):
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    flags = dict(smooth_eng_coeff=2e-3, barrier_coeff=0.8, increase_order_iter=100, deterministic=deterministic)
    if twice is not None:
        flags["twice_differentiable"] = twice
    return SmoothnessBarrierEnergy(V, T.reshape(-1, 4), flags)


@pytest.mark.gpu
@pytest.mark.parametrize("it", [10, 500], ids=["order2", "order4"])
def test_twice_differentiable_autograd(ext, it):
    torch = _torch()
    V, T, _, inputs, v = _mesh("shuffled")
    E_mod = _energy(ext, V, T, True)
    c1, c2 = E_mod.coeff_scheduler(it)
    x = torch.from_numpy(inputs["inverted_o2"][0]).cuda().requires_grad_(True)
    w = torch.from_numpy(v).cuda()
    ref = E_mod.hvp(x, w, it)
    E = E_mod(x, it, c1, c2)
    assert "SmoothnessBarrierFunc2" in type(E.grad_fn).__name__
    (g,) = torch.autograd.grad(E, x, create_graph=True)
    _, g_ref = E_mod.tet_sp.energy_grad(x.detach(), c1, c2, E_mod.order_at(it))
    assert torch.equal(g.detach(), g_ref)
    (hw,) = torch.autograd.grad((g * w).sum(), x)
    assert torch.allclose(hw, ref, rtol=0, atol=1e-6 * float(ref.abs().max()))
    # torch.autograd.functional.vhp
    _, vh = torch.autograd.functional.vhp(lambda xx: E_mod(xx, it, c1, c2), x.detach(), w)
    assert torch.allclose(vh, ref, rtol=0, atol=1e-6 * float(ref.abs().max()))
    # a scale s that requires grad: d/ds sum(s grad E . w) = grad E . w, and d/dx = s H w
    s = torch.tensor(0.7, device="cuda", requires_grad=True)
    E = E_mod(x, it, c1, c2)
    (g,) = torch.autograd.grad(E, x, grad_outputs=s, create_graph=True)
    gx, gs = torch.autograd.grad((g * w).sum(), (x, s))
    assert float(gs) == pytest.approx(float((g_ref.double() * w.double()).sum()), rel=1e-5)
    assert torch.allclose(gx, 0.7 * ref, rtol=0, atol=1e-6 * float(ref.abs().max()))
    # a third derivative raises
    E = E_mod(x, it, c1, c2)
    (g,) = torch.autograd.grad(E, x, create_graph=True)
    (h,) = torch.autograd.grad((g * w).sum(), x, create_graph=True)
    with pytest.raises(RuntimeError):
        torch.autograd.grad(h.sum(), x)


@pytest.mark.gpu
@pytest.mark.parametrize("twice", [None, False])
def test_default_route_unchanged(ext, twice, monkeypatch):
    torch = _torch()
    from tssplat_b200 import energies
    V, T, _, inputs, _ = _mesh("shuffled")
    E_mod = _energy(ext, V, T, twice, deterministic=False)

    def boom(*a, **k):
        raise AssertionError("the twice-differentiable route ran without the flag")

    monkeypatch.setattr(energies.SmoothnessBarrierFunc2, "apply", boom)
    x = torch.from_numpy(inputs["benign_o2"][0]).cuda().requires_grad_(True)
    E = E_mod(x, 10, 2e-3, 0.8)
    assert "SmoothnessBarrierFunc2" not in type(E.grad_fn).__name__
    E.backward()
    _, g_ref = E_mod.tet_sp.energy_grad(x.detach(), 2e-3, 0.8, 2)
    assert torch.equal(x.grad, g_ref)

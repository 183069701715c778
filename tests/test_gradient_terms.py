"""Per-term and per-row gradient parity against the fp64 oracle, and row ids at the top of the 24-bit range.

The other parity tests take one metric, ||g - g_oracle||_2 <= 1e-5 ||g_oracle||_2 over the whole pack with every energy
term summed.  It has two blind spots: an error confined to a small term hides under a large one (the smoothness term
is 0.4 % of the 16 x 4096 order-4 gradient, so a 2.6e-3 error in it passes), and an error confined to a few rows
vanishes in the norm (one row 1e-3 wrong among 13 k rows).  Here:

* each term runs alone (one coefficient non-zero) against the oracle's gradient and energy of that term, relative to
  that term's own norm;
* every row of the gradient is checked against a per-row, per-coordinate scale A (RowScale): the sums of the gradient
  with every product and difference replaced by its magnitude, |g - g_oracle|[i, c] <= KAPPA 2^-24 A[i, c], and
  vertices no tet references must be exactly 0;
* a mesh of n = 0xFFFFFE vertices (the largest a handle accepts) puts row ids with bits 20..23 set in the row-block
  headers (rid | len4 << 24 | log2(L) << 30), with about 16.7 M orphan rows to zero.

KAPPA is calibrated on the CPU with emulate_kernel(dtype=np.float32), the kernel's fp32 operations in its order, on
the inputs of the GPU tests (test_kappa_calibration)."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sps

from _helpers import COracle, build_host_plan, emulate_kernel, mirror_components, plan_shape_mesh, walk_streams
from oracle.tet_energy_oracle import build_G, rest_inverse, tet_laplacian
from tssplat_b200.mesh import connected_components, make_pack, perturb

U24 = 2.0 ** -24
# |g - g_oracle| <= KAPPA 2^-24 A per row and coordinate.  Largest err / (2^-24 A) observed: 2.31 in the fp32
# re-enactment (test_kappa_calibration: tiny components, AMIPS input, order 4); 2.75 on an H100 80GB HBM3 (700 W power
# limit), every plan and input of the GPU tests below (same mesh and input).  Before A took the corner order of the streamed tets into
# account (the barrier corner streamed first is minus the sum of the other three) both were near 24 and 33.
KAPPA = 16.0
REL = 1e-5                  # per-term gradient and energy tolerance (2e-5 for AMIPS, as in test_gpu_parity)
GH = 0.7                    # gradH of every run


# ---------------------------------------------------------------------------------------------------------------------
# The per-row scale


def _mag_cross(a, b):
    """|a| x |b| with every product and difference replaced by its magnitude (a, b: [..., 3] magnitudes)."""
    return np.stack([a[..., 1] * b[..., 2] + a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] + a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0]], axis=-1)


class RowScale:
    """The fp64 gradient of one mesh split into its terms, and the per-row scale A of each term.

    Smoothness: g_s[i] = gradH c1 sum_j M_ij (u_j - u_i), M = G^T L^T L G per coordinate; A_s[i] = |gradH c1|
    sum_j |M_ij| (|u_j - u_i| + |u_j| + |u_i|), the last two for the rounding of the staged displacements
    u = (x - X) - (x_r - X_r) (r: the component's reference vertex, its smallest vertex id).
    Barrier: per inverted tet, the corner vectors k (e2 x e3), k (e3 x e1), k (e1 x e2) and minus their sum, k = -gradH
    c2 p m^(p-1) / det(Dm), m = -J; A_b takes |e|, magnitude cross products and p m^(p-1) + p (p-1) m^(p-2) Jmag for
    the coefficient (Jmag: the magnitude form of J), for whichever corner the plan streams first.  Tets with J a few
    roundings above 0 count as inverted.
    AMIPS: per J > 0 tet, P B^T with P = 2 / (3 J^(2/3)) (F - tr / (3 J) cof F); A_a takes |F|, |cof F| in magnitude
    form and a factor 1 + Jmag / J for the rounding of J."""

    def __init__(self, verts, tets, ids=None):
        X = np.asarray(verts, np.float32).reshape(-1, 3).astype(np.float64)
        T = np.asarray(tets, np.int64).reshape(-1, 4)
        self.n, self.X, self.T = len(X), X, T
        L9 = sps.kron(tet_laplacian(T), sps.identity(9, format="csr"), format="csr")
        LG = (L9 @ build_G(X, T)).tocsr()
        M = (LG.T @ LG).tocsr()[0::3, 0::3].tocoo()          # M acts on each coordinate alike
        off = M.row != M.col
        self.Mi, self.Mj, self.Mv = M.row[off], M.col[off], M.data[off]
        self.B = rest_inverse(X, T)                           # rows: the hat gradients of corners 1..3
        self.idet = np.linalg.det(self.B)                     # 1 / det(Dm)
        # reference vertex per vertex: the smallest id of its component (in `ids` numbering when given)
        ids = np.arange(self.n) if ids is None else np.asarray(ids, np.int64)
        lab = connected_components(self.n, T)
        first = np.full(lab.max() + 1, np.iinfo(np.int64).max)
        np.minimum.at(first, lab, ids)
        where = {int(i): k for k, i in enumerate(ids)}
        self.ref = np.array([where[int(f)] for f in first])[lab]

    def _rows(self, w):
        return np.stack([np.bincount(self.Mi, weights=w[:, c], minlength=self.n) for c in range(3)], axis=1)

    def _scatter(self, corners):
        """[T, 4, 3] corner vectors -> [n, 3] per-vertex sums."""
        out = np.zeros((self.n, 3))
        for k in range(4):
            for c in range(3):
                out[:, c] += np.bincount(self.T[:, k], weights=corners[:, k, c], minlength=self.n)
        return out

    def tet_terms(self, x, c2, c3, order, gradH=GH):
        """Corner vectors and their magnitude forms, [T, 4, 3] each: (barrier, barrier A, AMIPS, AMIPS A), with the
        masks of the tets the oracle counts (J < 0 and J > 0)."""
        P = np.asarray(x, np.float32).reshape(-1, 3).astype(np.float64)[self.T]
        e = P[:, 1:] - P[:, :1]                                # e[:, k] = e_{k+1}
        e1, e2, e3 = e[:, 0], e[:, 1], e[:, 2]
        cr = [np.cross(e2, e3), np.cross(e3, e1), np.cross(e1, e2)]
        J = np.einsum("tr,tr->t", e1, cr[0]) * self.idet
        a = np.abs(e)
        Jmag = np.einsum("tr,tr->t", a[:, 0], _mag_cross(a[:, 1], a[:, 2])) * np.abs(self.idet)   # symmetric in the edges
        inv = J < 0
        m = np.where(inv, -J, 0.0)
        k = -order * m ** (order - 1) * self.idet * c2 * gradH
        bar = np.zeros((len(J), 4, 3))
        for q in range(3):
            bar[:, q + 1] = k[:, None] * cr[q]
        bar[:, 0] = -bar[:, 1:].sum(axis=1)
        bar[~inv] = 0.0
        # The staged plan streams a tet with its corners in another even order, and the corner streamed first gets minus
        # the sum of the other three: every corner takes the largest magnitude form over the four choices of first corner
        barA = np.zeros_like(bar)
        for b in range(4):
            o = [j for j in range(4) if j != b]
            f = np.abs(P[:, o] - P[:, b:b + 1])                    # |edges| from corner b
            pm = [_mag_cross(f[:, 1], f[:, 2]), _mag_cross(f[:, 2], f[:, 0]), _mag_cross(f[:, 0], f[:, 1])]
            Jb = np.einsum("tr,tr->t", f[:, 0], pm[0]) * np.abs(self.idet)
            near = J < 4 * U24 * Jb
            me = np.maximum(-J, 0.0) + 4 * U24 * Jb
            kA = np.where(near, order * me ** (order - 1) + order * (order - 1) * me ** (order - 2) * Jb, 0.0)
            kA = kA * np.abs(self.idet * c2 * gradH)
            Ab = np.zeros_like(bar)
            for q in range(3):
                Ab[:, o[q]] = kA[:, None] * pm[q]
            Ab[:, b] = Ab[:, o].sum(axis=1)
            barA = np.maximum(barA, Ab)
        am, amA = np.zeros_like(bar), np.zeros_like(bar)
        ok = J > 0
        if c3:
            Ds, B = e[ok].transpose(0, 2, 1), self.B[ok]           # Ds: edges as columns
            F = Ds @ B
            Fm = np.abs(Ds) @ np.abs(B)                            # the scale of F's rounding
            Jp, Jm = J[ok], Jmag[ok]
            tr = (F * F).sum(axis=(1, 2))
            cof = np.stack([np.cross(F[:, 1], F[:, 2]), np.cross(F[:, 2], F[:, 0]), np.cross(F[:, 0], F[:, 1])], axis=1)
            j23 = np.cbrt(Jp) ** 2
            s = (2 / (3 * j23) * c3 * gradH)[:, None, None]
            Q = F - (tr / (3 * Jp))[:, None, None] * cof
            Pk = s * Q
            # P moves by F's rounding (Fm) to first order: through F, through tr / (3 J) (tr and J) and through
            # cof F; plus J's rounding in the prefactor; plus the rounding of P itself
            aF = np.abs(F)
            dcof = np.stack([_mag_cross(aF[:, 1], Fm[:, 2]) + _mag_cross(Fm[:, 1], aF[:, 2]),
                             _mag_cross(aF[:, 2], Fm[:, 0]) + _mag_cross(Fm[:, 2], aF[:, 0]),
                             _mag_cross(aF[:, 0], Fm[:, 1]) + _mag_cross(Fm[:, 0], aF[:, 1])], axis=1)
            dtr = 2 * (aF * Fm).sum(axis=(1, 2))
            r = lambda v: v[:, None, None]
            PA = np.abs(s) * (Fm + r(tr / (3 * Jp)) * dcof + np.abs(cof) * r((dtr + tr * Jm / Jp) / (3 * Jp))
                              + (1 + r(Jm / Jp)) * np.abs(Q))
            gk = (Pk @ B.transpose(0, 2, 1)).transpose(0, 2, 1)      # [tet][corner k + 1][r]
            gA = ((PA @ np.abs(B).transpose(0, 2, 1)) + np.abs(Pk) @ np.abs(B).transpose(0, 2, 1)).transpose(0, 2, 1)
            am[ok] = np.concatenate([-gk.sum(axis=1, keepdims=True), gk], axis=1)
            amA[ok] = np.concatenate([gA.sum(axis=1, keepdims=True), gA], axis=1)
        return bar, barA, am, amA, inv, ok

    def terms(self, x, c, order, gradH=GH):
        """({term: fp64 gradient}, {term: A}) for c = (c1, c2, c3); terms 'smooth', 'barrier', 'amips'."""
        x64 = np.asarray(x, np.float32).reshape(-1, 3).astype(np.float64)
        dX = x64 - self.X
        u = dX - dX[self.ref]
        d = u[self.Mj] - u[self.Mi]
        s1 = c[0] * gradH
        g = {"smooth": s1 * self._rows(self.Mv[:, None] * d)}
        A = {"smooth": abs(s1) * self._rows(np.abs(self.Mv)[:, None] * (np.abs(d) + np.abs(u[self.Mj]) + np.abs(u[self.Mi])))}
        bar, barA, am, amA, _, _ = self.tet_terms(x, c[1], c[2], order, gradH)
        g["barrier"], A["barrier"] = self._scatter(bar), self._scatter(barA)
        g["amips"], A["amips"] = self._scatter(am), self._scatter(amA)
        return g, A

    def smooth_energy_scale(self, x):
        """Magnitude form of the smoothness energy 1/2 sum_i u_i . (M u)_i: 1/2 sum_i |u_i| A_s[i] / |gradH c1|.  Where
        the displacement is near the operator's null space (an affine stretch) the energy is a small residual of
        large products, and its fp32 rounding is relative to this scale, not to the energy."""
        x64 = np.asarray(x, np.float32).reshape(-1, 3).astype(np.float64)
        dX = x64 - self.X
        u = dX - dX[self.ref]
        return 0.5 * float((np.abs(u) * self.terms(x, (1.0, 0.0, 0.0), 2, 1.0)[1]["smooth"]).sum())

    def bound(self, x, c, order, gradH=GH):
        A = self.terms(x, c, order, gradH)[1]
        return A["smooth"] + A["barrier"] + A["amips"]


def row_ratio(g, go, A):
    """max over rows and coordinates of |g - go| / (2^-24 A), and where it is reached; a row with A = 0 must match
    exactly (inf otherwise), a NaN gives NaN."""
    err = np.abs(np.asarray(g, np.float64) - go)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(A > 0, err / (U24 * A), np.where(err == 0, 0.0, np.inf))
    if np.isnan(r).any():
        return np.nan, int(np.argwhere(np.isnan(r))[0, 0])
    i = int(np.argmax(r.max(axis=1)))
    return float(r[i].max()), i


def assert_rows(g, go, A, kappa=KAPPA, what=""):
    r, i = row_ratio(g, go, A)
    assert r <= kappa, f"{what}: row {i}: |g - g_oracle| = {np.abs(np.asarray(g, np.float64)[i] - go[i])}, " \
                       f"{r:.3g} x 2^-24 A (A = {A[i]}); bound {kappa}"
    return r


def old_metric_passes(g, go):
    return np.linalg.norm(np.asarray(g, np.float64) - go) <= 1e-5 * np.linalg.norm(go)


# ---------------------------------------------------------------------------------------------------------------------
# Inputs (the suite's own: test_gpu_parity, test_deterministic)

C2 = (2e-4 / 3, 2e-4, 0.0)            # smoothness + barrier (test_parity_small_pack)
C3 = (2e-4, 3e-4, 1e-4)               # with AMIPS (_check_amips)


def _pack_inputs(pack):
    """(name, x, c, order) of a pack: benign and inverted at orders 2 and 4, the mirrored AMIPS input at orders 2 and 4."""
    out = [(f"sig{sig}-o{order}", perturb(pack, sigma_rel=sig, seed=1), C2, order) for sig, order in ((0.02, 2), (0.35, 2), (0.35, 4))]
    xm = mirror_components(perturb(pack, sigma_rel=0.05, seed=0), pack.tets)
    return out + [(f"mirrored-o{order}", xm, C3, order) for order in (2, 4)]


def _mesh_inputs(V, T, mirror):
    """Inputs of a single mesh (whole-area meshes, the tiny-component pack): perturb(V, T, sigma, 4) as
    test_whole_area_staging uses them, the AMIPS input mirrored where the mesh has several components."""
    out = [(f"sig{sig}-o{order}", perturb(V, T, sig, 4), (2e-4, 3e-4, 0.0), order) for sig, order in ((0.02, 2), (0.35, 2), (0.35, 4))]
    xa = perturb(V, T, 0.05, 4)
    if mirror:
        xa = mirror_components(xa, T)
    return out + [(f"amips-o{order}", xa, C3, order) for order in (2, 4)]


def _ragged_inputs(seed):
    """test_randomised_ragged_meshes_on_gpu's mesh and inputs for one seed."""
    from test_host_logic import _ragged_mesh
    rng = np.random.default_rng(100 + seed)
    V, T = _ragged_mesh(rng, int(rng.integers(1, 7)), 1200)
    out = []
    for sig, order in ((0.03, 2), (0.4, 4)):
        out.append((f"sig{sig}-o{order}", (V + rng.normal(0, sig * 0.2, V.shape)).astype(np.float32), (3e-4, 2e-4, 0.0), order))
    xa = V * np.array([1.3, 1.0, 0.8], dtype=np.float32) + rng.normal(0, 0.002, V.shape)
    out.append(("amips-o2", mirror_components(xa, T).astype(np.float32), (3e-4, 2e-4, 1e-4), 2))
    return V, T, out


def _inputs(name):
    """(verts, tets, inputs) of each mesh of the GPU tests."""
    if name == "pack3x1024":
        pk = make_pack(3, 1024, seed=1)
        return pk.verts, pk.tets, _pack_inputs(pk)
    if name == "amips_pack":                 # test_amips_term_default_off's pack and AMIPS inputs
        pk = make_pack(3, 1024, seed=8)
        return pk.verts, pk.tets, [(f"amips-sig{sig}-o{order}", perturb(pk, sigma_rel=sig, seed=4), (2e-4, 3e-4, 1e-4), order)
                                   for sig, order in ((0.05, 2), (0.2, 4))]
    if name == "pack16x4096":
        pk = make_pack(16, 4096, seed=0, unique=4)
        return pk.verts, pk.tets, [(f"sig{sig}-o{order}", perturb(pk, sigma_rel=sig, seed=1), (2e-4 / 16, 2e-4, 0.0), order)
                                   for sig, order in ((0.02, 2), (0.35, 4))]
    if name.startswith("ragged"):
        return _ragged_inputs(int(name[len("ragged"):]))
    V, T = plan_shape_mesh(name)
    return V, T, _mesh_inputs(V, T, name in ("mixed", "tiny2600"))


_CACHE = {}


def _mesh(name):
    """(verts, tets, inputs, RowScale, COracle), built once per mesh."""
    if name not in _CACHE:
        V, T, inputs = _inputs(name)
        _CACHE.clear()                         # one mesh at a time: the big ones hold a large operator
        _CACHE[name] = (V, T, inputs, RowScale(V, T), COracle(V, T))
    return _CACHE[name]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the scale itself, KAPPA, and what the old metric misses


def test_row_scale_terms_sum_to_the_oracle():
    """RowScale's fp64 terms are the oracle's gradient, term by term; A bounds each term's magnitude."""
    V, T, inputs, rs, orc = _mesh("pack3x1024")
    for name, x, c, order in inputs:
        g, A = rs.terms(x, c, order)
        for k, term in enumerate(("smooth", "barrier", "amips")):
            ck = [0.0, 0.0, 0.0]
            ck[k] = c[k]
            go = orc.energy_grad_ex(x, *ck, order, gradH=GH)[2]
            assert np.linalg.norm(g[term] - go) <= 1e-12 * max(np.linalg.norm(go), 1e-300), (name, term)
            assert np.all(np.abs(g[term]) <= A[term] * (1 + 1e-12)), (name, term)
        assert (np.linalg.norm(g["amips"]) > 0) == (c[2] > 0)


def _emulated(V, T, x, c, order, smooth_energy=False, **kw):
    """emulate_kernel in fp32 on the host plan of (V, T); returns the gradient in fp64 (and the smoothness energy)."""
    plan = build_host_plan(V, T, enable_amips=int(c[2] != 0), **kw)
    extra = dict(c3=c[2]) if c[2] else {}
    res = emulate_kernel(plan, x, c[0], c[1], order, gradH=GH, dtype=np.float32, **extra)
    return (res[-1].astype(np.float64), float(res[1])) if smooth_energy else res[-1].astype(np.float64)


CALIB_PLANS = [dict(nw=16, grid=132), dict(nw=8, grid=264, force_global=1), dict(nw=8, grid=264, ring_slots=4)]


def test_kappa_calibration():
    """The fp32 re-enactment of the kernel against the oracle on every mesh and input of the GPU tests: the largest
    err / (2^-24 A) stays below KAPPA, for the summed gradient and for each term alone; each term's L2 error stays
    below 1e-5 of its norm or 2^-24 ||A||; the smoothness energy's error stays below KAPPA 2^-24 of its magnitude form
    (RowScale.smooth_energy_scale)."""
    worst = {}
    for mesh in ("pack3x1024", "amips_pack", "alone", "mixed", "near_cap", "tiny2600", "ragged0", "ragged1", "pack16x4096"):
        V, T, inputs, rs, orc = _mesh(mesh)
        plans = CALIB_PLANS if mesh == "pack3x1024" else CALIB_PLANS[:1]
        for kw in plans:
            for name, x, c, order in inputs:
                A = rs.terms(x, c, order)[1]
                _, terms, go = orc.energy_grad_ex(x, *c, order, gradH=GH)
                g, es = _emulated(V, T, x, c, order, smooth_energy=True, **kw)
                r = assert_rows(g, go, sum(A.values()), what=f"{mesh} {kw} {name}")
                worst[(mesh, name, "all")] = max(worst.get((mesh, name, "all"), 0.0), r)
                r = abs(es - terms[0]) / (U24 * rs.smooth_energy_scale(x))
                assert r <= KAPPA, (mesh, kw, name, es, terms[0])
                worst[(mesh, name, "smooth energy")] = max(worst.get((mesh, name, "smooth energy"), 0.0), r)
                for k, term in enumerate(("smooth", "barrier", "amips")):
                    if c[k] == 0:
                        continue
                    ck = [0.0, 0.0, 0.0]
                    ck[k] = c[k]
                    go = orc.energy_grad_ex(x, *ck, order, gradH=GH)[2]
                    g = _emulated(V, T, x, ck, order, **kw)
                    assert np.linalg.norm(g - go) <= max(REL * np.linalg.norm(go), U24 * np.linalg.norm(A[term]))
                    r = assert_rows(g, go, A[term], what=f"{mesh} {kw} {name} {term}")
                    worst[(mesh, name, term)] = max(worst.get((mesh, name, term), 0.0), r)
    print("\n".join(f"{k}: {v:.2f}" for k, v in sorted(worst.items(), key=lambda kv: -kv[1])[:12]))


def _emulated_terms(mesh, input_name, **kw):
    """(x, c, order, RowScale, oracle gradient, emulated gradient, {term: emulated gradient of that term alone})."""
    V, T, inputs, rs, orc = _mesh(mesh)
    _, x, c, order = next(i for i in inputs if i[0] == input_name)
    go = orc.energy_grad_ex(x, *c, order, gradH=GH)[2]
    g = _emulated(V, T, x, c, order, **kw)
    gt = {}
    for k, term in enumerate(("smooth", "barrier", "amips")):
        ck = [0.0, 0.0, 0.0]
        ck[k] = c[k]
        gt[term] = _emulated(V, T, x, ck, order, **kw) if c[k] else None
    assert old_metric_passes(g, go) and assert_rows(g, go, rs.bound(x, c, order)) <= KAPPA
    return x, c, order, rs, go, g, gt


def test_old_metric_misses_one_row_of_smoothness():
    """One row's smoothness sum scaled by 1 + 1e-4: the whole-pack L2 check passes it, the per-row bound does not."""
    x, c, order, rs, go, g, gt = _emulated_terms("pack3x1024", "sig0.35-o2", nw=16, grid=132)
    A = rs.bound(x, c, order)
    score = (np.abs(gt["smooth"]) / np.maximum(A, 1e-300)).max(axis=1)
    small = 1e-4 * np.linalg.norm(gt["smooth"], axis=1) < 5e-6 * np.linalg.norm(go)     # rows the old metric misses
    i = int(np.argmax(np.where(small, score, 0.0)))
    bad = g.copy()
    bad[i] += 1e-4 * gt["smooth"][i]
    assert old_metric_passes(bad, go)
    assert row_ratio(bad, go, A)[0] > KAPPA


def test_old_metric_misses_a_dropped_barrier_corner():
    """One inverted tet's corner vector dropped from one of its vertices (sigma 0.35, order 2: many slightly inverted
    tets, whose corner vectors are small)."""
    x, c, order, rs, go, g, gt = _emulated_terms("pack3x1024", "sig0.35-o2", nw=16, grid=132)
    A = rs.bound(x, c, order)
    bar, _, _, _, inv, _ = rs.tet_terms(x, c[1], c[2], order)
    t, k = np.nonzero(inv[:, None] & (np.linalg.norm(bar, axis=2) < 5e-6 * np.linalg.norm(go)))
    assert len(t), "no corner small enough for the old metric to miss"
    v = rs.T[t, k]
    score = (np.abs(bar[t, k]) / (U24 * A[v])).max(axis=1)
    j = int(np.argmax(score))
    bad = g.copy()
    bad[v[j]] -= bar[t[j], k[j]]
    assert old_metric_passes(bad, go)
    assert row_ratio(bad, go, A)[0] > KAPPA


def test_old_metric_misses_one_amips_tet():
    """One tet's AMIPS contribution scaled by 1 + 1e-3 (the mirrored input of every deterministic-mode AMIPS check)."""
    x, c, order, rs, go, g, gt = _emulated_terms("pack3x1024", "mirrored-o2", nw=16, grid=132)
    A = rs.bound(x, c, order)
    _, _, am, _, _, ok = rs.tet_terms(x, c[1], c[2], order)
    score = (np.abs(am) / np.maximum(U24 * A[rs.T], 1e-300)).max(axis=(1, 2))
    small = 1e-3 * np.linalg.norm(am, axis=(1, 2)) < 5e-6 * np.linalg.norm(go)          # tets the old metric misses
    t = int(np.argmax(np.where(ok & small, score, 0.0)))
    bad = g.copy()
    np.add.at(bad, rs.T[t], 1e-3 * am[t])
    assert old_metric_passes(bad, go)
    assert row_ratio(bad, go, A)[0] > KAPPA


def test_old_metric_misses_a_scaled_smoothness_term():
    """The whole smoothness term scaled by 1 + 5e-4 on the 16 x 4096 order-4 input, where the barrier is 99.9 % of
    the gradient: the per-term check and the per-row bound both catch it."""
    x, c, order, rs, go, g, gt = _emulated_terms("pack16x4096", "sig0.35-o4", nw=16, grid=132)
    bad = g + 5e-4 * gt["smooth"]
    assert old_metric_passes(bad, go)
    assert row_ratio(bad, go, rs.bound(x, c, order))[0] > KAPPA
    go_s = _mesh("pack16x4096")[4].energy_grad_ex(x, c[0], 0, 0, order, gradH=GH)[2]
    assert np.linalg.norm(gt["smooth"] - go_s) <= REL * np.linalg.norm(go_s)
    assert np.linalg.norm(gt["smooth"] * (1 + 5e-4) - go_s) > REL * np.linalg.norm(go_s)


# ---------------------------------------------------------------------------------------------------------------------
# Row ids at the top of the 24-bit range

TOP_N = 0xFFFFFE            # the largest vertex count a handle accepts (0xFFFFFF is the idle-lane row id)


def _top_mesh():
    """n = 0xFFFFFE vertices; four 1024-tet spheres relabelled: one contiguous at the very top (last id 0xFFFFFD),
    one scattered over [2^23, its start) (no contiguous base: staged through vlist), one straddling 2^20, one low.
    Every other vertex is an orphan.  Returns (pack, ids: compact vertex -> id, rest [n, 3], tets)."""
    pk = make_pack(4, 1024, seed=9)
    nv = np.diff(pk.vert_offsets)
    rng = np.random.default_rng(9)
    top = np.arange(TOP_N - nv[0], TOP_N)
    scattered = (1 << 23) + rng.choice(int(top[0]) - (1 << 23), size=int(nv[1]), replace=False)
    straddle = (1 << 20) - nv[2] // 2 + np.arange(nv[2])
    low = 3 + np.arange(nv[3])
    ids = np.concatenate([top, scattered, straddle, low]).astype(np.int64)
    assert ids.max() == 0xFFFFFD and scattered.min() >= 1 << 23 and len(np.unique(ids)) == pk.n
    rest = np.zeros((TOP_N, 3), np.float32)
    rest[ids] = pk.verts
    return pk, ids, rest, ids[pk.tets].astype(np.int32)


def _top_inputs(pk):
    """(name, compact x, c, order): inverted at orders 2 and 4, and the mirrored AMIPS input."""
    xi = perturb(pk, sigma_rel=0.35, seed=2)
    xa = mirror_components(perturb(pk, sigma_rel=0.05, seed=2), pk.tets)
    return [("inverted-o2", xi, (1e-4, 2e-4, 0.0), 2), ("inverted-o4", xi, (1e-4, 2e-4, 0.0), 4), ("amips-o4", xa, C3, 4)]


@pytest.fixture(scope="module")
def top():
    pk, ids, rest, T = _top_mesh()
    return pk, ids, rest, T, RowScale(pk.verts, pk.tets, ids=ids), COracle(pk.verts, pk.tets)


@pytest.mark.parametrize("force_global", [0, 1])
def test_top_range_plan_headers(top, force_global):
    """The block headers' row ids are the relabelled vertex ids (bits 20..23 set), and every header read as fp32 is
    finite (for ids >= 2^23 bit 23 is the float's exponent LSB)."""
    pk, ids, rest, T, _, _ = top
    plan = build_host_plan(rest, T, force_global=force_global)
    assert plan["n"] == TOP_N and plan["mode_global"] == force_global and len(plan["orphans"]) == TOP_N - pk.n
    if not force_global:
        assert any(s["vbase"] < 0 for s in plan["segs"]) and any(s["vbase"] >= 1 << 23 for s in plan["segs"])
    hdr = np.array([h for _, h in walk_streams(plan)[0]])   # the 32 lanes' header words of every row block
    rid = hdr & 0xFFFFFF
    assert np.array_equal(np.unique(rid[rid != 0xFFFFFF]), np.sort(ids))
    assert np.isfinite(hdr.view(np.float32)).all()
    assert ((hdr[rid != 0xFFFFFF] >> 23) & 1).any(), "no header with bit 23 set"


def test_top_range_reenactment_and_limit(top):
    """The fp32 re-enactment on the n = 0xFFFFFE plan against the oracle (on the compacted mesh: the energy does not
    depend on the labels), with the per-row bound; orphans exactly 0.  n = 0xFFFFFF is rejected."""
    pk, ids, rest, T, rs, orc = top
    orphan = np.ones(TOP_N, bool)
    orphan[ids] = False
    for name, xc, c, order in _top_inputs(pk)[1:]:
        plan = build_host_plan(rest, T, enable_amips=int(c[2] != 0))
        x = rest.copy()
        x[ids] = xc
        extra = dict(c3=c[2]) if c[2] else {}
        res = emulate_kernel(plan, x, c[0], c[1], order, gradH=GH, dtype=np.float32, **extra)
        g = res[-1]
        eo, terms, go = orc.energy_grad_ex(xc, *c, order, gradH=GH)
        assert res[0] == pytest.approx(eo, rel=REL)
        assert not g[orphan].any()
        assert_rows(g[ids].astype(np.float64), go, rs.bound(xc, c, order), what=name)
        del plan, x, g, res
    big = np.zeros((0xFFFFFF, 3), np.float32)
    with pytest.raises(RuntimeError, match="16.7 M"):
        build_host_plan(big, T)


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


GPU_WORST = {}              # largest err / (2^-24 A) per plan and input


@pytest.fixture(scope="module", autouse=True)
def _report_gpu_worst():
    """Prints the largest err / (2^-24 A) the GPU tests of this module saw (visible with -s)."""
    yield
    for k, v in sorted(GPU_WORST.items(), key=lambda kv: -kv[1])[:12]:
        print(f"gpu worst {v:8.2f}  {k}")
    if GPU_WORST:
        print(f"gpu worst overall {max(GPU_WORST.values()):.2f} (KAPPA {KAPPA})")


def _note(key, r):
    GPU_WORST[key] = max(GPU_WORST.get(key, 0.0), r)


def _handle(ext, V, T, **kw):
    sp = ext.TetSpheres(np.ascontiguousarray(V, np.float32).reshape(-1), np.ascontiguousarray(T, np.int32).reshape(-1), **kw)
    if kw.get("ring_slots"):
        assert sp.info["ring_slots"] == kw["ring_slots"], "the ring was shrunk: this variant would not test its depth"
    return sp


def _term_parity(sp, rs, orc, x_np, c, order, key, tensor_gradH=False):
    """Each term alone against the oracle's term (relative to its own norm, and per row), then all terms together
    (per row), and the sum of the single-term gradients equal to the combined one (per row, both sides' error).  A term
    near the operator's null space (the affine-stretched AMIPS input of the ragged meshes) is a small residual of large
    products: its L2 error and the smoothness energy's are also allowed their own fp32 rounding scale."""
    torch = _torch()
    x = torch.from_numpy(np.ascontiguousarray(x_np, np.float32)).cuda()
    _, A = rs.terms(x_np, c, order)
    Atot = A["smooth"] + A["barrier"] + A["amips"]
    es_slack = KAPPA * U24 * rs.smooth_energy_scale(x_np)           # the smoothness energy's own rounding scale
    parts = []
    for k, term in enumerate(("smooth", "barrier", "amips")):
        if c[k] == 0:
            continue
        ck = [0.0, 0.0, 0.0]
        ck[k] = c[k]
        rel = 2e-5 if term == "amips" else REL
        e, g = sp.energy_grad(x, ck[0], ck[1], order, GH, c3=ck[2])
        eo, _, go = orc.energy_grad_ex(x_np, *ck, order, gradH=GH)
        e, g = e.cpu().numpy().astype(np.float64), g.cpu().numpy().astype(np.float64)
        assert abs(e[0] - eo) <= max(rel * abs(eo), abs(ck[0]) * es_slack), (key, term, e[0], eo)
        ng = np.linalg.norm(go)
        assert np.linalg.norm(g - go) <= max(rel * ng, U24 * np.linalg.norm(A[term])), \
            (key, term, np.linalg.norm(g - go) / max(ng, 1e-300))
        _note(key + ("term",), assert_rows(g, go, A[term], what=f"{key} {term} alone"))
        parts.append(g)
    eo, terms, go = orc.energy_grad_ex(x_np, *c, order, gradH=GH)
    for gh in ((GH, torch.tensor(GH, device="cuda")) if tensor_gradH else (GH,)):
        e, g = sp.energy_grad(x, c[0], c[1], order, gh, c3=c[2])
        e, g = e.cpu().numpy().astype(np.float64), g.cpu().numpy().astype(np.float64)
        assert abs(e[0] - eo) <= max(REL * abs(eo), c[0] * es_slack), (key, e[0], eo)
        assert abs(e[1] - terms[0]) <= max(REL * abs(terms[0]), es_slack), (key, e[1], terms[0])
        assert e[2] == pytest.approx(terms[1], rel=REL, abs=1e-30), key
        if c[2]:
            assert e[3] == pytest.approx(terms[2], rel=2e-5), key
        _note(key + ("all",), assert_rows(g, go, Atot, what=f"{key} all terms, gradH {type(gh).__name__}"))
        assert_rows(g, sum(parts), Atot, kappa=2 * KAPPA, what=f"{key} all terms vs the sum of the terms")


def _run_plans(ext, mesh, kw):
    V, T, inputs, rs, orc = _mesh(mesh)
    plain = _handle(ext, V, T, **kw)
    amips = _handle(ext, V, T, enable_amips=True, **kw)
    for i, (name, x, c, order) in enumerate(inputs):
        _term_parity(amips if c[2] else plain, rs, orc, x, c, order, (mesh, str(kw), name), tensor_gradH=i == 0)


def _kw_id(k):
    return "-".join(f"{a}{b}" for a, b in k.items()) or "default"


def _variants():
    from test_gpu_parity import VARIANTS
    return VARIANTS


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True], ids=["atomic", "det"])
@pytest.mark.parametrize("kw", _variants(), ids=_kw_id)
def test_terms_and_rows_every_variant(ext, kw, det):
    """Every kernel variant, default and deterministic, on the 3 x 1024 pack."""
    _run_plans(ext, "pack3x1024", dict(kw, deterministic=det))


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True], ids=["atomic", "det"])
@pytest.mark.parametrize("kw", [dict(), dict(warps_per_cta=8), dict(force_global=True)], ids=_kw_id)
def test_terms_and_rows_amips_pack(ext, kw, det):
    """test_amips_term_default_off's pack and AMIPS inputs (sigma 0.05 order 2, sigma 0.2 order 4)."""
    _run_plans(ext, "amips_pack", dict(kw, deterministic=det))


@pytest.mark.gpu
@pytest.mark.parametrize("nw", [16, 8])
@pytest.mark.parametrize("mesh", ["alone", "mixed", "near_cap"])
def test_terms_and_rows_whole_area_staging(ext, mesh, nw):
    _run_plans(ext, mesh, dict(warps_per_cta=nw))


@pytest.mark.gpu
@pytest.mark.parametrize("mesh", ["tiny2600", "ragged0", "ragged1", "pack16x4096"])
def test_terms_and_rows_other_meshes(ext, mesh):
    """2600 twelve-tet components, two ragged relabelled meshes, and the 16 x 4096 pack."""
    _run_plans(ext, mesh, {})


def _raw_launch(sp, x, c, order):
    """tsb_energy_grad(_ex) through the C ABI into a gradient buffer pre-filled with NaN: rows the kernel does not
    write stay NaN."""
    torch = _torch()
    from tssplat_b200 import _capi
    g = torch.full((sp.n, 3), float("nan"), device="cuda")
    e = torch.zeros(4, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    if c[2]:
        terms = _capi.tsb_terms_t(c1=c[0], c2=c[1], order=order, c3=c[2])
        rc = _capi.lib.tsb_energy_grad_ex(sp._h, x.data_ptr(), C.byref(terms), GH, None, e.data_ptr(), g.data_ptr(), st)
    else:
        rc = _capi.lib.tsb_energy_grad(sp._h, x.data_ptr(), c[0], c[1], order, GH, None, e.data_ptr(), g.data_ptr(), st)
    _capi.check(rc, sp._h)
    torch.cuda.synchronize()
    return e.cpu().numpy().astype(np.float64), g


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(warps_per_cta=8), dict(force_global=True), dict(deterministic=True),
                                dict(enable_amips=True)], ids=_kw_id)
def test_top_range_on_gpu(ext, top, kw):
    """n = 0xFFFFFE: the referenced rows against the oracle with the per-row bound, energies at 1e-5, and all
    ~16.7 M orphan rows written to exactly 0 (the buffer starts as NaN)."""
    torch = _torch()
    pk, ids, rest, T, rs, orc = top
    sp = _handle(ext, rest, T, **kw)
    assert sp.n == TOP_N and sp.info["mode_global"] == int(bool(kw.get("force_global")))
    ids_t = torch.from_numpy(ids).cuda()
    orphan = torch.ones(TOP_N, dtype=torch.bool, device="cuda")
    orphan[ids_t] = False
    x = torch.from_numpy(rest).cuda()
    for name, xc, c, order in _top_inputs(pk):
        if c[2] and not kw.get("enable_amips"):
            continue
        x[ids_t] = torch.from_numpy(xc).cuda()
        e, g = _raw_launch(sp, x, c, order)
        eo, terms, go = orc.energy_grad_ex(xc, *c, order, gradH=GH)
        assert e[0] == pytest.approx(eo, rel=REL) and e[1] == pytest.approx(terms[0], rel=REL), (kw, name)
        assert e[2] == pytest.approx(terms[1], rel=REL, abs=1e-30), (kw, name)
        if c[2]:
            assert e[3] == pytest.approx(terms[2], rel=2e-5), (kw, name)
        assert int(torch.count_nonzero(g[orphan])) == 0, "an orphan row is not exactly 0"
        _note(("top", str(kw), name), assert_rows(g[ids_t].cpu().numpy().astype(np.float64), go, rs.bound(xc, c, order),
                                                  what=f"{kw} {name}"))
        del g
    with pytest.raises(RuntimeError, match="16.7 M"):
        _handle(ext, np.zeros((0xFFFFFF, 3), np.float32), T, **kw)

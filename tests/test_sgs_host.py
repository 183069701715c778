"""The symmetric Gauss-Seidel preconditioner on the CPU: the host colouring and sweep tables of tsb_pcg_enable_sgs
(tsb::build_sgs_tables through the test-only inspection library), and the algorithm in fp64 (tests/_sgs_model.py)."""
import numpy as np
import pytest

from _newton_model import (CONVERGED, _shuffled_mesh, batched_pcg_reference, block_preconditioner,
                           jacobi_inverse_blocks, reference_problem)
from _sgs_model import block, sgs_apply, sgs_matrix, sgs_tables
from tssplat_b200.mesh import make_pack


def _orphan_mesh():
    """make_pack(4, 512) with 37 vertices no tet references interleaved into the numbering."""
    pk = make_pack(4, 512, seed=5)
    rng = np.random.default_rng(3)
    n = len(pk.verts) + 37
    ids = np.sort(rng.permutation(n)[:len(pk.verts)])
    V = rng.normal(size=(n, 3)).astype(np.float32)
    V[ids] = pk.verts
    return V, ids[pk.tets].astype(np.int32)


def _mesh(name):
    if name == "pack":
        pk = make_pack(3, 512, seed=4)
        return pk.verts, pk.tets
    if name == "shuffled":
        V, T, _ = _shuffled_mesh()
        return V, T
    return _orphan_mesh()


MESHES = ("pack", "shuffled", "orphans")


@pytest.mark.parametrize("name", MESHES)
def test_colouring_is_proper_and_complete(name):
    V, T = _mesh(name)
    t = sgs_tables(V, T)
    color, crow, col = t["color"], t["crow"], t["col"]
    used = np.zeros(len(V), bool)
    used[np.unique(T)] = True
    assert (color[used] >= 0).all() and (color[~used] == -1).all()
    # no two vertices of one tet share a colour, nor any two vertices the pattern couples
    tc = color[T]
    for k in range(4):
        for m in range(k + 1, 4):
            assert (tc[:, k] != tc[:, m]).all()
    rows = np.repeat(np.arange(len(V)), np.diff(crow))
    off = rows != col
    assert (color[rows[off]] != color[col[off]]).all()
    # at most max degree + 1 colours, and n_colors is the largest count any component uses
    deg = np.diff(crow) - used
    assert t["n_colors"] == color.max() + 1 <= deg.max() + 1
    # greedy in ascending order: every vertex's colour is the smallest one its earlier neighbours leave free
    for v in np.flatnonzero(used)[:400]:
        nb = col[crow[v]:crow[v + 1]]
        taken = set(color[nb[nb < v]].tolist())
        assert color[v] == min(set(range(len(taken) + 1)) - taken)


@pytest.mark.parametrize("name", MESHES)
def test_tables_are_deterministic(name):
    V, T = _mesh(name)
    ref = sgs_tables(V, T, nth=1)
    for nth in (2, 7, 0, 0):
        t = sgs_tables(V, T, nth=nth)
        for k, a in ref.items():
            assert np.array_equal(np.asarray(a), np.asarray(t[k])), (nth, k)


@pytest.mark.parametrize("name", MESHES)
def test_row_lists_partition_the_off_diagonal_blocks(name):
    V, T = _mesh(name)
    t = sgs_tables(V, T)
    color, crow, col, vert, comp_off = t["color"], t["crow"], t["col"], t["vert"], t["comp_off"]
    lo, hi = t["lo"].reshape(-1, 2), t["hi"].reshape(-1, 2)
    comp = np.searchsorted(comp_off, np.arange(len(vert)), side="right") - 1
    for e, v in enumerate(vert):
        blocks = np.arange(crow[v], crow[v + 1])
        off = blocks[col[blocks] != v]
        L, H = lo[t["lo_ptr"][e]:t["lo_ptr"][e + 1]], hi[t["hi_ptr"][e]:t["hi_ptr"][e + 1]]
        # a partition of the row's off-diagonal blocks, each list in column order
        assert np.array_equal(np.sort(np.concatenate([L[:, 0], H[:, 0]])), off)
        assert (np.diff(L[:, 0]) > 0).all() and (np.diff(H[:, 0]) > 0).all()
        assert (color[col[L[:, 0]]] < color[v]).all() and (color[col[H[:, 0]]] > color[v]).all()
        # the column positions are those of the solver's vertex list, relative to the component
        for q in (L, H):
            assert np.array_equal(vert[comp_off[comp[e]] + q[:, 1]], col[q[:, 0]])
    # the schedule: every component's rows grouped by colour, ascending in each
    for c in range(len(comp_off) - 1):
        offs = t["color_off"][t["color_ptr"][c]:t["color_ptr"][c + 1]]
        assert offs[0] == comp_off[c] and offs[-1] == comp_off[c + 1]
        for k in range(len(offs) - 1):
            rows = t["sched"][offs[k]:offs[k + 1]]
            assert len(rows) > 0 and (np.diff(rows) > 0).all() and (color[vert[rows]] == k).all()


# ---------------------------------------------------------------------------------------------------------------------
# the algorithm in fp64, on the small mixed pack of the Newton references (sphere 0 has inverted tets: indefinite H)


def _sphere_problem(amips=False):
    P, x, _, o = reference_problem(amips=amips)
    H = P.hess_blocks(x.reshape(-1))
    t = sgs_tables(P.pk.verts, P.pk.tets)
    b = -P.grad(x.reshape(-1))
    out = []
    for s, Hs in enumerate(H):
        v0, v1 = P.vo[s], P.vo[s + 1]
        out.append((Hs, t["color"][v0:v1], b[3 * v0:3 * v1]))
    return out, o


def _dinv(Hs, shift, rel_floor=1e-6):
    m = len(Hs) // 3
    D = np.stack([Hs[3 * i:3 * i + 3, 3 * i:3 * i + 3] for i in range(m)]) + shift * np.eye(3)
    return np.stack([block(q) for q in jacobi_inverse_blocks(D, rel_floor)])


@pytest.mark.parametrize("shift", [0.0, 1e-3])
def test_sgs_model_is_spd(shift):
    spheres, _ = _sphere_problem()
    for s, (Hs, colors, _) in enumerate(spheres):
        A = Hs + shift * np.eye(len(Hs))
        Dinv = _dinv(Hs, shift)
        Minv = sgs_matrix(A, Dinv, colors)
        sc = np.abs(Minv).max()
        assert np.abs(Minv - Minv.T).max() <= 1e-12 * sc, s
        assert np.linalg.eigvalsh(0.5 * (Minv + Minv.T)).min() > 0.0, s
        if s == 0 and shift == 0.0:
            assert np.linalg.eigvalsh(A).min() < 0.0       # the rough sphere is indefinite, M^-1 is SPD all the same


def test_sgs_model_zero_blocks():
    Hs, colors, b = _sphere_problem()[0][1]
    Dinv = _dinv(Hs, 0.0)
    dead = np.arange(0, len(colors), 5)
    Dinv[dead] = 0.0
    z = sgs_apply(Hs, Dinv, colors, b).reshape(-1, 3)
    assert not z[dead].any() and z.any()
    Minv = sgs_matrix(Hs, Dinv, colors)
    assert np.abs(Minv - Minv.T).max() <= 1e-12 * np.abs(Minv).max()
    assert np.linalg.eigvalsh(0.5 * (Minv + Minv.T)).min() > -1e-12 * np.abs(Minv).max()


@pytest.mark.parametrize("amips", [False, True])
def test_sgs_model_needs_fewer_products(amips):
    """fp64 PCG to rtol = 1e-3 on the small mixed pack: the quiet spheres unshifted, every sphere with an LM shift that
    makes it positive definite; SGS never needs more products than block Jacobi, and fewer in total."""
    spheres, _ = _sphere_problem(amips)
    for shifted in (False, True):
        H, bs, Pj, Ps = [], [], [], []
        for s, (Hs, colors, b) in enumerate(spheres):
            if not shifted and s == 0:
                continue
            mu = max(0.0, -np.linalg.eigvalsh(Hs).min()) * 1.5 + 1e-6 * np.abs(np.diag(Hs)).max() if shifted else 0.0
            A = Hs + mu * np.eye(len(Hs))
            m = len(Hs) // 3
            D = np.stack([Hs[3 * i:3 * i + 3, 3 * i:3 * i + 3] for i in range(m)])
            H.append(A)
            bs.append(b)
            Pj.append(block_preconditioner(D, mu, 1e-6))
            Ps.append(sgs_matrix(A, _dinv(Hs, mu), colors))
        rj = batched_pcg_reference(H, bs, Pj, 400, 1e-3)
        rs = batched_pcg_reference(H, bs, Ps, 400, 1e-3)
        assert all(r["status"] == CONVERGED for r in rj + rs)
        nj, ns = [r["n_hvp"] for r in rj], [r["n_hvp"] for r in rs]
        assert all(a <= b for a, b in zip(ns, nj)) and sum(ns) < sum(nj), (shifted, nj, ns)

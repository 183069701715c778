"""The assembled Hessian (tsb_hessian_create / tsb_hessian_assemble, tssplat_b200.hessian.DeviceHessian): the matrix a
solver workspace multiplies by, as 3x3 block-CSR over all vertices, exact or with PSD-projected tet blocks.

CPU: the host block pattern (through the plan inspection library) against the oracle's M, the plan's streamed weights,
the components and the tets; an fp64 numpy restatement of the kernel's per-tet 12 x 12 closed form against G^T Hess(psi) G,
off-diagonal corner blocks included.  GPU: per-sphere blocks against a dense fp64 assembly (the oracle's M, the tet terms
on the kernels' rounded inputs), H v against tsb_hvp_ex and
tsb_pcg_hvp_psd, the diagonal against tsb_hess_diag, bitwise invariants, a sparse direct solve against the device PCG,
argument errors and memory."""
import ctypes as C
import functools

import numpy as np
import pytest

from _helpers import CELL_FORMAT, PLAN_DEBUG_SO, build_host_plan, walk_streams
from _newton_model import C3, COEF, _cuda, _handle, _pack, _psd_pack, _small_mixed, _torch, ext  # noqa: F401
from test_hess_diag import psi_hessians, tet_hessians
from tssplat_b200.mesh import make_pack

U = 2.0 ** -24
KAPPA = 64              # diagonal blocks against tsb_hess_diag: its per-row bound (test_hess_diag)
# exact blocks: |H - H64|_max <= KAPPA_BLOCK u A_ij.  A block is a recursive fp32 sum of up to 39 addends in these packs
# (gamma_39 ~ 41 u) of fp32-rounded fp64 tet blocks, and near-flat AMIPS tets amplify fp64 rounding on both sides; the
# largest ratio measured on an H100 is 63 (mixed64)
KAPPA_BLOCK = 128
KAPPA_PSD = 1024        # projected blocks: the fp32 operator carries the projection's own error (test_psd_edges); worst 86
REL = 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# host pattern


def hess_pattern(rest, tets, laplacian_scale=0):
    lib = C.CDLL(PLAN_DEBUG_SO)
    lib.tsbdbg_hess_build.restype = C.c_int
    lib.tsbdbg_hess_build.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p),
                                      C.POINTER(C.c_int64)]
    lib.tsbdbg_hess_array.restype = C.c_int
    lib.tsbdbg_hess_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]
    lib.tsbdbg_hess_free.argtypes = [C.c_void_p]
    lib.tsbdbg_last_error.restype = C.c_char_p
    rest = np.ascontiguousarray(np.asarray(rest, np.float32).reshape(-1))
    tets = np.ascontiguousarray(np.asarray(tets, np.int32).reshape(-1))
    d, nnzb = C.c_void_p(), C.c_int64()
    rc = lib.tsbdbg_hess_build(rest.ctypes.data, tets.ctypes.data, rest.size // 3, tets.size // 4, int(laplacian_scale),
                               C.byref(d), C.byref(nnzb))
    if rc:
        raise RuntimeError(lib.tsbdbg_last_error().decode())
    out = {"nnzb": int(nnzb.value)}
    try:
        for name, dt in (("crow", np.int32), ("col", np.int32), ("w", np.float32), ("tblk", np.int32),
                         ("inc_ptr", np.int32), ("inc", np.int32), ("B", np.float32), ("comp_label", np.int32)):
            ptr, cnt = C.c_void_p(), C.c_int64()
            assert lib.tsbdbg_hess_array(d, name.encode(), C.byref(ptr), C.byref(cnt)) == 0, name
            out[name] = np.ctypeslib.as_array((C.c_char * (cnt.value * 4)).from_address(ptr.value)).view(dt).copy() \
                if cnt.value else np.zeros(0, dt)
    finally:
        lib.tsbdbg_hess_free(d)
    return out


def streamed_weights(rest, tets):
    """{(row, col): fp32 weight} of every non-zero off-diagonal entry the GLOBAL plan streams."""
    plan = build_host_plan(rest, tets, force_global=1)
    CELL, IB, _ = CELL_FORMAT[True]
    WOFF = 128 * IB
    st = plan["stream"]
    blocks, _ = walk_streams(plan)
    out = {}
    for p, hdr in blocks:
        len4, L = int((hdr[0] >> 24) & 63), 1 << int(hdr[0] >> 30)
        rid = (hdr & 0xFFFFFF).astype(np.int64)
        for q in range(len4):
            j = st[p + q * CELL:p + q * CELL + 128 * IB].view(np.uint32).reshape(32, 4)
            w = st[p + q * CELL + WOFF:p + q * CELL + WOFF + 512].view(np.float32).reshape(32, 4)
            for lane in range(32):
                row = int(rid[(lane // L) * L])
                if row == 0xFFFFFF:
                    continue
                for c in range(4):
                    if w[lane, c] != 0 and int(j[lane, c]) != row:
                        out[(row, int(j[lane, c]))] = w[lane, c]
    return out


@functools.lru_cache(maxsize=None)
def _meshes():
    from test_hvp_amips import _mesh
    pk = make_pack(3, 256, seed=4)
    out = {"pack3x256": (pk.verts, pk.tets), "pack8x1024": (make_pack(8, 1024, seed=2).verts, make_pack(8, 1024, seed=2).tets)}
    for name in ("shuffled", "a_veg"):
        V, T, *_ = _mesh(name)
        out[name] = (V, T)
    return out


@pytest.mark.parametrize("name", ["pack3x256", "pack8x1024", "shuffled", "a_veg"])
def test_pattern(name):
    from oracle.tet_energy_oracle import ReferenceEnergyOracle
    V, T = _meshes()[name]
    T = np.asarray(T, np.int64).reshape(-1, 4)
    n = len(V)
    H = hess_pattern(V, T)
    crow, col, w = H["crow"], H["col"], H["w"]
    assert len(crow) == n + 1 and crow[-1] == H["nnzb"] == len(col)
    rows = np.repeat(np.arange(n), np.diff(crow))
    # columns strictly ascending inside a row; a diagonal block in every referenced row; orphan rows empty
    same = rows[1:] == rows[:-1]
    assert (col[1:][same] > col[:-1][same]).all()
    used = np.zeros(n, bool)
    used[T.reshape(-1)] = True
    assert ((np.diff(crow) > 0) == used).all()
    diag = rows == col
    assert diag.sum() == used.sum()
    # block-diagonal by sphere
    lab = H["comp_label"]
    assert (lab[rows] == lab[col]).all() and (lab[~used] == -1).all()
    # the oracle M's sparsity plus the diagonal (entries the operator keeps structurally are exact or rounding zeros)
    orc = ReferenceEnergyOracle(V, T)
    M1 = orc.M[0::3, 0::3].tocsr()
    M1.eliminate_zeros()
    Mc = M1.tocoo()
    pat = set(zip(rows.tolist(), col.tolist()))
    assert set(zip(Mc.row.tolist(), Mc.col.tolist())) <= pat
    Md = np.asarray(M1[rows, col]).ravel()
    scale = np.asarray(abs(M1).max(axis=1).todense()).ravel()[rows]
    assert (np.abs(w[~diag] - Md[~diag]) <= 1e-6 * scale[~diag]).all()
    # the off-diagonal weights are the plan's, bit for bit; the diagonal is -sum in fp64, in column order
    sw = streamed_weights(V, T)
    offd = {(r, c): x for r, c, x in zip(rows[~diag].tolist(), col[~diag].tolist(), w[~diag]) if x != 0}
    assert offd.keys() == sw.keys()
    assert all(offd[k].tobytes() == sw[k].tobytes() for k in offd)
    for i in np.nonzero(used)[0][:: max(1, used.sum() // 400)]:
        b = np.arange(crow[i], crow[i + 1])
        ref = np.float32(-sum(float(x) for x in w[b][col[b] != i]))
        assert w[b][col[b] == i][0].tobytes() == ref.tobytes()
    # mirror weights equal, so mirror blocks can be
    Wm = {(r, c): x for r, c, x in zip(rows.tolist(), col.tolist(), w)}
    assert all(Wm[(c, r)].tobytes() == x.tobytes() for (r, c), x in Wm.items())
    # every corner pair of every tet is a block of the row of its first corner
    tb = H["tblk"].reshape(-1, 4, 4)
    assert (col[tb] == T[:, None, :]).all()
    assert ((crow[T][:, :, None] <= tb) & (tb < crow[T + 1][:, :, None])).all()
    # incidence lists: 4 t + k, ascending within a row
    ip, inc = H["inc_ptr"], H["inc"]
    assert (np.repeat(np.arange(n), np.diff(ip)) == T.reshape(-1)[inc]).all()
    assert all((np.diff(inc[ip[i]:ip[i + 1]]) > 0).all() for i in range(n))


# ---------------------------------------------------------------------------------------------------------------------
# per-tet closed form (fp64 restatement of hessian_blocks_kernel)


def closed_form_blocks(F, a, order=None):
    """12 x 12 tet Hessian from the kernel's formula: H_kl = al (a_k.a_l) I + be (f_k g_l^T + g_k f_l^T) + ga g_k g_l^T
    + sk S(F (a_k x a_l)); a: [4, 3] corner vectors."""
    J = np.linalg.det(F)
    Cf = J * np.linalg.inv(F).T
    if order is not None:
        m = -J
        al = be = 0.0
        ga, sk = order * (order - 1) * m ** (order - 2), -order * m ** (order - 1)
    else:
        tr = (F * F).sum()
        al = 2.0 / (3.0 * np.cbrt(J) ** 2)
        be, ga, sk = -2.0 * al / (3.0 * J), 5.0 * al * tr / (9.0 * J * J), -al * tr / (3.0 * J)
    g, f = a @ Cf.T, a @ F.T
    H = np.zeros((12, 12))
    for k in range(4):
        for l in range(4):
            w = F @ np.cross(a[k], a[l])
            S = np.array([[0, w[2], -w[1]], [-w[2], 0, w[0]], [w[1], -w[0], 0]])
            H[3 * k:3 * k + 3, 3 * l:3 * l + 3] = (al * (a[k] @ a[l]) * np.eye(3) + be * (np.outer(f[k], g[l]) + np.outer(g[k], f[l]))
                                                   + ga * np.outer(g[k], g[l]) + sk * S)
    return H


@pytest.mark.parametrize("term", ["barrier2", "barrier4", "amips"])
def test_tet_closed_form_against_psi_hessians(term):
    rng = np.random.default_rng(11)
    order = {"barrier2": 2, "barrier4": 4, "amips": None}[term]
    X = np.array([[0.0, 0.0, 0.0], [1.1, 0.1, -0.3], [0.3, 0.9, 0.2], [-0.2, 0.4, 1.3]])
    B = np.linalg.inv((X[1:] - X[0]).T)
    a = np.concatenate([-B.sum(axis=0, keepdims=True), B])       # rows of B, a_0 = -sum
    K = np.zeros((9, 12))                                         # vec F (row-major) = K x, F = sum_k x_k a_k^T
    for k in range(4):
        for r in range(3):
            K[3 * r:3 * r + 3, 3 * k + r] = a[k]
    Q = np.linalg.qr(rng.standard_normal((3, 3)))[0]
    cases = [rng.standard_normal((3, 3)) for _ in range(4)] + [Q, 1.7 * Q, np.eye(3) + 1e-4 * rng.standard_normal((3, 3)),
                                                                Q @ np.diag([1.4, 0.75, -1.0]), Q @ np.diag([1.2, 0.9, -1e-3])]
    off = 0
    for F in cases:
        if (order is None) != (np.linalg.det(F) > 0):
            F = F @ np.diag([1.0, 1.0, -1.0])
        H9 = psi_hessians(F[None], order=order, amips=order is None)[0]
        ref = K.T @ H9 @ K
        got = closed_form_blocks(F, a, order)
        scale = np.abs(ref).max()
        assert np.abs(got - ref).max() <= 1e-10 * scale, (term, np.abs(got - ref).max() / scale)
        off += np.abs(ref[:3, 3:]).max() > 1e-3 * scale           # the cross-corner blocks are not zero
    assert off == len(cases)


# ---------------------------------------------------------------------------------------------------------------------
# GPU


def _dev_hessian(sp, hessian="exact"):
    from tssplat_b200.hessian import DeviceHessian
    from tssplat_b200.newton import DevicePCG
    return DeviceHessian(DevicePCG(sp, hessian=hessian))


def _bsr_hv(torch, hs, values, v):
    """fp64 H v by an index gather (not torch's sparse kernels), and the magnitude |H| |v|."""
    crow = hs.crow.long()
    rows = torch.repeat_interleave(torch.arange(len(crow) - 1, device=crow.device), crow[1:] - crow[:-1])
    vals = values.double().reshape(-1, 3, 3)
    vc = v.double().reshape(-1, 3)[hs.col.long()]
    y = torch.zeros(len(crow) - 1, 3, dtype=torch.float64, device=vals.device)
    y.index_add_(0, rows, torch.einsum("bij,bj->bi", vals, vc))
    m = torch.zeros_like(y)
    m.index_add_(0, rows, torch.einsum("bij,bj->bi", vals.abs(), vc.abs()))
    return y.reshape(-1).cpu().numpy(), m.reshape(-1).cpu().numpy()


def kernel_input_dense(orc, pk, x, c1, c2, c3, order, project, nsph):
    """Per-sphere dense fp64 c1 M + sum_t K_t^T (c2 H_b + c3 H_a) K_t and the magnitude sums c1 |M| + sum_t |K_t^T H K_t|,
    with the tet terms of tet_hessians (on the kernels' inputs)."""
    T = np.asarray(pk.tets, np.int64)
    Ht, At = tet_hessians(pk.verts, T, x, c2, c3, order, project=project)
    M = orc.M.toarray()
    rowsum = np.abs(c1) * (np.abs(M).sum(axis=1) - np.abs(np.diag(M)))     # M_ii = -sum_j M_ij cancels: its error scales so
    refs, mags = [], []
    for s in range(nsph):
        v0, v1 = pk.vert_offsets[s], pk.vert_offsets[s + 1]
        H = c1 * M[3 * v0:3 * v1, 3 * v0:3 * v1]
        A = np.abs(H) + np.diag(rowsum[3 * v0:3 * v1])
        for t in np.nonzero((T[:, 0] >= v0) & (T[:, 0] < v1))[0]:
            idx = np.concatenate([3 * (T[t, k] - v0) + np.arange(3) for k in range(4)])
            H[np.ix_(idx, idx)] += Ht[t]
            A[np.ix_(idx, idx)] += At[t]
        refs.append(H)
        mags.append(A)
    return refs, mags


def _blockmax(A):
    n = A.shape[0] // 3
    return np.abs(A).reshape(n, 3, n, 3).max(axis=(1, 3))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "mixed8", "mixed64"])
@pytest.mark.parametrize("hessian", ["exact", "psd"])
def test_blocks_against_fp64_oracle(ext, name, hessian):
    torch = _torch()
    from oracle.tet_energy_oracle import ReferenceEnergyOracle, _det3
    if name == "small":
        pk, x_np = _small_mixed()
        sub, nsph = pk, pk.num_spheres
    else:
        pk, x_np = _psd_pack(name)
        sub, nsph = pk.slice_spheres(0, 8), 8
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True)
    hs = _dev_hessian(sp, hessian)
    orc = ReferenceEnergyOracle(sub.verts, sub.tets)
    xs = np.asarray(x_np[:sub.n], np.float64)
    J = _det3((orc.G @ xs.reshape(-1)).reshape(-1, 3, 3))
    near = np.abs(J) <= 1e-6 * np.abs(J).max()                  # within fp32 rounding of J = 0: activity may differ
    x = _cuda(x_np)
    c1, c2 = COEF
    worst = 0.0
    for order in (2, 4):
        for c3 in (0.0, C3):
            vals = hs.assemble(x, c1, c2, order, c3=c3)
            ref, mag = kernel_input_dense(orc, sub, xs, c1, c2, c3, order, hessian == "psd", nsph)
            for s in range(nsph):
                got = hs.sphere(vals, s).toarray().astype(np.float64)
                v0, v1 = sub.vert_offsets[s], sub.vert_offsets[s + 1]
                assert (hs.sphere_vertices(s) == np.arange(v0, v1)).all()
                skip = np.zeros(v1 - v0, bool)
                tl = np.nonzero(near & (orc.tets[:, 0] >= v0) & (orc.tets[:, 0] < v1))[0]
                skip[(orc.tets[tl] - v0).reshape(-1)] = True
                err = _blockmax(got - ref[s]) / (U * np.maximum(_blockmax(mag[s]), 1e-300))
                err[skip, :] = 0
                err[:, skip] = 0
                worst = max(worst, err.max())
                assert err.max() <= (KAPPA_PSD if hessian == "psd" else KAPPA_BLOCK), (name, hessian, order, c3, s, err.max())
    print(f"{name} {hessian}: worst |H - H64| / (u A_ij) = {worst:.3g}")


def _skip_spheres(pk, x, amips_fp32):
    """Spheres with a tet within fp32 rounding of J = 0 (the two calls may classify it differently), and with
    amips_fp32 also those with |J| <= 0.05: the fp32 AMIPS product (tsb_hvp_ex) forms F from rounded edges and its Hessian
    grows like 1 / J^2 (the rule of test_hvp_amips)."""
    from oracle.tet_energy_oracle import _det3
    T = np.asarray(pk.tets, np.int64)
    X, xx = np.asarray(pk.verts, np.float64)[T], np.asarray(x, np.float32).astype(np.float64)[T]
    J = _det3(np.einsum("tki,tkc->tic", xx[:, 1:] - xx[:, :1], np.linalg.inv(X[:, 1:] - X[:, :1])))
    lab = np.searchsorted(pk.vert_offsets, T[:, 0], side="right") - 1
    bad = np.abs(J) <= (0.05 if amips_fp32 else 1e-6 * np.abs(J).max())
    return set(lab[bad].tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("hessian", ["exact", "psd"])
def test_product_and_diagonal_match_the_operator_calls(ext, hessian):
    """H_bsr v (fp64 gather) equals tsb_hvp_ex or tsb_pcg_hvp_psd per sphere to REL; the diagonal blocks equal
    tsb_hess_diag (exact) within its per-row bound."""
    torch = _torch()
    from test_hvp_amips import _mesh
    from tssplat_b200.hessian import DeviceHessian
    from tssplat_b200.newton import DevicePCG, hess_blocks
    cases = [("mixed64", *_pack("mixed"), dict())]
    for name, kw in (("a_veg", dict(force_global=True)), ("shuffled", dict())):
        V, T, _, inputs, _ = _mesh(name)
        cases.append((name, V, T, next(iter(inputs.values()))[0], kw))
    cases = [(c[0], c[1].verts, c[1].tets, c[2], c[3]) if c[0] == "mixed64" else c for c in cases]
    rng = np.random.default_rng(3)
    c1, c2 = COEF
    for name, V, T, x_np, kw in cases:
        sp = _handle(ext, V, T, enable_amips=True, **kw)
        pcg = DevicePCG(sp, hessian=hessian)
        hs = DeviceHessian(pcg)
        x, v = _cuda(x_np), _cuda(rng.standard_normal((len(V), 3)))
        for order, c3 in ((2, 0.0), (4, C3), (2, C3)):
            vals = hs.assemble(x, c1, c2, order, c3=c3)
            y, mag = _bsr_hv(torch, hs, vals, v)
            ref = (sp.hvp(x, v, c1, c2, order, c3=c3)[0] if hessian == "exact" else pcg.hvp_psd(x, v, c1, c2, order, c3=c3)[0])
            ref = ref.double().cpu().numpy().reshape(-1)
            if name == "mixed64":
                pk = _pack("mixed")[0]
                skip = _skip_spheres(pk, x_np, hessian == "exact" and c3 != 0)
                assert len(skip) < pk.num_spheres
                for s in range(pk.num_spheres):
                    if s in skip:
                        continue
                    sl = slice(3 * pk.vert_offsets[s], 3 * pk.vert_offsets[s + 1])
                    assert np.linalg.norm(y[sl] - ref[sl]) <= REL * np.linalg.norm(mag[sl]), (name, s, order, c3)
            else:
                assert np.linalg.norm(y - ref) <= REL * np.linalg.norm(mag), (name, order, c3)
            if hessian == "exact":
                D = hess_blocks(sp.hess_diag(x, c1, c2, order, c3=c3)).double().cpu().numpy()
                crow, col = hs.crow.cpu().numpy(), hs.col.cpu().numpy()
                vh = vals.double().cpu().numpy()
                rows = np.repeat(np.arange(len(V)), np.diff(crow))
                A = np.zeros(len(V))
                np.add.at(A, rows, np.abs(vh).max(axis=(1, 2)))
                got = np.zeros_like(D)
                got[rows[rows == col]] = vh[rows == col]
                ok = np.ones(len(V), bool)
                if name == "mixed64":                                   # tsb_hess_diag is fp32 too: the same exclusions
                    for s in skip:
                        ok[pk.vert_offsets[s]:pk.vert_offsets[s + 1]] = False
                assert (np.abs(got - D).max(axis=(1, 2)) <= KAPPA * U * A)[ok].all(), (name, order, c3)


def _mirror_index(hs):
    import scipy.sparse as sps
    crow, col = hs.crow.cpu().numpy(), hs.col.cpu().numpy()
    n = len(crow) - 1
    m = sps.csr_matrix((np.arange(len(col)) + 1, col, crow), shape=(n, n)).T.tocsr()
    m.sort_indices()
    assert (m.indptr == crow).all() and (m.indices == col).all()
    return m.data - 1


@pytest.mark.gpu
@pytest.mark.parametrize("hessian", ["exact", "psd"])
def test_bitwise_invariants(ext, hessian):
    torch = _torch()
    pk, x_np = _psd_pack("mixed64")
    c1, c2 = COEF
    x = _cuda(x_np)
    hss = [_dev_hessian(_handle(ext, pk.verts, pk.tets, enable_amips=True, **kw), hessian)
           for kw in (dict(), dict(deterministic=True), dict(force_global=True))]
    hs = hss[0]
    mir = torch.from_numpy(_mirror_index(hs)).long().cuda()
    for order, c3 in ((2, 0.0), (4, C3)):
        a = hs.assemble(x, c1, c2, order, c3=c3)
        assert torch.equal(a, a[mir].transpose(1, 2))                      # (i, j) = (j, i)^T bitwise
        assert torch.equal(a, hs.assemble(x, c1, c2, order, c3=c3))       # repeatable
        for other in hss[1:]:
            assert torch.equal(other.crow, hs.crow) and torch.equal(other.col, hs.col)
            assert torch.equal(a, other.assemble(x, c1, c2, order, c3=c3))
        s2 = torch.cuda.Stream()
        out = torch.empty_like(a)
        s2.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s2):
            hs.assemble(x, c1, c2, order, c3=c3, out=out)
        torch.cuda.current_stream().wait_stream(s2)
        assert torch.equal(a, out)
        # CUDA graph
        g = torch.cuda.CUDAGraph()
        out2 = torch.zeros_like(a)
        with torch.cuda.graph(g):
            hs.assemble(x, c1, c2, order, c3=c3, out=out2)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(a, out2)
    # changing one sphere's x changes only that sphere's blocks
    vo = pk.vert_offsets
    x2 = x.clone()
    x2[vo[5]:vo[6]] += 0.01 * torch.randn((vo[6] - vo[5], 3), device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    a, b = hs.assemble(x, c1, c2, 4, c3=C3), hs.assemble(x2, c1, c2, 4, c3=C3)
    crow = hs.crow.cpu().numpy()
    rows = torch.from_numpy(np.repeat(np.arange(pk.n), np.diff(crow))).cuda()
    inside = (rows >= int(vo[5])) & (rows < int(vo[6]))
    assert torch.equal(a[~inside], b[~inside]) and not torch.equal(a[inside], b[inside])


@pytest.mark.gpu
def test_sparse_direct_solve_matches_device_pcg(ext):
    import scipy.sparse.linalg as spla
    torch = _torch()
    from tssplat_b200.hessian import DeviceHessian
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _small_mixed()
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True)
    pcg = DevicePCG(sp, hessian="psd")
    hs = DeviceHessian(pcg)
    he = DeviceHessian(DevicePCG(sp))
    x = _cuda(x_np)
    c1, c2 = COEF
    vals = hs.assemble(x, c1, c2, 2, c3=C3)
    Hp = hs.sphere(vals, 0).toarray().astype(np.float64)
    He = he.sphere(he.assemble(x, c1, c2, 2, c3=C3), 0).toarray().astype(np.float64)
    wp, we = np.linalg.eigvalsh(0.5 * (Hp + Hp.T)), np.linalg.eigvalsh(0.5 * (He + He.T))
    assert wp.min() >= -1e-6 * wp.max(), (wp.min(), wp.max())
    assert we.min() < -1e-6 * we.max(), (we.min(), we.max())           # the rough sphere's exact Hessian is not PSD
    mu = 1e-3 * wp.max()
    b_np = np.zeros((pk.n, 3), np.float32)
    v0, v1 = pk.vert_offsets[0], pk.vert_offsets[1]
    b_np[v0:v1] = np.random.default_rng(4).standard_normal((v1 - v0, 3))
    import scipy.sparse as sps
    Hs = hs.sphere(vals, 0).astype(np.float64) + mu * sps.identity(Hp.shape[0])
    d_ref = spla.spsolve(Hs.tocsc(), b_np[v0:v1].reshape(-1).astype(np.float64))
    res = pcg.solve(x, _cuda(b_np), c1, c2, 2, c3=C3, max_iter=2000, rtol=1e-6, shift=float(mu))
    d = res.d.double().cpu().numpy()[v0:v1].reshape(-1)
    assert int(res.status[0]) == 1
    assert np.linalg.norm(d - d_ref) <= 1e-4 * np.linalg.norm(d_ref), np.linalg.norm(d - d_ref) / np.linalg.norm(d_ref)


@pytest.mark.gpu
def test_errors_memory_and_module(ext):
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    from tssplat_b200.hessian import DeviceHessian
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _small_mixed()
    sp = _handle(ext, pk.verts, pk.tets)
    info0 = dict(sp.info)
    pcg = DevicePCG(sp)
    pb = pcg.device_bytes
    hs = DeviceHessian(pcg)
    assert dict(sp.info) == info0 and int(_capi.lib.tsb_pcg_device_bytes(pcg._s)) == pb
    n, nele = pk.n, len(pk.tets)
    assert hs.device_bytes == 8 * (n + 1) + 8 * hs.nnzb + 493 * nele
    spa = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    hp = DeviceHessian(DevicePCG(spa, hessian="psd"))
    assert hp.device_bytes == 8 * (n + 1) + 8 * hs.nnzb + 561 * nele and hp.nnzb == hs.nnzb
    x = _cuda(x_np)
    c1, c2 = COEF
    with pytest.raises(RuntimeError, match="float32"):
        hs.assemble(x.double(), c1, c2, 2)
    with pytest.raises(RuntimeError, match="float32"):
        hs.assemble(x[:-1], c1, c2, 2)
    with pytest.raises(RuntimeError, match="out"):
        hs.assemble(x, c1, c2, 2, out=torch.empty(9 * hs.nnzb - 1, device="cuda"))
    with pytest.raises(RuntimeError, match="order"):
        hs.assemble(x, c1, c2, 3)
    with pytest.raises(RuntimeError, match="enable_amips"):
        hs.assemble(x, c1, c2, 2, c3=C3)
    with pytest.raises(RuntimeError, match=">= 0"):
        hp.assemble(x, c1, -c2, 2)
    with pytest.raises(RuntimeError, match="psd"):
        DeviceHessian(pcg, hessian="psd")
    hs.assemble(x, -c1, c2, 2)                                          # negative weights are fine in exact mode
    # the module route: scheduler coefficients, order at it, amips_coeff, newton_hessian
    flags = dict(smooth_eng_coeff=2e-4, barrier_coeff=2e-4, increase_order_iter=100, amips_coeff=C3, newton_hessian="psd")
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    for it in (10, 200):
        got = E.hessian(x, it)
        cc1, cc2 = E.coeff_scheduler(it)
        ref = E.device_hessian.assemble(x, cc1, cc2, E.order_at(it), c3=C3)
        assert torch.equal(got, ref) and E.device_hessian.hessian == "psd" and E.device_hessian.pcg is E.device_pcg


# ---------------------------------------------------------------------------------------------------------------------
# the plan-shape meshes: a sparse fp64 reference on the block pattern (a dense one would need 11 GB for mixed, 125 GB
# for tiny2600)


def sparse_reference(V, T, x, c1, c2, c3, order, project, pattern, rest64=False):
    """fp64 blocks [nnzb, 3, 3] of c1 M_ij I plus the tet blocks of tet_hessians scattered to their (crow, col) blocks,
    the magnitudes as kernel_input_dense forms them (|c1 M_ij| I, c1 sum_{j != i} |M_ij| on the diagonal, sum_t |K_t^T H
    K_t|), and each block's number of fp32 addends n_ij: its active tets + 1 (c1 M_ij I)."""
    from oracle.tet_energy_oracle import ReferenceEnergyOracle
    T = np.asarray(T, np.int64).reshape(-1, 4)
    crow, col, tblk = pattern["crow"], pattern["col"], pattern["tblk"].reshape(-1)
    n, nnzb = len(crow) - 1, len(col)
    rows = np.repeat(np.arange(n), np.diff(crow))
    M1 = ReferenceEnergyOracle(V, T).M[0::3, 0::3].tocsr()
    Mij = np.asarray(M1[rows, col]).ravel()
    rowsum = np.abs(c1) * (np.asarray(abs(M1).sum(axis=1)).ravel() - np.abs(M1.diagonal()))
    eye = np.eye(3)
    ref = (c1 * Mij)[:, None, None] * eye
    mag = (np.abs(c1 * Mij) + np.where(rows == col, rowsum[rows], 0.0))[:, None, None] * eye
    Ht, At = tet_hessians(V, T, x, c2, c3, order, project=project, rest64=rest64)
    blk = lambda H: H.reshape(-1, 4, 3, 4, 3).transpose(0, 1, 3, 2, 4).reshape(-1, 3, 3)      # [t, k, l] blocks
    np.add.at(ref, tblk, blk(Ht))
    np.add.at(mag, tblk, blk(At))
    active = np.repeat(At.reshape(len(T), -1).max(axis=1) > 0, 16)
    return ref, mag, np.bincount(tblk[active], minlength=nnzb) + 1


def _bsr_mul(pattern, blocks, v):
    crow, col = pattern["crow"], pattern["col"]
    rows = np.repeat(np.arange(len(crow) - 1), np.diff(crow))
    y = np.zeros((len(crow) - 1, 3))
    np.add.at(y, rows, np.einsum("bij,bj->bi", blocks, np.asarray(v, np.float64).reshape(-1, 3)[col]))
    return y


@pytest.mark.parametrize("name", ["pole", "near_cap"])
def test_sparse_reference_is_the_products(name):
    """With fp64 rest inverses, sparse_reference times v is c1 M v + c2 H_b v + c3 H_a v of the fp64 matrix-form
    products (test_hvp, test_hvp_amips) on every input of the suites: the scatter puts every tet block where it belongs."""
    from test_hvp import hvp_terms
    from test_hvp_amips import _mesh, amips_hvp_terms
    V, T, orc, inputs, v = _mesh(name)
    pattern = hess_pattern(V, T)
    vv = v.astype(np.float64)
    c1, c2, c3 = 2e-3, 0.8, 0.5
    for case, (x, _) in inputs.items():
        Hav, _ = amips_hvp_terms(orc, x.astype(np.float64), vv)
        for order in (2, 4):
            Mv, Hbv, _, _ = hvp_terms(orc, x.astype(np.float64), vv, order)
            ref = (c1 * Mv + c2 * Hbv + c3 * Hav).reshape(-1, 3)
            blocks, _, _ = sparse_reference(V, T, x, c1, c2, c3, order, False, pattern, rest64=True)
            y = _bsr_mul(pattern, blocks, v)
            assert np.linalg.norm(y - ref) <= 1e-12 * np.linalg.norm(ref), (case, order, np.linalg.norm(y - ref) / np.linalg.norm(ref))


@pytest.mark.gpu
@pytest.mark.parametrize("hessian", ["exact", "psd"])
@pytest.mark.parametrize("mesh", ["pole", "near_cap", "tiny2600", "mixed"])
def test_blocks_plan_shapes(ext, mesh, hessian):
    """The assembled blocks of the plan-shape meshes against sparse_reference, block by block, within (KAPPA_BLOCK +
    n_ij) u A_ij (KAPPA_PSD projected): the pole's row 0 has 989 blocks (31 passes of the row gather) and block (0, 0)
    is a recursive fp32 sum of 1973 addends; near_cap's and the pole's last block-kernel CTA is partial; tiny2600 has 2600
    spheres (also checked through hs.sphere on a sample) and mixed whole-area and twelve-tet spheres side by side."""
    from _helpers import assert_plan_shape, cpu_plan
    from test_hvp_amips import _mesh
    V, T, _, inputs, _ = _mesh(mesh)
    sp = _handle(ext, V, T, enable_amips=True)
    assert_plan_shape(mesh, cpu_plan(sp, V, T, enable_amips=True), {})
    hs = _dev_hessian(sp, hessian)
    pattern = hess_pattern(V, T)
    crow = hs.crow.cpu().numpy()
    assert (crow == pattern["crow"]).all() and (hs.col.cpu().numpy() == pattern["col"]).all()
    if mesh == "pole":
        assert crow[1] - crow[0] == 989 and pattern["inc_ptr"][1] - pattern["inc_ptr"][0] == 1972
    assert len(T) % 128 != 0                                        # the block kernel's last CTA (kHessT tets) is partial
    mirror = _torch().from_numpy(_mirror_index(hs)).long().cuda() if mesh == "pole" else None
    rows = np.repeat(np.arange(len(V)), np.diff(crow))
    c1, c2 = COEF
    kappa = KAPPA_PSD if hessian == "psd" else KAPPA_BLOCK
    worst, worst_frac = 0.0, 0.0
    for case, c3 in (("inverted_o2", 0.0), ("inverted_o2", C3), ("stretched_o2", C3)):
        x_np = inputs[case][0]
        x = _cuda(x_np)
        for order in (2, 4):
            vals = hs.assemble(x, c1, c2, order, c3=c3)
            if mirror is not None:                               # row 0 in 31 passes, its mirrors from 988 short rows
                assert _torch().equal(vals, vals[mirror].transpose(1, 2))
            got = vals.double().cpu().numpy()
            ref, mag, nadd = sparse_reference(V, T, x_np, c1, c2, c3, order, hessian == "psd", pattern)
            r = np.abs(got - ref).max(axis=(1, 2)) / (U * np.maximum(np.abs(mag).max(axis=(1, 2)), 1e-300))
            key = (mesh, hessian, case, order, c3)
            assert (r <= kappa + nadd).all(), (key, r.max(), int(np.argmax(r / (kappa + nadd))))
            worst, worst_frac = max(worst, r.max()), max(worst_frac, (r / (kappa + nadd)).max())
            if mesh == "tiny2600":
                for s in np.random.default_rng(order).choice(sp.info["n_components"], 12, replace=False):
                    vs = hs.sphere_vertices(int(s))
                    loc = np.full(len(V), -1)
                    loc[vs] = np.arange(len(vs))
                    inside = np.isin(rows, vs)
                    dense = np.zeros((3 * len(vs), 3 * len(vs)))
                    for b in np.nonzero(inside)[0]:
                        i, j = loc[rows[b]], loc[pattern["col"][b]]
                        dense[3 * i:3 * i + 3, 3 * j:3 * j + 3] = ref[b]
                    gs = hs.sphere(vals, int(s)).toarray().astype(np.float64)
                    bound = (kappa + nadd[inside].max()) * U * np.abs(mag[inside]).max()
                    assert np.abs(gs - dense).max() <= bound, (key, int(s))
    print(f"{mesh} {hessian}: worst |H - H64| / (u A_ij) = {worst:.3g}, of the bound (KAPPA + n_ij): {worst_frac:.3g}")

"""The device-resident per-sphere PCG solver (tsb_pcg_*, tsb_sphere_axpy, newton.DevicePCG,
SmoothnessBarrierEnergy.newton_direction).

CPU: the fp64 numpy restatement of the batched state machine the kernels implement (_newton_model), against dense
solves per component and step for step against newton.pcg; its status semantics; the kernel's 3x3 Jacobi eigen /
clamp / inverse algorithm re-enacted in numpy against newton.block_jacobi; the host builder's component lists and chunk
table.  GPU: the
preconditioner kernel, the solve (true residuals, records, energy decrease, product counts), a mixed pack where the
global CG is truncated by one sphere, independence and bitwise repeatability, handle variants, the per-sphere axpy,
chaining, handle info, argument errors and the module route end to end."""
import ctypes as C

import numpy as np
import pytest

from _helpers import GOLDEN, PLAN_DEBUG_SO
from _newton_model import (CHUNK, COEF, CONVERGED, MAXITER, NEGCURV, NEGCURV_FIRST, ZERO_RHS, _cuda, _handle,  # noqa: F401
                           _shuffled_mesh, _spd, _torch, batched_pcg_reference, ext, jacobi_inverse_blocks, planes_of, sym6)
from tssplat_b200.mesh import connected_components, make_pack, perturb


# ---------------------------------------------------------------------------------------------------------------------
# CPU


@pytest.fixture(scope="module")
def assembled():
    """H = c1 M + c2 sum_t H_t of a 3-sphere pack with one sphere mirrored, dense per component, column by column from
    test_hvp.hvp_terms."""
    from _helpers import mirror_components
    from oracle.tet_energy_oracle import ReferenceEnergyOracle
    from test_hvp import hvp_terms
    pk = make_pack(3, 96, seed=4)
    orc = ReferenceEnergyOracle(pk.verts, pk.tets)
    x = mirror_components(perturb(pk, sigma_rel=0.02, seed=2), pk.tets, every=3).astype(np.float64)   # sphere 0 inverted
    c1, c2 = 1e-3, 1.0
    n3 = 3 * len(pk.verts)
    H = np.zeros((n3, n3))
    for j in range(n3):
        e = np.zeros(n3)
        e[j] = 1.0
        Mv, Hbv, _, _ = hvp_terms(orc, x, e, 2)
        H[:, j] = c1 * Mv + c2 * Hbv
    assert np.abs(H - H.T).max() <= 1e-12 * np.abs(H).max()
    vo = pk.vert_offsets
    blocks = [H[3 * vo[s]:3 * vo[s + 1], 3 * vo[s]:3 * vo[s + 1]] for s in range(3)]
    off = H.copy()
    for s in range(3):
        off[3 * vo[s]:3 * vo[s + 1], 3 * vo[s]:3 * vo[s + 1]] = 0
    assert not off.any(), "spheres share no vertices: H is block diagonal"
    g = orc.backward(1.0, x, c1, c2, 2).reshape(-1)
    return blocks, [-g[3 * vo[s]:3 * vo[s + 1]] for s in range(3)], pk


def _block_precond(Hc):
    """Dense block-Jacobi preconditioner of a dense block, with newton.block_jacobi's semantics."""
    import torch
    from tssplat_b200.newton import block_jacobi
    m = len(Hc) // 3
    D = np.stack([Hc[3 * i:3 * i + 3, 3 * i:3 * i + 3] for i in range(m)])
    Pb = block_jacobi(torch.from_numpy(planes_of(D))).numpy()
    P = np.zeros_like(Hc)
    for i in range(m):
        P[3 * i:3 * i + 3, 3 * i:3 * i + 3] = Pb[i]
    return P, Pb


def test_reference_against_dense_solves(assembled):
    blocks, b, _ = assembled
    P = [_block_precond(Hc)[0] for Hc in blocks]
    rtol = 1e-8
    res = batched_pcg_reference(blocks, b, P, 2000, rtol)
    assert any(r["status"] == CONVERGED for r in res)
    for c, r in enumerate(res):
        if r["status"] != CONVERGED:
            assert r["status"] in (NEGCURV, NEGCURV_FIRST) and np.linalg.eigvalsh(blocks[c]).min() < 0   # the mirrored sphere
            continue
        Hc = blocks[c]
        assert np.linalg.norm(Hc @ r["d"] - b[c]) <= 10 * rtol * np.linalg.norm(b[c])
        # M's null space (rigid translations at least): compare on the range of H
        w, Q = np.linalg.eigh(Hc)
        R = Q[:, w > 1e-10 * w.max()]
        exact = R @ ((R.T @ b[c]) / w[w > 1e-10 * w.max()])
        assert np.linalg.norm(R @ (R.T @ r["d"]) - exact) <= 1e-5 * np.linalg.norm(exact)
        assert abs(r["d_H_d"] - r["d"] @ Hc @ r["d"]) <= 1e-6 * abs(r["d_H_d"])
        assert abs(r["b_dot_d"] - b[c] @ r["d"]) <= 1e-12 * abs(r["b_dot_d"])


@pytest.mark.parametrize("comp", [0, 1])
def test_reference_step_for_step_against_newton_pcg(assembled, comp):
    """One component: after every number of iterations the restatement returns what newton.pcg returns."""
    import torch
    from tssplat_b200.newton import pcg
    blocks, b, _ = assembled
    Hc, bc = blocks[comp], b[comp]
    P, Pb = _block_precond(Hc)
    Ht, bt = torch.from_numpy(Hc), torch.from_numpy(bc).reshape(-1, 3)
    hv = lambda p: (Ht @ p.reshape(-1)).reshape(p.shape)
    for k in (1, 2, 3, 5, 8, 13, 40):
        ref = pcg(hv, bt, torch.from_numpy(Pb), max_iter=k, rtol=1e-6)
        got = batched_pcg_reference([Hc], [bc], [P], k, 1e-6)[0]
        assert got["n_hvp"] == ref.n_hvp
        assert (got["status"] == CONVERGED) == ref.converged and (got["status"] in (NEGCURV, NEGCURV_FIRST)) == ref.negative_curvature
        # the same recurrence with differently ordered fp64 sums: rounding differences grow with the iteration count
        assert np.allclose(got["d"], ref.x.numpy().reshape(-1), rtol=0, atol=1e-6 * np.abs(got["d"]).max())
        assert abs(got["rel_residual"] - ref.rel_residual) <= 1e-2 * ref.rel_residual


def test_reference_status_semantics():
    rng = np.random.default_rng(0)
    m = 12
    H = [_spd(rng, m) for _ in range(5)]
    b = [rng.normal(size=m) for _ in range(5)]
    b[1][:] = 0.0                                                      # zero right-hand side
    H[2] = -_spd(rng, m)                                               # negative curvature at the first direction
    Q = np.linalg.qr(rng.normal(size=(m, m)))[0]                       # indefinite: one negative direction, found later
    H[3] = (Q * np.r_[-3.0, rng.uniform(0.5, 20, m - 1)]) @ Q.T
    b[3] = Q @ np.r_[1e-3, rng.normal(size=m - 1)]
    P = [None] * 5
    res = batched_pcg_reference(H, b, P, 50, 1e-10)
    assert [r["status"] for r in res] == [CONVERGED, ZERO_RHS, NEGCURV_FIRST, NEGCURV, CONVERGED]
    assert res[1]["n_hvp"] == 0 and not res[1]["d"].any() and res[1]["rel_residual"] == 0.0
    assert res[2]["n_hvp"] == 1 and np.array_equal(res[2]["d"], b[2]) and res[2]["rel_residual"] == 1.0 and res[2]["d_H_d"] == 0.0
    assert res[3]["n_hvp"] > 1 and res[3]["d"].any() and res[3]["b_dot_d"] > 0
    for c in (0, 4):
        assert np.allclose(res[c]["d"], np.linalg.solve(H[c], b[c]), rtol=1e-8)
        alone = batched_pcg_reference([H[c]], [b[c]], [None], 50, 1e-10)[0]
        assert np.array_equal(alone["d"], res[c]["d"]) and alone["n_hvp"] == res[c]["n_hvp"]    # bitwise: no coupling
    # max_iter: the iterate after k steps, status MAXITER
    r2 = batched_pcg_reference(H[:1], b[:1], [None], 2, 1e-10)[0]
    assert r2["status"] == MAXITER and r2["n_hvp"] == 2 and 0 < r2["rel_residual"] < 1


def _jacobi_cases():
    rng = np.random.default_rng(3)
    Q = np.linalg.qr(rng.normal(size=(200, 3, 3)))[0]
    lam = np.concatenate([rng.uniform(0.1, 10, size=(60, 3)),                       # SPD
                          rng.uniform(-5, 5, size=(60, 3)),                         # indefinite
                          np.c_[np.zeros((20, 2)), rng.uniform(0.1, 5, size=20)],   # rank 1 (a barrier block)
                          np.repeat(rng.uniform(1e-4, 3, size=(20, 1)), 3, axis=1),  # c I (the smoothness block)
                          np.zeros((20, 3)),                                        # zero
                          -rng.uniform(0.1, 5, size=(20, 3))])                      # negative definite
    D = np.einsum("nij,nj,nkj->nik", Q, lam, Q)
    D[140:160] = np.einsum("n,ij->nij", lam[140:160, 0], np.eye(3))                 # exactly diagonal
    D[160:180] = 0.0
    return 0.5 * (D + D.transpose(0, 2, 1)), lam


def test_jacobi_blocks_against_block_jacobi():
    """The kernel's algorithm in fp64 is block_jacobi to rounding; on fp32 inputs (what tsb_hess_diag hands it) the
    result rounded to fp32 stays within 8 fp32 ulps of the largest entry of the block: the bound of the GPU check."""
    import torch
    from tssplat_b200.newton import block_jacobi
    D, lam = _jacobi_cases()
    for rel_floor in (1e-6, 1e-2):
        ref = sym6(block_jacobi(torch.from_numpy(planes_of(D)), rel_floor=rel_floor).numpy())
        got = jacobi_inverse_blocks(D, rel_floor)
        scale = np.abs(ref).max(axis=1, keepdims=True)
        assert (np.abs(got - ref) <= 1e-9 * scale + 1e-300).all()
        assert not got[160:].any() and not ref[160:].any()              # zero and negative definite blocks -> 0
    D32 = D.astype(np.float32).astype(np.float64)
    ref = sym6(block_jacobi(torch.from_numpy(planes_of(D32)), rel_floor=1e-6).numpy())
    got = jacobi_inverse_blocks(D32, np.float64(np.float32(1e-6))).astype(np.float32).astype(np.float64)
    scale = np.abs(ref).max(axis=1, keepdims=True)
    assert (np.abs(got - ref) <= 8 * 2.0 ** -24 * scale + 1e-300).all()


def _pcg_lists(V, T):
    lib = C.CDLL(PLAN_DEBUG_SO)
    lib.tsbdbg_build_det.restype = C.c_int
    lib.tsbdbg_build_det.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int32] * 8 + [C.c_float] + [C.c_int32] * 3 + [C.POINTER(C.c_void_p)]
    lib.tsbdbg_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_int32)]
    lib.tsbdbg_free.argtypes = [C.c_void_p]
    V = np.ascontiguousarray(V, np.float32).reshape(-1)
    T = np.ascontiguousarray(T, np.int32).reshape(-1)
    d = C.c_void_p()
    assert lib.tsbdbg_build_det(V.ctypes.data, T.ctypes.data, V.size // 3, T.size // 4, 16, 132, 0, 0, 0, 0, 0.0, 0, 0, 0, C.byref(d)) == 0
    out = {}
    try:
        for name in ("comp_label", "pcg_vert", "pcg_comp_off", "pcg_chunk", "pcg_comp_chunk", "comp_first_vertex", "orphans"):
            ptr, cnt, eb = C.c_void_p(), C.c_int64(), C.c_int32()
            assert lib.tsbdbg_array(d, name.encode(), C.byref(ptr), C.byref(cnt), C.byref(eb)) == 0, name
            out[name] = np.frombuffer(bytes((C.c_char * (cnt.value * eb.value)).from_address(ptr.value)) if cnt.value else b"",
                                      dtype=np.int32).copy()
    finally:
        lib.tsbdbg_free(d)
    return out


@pytest.mark.parametrize("mesh", ["pack", "shuffled"])
def test_component_lists_and_chunk_table(mesh):
    if mesh == "pack":
        pk = make_pack(5, 700, seed=2)
        V, T = pk.verts, pk.tets
    else:
        V, T, _ = _shuffled_mesh()
    L = _pcg_lists(V, T)
    n = len(V)
    used = np.zeros(n, bool)
    used[np.unique(T)] = True
    lab = connected_components(n, T)
    label, vert, off, chunk, cchunk = L["comp_label"], L["pcg_vert"], L["pcg_comp_off"], L["pcg_chunk"].reshape(-1, 3), L["pcg_comp_chunk"]
    S = len(off) - 1
    # a partition of the non-orphan vertices; orphans belong to no component
    assert np.array_equal(np.sort(vert), np.flatnonzero(used)) and np.array_equal(np.sort(L["orphans"]), np.flatnonzero(~used))
    assert (label[~used] == -1).all() and (label[used] >= 0).all()
    first = []
    for c in range(S):
        vs = vert[off[c]:off[c + 1]]
        assert (np.diff(vs) > 0).all() and (label[vs] == c).all() and len(set(lab[vs])) == 1
        assert np.array_equal(np.sort(np.flatnonzero((lab == lab[vs[0]]) & used)), vs)
        first.append(vs[0])
    assert (np.diff(first) > 0).all() and np.array_equal(first, L["comp_first_vertex"])     # component order: lowest id
    # chunks: <= 256 entries, never across a component, in order, covering every entry once
    assert (chunk[:, 2] - chunk[:, 1] <= CHUNK).all() and (chunk[:, 2] > chunk[:, 1]).all()
    assert chunk[0, 1] == 0 and chunk[-1, 2] == len(vert) and np.array_equal(chunk[1:, 1], chunk[:-1, 2])
    for c in range(S):
        ck = chunk[cchunk[c]:cchunk[c + 1]]
        assert (ck[:, 0] == c).all() and ck[0, 1] == off[c] and ck[-1, 2] == off[c + 1]
        assert len(ck) == -(-(off[c + 1] - off[c]) // CHUNK)
    if mesh == "shuffled":
        assert (~used).sum() == 500 and any((np.diff(vert[off[c]:off[c + 1]]) > 1).any() for c in range(S))


# ---------------------------------------------------------------------------------------------------------------------
# GPU



_PACKS = {}


def _pack(name):
    """(pack, x): "small" = make_pack(3, 512, seed=4) near rest, "big" = the 64 x 4096 pack near rest, "mixed" = 8 x 1024
    with every fourth sphere perturbed at 0.35 h (inverted tets) and the rest at 0.02 h."""
    if name not in _PACKS:
        if name == "small":
            pk = make_pack(3, 512, seed=4)
            x = perturb(pk, sigma_rel=0.02, seed=1)
        elif name == "big":
            pk = make_pack(64, 4096, seed=0, unique=8)
            x = perturb(pk, sigma_rel=0.02, seed=1)
        else:
            pk = make_pack(8, 1024, seed=5)
            x, rough = perturb(pk, sigma_rel=0.02, seed=1), perturb(pk, sigma_rel=0.35, seed=3)
            for s in range(0, pk.num_spheres, 4):
                x[pk.vert_offsets[s]:pk.vert_offsets[s + 1]] = rough[pk.vert_offsets[s]:pk.vert_offsets[s + 1]]
        _PACKS[name] = (pk, x)
    return _PACKS[name]


def _sphere_of(pk):
    return np.repeat(np.arange(pk.num_spheres), np.diff(pk.vert_offsets))


def _sphere_norms(torch, v, sid, S):
    return torch.zeros(S, dtype=torch.float64, device=v.device).index_add_(0, sid, (v.double() ** 2).sum(dim=1)).sqrt()


def _sphere_dots(torch, a, b, sid, S):
    return torch.zeros(S, dtype=torch.float64, device=a.device).index_add_(0, sid, (a.double() * b.double()).sum(dim=1))


@pytest.mark.gpu
@pytest.mark.parametrize("mesh", ["big", "shuffled"])
def test_set_blocks_against_block_jacobi(ext, mesh):
    torch = _torch()
    from tssplat_b200.newton import DevicePCG, block_jacobi
    if mesh == "big":
        pk, x = _pack("big")
        V, T = pk.verts, pk.tets
    else:
        V, T, x = _shuffled_mesh()
    sp = _handle(ext, V, T, enable_amips=True)
    planes = sp.hess_diag(_cuda(x), 2e-3, 0.8, 2, c3=0.5)
    ws = DevicePCG(sp)
    for rel_floor in (1e-6, 1e-2):
        got = ws.set_blocks(planes, rel_floor=rel_floor, want_inverse=True).double().cpu().numpy()
        ref = sym6(block_jacobi(planes.double().cpu(), rel_floor=rel_floor).numpy())
        scale = np.abs(ref).max(axis=1, keepdims=True)
        assert (np.abs(got - ref) <= 8 * 2.0 ** -24 * scale).all()       # the bound test_jacobi_blocks_against_block_jacobi calibrates
    if mesh == "shuffled":
        orphans = np.ones(len(V), bool)
        orphans[np.unique(T)] = False
        assert orphans.sum() == 500 and not got[orphans].any()
    ident = ws.set_blocks(None, want_inverse=True).cpu().numpy()
    assert (ident == np.array([1, 1, 1, 0, 0, 0], np.float32)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "big"])
def test_solve_residuals_records_and_energy(ext, name):
    torch = _torch()
    from tssplat_b200.newton import DevicePCG, block_jacobi, pcg
    pk, x_np = _pack(name)
    sp = _handle(ext, pk.verts, pk.tets)
    x = _cuda(x_np)
    c1, c2 = COEF
    S, rtol = pk.num_spheres, 1e-3
    sid = torch.from_numpy(_sphere_of(pk)).cuda()
    e0, g = sp.energy_grad(x, c1, c2, 2)
    e0, b = float(e0[0]), -g
    planes = sp.hess_diag(x, c1, c2, 2)
    ws = DevicePCG(sp)
    ws.set_blocks(planes)
    res = ws.solve(x, b, c1, c2, 2, max_iter=1000, rtol=rtol, check_every=10)
    assert (res.status == CONVERGED).all() and res.iters_run < 1000 and res.iters_run % 10 == 0
    Hd = sp.hvp(x, res.d, c1, c2, 2)[0]
    bn = _sphere_norms(torch, b, sid, S)
    true_res = _sphere_norms(torch, b - Hd, sid, S) / bn
    # the recurrence's fp32 residual drifts from b - H d by a few fp32 roundings of |b| per iteration: 20 % slack
    assert (true_res <= 1.2 * rtol).all(), float(true_res.max())
    assert torch.allclose(res.rel_residual.double(), true_res, rtol=0.2, atol=0.2 * rtol)
    bd = _sphere_dots(torch, b, res.d, sid, S)
    assert torch.allclose(res.b_dot_d.double(), bd, rtol=1e-5) and (bd > 0).all()
    dHd = _sphere_dots(torch, res.d, Hd, sid, S)
    assert torch.allclose(res.d_H_d.double(), dHd, rtol=2e-2)                # fp32 CG loses some conjugacy
    e1, _ = sp.energy_grad(x + res.d, c1, c2, 2, want_grad=False)
    assert float(e1[0]) < e0
    ref = pcg(lambda p: sp.hvp(x, p, c1, c2, 2)[0], b, block_jacobi(planes.cpu()).cuda(), max_iter=1000, rtol=rtol)
    assert ref.converged
    print(f"{name}: newton.pcg {ref.n_hvp} products; per sphere max {int(res.n_hvp.max())}, mean {float(res.n_hvp.float().mean()):.1f}")
    # every sphere's own Krylov space resolves only its own spectrum; the margin (10 % + 2 products) is for the stopping
    # tests: |r_c| <= rtol |b_c| for every sphere is stricter than the pooled test for the slowest one
    assert int(res.n_hvp.max()) <= int(1.1 * ref.n_hvp) + 2


@pytest.mark.gpu
def test_mixed_pack_one_sphere_does_not_truncate_the_others(ext):
    torch = _torch()
    from tssplat_b200.newton import DevicePCG, block_jacobi, pcg
    pk, x_np = _pack("mixed")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    x = _cuda(x_np)
    c1, c2 = COEF
    c3 = 1e-4
    _, g = sp.energy_grad(x, c1, c2, 2, c3=c3)
    planes = sp.hess_diag(x, c1, c2, 2, c3=c3)
    ws = DevicePCG(sp)
    ws.set_blocks(planes)
    res = ws.solve(x, -g, c1, c2, 2, c3=c3, max_iter=600, rtol=1e-3)
    st = res.status.cpu().numpy()
    rough = np.arange(pk.num_spheres) % 4 == 0
    assert np.isin(st[rough], (NEGCURV, NEGCURV_FIRST)).any(), st
    assert (st[~rough] == CONVERGED).all(), st
    ref = pcg(lambda p: sp.hvp(x, p, c1, c2, 2, c3=c3)[0], -g, block_jacobi(planes.cpu()).cuda(), max_iter=600, rtol=1e-3)
    assert ref.negative_curvature and not ref.converged


def _solve_raw(torch, ws, x, b, terms_kw, max_iter, rtol, check_every=0, stream=None, d=None, rec=None):
    from tssplat_b200 import _capi
    S = ws.n_spheres
    d = torch.full((ws.tet_sp.n, 3), float("nan"), device="cuda") if d is None else d
    rec = torch.zeros((S, 8), dtype=torch.int32, device="cuda") if rec is None else rec
    terms = _capi.tsb_terms_t(**terms_kw)
    opt = _capi.tsb_pcg_options_t(max_iter=max_iter, rtol=rtol, check_every=check_every)
    it = C.c_int32(-1)
    st = torch.cuda.current_stream().cuda_stream if stream is None else stream
    rc = _capi.lib.tsb_pcg_solve(ws._s, x.data_ptr(), b.data_ptr(), C.byref(terms), C.byref(opt), d.data_ptr(), rec.data_ptr(),
                                 C.byref(it), st)
    assert rc == 0, ws._error(ws._s)
    return d, rec, it.value


@pytest.mark.gpu
def test_independence_and_bitwise_repeatability(ext):
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _pack("mixed")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    x = _cuda(x_np)
    c1, c2 = COEF
    tk = dict(c1=c1, c2=c2, order=2, c3=1e-4)
    _, g = sp.energy_grad(x, c1, c2, 2, c3=1e-4)
    b = -g
    ws = DevicePCG(sp)
    ws.set_blocks(sp.hess_diag(x, c1, c2, 2, c3=1e-4))
    d0, r0, it0 = _solve_raw(torch, ws, x, b, tk, 40, 1e-3)
    assert it0 == 40 and not torch.isnan(d0).any()
    d1, r1, _ = _solve_raw(torch, ws, x, b, tk, 40, 1e-3)                    # again
    assert torch.equal(d0, d1) and torch.equal(r0, r1)
    other = torch.cuda.Stream()                                              # another stream
    torch.cuda.synchronize()
    with torch.cuda.stream(other):
        d2, r2, _ = _solve_raw(torch, ws, x, b, tk, 40, 1e-3, stream=other.cuda_stream)
    other.synchronize()
    assert torch.equal(d0, d2) and torch.equal(r0, r2)
    dg, rg = torch.empty_like(d0), torch.zeros_like(r0)                      # CUDA graph, replayed twice
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _solve_raw(torch, ws, x, b, tk, 40, 1e-3, stream=torch.cuda.current_stream().cuda_stream, d=dg, rec=rg)
    for _ in range(2):
        dg.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(d0, dg) and torch.equal(r0, rg)
    # zero the right-hand side of sphere 2: ZERO_RHS there, every other sphere bitwise unchanged
    vo = pk.vert_offsets
    bz = b.clone()
    bz[vo[2]:vo[3]] = 0
    dz, rz, _ = _solve_raw(torch, ws, x, bz, tk, 40, 1e-3)
    keep = torch.ones(len(x), dtype=torch.bool, device="cuda")
    keep[vo[2]:vo[3]] = False
    assert torch.equal(dz[keep], d0[keep]) and not dz[~keep].any() and not torch.isnan(dz).any()
    sk = torch.arange(pk.num_spheres, device="cuda") != 2
    assert torch.equal(rz[sk], r0[sk]) and int(rz[2, 4]) == ZERO_RHS and int(rz[2, 3]) == 0
    # check_every stops early and gives what a fixed number of iterations gives
    d5, r5, it5 = _solve_raw(torch, ws, x, b, tk, 300, 1e-3, check_every=5)
    assert it5 % 5 == 0 or it5 == 300
    d6, r6, _ = _solve_raw(torch, ws, x, b, tk, it5, 1e-3)
    assert torch.equal(d5, d6) and torch.equal(r5, r6)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(warps_per_cta=8), dict(deterministic=True), dict(warps_per_cta=8, deterministic=True)],
                         ids=["w16", "w8", "w16-det", "w8-det"])


def test_staged_handle_variants(ext, kw):
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, **kw)
    assert sp.info["mode_global"] == 0
    _check_converges(torch, sp, DevicePCG(sp), _cuda(x_np), torch.from_numpy(_sphere_of(pk)).cuda(), pk.num_spheres)


def _check_converges(torch, sp, ws, x, sid, S):
    c1, c2 = COEF
    _, g = sp.energy_grad(x, c1, c2, 2)
    ws.set_blocks(sp.hess_diag(x, c1, c2, 2))
    res = ws.solve(x, -g, c1, c2, 2, max_iter=3000, rtol=1e-3, check_every=50)
    assert (res.status == CONVERGED).all(), res.status
    Hd = sp.hvp(x, res.d, c1, c2, 2)[0]
    true_res = _sphere_norms(torch, -g - Hd, sid, S) / _sphere_norms(torch, -g, sid, S)
    assert (true_res <= 1.2e-3).all(), float(true_res.max())
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
def test_a_veg_global_handle(ext, det):
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    d = np.load(GOLDEN + "/a_veg_mesh.npz")
    V, T = d["verts"].astype(np.float32), d["tets"].astype(np.int32)
    h = np.linalg.norm(V[T[:, 1]] - V[T[:, 0]], axis=1).mean()
    x = (V + np.random.default_rng(6).normal(scale=0.02 * h, size=V.shape)).astype(np.float32)
    sp = _handle(ext, V, T, force_global=True, deterministic=det)
    assert sp.info["mode_global"] == 1
    lab = connected_components(len(V), T)
    used = np.zeros(len(V), bool)
    used[np.unique(T)] = True
    S = sp.info["n_components"]
    sid = np.where(used, np.searchsorted(np.unique(lab[used]), lab), 0)
    res = _check_converges(torch, sp, DevicePCG(sp), _cuda(x), torch.from_numpy(sid).cuda(), S)
    assert not res.d[torch.from_numpy(~used).cuda()].any()


@pytest.mark.gpu
def test_shuffled_ids_with_orphans_solve_and_axpy(ext):
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    V, T, x_np = _shuffled_mesh()
    sp = _handle(ext, V, T)
    ws = DevicePCG(sp)
    used = np.zeros(len(V), bool)
    used[np.unique(T)] = True
    lab = connected_components(len(V), T)                                    # labels in order of first vertex
    firsts = np.array([np.flatnonzero(lab == c)[0] for c in np.unique(lab[used])])
    sid_np = np.where(used, np.searchsorted(np.unique(lab[used]), lab), 0)
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(~used).cuda()
    x = _cuda(x_np)
    c1, c2 = COEF
    _, g = sp.energy_grad(x, c1, c2, 2)
    ws.set_blocks(sp.hess_diag(x, c1, c2, 2))
    res = ws.solve(x, -g, c1, c2, 2, max_iter=400, rtol=1e-3, check_every=20)
    assert (res.status == CONVERGED).all() and not res.d[orph].any() and not torch.isnan(res.d).any()
    raw = torch.zeros((3, 8), dtype=torch.int32, device="cuda")
    _solve_raw(torch, ws, x, -g, dict(c1=c1, c2=c2, order=2, c3=0.0), 5, 1e-3, rec=raw)
    assert raw[:, 5].cpu().tolist() == firsts.tolist()                       # first_vertex
    assert raw[:, 6].cpu().tolist() == [int(((sid_np == k) & used).sum()) for k in range(3)]
    # axpy against torch indexing, orphans copied, in place
    a = torch.tensor([0.5, -1.25, 2.0], device="cuda")
    expect = torch.where(orph[:, None], x, x + a[sid][:, None] * res.d)
    out = ws.axpy(x, a, res.d)
    # the kernel's x + a d is one fused multiply-add, torch's two roundings: within one ulp of the result
    assert ((out - expect).abs() <= 2.0 ** -23 * expect.abs()).all() and torch.equal(out[orph], x[orph])
    xc = x.clone()
    assert ws.axpy(xc, a, res.d, out=xc) is xc and torch.equal(xc, out)


@pytest.mark.gpu
def test_more_chunks_than_one_resident_wave(ext):
    """1100 x 4096: about 4400 chunk CTAs per kernel, several times what the GPU holds at once, so the chunks of many
    spheres run in different waves.  Every sphere's true residual meets the test, and a sphere's step and record are
    bitwise the same when every other sphere's right-hand side is zeroed."""
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    pk = make_pack(1100, 4096, seed=0, unique=8)
    S = pk.num_spheres
    chunks = int(sum(-(-int(m) // CHUNK) for m in np.diff(pk.vert_offsets)))
    props = torch.cuda.get_device_properties(0)
    assert chunks > props.multi_processor_count * (props.max_threads_per_multi_processor // CHUNK), "not more than one wave"
    sp = _handle(ext, pk.verts, pk.tets, deterministic=True)
    x = _cuda(perturb(pk, sigma_rel=0.02, seed=1))
    sid = torch.from_numpy(_sphere_of(pk)).cuda()
    c1, c2 = COEF
    tk = dict(c1=c1, c2=c2, order=2, c3=0.0)
    _, g = sp.energy_grad(x, c1, c2, 2)
    b = -g
    ws = DevicePCG(sp)
    ws.set_blocks(sp.hess_diag(x, c1, c2, 2))
    res = ws.solve(x, b, c1, c2, 2, max_iter=1000, rtol=1e-3, check_every=25)
    assert (res.status == CONVERGED).all() and res.iters_run < 1000
    Hd = sp.hvp(x, res.d, c1, c2, 2)[0]
    true_res = _sphere_norms(torch, b - Hd, sid, S) / _sphere_norms(torch, b, sid, S)
    assert (true_res <= 1.2e-3).all(), float(true_res.max())
    d0, r0, _ = _solve_raw(torch, ws, x, b, tk, res.iters_run, 1e-3)
    assert torch.equal(d0, res.d)
    odd = (sid % 2 == 1)
    bz = torch.where(odd[:, None], torch.zeros_like(b), b)
    dz, rz, _ = _solve_raw(torch, ws, x, bz, tk, res.iters_run, 1e-3)
    assert torch.equal(dz[~odd], d0[~odd]) and not dz[odd].any()
    assert torch.equal(rz[0::2], r0[0::2]) and (rz[1::2, 4] == ZERO_RHS).all()


@pytest.mark.gpu
def test_component_with_more_than_32_chunks(ext):
    """One sphere of 50 000 tets (about 10 000 vertices, 40 chunks: the fold's lanes each add more than one partial)
    next to three small ones, on a GLOBAL deterministic handle."""
    torch = _torch()
    from tssplat_b200.mesh import concat_spheres, make_tet_sphere
    from tssplat_b200.newton import DevicePCG
    small = make_pack(3, 512, seed=4)
    vo, to = small.vert_offsets, small.tet_offsets
    parts = [(small.verts[vo[k]:vo[k + 1]], small.tets[to[k]:to[k + 1]] - vo[k]) for k in range(3)]
    parts.insert(1, make_tet_sphere(7, n_tets=50000))
    pk = concat_spheres(parts)
    nv = np.diff(pk.vert_offsets)
    assert -(-int(nv[1]) // CHUNK) > 32
    sp = _handle(ext, pk.verts, pk.tets, deterministic=True)
    assert sp.info["mode_global"] == 1 and sp.info["n_components"] == 4
    x = _cuda(perturb(pk, sigma_rel=0.02, seed=1))
    sid = torch.from_numpy(_sphere_of(pk)).cuda()
    c1, c2 = COEF
    tk = dict(c1=c1, c2=c2, order=2, c3=0.0)
    _, g = sp.energy_grad(x, c1, c2, 2)
    b = -g
    ws = DevicePCG(sp)
    ws.set_blocks(sp.hess_diag(x, c1, c2, 2))
    rtol = 1e-2
    res = ws.solve(x, b, c1, c2, 2, max_iter=5000, rtol=rtol, check_every=50)
    assert (res.status == CONVERGED).all(), (res.status, res.rel_residual)
    Hd = sp.hvp(x, res.d, c1, c2, 2)[0]
    true_res = _sphere_norms(torch, b - Hd, sid, 4) / _sphere_norms(torch, b, sid, 4)
    assert (true_res <= 1.2 * rtol).all(), true_res
    d0, r0, _ = _solve_raw(torch, ws, x, b, tk, res.iters_run, rtol)
    big = sid == 1
    bz = torch.where(big[:, None], b, torch.zeros_like(b))
    dz, rz, _ = _solve_raw(torch, ws, x, bz, tk, res.iters_run, rtol)
    assert torch.equal(dz[big], d0[big]) and torch.equal(rz[1], r0[1]) and not dz[~big].any()


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(deterministic=True)], ids=["default", "det"])
def test_chaining_and_handle_info(ext, kw):
    """The other calls of the handle give bitwise the same outputs after a solve on the same stream as on a handle that
    never ran one; creating a workspace leaves tsb_get_info unchanged; tsb_pcg_device_bytes is the documented sum."""
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _pack("small")
    det = bool(kw)
    x = _cuda(x_np)
    c1, c2 = COEF
    c3 = 1e-4 if det else 0.0
    a, b_ = _handle(ext, pk.verts, pk.tets, enable_amips=True, **kw), _handle(ext, pk.verts, pk.tets, enable_amips=True, **kw)
    info0 = dict(a.info)
    ws = DevicePCG(a)
    info = _capi.tsb_info_t()
    _capi.check(_capi.lib.tsb_get_info(a._h, C.byref(info)), a._h)
    assert {k: getattr(info, k) for k, _ in _capi.tsb_info_t._fields_} == info0 == dict(b_.info)
    n, S = a.n, a.info["n_components"]
    chunks = int(sum(-(-int(m) // CHUNK) for m in np.diff(pk.vert_offsets)))
    assert ws.device_bytes == 72 * n + 4 * n + 36 * chunks + 64 * S + 4 * (S + 1) + 4
    w = _cuda(np.random.default_rng(2).normal(size=x_np.shape))
    res = []
    for h, run in ((a, True), (b_, False)):
        if run:
            _, g = h.energy_grad(x, c1, c2, 2, c3=c3)
            ws.set_blocks(h.hess_diag(x, c1, c2, 2, c3=c3))
            ws.solve(x, -g, c1, c2, 2, c3=c3, max_iter=7)
        e, g = h.energy_grad(x, c1, c2, 2, c3=c3)
        e = e.clone()
        hv, cv = h.hvp(x, w, c1, c2, 2, want_curv=True, c3=c3)
        ls = h.line_search(x, w, [1e-4, 1e-3], c1, c2, 2, c3=c3, per_sphere=True)
        dg = h.hess_diag(x, c1, c2, 2, c3=c3)
        res.append((e, g, hv, cv, ls.delta, ls.max_step, ls.sphere_delta, ls.sphere_max_step, dg))
    torch.cuda.synchronize()
    for p, q in zip(*res):
        assert torch.equal(p, q)


@pytest.mark.gpu
def test_bad_arguments(ext):
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _pack("small")
    plain = _handle(ext, pk.verts, pk.tets)
    ws = DevicePCG(plain)
    x, b = _cuda(x_np), _cuda(np.random.default_rng(1).normal(size=x_np.shape))
    d = torch.full((len(x_np), 3), float("nan"), device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    E = _capi.TSB_E_INVALID
    T_ = lambda **k: _capi.tsb_terms_t(**{**dict(c1=1.0, c2=1.0, order=2, c3=0.0), **k})
    O_ = lambda **k: _capi.tsb_pcg_options_t(**{**dict(max_iter=5, rtol=1e-3, check_every=0), **k})

    def call(xp, bp, terms, opt, dp, s=ws._s):
        return _capi.lib.tsb_pcg_solve(s, xp, bp, C.byref(terms) if terms else None, C.byref(opt) if opt else None, dp, None, None, st)

    X, B, D = x.data_ptr(), b.data_ptr(), d.data_ptr()
    assert call(None, B, T_(), O_(), D) == E and call(X, None, T_(), O_(), D) == E and call(X, B, T_(), O_(), None) == E
    assert call(X, B, None, O_(), D) == E and call(X, B, T_(), None, D) == E
    assert call(X, B, T_(), O_(max_iter=0), D) == E and call(X, B, T_(), O_(rtol=-1.0), D) == E
    assert call(X, B, T_(), O_(check_every=-1), D) == E and call(X, B, T_(order=3), O_(), D) == E
    assert call(X, B, T_(c3=0.5), O_(), D) == E and b"enable_amips" in _capi.lib.tsb_pcg_last_error(ws._s)
    assert call(X, B, T_(), O_(), D, s=None) == E
    a = torch.ones(3, device="cuda")
    assert _capi.lib.tsb_sphere_axpy(ws._s, X, None, B, D, st) == E and _capi.lib.tsb_sphere_axpy(ws._s, X, a.data_ptr(), B, None, st) == E
    out = C.c_void_p()
    assert _capi.lib.tsb_pcg_create(None, C.byref(out)) == E and _capi.lib.tsb_pcg_create(plain._h, None) == E
    # check_every > 0 waits on the host: refused on a capturing stream before anything is recorded; the capture survives
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        d.fill_(float("nan"))
        cs = torch.cuda.current_stream().cuda_stream
        assert _capi.lib.tsb_pcg_solve(ws._s, X, B, C.byref(T_()), C.byref(O_(check_every=2)), D, None, None, cs) == E
    assert b"captured" in _capi.lib.tsb_pcg_last_error(ws._s)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.isnan(d).all()                                              # nothing was launched
    with pytest.raises(RuntimeError, match="enable_amips"):
        ws.solve(x, b, 1.0, 1.0, 2, c3=0.5)
    # a solve before set_blocks is not an error: the identity preconditioner
    fresh = DevicePCG(plain)
    c1, c2 = COEF
    r = fresh.solve(x, b, c1, c2, 2, max_iter=3)
    assert (r.n_hvp == 3).all() and not torch.isnan(r.d).any()


@pytest.mark.gpu
def test_module_newton_direction_with_per_sphere_armijo(ext):
    """Five Newton steps of the INTEGRATION.md loop on the mixed pack: the energy falls monotonically and the number of
    inverted tets never grows."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    pk, x_np = _pack("mixed")
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000,
                                                        amips_coeff=1e-4, deterministic=True))
    x = _cuda(x_np)
    it = 10
    alphas = torch.tensor([1.0, 0.5, 0.25, 0.125, 1 / 16, 1 / 32, 1 / 64, 1 / 128], device="cuda")

    def state(x):
        st = E.sphere_stats(x, it)
        c1, c2 = E.coeff_scheduler(it)
        return float((c1 * st.smooth + c2 * st.barrier + E.amips_coeff * st.amips).sum()), int(st.n_inverted.sum())

    e_prev, inv_prev = state(x)
    assert inv_prev > 0
    for _ in range(5):
        res = E.newton_direction(x, it, max_iter=50, rtol=1e-2)
        ls = E.line_search(x, res.d, it, alphas, per_sphere=True)
        # per sphere: the largest alpha_k below the inversion bound with E(x + alpha d) - E(x) <= -1e-4 alpha b.d
        ok = (ls.sphere_delta[:, :, 0] <= -1e-4 * alphas[None, :] * res.b_dot_d[:, None]) & \
             (alphas[None, :] < ls.sphere_max_step[:, None]) & (res.b_dot_d > 0)[:, None]
        a = (ok * alphas[None, :]).max(dim=1).values                         # 0 where no step size passes
        x = E.device_pcg.axpy(x, a, res.d)
        e, inv = state(x)
        assert e < e_prev and inv <= inv_prev, (e, e_prev, inv, inv_prev)
        e_prev, inv_prev = e, inv

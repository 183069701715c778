"""The deterministic gradient mode (tsb_options_t.deterministic).

CPU: the plan's vertex -> (tet slot, corner) lists against the tet cells of the stream, the shared plan arrays against
a default plan, and a numpy re-enactment of the store-then-gather sequence against the fp64 oracle.
GPU (marked): parity in every kernel variant, bitwise agreement with the default path where it must hold, bitwise
repeatability (launches, handles, CUDA-graph replays), no state carried between launches, and every entry point."""
import ctypes as C

import numpy as np
import pytest

import _helpers as H
from _helpers import COracle, build_host_plan, emulate_kernel, min_abs_J, mirror_components
from tssplat_b200.mesh import connected_components, make_pack, perturb

CHUNK_ROWS = 256            # tsb_plan.h kDetChunkRows
SHARED = ("stream", "X4", "vlist", "segs", "cta_seg", "wdesc", "wseg", "orphans", "pos16", "pos_gid", "Bt")


def stream_tets(plan):
    """Walk every warp's stream as the kernel does and return, per tet slot (wtc0[s, w] + tc) * TPC + lane * TPL + t,
    the global ids of its four streamed corners (-1 for padding tets) and its 1/det(Dm)."""
    glob = bool(plan["mode_global"])
    TPC = 32 * H.CELL_FORMAT[glob][2]
    wtc0 = plan["wtc0"].reshape(-1, plan["nw"])
    cta_seg = plan["cta_seg"].reshape(-1, 2)
    verts = np.full((plan["n_tetcells"] * TPC, 4), -2, np.int64)
    idet = np.zeros(plan["n_tetcells"] * TPC, np.float32)
    for p, b, s, w, tc in H.walk_streams(plan)[1]:
        idx, d = H.tet_cell(plan, p)
        if not glob:
            h = plan["segs"][s]
            li = s - cta_seg[b, 0]
            xb = h["npos"] if h["whole"] else (li & 1) * 2 * plan["vh"] + plan["vh"]
            idx = plan["pos_gid"][h["p4off"] + idx // 16 - xb].astype(np.int64)
        sl = (int(wtc0[s, w]) + tc) * TPC
        verts[sl:sl + TPC] = np.where((d == 0)[:, None], -1, idx)
        idet[sl:sl + TPC] = d
    assert (verts >= -1).all(), "a tet cell was not visited"
    return verts, idet


def _ragged(seed):
    from test_host_logic import _ragged_mesh
    return _ragged_mesh(np.random.default_rng(seed), 4, 400)


def _noncontiguous():
    pk = make_pack(2, 400, seed=11)
    perm = np.random.default_rng(0).permutation(pk.n)
    verts = np.empty_like(pk.verts)
    verts[perm] = pk.verts
    return verts, perm[pk.tets].astype(np.int32)


def _mesh(name):
    if name == "pack":
        pk = make_pack(3, 768, seed=2)
        return pk.verts, pk.tets
    if name == "a_veg":
        d = np.load(H.os.path.join(H.GOLDEN, "a_veg_mesh.npz"))
        return d["verts"], d["tets"]
    if name == "tiny_components":
        pk = make_pack(2600, 12, seed=3, unique=6)
        return pk.verts, pk.tets
    if name == "noncontiguous":
        return _noncontiguous()
    return _ragged(int(name.split("_")[1]))


STRUCT_CASES = [("pack", dict(nw=16, grid=132)), ("pack", dict(nw=8, grid=5)), ("pack", dict(nw=16, grid=7, force_global=1)),
                ("pack", dict(nw=8, grid=3, vh_cap=100, area_cap=300)), ("a_veg", dict(nw=16, grid=132)),
                ("ragged_3", dict(nw=8, grid=9)), ("ragged_5", dict(nw=16, grid=4, force_global=1)),
                ("tiny_components", dict(nw=16, grid=132)), ("noncontiguous", dict(nw=8, grid=6))]


@pytest.mark.parametrize("mesh,kw", STRUCT_CASES, ids=[f"{m}-" + "-".join(f"{a}{b}" for a, b in k.items()) for m, k in STRUCT_CASES])
@pytest.mark.parametrize("amips", [0, 1])
def test_det_lists_structure(mesh, kw, amips):
    """Every (non-padding streamed tet, corner) is listed exactly once, under the global vertex the stream names; lists
    are ascending; padding and orphans are absent; rows are grouped by component; the default plan is unchanged."""
    V, T = _mesh(mesh)
    plan = build_host_plan(V, T, enable_amips=amips, deterministic=1, **kw)
    ref = build_host_plan(V, T, enable_amips=amips, **kw)
    for k in SHARED:
        if k == "segs":
            assert plan["segs"] == ref["segs"]
        else:
            assert plan[k].tobytes() == ref[k].tobytes(), k
    assert all(plan[k] == ref[k] for k in H._SCALARS)
    if amips:
        assert np.array_equal(plan["wtc0"], ref["wtc0"])
    else:
        assert len(ref["wtc0"]) == 0 and len(plan["wtc0"]) == len(plan["segs"]) * plan["nw"]

    verts, _ = stream_tets(plan)
    n, nele = plan["n"], len(np.asarray(T).reshape(-1, 4))
    rowptr, vert, ent, comp_row = plan["det_rowptr"], plan["det_vert"], plan["det_ent"], plan["det_comp_row"]
    rows = len(vert)
    used = np.unique(np.asarray(T))
    assert rows == len(used) == n - len(plan["orphans"]) and np.array_equal(np.sort(vert), used)
    assert not np.isin(plan["orphans"], vert).any()
    assert rowptr[0] == 0 and np.all(np.diff(rowptr) > 0) and rowptr[-1] == len(ent) == 4 * nele
    slot, corner = ent >> 2, ent & 3
    assert len(np.unique(ent)) == len(ent)
    row_of_ent = np.repeat(np.arange(rows), np.diff(rowptr))
    assert np.array_equal(verts[slot, corner], vert[row_of_ent]), "a list names a corner the stream gives another vertex"
    live = verts[:, 0] >= 0
    assert live.sum() == nele and (verts[live] >= 0).all() and (verts[~live] == -1).all()
    assert live[slot].all(), "padding tets must not be listed"
    assert np.all((np.diff(ent.astype(np.int64)) > 0) | (np.diff(row_of_ent) > 0)), "lists must be ascending"
    # the streamed tets are the mesh's tets (as vertex sets, with multiplicity)
    def rows_sorted(a):
        a = np.sort(np.asarray(a, np.int64).reshape(-1, 4), axis=1)
        return a[np.lexsort(a.T[::-1])]
    assert np.array_equal(rows_sorted(verts[live]), rows_sorted(T))
    # rows grouped by component, vertices ascending inside a component, one component per row range
    assert comp_row[0] == 0 and comp_row[-1] == rows and np.all(np.diff(comp_row) > 0)
    assert len(comp_row) == plan["n_components"] + 1
    lab = connected_components(n, np.asarray(T).reshape(-1, 4))
    for c in range(plan["n_components"]):
        vs = vert[comp_row[c]:comp_row[c + 1]]
        assert np.all(np.diff(vs) > 0) and len(np.unique(lab[vs])) == 1 and (lab[used] == lab[vs[0]]).sum() == len(vs)
    ch = plan["det_chunk"].reshape(-1, 2)
    expect = [(c, r) for c in range(plan["n_components"]) for r in range(comp_row[c], comp_row[c + 1], CHUNK_ROWS)]
    assert [tuple(x) for x in ch.tolist()] == expect


def emulate_det(plan, x, c1, c2, order, gradH=1.0, c3=None):
    """The deterministic sequence re-enacted: operator rows as emulate_kernel walks them, every tet's corner vectors at
    its slot (the kernel's formulas, fp64), then per vertex the active entries of its list summed in list order."""
    TPL = 1 if plan["mode_global"] else 2
    kw = dict(c3=0.0) if c3 is not None else {}
    rows_grad = emulate_kernel(plan, x, c1, 0.0, order, gradH, **kw)[-1]          # c2 = c3 = 0: the rows alone
    verts, idet = stream_tets(plan)
    live = verts[:, 0] >= 0
    xs = np.asarray(x, np.float32).reshape(-1, 3).astype(np.float64)
    q = xs[np.where(live[:, None], verts, 0)]
    e1, e2, e3 = q[:, 1] - q[:, 0], q[:, 2] - q[:, 0], q[:, 3] - q[:, 0]
    c23 = np.cross(e2, e3)
    J = np.einsum("lr,lr->l", e1, c23) * idet
    corners = np.zeros((len(J), 4, 3))
    inv = live & (J < 0)
    m = np.where(inv, -J, 0.0)
    k = (-(order * m ** (order - 1)) * idet * c2 * gradH)[:, None]
    g1, g2, g3 = k * c23, k * np.cross(e3, e1), k * np.cross(e1, e2)
    corners[inv] = np.stack([-(g1 + g2 + g3), g1, g2, g3], axis=1)[inv]
    active = inv.copy()
    if c3 is not None:
        ok = live & (J > 0)
        Bt = plan["Bt"].reshape(-1, 3, 32 * TPL, 4)[..., :3]                        # [cell][row][slot in cell][c]
        B = Bt.transpose(0, 2, 1, 3).reshape(-1, 3, 3)[ok]                          # per slot: rows of Dm^-1
        F = np.stack([e1[ok], e2[ok], e3[ok]], axis=2) @ B
        Jp, tr = J[ok], (F * F).sum(axis=(1, 2))
        j23 = np.cbrt(Jp) ** 2
        cof = np.linalg.det(F)[:, None, None] * np.linalg.inv(F).transpose(0, 2, 1)
        P = (2 / (3 * j23) * c3 * gradH)[:, None, None] * (F - (tr / (3 * Jp))[:, None, None] * cof)
        gk = (P @ B.transpose(0, 2, 1)).transpose(0, 2, 1)                          # [tet][corner k+1][r]
        corners[ok] = np.concatenate([-gk.sum(axis=1, keepdims=True), gk], axis=1)
        active |= ok
    g = rows_grad.copy()
    rowptr, vert, ent = plan["det_rowptr"], plan["det_vert"], plan["det_ent"]
    for r in range(len(vert)):
        e = ent[rowptr[r]:rowptr[r + 1]]
        s, c = e >> 2, e & 3
        a = active[s]
        if a.any():
            g[vert[r]] += corners[s[a], c[a]].sum(axis=0)
    return g


@pytest.mark.parametrize("kw", [dict(nw=16, grid=132), dict(nw=8, grid=5), dict(nw=16, grid=7, force_global=1),
                                dict(nw=8, grid=3, vh_cap=100, area_cap=300)],
                         ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()))
def test_det_reenactment_matches_oracle(kw):
    """Store at the slots, gather in list order: the result is the oracle's gradient (barrier orders 2 and 4 on
    inverted input; AMIPS beside the barrier)."""
    pack = make_pack(3, 768, seed=2)
    plan = build_host_plan(pack.verts, pack.tets, enable_amips=1, deterministic=1, **kw)
    orc = COracle(pack.verts, pack.tets)
    for order in (2, 4):
        x = perturb(pack, sigma_rel=0.35, seed=1)
        g = emulate_det(plan, x, 2e-4, 3e-4, order, gradH=0.7)
        _, terms, go = orc.energy_grad(x, 2e-4, 3e-4, order, gradH=0.7)
        assert terms[1] > 0 and np.linalg.norm(g - go) <= 2e-6 * np.linalg.norm(go)
        assert min_abs_J(pack.verts, pack.tets, x) > 1e-4
        g = emulate_det(plan, x, 2e-4, 3e-4, order, gradH=0.7, c3=1e-4)
        _, terms, go = orc.energy_grad_ex(x, 2e-4, 3e-4, 1e-4, order, gradH=0.7)
        assert terms[2] > 0 and np.linalg.norm(g - go) <= 2e-6 * np.linalg.norm(go)


def test_options_struct_mirrors_header():
    import re
    from tssplat_b200 import _capi
    hdr = open(H.os.path.join(H.ROOT, "include", "tssplat_b200.h")).read()
    body = hdr[hdr.index("typedef struct {\n  int32_t warps_per_cta;"):hdr.index("} tsb_options_t;")]
    assert re.findall(r"int32_t\s+([a-z_0-9]+)", body) == [f for f, _ in _capi.tsb_options_t._fields_]
    assert C.sizeof(_capi.tsb_options_t) == 32


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


def _run(sp, x_np, c=(2e-4 / 3, 2e-4, 0.0), order=2, gradH=0.7, want_grad=True):
    torch = _torch()
    e, g = sp.energy_grad(torch.from_numpy(np.ascontiguousarray(x_np, np.float32)).cuda(), c[0], c[1], order, gradH,
                          want_grad=want_grad, c3=c[2])
    torch.cuda.synchronize()
    return e.clone(), (g.clone() if g is not None else None)


def _amips_input(pack):
    """Every other component mirrored (J near -1: barrier) beside AMIPS components, |J| clear of 0."""
    return mirror_components(perturb(pack, sigma_rel=0.05, seed=0), pack.tets)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", __import__("test_gpu_parity").VARIANTS, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()) or "default")
def test_det_parity(ext, kw):
    """A deterministic handle in every kernel variant against the oracle: benign and inverted inputs, orders 2 and 4,
    AMIPS, and a CUDA gradH tensor."""
    torch = _torch()
    from test_gpu_parity import _check, _check_amips
    pack = make_pack(3, 1024, seed=1)
    for sig, order in ((0.02, 2), (0.35, 2), (0.35, 4)):
        sp, _, g = _check(ext, pack.verts, pack.tets, perturb(pack, sigma_rel=sig, seed=1), 2e-4 / 3, 2e-4, order, gradH=0.7,
                          deterministic=True, **kw)
        assert sp.deterministic
    sp = _handle(ext, pack.verts, pack.tets, deterministic=True, enable_amips=True, **kw)
    x = _amips_input(pack)
    for order in (2, 4):
        _check_amips(sp, pack.verts, pack.tets, x, order)
    xt = torch.from_numpy(perturb(pack, sigma_rel=0.35, seed=1)).cuda()
    e1, g1 = sp.energy_grad(xt, 1e-4, 2e-4, 4, 0.7, c3=1e-4)
    e2, g2 = sp.energy_grad(xt, 1e-4, 2e-4, 4, torch.tensor(0.7, device="cuda"), c3=1e-4)
    torch.cuda.synchronize()
    assert torch.equal(g1, g2) and torch.equal(e1, e2)


@pytest.mark.gpu
def test_det_parity_whole_area_staging(ext):
    from _helpers import whole_area_meshes
    from test_gpu_parity import _check, _check_amips
    for name, (V, T) in whole_area_meshes().items():
        x_amips = perturb(V, T, 0.05, 4)
        if name == "mixed":
            x_amips = mirror_components(x_amips, T)
        for nw in (16, 8):
            for sig, order in ((0.02, 2), (0.35, 4)):
                _check(ext, V, T, perturb(V, T, sig, 4), 2e-4 / 3, 2e-4, order, gradH=0.7, deterministic=True, warps_per_cta=nw)
            sp = _handle(ext, V, T, deterministic=True, enable_amips=True, warps_per_cta=nw)
            _check_amips(sp, V, T, x_amips, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(warps_per_cta=8), dict(force_global=True)],
                         ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()) or "default")
def test_det_bitwise_equal_to_default_where_it_must_be(ext, kw):
    """Same grid; energies bitwise equal; gradient rows no contributing tet touches bitwise equal; the rest to 1e-6."""
    torch = _torch()
    from tssplat_b200.mesh import _signed_volumes
    pack = make_pack(4, 2048, seed=6)
    a = _handle(ext, pack.verts, pack.tets, enable_amips=True, **kw)
    d = _handle(ext, pack.verts, pack.tets, enable_amips=True, deterministic=True, **kw)
    assert a.info["grid"] == d.info["grid"] and a.info["ctas_per_sm"] == d.info["ctas_per_sm"]
    assert d.info["device_bytes"] > a.info["device_bytes"] + 60 * pack.nele
    T = pack.tets.astype(np.int64)
    for x_np, c in ((perturb(pack, sigma_rel=0.35, seed=5), (1e-4, 2e-4, 0.0)), (_amips_input(pack), (1e-4, 2e-4, 1e-4))):
        ea, ga = _run(a, x_np, c)
        ed, gd = _run(d, x_np, c)
        assert torch.equal(ea, ed)
        J = _signed_volumes(x_np.astype(np.float64), T) / _signed_volumes(pack.verts.astype(np.float64), T)
        # every tet that may contribute, with a margin: with AMIPS on, J < 0 (barrier) and J > 0 (AMIPS) both do
        contrib = np.ones(len(T), bool) if c[2] else (J < 1e-3)
        quiet = np.ones(pack.n, bool)
        quiet[np.unique(T[contrib])] = False
        ga, gd = ga.cpu().numpy(), gd.cpu().numpy()
        assert np.array_equal(ga[quiet], gd[quiet]) and (quiet.sum() > 100 or c[2])
        assert np.linalg.norm(gd - ga) <= 1e-6 * np.linalg.norm(ga)


@pytest.mark.gpu
def test_det_repeatable_launches_handles_and_graph_replays(ext):
    torch = _torch()
    pack = make_pack(4, 2048, seed=6)
    x_np = mirror_components(perturb(pack, sigma_rel=0.35, seed=5), pack.tets)       # inverted tets and AMIPS
    kw = dict(enable_amips=True, deterministic=True)
    sp = _handle(ext, pack.verts, pack.tets, **kw)
    c = (1e-4, 2e-4, 1e-4)
    e0, g0 = _run(sp, x_np, c, order=4)
    assert float(e0[2]) > 0 and float(e0[3]) > 0
    for _ in range(10):
        e, g = _run(sp, x_np, c, order=4)
        assert torch.equal(e, e0) and torch.equal(g, g0)
    e, g = _run(_handle(ext, pack.verts, pack.tets, **kw), x_np, c, order=4)
    assert torch.equal(e, e0) and torch.equal(g, g0)
    side = torch.cuda.Stream()                                                        # another stream
    with torch.cuda.stream(side):
        e, g = _run(sp, x_np, c, order=4)
    assert torch.equal(e, e0) and torch.equal(g, g0)
    xs = torch.from_numpy(x_np).cuda()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        eg, gg = sp.energy_grad(xs, *c[:2], 4, 0.7, c3=c[2])
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(eg, e0) and torch.equal(gg, g0)


@pytest.mark.gpu
def test_det_no_stale_state(ext):
    """Inverted -> benign -> energy only -> benign on one handle: each result equals a fresh handle's, bitwise."""
    torch = _torch()
    pack = make_pack(3, 1024, seed=2)
    kw = dict(enable_amips=True, deterministic=True)
    sp = _handle(ext, pack.verts, pack.tets, **kw)
    benign = perturb(pack, sigma_rel=0.02, seed=1)
    for x_np, c3, want in ((perturb(pack, sigma_rel=0.35, seed=1), 0.0, True), (benign, 0.0, True),
                           (perturb(pack, sigma_rel=0.35, seed=2), 1e-4, False), (benign, 0.0, True),
                           (_amips_input(pack), 1e-4, True), (benign, 0.0, True)):
        e, g = _run(sp, x_np, (1e-4, 2e-4, c3), want_grad=want)
        ef, gf = _run(_handle(ext, pack.verts, pack.tets, **kw), x_np, (1e-4, 2e-4, c3), want_grad=want)
        assert torch.equal(e, ef) and (g is None or torch.equal(g, gf))


@pytest.mark.gpu
def test_det_every_entry_point(ext):
    """Host buffers (both internal streams and a stream capture), the autograd surface (Python Function and C++ bridge,
    with `deterministic` in FLAGS) and ShardedEnergy at world size 1 give the device entry point's bits."""
    torch = _torch()
    from tssplat_b200 import energies
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    from tssplat_b200.sharding import ShardedEnergy
    pack = make_pack(3, 1024, seed=5)
    x_np = perturb(pack, sigma_rel=0.35, seed=4)
    sp = _handle(ext, pack.verts, pack.tets, deterministic=True)
    e0, g0 = _run(sp, x_np, (1e-4, 2e-4, 0.0), order=4, gradH=0.5)
    x_host = torch.from_numpy(x_np).pin_memory()
    for _ in range(3):                                        # alternates the two internal streams
        g_host, e_host = torch.empty((pack.n, 3)).pin_memory(), torch.empty(3).pin_memory()
        ext.energy_grad_host(sp, x_host, 1e-4, 2e-4, 4, 0.5, e_host, g_host)
        torch.cuda.synchronize()
        assert torch.equal(e_host, e0[:3].cpu()) and torch.equal(g_host, g0.cpu())
    graph = torch.cuda.CUDAGraph()
    g_host.zero_()
    with torch.cuda.graph(graph):
        ext.energy_grad_host(sp, x_host, 1e-4, 2e-4, 4, 0.5, e_host, g_host)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g_host, g0.cpu())

    flags = dict(smooth_eng_coeff=2e-4 / 3, barrier_coeff=2e-4, increase_order_iter=1000, deterministic=True)
    eng = SmoothnessBarrierEnergy(pack.verts, pack.tets, flags)
    assert eng.tet_sp.deterministic and eng.tet_sp.native_state() is not None
    grads = {}
    for native in (True, False, True):
        energies.use_native_autograd = native
        try:
            x = torch.nn.Parameter(torch.from_numpy(x_np).cuda())
            e = eng(x, 10, 1e-4, 2e-4)
            (3.0 * e).backward()
            torch.cuda.synchronize()
        finally:
            energies.use_native_autograd = True
        if native in grads:
            assert torch.equal(grads[native], x.grad)
        grads[native] = x.grad.clone()
    assert torch.equal(grads[True], grads[False])
    _, _, go = COracle(pack.verts, pack.tets).energy_grad(x_np, 1e-4, 2e-4, 2, gradH=3.0)
    assert np.linalg.norm(grads[True].cpu().numpy() - go) <= 1e-5 * np.linalg.norm(go)

    sh = ShardedEnergy(pack, rank=0, world_size=1, deterministic=True)
    assert sh.tet_sp.deterministic
    e, g = sh.energy_grad(torch.from_numpy(x_np).cuda(), 1e-4, 2e-4, 4, 0.5)
    sh.wait()
    torch.cuda.synchronize()
    assert torch.equal(e, e0[:3]) and torch.equal(g, g0)

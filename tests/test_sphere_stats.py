"""Per-sphere geometry statistics (tsb_energy_grad_spheres, TetSpheres.energy_grad_spheres,
SmoothnessBarrierEnergy.sphere_stats): the plan's per-component tables on the CPU, the records against the fp64 oracle
and against the launch's own totals on the GPU."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest

import _helpers as H
from _helpers import COracle, build_host_plan, min_abs_J, mirror_components
from tssplat_b200.mesh import connected_components, load_veg, make_pack, perturb

REL = 1e-5


# ---- helpers -------------------------------------------------------------------------------------------------------
def _components(n, tets):
    """(vertex ids, tet ids) of every connected component, in order of the lowest vertex id."""
    t = np.asarray(tets).reshape(-1, 4)
    lab = connected_components(n, t)
    used = np.zeros(n, bool)
    used[t.reshape(-1)] = True
    labs = np.unique(lab[used])
    first = {int(c): int(np.flatnonzero((lab == c) & used)[0]) for c in labs}
    order = sorted(labs, key=lambda c: first[int(c)])
    tlab = lab[t[:, 0]]
    return [(np.flatnonzero((lab == c) & used), np.flatnonzero(tlab == c)) for c in order]


def _noncontiguous(num=3, n_tets=400, seed=11, orphans=5):
    """A pack whose vertex ids are shuffled (no component is contiguous), with orphan vertices mixed in."""
    pk = make_pack(num, n_tets, seed=seed)
    n = pk.n + orphans
    perm = np.random.default_rng(0).permutation(n)[:pk.n]
    verts = np.random.default_rng(1).uniform(-1, 1, (n, 3)).astype(np.float32)
    verts[perm] = pk.verts
    return verts, perm[pk.tets].astype(np.int32)


def _a_veg():
    v, t = load_veg(os.path.join(H.GOLDEN, "a_veg_excerpt.veg"))
    return v.astype(np.float32), t.astype(np.int32)


def _tet_cells(plan):
    """(streamed ids [slots, 4], 1/det(Dm) [slots]) of every tet slot of every tet cell, walking each warp's stream."""
    ids, idets = zip(*(H.tet_cell(plan, c[0]) for c in H.walk_streams(plan)[1]))
    return np.concatenate(ids), np.concatenate(idets)


PLAN_CASES = {
    "pack64": lambda: (lambda pk: (pk.verts, pk.tets, {}))(make_pack(64, 256, seed=2, unique=8)),
    "shuffled_orphans": lambda: _noncontiguous() + ({},),
    "large_split": lambda: (lambda pk: (pk.verts, pk.tets, {"grid": 132}))(make_pack(3, 4096, seed=4)),
    "a_veg_global": lambda: _a_veg() + ({"force_global": 1},),
}


# ---- CPU: the plan's per-component tables ------------------------------------------------------------------------
@pytest.mark.parametrize("case", sorted(PLAN_CASES))
def test_component_tables(case):
    verts, tets, kw = PLAN_CASES[case]()
    plan = build_host_plan(verts, tets, **kw)
    comps = _components(len(verts), tets)
    NC, nseg = len(comps), len(plan["segs"])
    assert plan["n_components"] == NC and bool(plan["mode_global"]) == bool(kw.get("force_global"))
    cs = plan["comp_seg"]
    assert len(cs) == NC + 1 and cs[0] == 0 and cs[-1] == nseg
    assert np.all(np.diff(cs) >= 1), "every component has a segment"
    owner = np.repeat(np.arange(NC), np.diff(cs))          # each segment lies in exactly one component range
    assert np.array_equal(owner, [sg["comp"] for sg in plan["segs"]])
    assert np.array_equal(plan["comp_first_vertex"], [v[0] for v, _ in comps])
    assert np.array_equal(plan["comp_ntets"], [len(t) for _, t in comps])
    assert plan["comp_ntets"].sum() == len(np.asarray(tets).reshape(-1, 4))
    if case == "large_split":
        assert np.diff(cs).max() > 10, "the large spheres must be split over many CTAs"


@pytest.mark.parametrize("case", sorted(PLAN_CASES))
def test_padding_tets_have_zero_inverse_volume(case):
    """min_J skips tets whose 1/det(Dm) is 0: exactly the padding slots (four equal vertex entries), never a real tet."""
    verts, tets, kw = PLAN_CASES[case]()
    ids, idet = _tet_cells(build_host_plan(verts, tets, **kw))
    pad = (ids == ids[:, :1]).all(axis=1)
    assert np.count_nonzero(~pad) == len(np.asarray(tets).reshape(-1, 4))
    assert np.all(idet[pad] == 0.0) and np.all(idet[~pad] != 0.0)


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _stats_np(st):
    return {k: getattr(st, k).cpu().numpy() for k in st._fields}


def _oracle_spheres(verts, tets, x, order, c3=0.0):
    """Per component: (first vertex, n_tets, smooth, barrier, amips, n_inverted, min J), fp64 oracle."""
    from tssplat_b200.mesh import _signed_volumes
    out = []
    for vid, tid in _components(len(verts), tets):
        remap = np.full(len(verts), -1, np.int64)
        remap[vid] = np.arange(len(vid))
        t = remap[np.asarray(tets).reshape(-1, 4)[tid]].astype(np.int32)
        _, terms, _ = COracle(verts[vid], t).energy_grad_ex(x[vid], 1.0, 1.0, c3, order, want_grad=False)
        J = _signed_volumes(x[vid].astype(np.float64), t.astype(np.int64)) / _signed_volumes(verts[vid].astype(np.float64), t.astype(np.int64))
        out.append((vid[0], len(tid), terms[0], terms[1], terms[2], int((J < 0).sum()), J.min()))
    return out


def _check_against_oracle(st, verts, tets, x, order, c3=0.0):
    s = _stats_np(st)
    ref = _oracle_spheres(verts, tets, x, order, c3)
    assert len(s["smooth"]) == len(ref)
    for k, (fv, nt, sm, ba, am, ninv, mj) in enumerate(ref):
        assert s["first_vertex"][k] == fv and s["n_tets"][k] == nt
        assert abs(s["smooth"][k] - sm) <= REL * max(abs(sm), 1e-30), (k, s["smooth"][k], sm)
        assert s["barrier"][k] == pytest.approx(ba, rel=REL, abs=1e-30), k
        assert s["amips"][k] == pytest.approx(am, rel=2e-5, abs=1e-30), k
        assert s["n_inverted"][k] == ninv, k
        assert s["min_J"][k] == pytest.approx(mj, rel=1e-5), k


PARITY = [  # (name, mesh, sigma, order, c3, handle options)
    ("benign_o2", "pack", 0.02, 2, 0.0, {}),
    ("inverted_o4", "pack", 0.3, 4, 0.0, {}),
    ("inverted_o2_amips", "pack", 0.3, 2, 1e-4, {"enable_amips": True}),
    ("inverted_8warps", "pack", 0.3, 4, 0.0, {"warps_per_cta": 8}),
    ("inverted_global", "pack", 0.3, 2, 0.0, {"force_global": True}),
    ("noncontiguous", "shuffled", 0.3, 4, 0.0, {}),
    ("deterministic_amips", "pack", 0.3, 2, 1e-4, {"enable_amips": True, "deterministic": True}),
]


def _parity_mesh(kind):
    """Small meshes and seeds whose inverted inputs keep every |J| above 2e-3 (fp32 signs and min J well defined)."""
    if kind == "pack":
        pk = make_pack(4, 256, seed=21)
        return pk.verts, pk.tets, pk
    v, t = _noncontiguous(num=3, n_tets=256)
    return v, t, None


def _x_for(verts, tets, pk, sigma):
    x = perturb(pk, sigma_rel=sigma, seed=30) if pk is not None else perturb(verts, tets, sigma_rel=sigma, seed=1)
    used = np.unique(np.asarray(tets).reshape(-1))
    xx = np.array(verts, dtype=np.float32)
    xx[used] = x[used]
    return xx


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind,sigma,order,c3,opt", PARITY, ids=[p[0] for p in PARITY])
def test_parity_per_sphere(name, kind, sigma, order, c3, opt):
    import torch
    from tssplat_b200 import tet_spheres_ext as ext
    verts, tets, pk = _parity_mesh(kind)
    x_np = _x_for(verts, tets, pk, sigma)
    assert min_abs_J(verts, tets, x_np) > 1e-3, "test input: |J| must stay away from 0"
    sp = ext.TetSpheres(verts.reshape(-1), tets.reshape(-1), **opt)
    x = torch.from_numpy(x_np).cuda()
    e, g, st = sp.energy_grad_spheres(x, 2e-4, 3e-4, order, c3=c3)
    torch.cuda.synchronize()
    _check_against_oracle(st, verts, tets, x_np, order, c3)
    if pk is not None:   # spheres concatenated one after the other: record k is sphere k
        assert np.array_equal(st.first_vertex.cpu().numpy(), pk.vert_offsets[:-1])
        for k in (0, pk.num_spheres - 1):
            sl = pk.slice_spheres(k, k + 1)
            _, terms, _ = COracle(sl.verts, sl.tets).energy_grad_ex(x_np[pk.vert_offsets[k]:pk.vert_offsets[k + 1]], 1, 1, c3, order, want_grad=False)
            assert float(st.barrier[k]) == pytest.approx(terms[1], rel=REL, abs=1e-30)
    if sigma > 0.1:
        assert int(st.n_inverted.sum()) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("opt", [{}, {"warps_per_cta": 8}, {"force_global": True}], ids=["default", "8warps", "global"])
def test_known_answers(opt):
    import torch
    from tssplat_b200 import tet_spheres_ext as ext
    pk = make_pack(6, 512, seed=22)
    sp = ext.TetSpheres(pk.verts.reshape(-1), pk.tets.reshape(-1), **opt)
    nt = np.diff(pk.tet_offsets)
    # rest pose
    _, _, st = sp.energy_grad_spheres(torch.from_numpy(pk.verts.copy()).cuda(), 1.0, 1.0, 2)
    s = _stats_np(st)
    assert np.all(s["smooth"] == 0) and np.all(s["barrier"] == 0) and np.all(s["n_inverted"] == 0)
    assert np.allclose(s["min_J"], 1.0, rtol=1e-5) and np.array_equal(s["n_tets"], nt)
    # every other sphere mirrored: all of its tets at J = -1
    xm = mirror_components(pk.verts, pk.tets)
    mirrored = np.arange(pk.num_spheres) % 2 == 0
    for order in (2, 4):
        _, _, st = sp.energy_grad_spheres(torch.from_numpy(xm).cuda(), 1.0, 1.0, order)
        s = _stats_np(st)
        assert np.array_equal(s["n_inverted"], np.where(mirrored, nt, 0))
        assert np.allclose(s["barrier"], np.where(mirrored, nt, 0), rtol=1e-5, atol=0)
        assert np.allclose(s["min_J"], np.where(mirrored, -1.0, 1.0), rtol=1e-5)
    # a global reflection: the same answer for every sphere
    xr = pk.verts.copy()
    xr[:, 2] = -xr[:, 2]
    for order in (2, 4):
        _, _, st = sp.energy_grad_spheres(torch.from_numpy(xr).cuda(), 1.0, 1.0, order)
        s = _stats_np(st)
        assert np.array_equal(s["n_inverted"], nt) and np.allclose(s["barrier"], nt, rtol=1e-5)
        assert np.allclose(s["min_J"], -1.0, rtol=1e-5)


def _ulp_close(a, b, ulps=1):
    a, b = np.float32(a), np.float32(b)
    return abs(int(a.view(np.int32)) - int(b.view(np.int32))) <= ulps or a == b


@pytest.mark.gpu
@pytest.mark.parametrize("sigma,opt", [(0.02, {}), (0.35, {}), (0.35, {"warps_per_cta": 8, "enable_amips": True}),
                                       (0.35, {"force_global": True})], ids=["benign", "inverted", "8warps_amips", "global"])
def test_consistency_with_totals(sigma, opt):
    import torch
    from tssplat_b200 import tet_spheres_ext as ext
    pk = make_pack(12, 512, seed=23)
    sp = ext.TetSpheres(pk.verts.reshape(-1), pk.tets.reshape(-1), **opt)
    x = torch.from_numpy(perturb(pk, sigma_rel=sigma, seed=2)).cuda()
    c3 = 1e-4 if opt.get("enable_amips") else 0.0
    e, _, st = sp.energy_grad_spheres(x, 2e-4, 3e-4, 4, c3=c3)
    e_def, _ = sp.energy_grad(x, 2e-4, 3e-4, 4, c3=c3 if c3 else 0.0)
    e, e_def = e.cpu().numpy(), e_def.cpu().numpy()
    s = _stats_np(st)
    for k, key in ((1, "smooth"), (2, "barrier"), (3, "amips")):
        assert _ulp_close(s[key].sum(), e[k]), key                                             # the launch's own terms
    for k in range(len(e_def)):
        assert _ulp_close(e[k], e_def[k]), (k, e[k], e_def[k])                                   # the default launch's
    assert int(s["n_tets"].sum()) == pk.nele


@pytest.mark.gpu
def test_gradient_untouched():
    import torch
    from tssplat_b200 import tet_spheres_ext as ext
    pk = make_pack(6, 512, seed=24)
    sp = ext.TetSpheres(pk.verts.reshape(-1), pk.tets.reshape(-1))
    x = torch.from_numpy(perturb(pk, sigma_rel=0.02, seed=1)).cuda()
    assert min_abs_J(pk.verts, pk.tets, x.cpu().numpy()) > 0.05       # benign: no tet inverted, no atomics
    _, g0 = sp.energy_grad(x, 2e-4, 3e-4, 2)
    _, g1, _ = sp.energy_grad_spheres(x, 2e-4, 3e-4, 2)
    assert torch.equal(g0, g1)
    spd = ext.TetSpheres(pk.verts.reshape(-1), pk.tets.reshape(-1), deterministic=True, enable_amips=True)
    for sigma, c3 in ((0.02, 0.0), (0.35, 0.0), (0.35, 1e-4)):
        x = torch.from_numpy(perturb(pk, sigma_rel=sigma, seed=3)).cuda()
        _, g0 = spd.energy_grad(x, 2e-4, 3e-4, 4, c3=c3)
        _, g1, _ = spd.energy_grad_spheres(x, 2e-4, 3e-4, 4, c3=c3)
        assert torch.equal(g0, g1), (sigma, c3)


def _raw_call(sp, x, grad, energy, out, order=4, c3=0.0, stream=None):
    from tssplat_b200 import _capi
    from tssplat_b200.tet_spheres_ext import _stream_ptr
    terms = _capi.tsb_terms_t(c1=2e-4, c2=3e-4, order=order, c3=c3)
    return _capi.lib.tsb_energy_grad_spheres(sp._h, x.data_ptr(), C.byref(terms), 1.0, None, energy.data_ptr(),
                                             grad.data_ptr() if grad is not None else None,
                                             out.data_ptr() if out is not None else None,
                                             stream if stream is not None else _stream_ptr(x.device))


@pytest.mark.gpu
@pytest.mark.parametrize("opt", [{}, {"deterministic": True}, {"force_global": True}], ids=["default", "det", "global"])
def test_repeatable_no_carried_state(opt):
    import torch
    from tssplat_b200 import tet_spheres_ext as ext
    pk = make_pack(8, 512, seed=25)
    sp = ext.TetSpheres(pk.verts.reshape(-1), pk.tets.reshape(-1), **opt)
    S = sp.info["n_components"]
    x = torch.from_numpy(perturb(pk, sigma_rel=0.35, seed=4)).cuda()
    xb = torch.from_numpy(perturb(pk, sigma_rel=0.02, seed=4)).cuda()
    outs = [torch.empty((S, 40), dtype=torch.uint8, device="cuda") for _ in range(3)]
    e = torch.empty(4, device="cuda")
    g = torch.empty_like(x)
    assert _raw_call(sp, x, g, e, outs[0]) == 0
    ref = outs[0].clone()
    e_ref = e.clone()
    for _ in range(3):                                  # repeated launches, interleaved with default launches
        assert _raw_call(sp, x, g, e, outs[1]) == 0
        assert torch.equal(outs[1], ref) and torch.equal(e, e_ref)
        sp.energy_grad(xb, 2e-4, 3e-4, 4)
        sp.energy_grad(x, 2e-4, 3e-4, 4, want_grad=False)
    e_def, g_def = sp.energy_grad(xb, 2e-4, 3e-4, 4)
    assert _raw_call(sp, xb, g, e, outs[1]) == 0
    e_def2, g_def2 = sp.energy_grad(xb, 2e-4, 3e-4, 4)
    assert torch.equal(e_def, e_def2) and torch.equal(g_def, g_def2)
    assert _raw_call(sp, x, None, e, outs[2]) == 0     # no gradient: the same records
    assert torch.equal(outs[2], ref)
    # CUDA-graph replays
    outs[2].zero_()
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st):
        assert _raw_call(sp, x, g, e, outs[2], stream=st.cuda_stream) == 0
    for _ in range(3):
        outs[2].zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(outs[2], ref)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_errors():
    import torch
    from tssplat_b200 import _capi
    from tssplat_b200 import tet_spheres_ext as ext
    pk = make_pack(2, 256, seed=26)
    sp = ext.TetSpheres(pk.verts.reshape(-1), pk.tets.reshape(-1))
    x = torch.from_numpy(pk.verts.copy()).cuda()
    e = torch.empty(4, device="cuda")
    out = torch.empty((2, 40), dtype=torch.uint8, device="cuda")
    assert _raw_call(sp, x, None, e, None) == _capi.TSB_E_INVALID
    assert _raw_call(sp, x, None, e, out, c3=1e-4) == _capi.TSB_E_INVALID       # c3 without enable_amips
    assert _raw_call(sp, x, None, e, out, order=3) == _capi.TSB_E_INVALID
    with pytest.raises(RuntimeError):
        sp.energy_grad_spheres(x, 1.0, 1.0, 2, c3=1e-4)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_python_surface():
    import torch
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    verts, tets, pk = _parity_mesh("pack")
    flags = dict(smooth_eng_coeff=2e-4, barrier_coeff=2e-4, increase_order_iter=100)
    eng = SmoothnessBarrierEnergy(verts, tets, flags)
    x_np = _x_for(verts, tets, pk, 0.3)
    x = torch.nn.Parameter(torch.from_numpy(x_np).cuda())
    for it, order in ((10, 2), (101, 4)):
        st = eng.sphere_stats(x, it)
        c1, c2 = eng.coeff_scheduler(it)
        _, _, st2 = eng.tet_sp.energy_grad_spheres(x.detach(), c1, c2, order, want_grad=False)
        for a, b in zip(st, st2):
            assert torch.equal(a, b)
        assert x.grad is None and eng.tet_sp._cache_grad is None
        _check_against_oracle(st, verts, tets, x_np, order)
    assert st.smooth.dtype == torch.float64 and st.min_J.dtype == torch.float32 and st.n_tets.dtype == torch.int32
    torch.cuda.synchronize()

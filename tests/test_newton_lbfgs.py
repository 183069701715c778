"""The per-sphere L-BFGS step: tsb_newton_lbfgs_step, DeviceNewton.lbfgs_step / minimize(method="lbfgs") and
SmoothnessBarrierEnergy with FLAGS.newton_method = "lbfgs".

CPU: the model's two-loop recursion against the dense compact-form inverse-BFGS matrix (skipped pairs, ring
wraparound); the fp64 model of the step on the small mixed pack (the objective never increases, its change is the
record's, every sphere converges within the pinned step count, stationarity); the record and option structs.
GPU: the step against the public calls composed with the fp64 two-loop; convergence on the mixed 64 x 4096 pack within
the model's count plus a slack; the proximal objective (w = 0 is the plain step bitwise, unusable weights freeze);
determinism, another stream, CUDA graph replays and per-sphere independence; reset; orphans; every refusal; the module
route."""
import ctypes as C
import math

import numpy as np
import pytest

from _lbfgs_model import LBFGS_GPU_SLACK, LBFGS_OPTS, LBFGS_REF_STEPS, History, compact_inverse, lbfgs_reference_run, two_loop
from _newton_model import (ACTIVE, ALPHAS, C3, COEF, MAX_ROUNDING_FLIPS, N_CONVERGED, STALLED, _cuda, _handle,  # noqa: F401
                           _labels, _pack, _records, _shuffled_mesh, _torch, converged_at, dense_sphere_hessians, ext, f32,
                           jacobi_inverse_blocks, reference_problem)
from tssplat_b200.mesh import perturb


# ---------------------------------------------------------------------------------------------------------------------
# CPU


def _block_diag(inv6):
    """Dense block-diagonal matrix from [n, 6] = (xx, yy, zz, yz, xz, xy) blocks."""
    q = np.asarray(inv6, np.float64)
    B = np.zeros((3 * len(q), 3 * len(q)))
    for i, r in enumerate(q):
        B[3 * i:3 * i + 3, 3 * i:3 * i + 3] = [[r[0], r[5], r[4]], [r[5], r[1], r[3]], [r[4], r[3], r[2]]]
    return B


def test_two_loop_equals_compact_form():
    """On a quiet sphere of the small mixed pack, with H0 the kernel's block-Jacobi preconditioner of its Hessian's
    diagonal blocks: 11 pairs (y = H s plus noise) through a ring of m = 4, three of them with s.y < 0 (skipped), so
    the ring wraps twice; after every push the two-loop equals the compact-form matrix times b to 1e-12."""
    P, x0, _, _ = reference_problem()
    H = dense_sphere_hessians(P.orc, P.pk, x0, P.c1, P.c2, 0.0, P.order, False)[1]
    nv = len(H) // 3
    D = np.stack([H[3 * i:3 * i + 3, 3 * i:3 * i + 3] for i in range(nv)])
    H0 = _block_diag(jacobi_inverse_blocks(D, 1e-6))
    rng = np.random.default_rng(3)
    ring = History(4, 1e-8)
    b = rng.normal(size=len(H))
    kept = 0
    for i in range(11):
        s = rng.normal(size=len(H))
        y = -s if i in (2, 6, 7) else H @ s + 1e-3 * np.linalg.norm(H @ s) / np.sqrt(len(H)) * rng.normal(size=len(H))
        kept += ring.push(s, y)
        assert len(ring.pairs) == min(kept, 4)
        d = two_loop(b, ring.pairs, H0)
        ref = compact_inverse(ring.pairs, H0) @ b
        assert np.linalg.norm(d - ref) <= 1e-12 * np.linalg.norm(ref), i
    assert kept == 8


@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_model_on_small_mixed_pack(amips):
    """The fp64 model with the default options: the objective never increases and its change is the record's; every
    shorter step is an Armijo step below the inversion bound; no tet with J > 0 inverts; every sphere (the rough one
    with inverted tets included) is CONVERGED within LBFGS_REF_STEPS, the count the GPU budget derives from, and
    stationary to gtol; pairs are kept, and the ring fills."""
    from oracle.tet_energy_oracle import _det3
    P, x0, o, x, hist = lbfgs_reference_run(amips)
    assert hist[0][0]["inv0"] > 0
    for t, step in enumerate(hist):
        nxt = hist[t + 1] if t + 1 < len(hist) else None
        E1 = P.sphere_energy(x)[0]
        for s, h in enumerate(step):
            after = nxt[s]["E0"] if nxt else E1[s]
            assert after <= h["E0"] + 1e-12 * abs(h["E0"]), (t, s)
            assert abs((after - h["E0"]) - h["delta"]) <= 1e-9 * abs(h["E0"]), (t, s)
            if h["alpha"] > 0:
                assert h["alpha"] < f32(o["eta"]) * h["ahat"] and h["delta"] <= -f32(o["sigma"]) * h["alpha"] * h["bd"], (t, s)
    J0 = _det3((P.orc.G @ x0.reshape(-1)).reshape(-1, 3, 3))
    J = _det3((P.orc.G @ x).reshape(-1, 3, 3))
    assert not ((J0 > 0) & (J <= 0)).any()
    conv = converged_at(hist, P.S)
    kept = sum(h["pair"] == 1 for st in hist for h in st)
    print(f"L-BFGS amips={amips}: converged at {conv}, pairs kept {kept}, rejected {sum(h['pair'] == 0 for st in hist for h in st)}, "
          f"cleared {sum(h['cleared'] for st in hist for h in st)}")
    assert all(c is not None for c in conv) and max(conv) == LBFGS_REF_STEPS[amips], conv
    assert max(h["n_pairs"] for st in hist for h in st) == o["m"] and kept > 0
    g = P.grad(x)
    for s in range(P.S):
        assert np.linalg.norm(g[3 * P.vo[s]:3 * P.vo[s + 1]]) <= o["gtol"] * (1 + 1e-6), s


def test_record_and_option_structs():
    """Both structs are 64 bytes; record_fields reads every scalar field of the record at its offset; the Python
    defaults name exactly the option fields."""
    import torch
    from tssplat_b200 import _capi
    from tssplat_b200.newton import NEWTON_LBFGS_DEFAULTS, NewtonLBFGSStepResult
    R, O = _capi.tsb_newton_lbfgs_sphere_t, _capi.tsb_newton_lbfgs_options_t
    assert C.sizeof(R) == 64 and C.sizeof(O) == 64
    assert set(NEWTON_LBFGS_DEFAULTS) == {k for k, _ in O._fields_} - {"reserved"}
    S = 5
    recs = (R * S)()
    for c in range(S):
        recs[c] = R(grad_norm=1.5 + c, alpha=0.5 ** c, delta=-c - 0.25, b_dot_d=2.0 * c, d_norm=3.0 + c, k=c - 1, status=c % 3,
                    n_pairs=c, pair_kept=c % 3 - 1, history_cleared=c % 2, first_vertex=100 * c)
    raw = torch.from_numpy(np.frombuffer(bytes(recs), dtype=np.uint8).reshape(S, 64).copy())
    f = _capi.record_fields(raw, R)
    assert set(NewtonLBFGSStepResult._fields) <= set(f)
    for name, _ in R._fields_:
        if name != "reserved":
            assert f[name].tolist() == [getattr(recs[c], name) for c in range(S)], name


# ---------------------------------------------------------------------------------------------------------------------
# GPU


def _p_dense(inv, v0, v1):
    return _block_diag(inv[v0:v1].double().cpu().numpy())


@pytest.mark.gpu
def test_step_against_composition(ext):
    """Twelve steps on the small pack (sphere 0 with inverted tets; AMIPS on; m = 3, so the ring wraps) against the
    public calls: the gradient, hess_diag and set_blocks give b and P; the test keeps the fp32 s = x - x_prev and
    y = b_prev - b the device forms (x is the device's after every step) and runs the two-loop in fp64; the line
    search along that direction and the rule give alpha, k and status.  The pair decision and the history length are
    exact; b.d agrees to 1e-4; alpha, k and status agree wherever every Armijo and eta alpha^ margin the rule looked at
    exceeds 1e-3 (relative).  The device's two-loop rounds its vectors to fp32 after every one of its 2m + 1 updates, so
    its d differs from the fp64 one by a few hundred fp32 roundings of d at most: x agrees to 1e-3 alpha max|d| +
    2^-22 max|x| per sphere."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    S, vo = pk.num_spheres, pk.vert_offsets
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    o = dict(LBFGS_OPTS, m=3)
    x = _cuda(x_np)
    ring = [History(o["m"], f32(o["curv_eps"])) for _ in range(S)]
    xp = bp = None
    moved, status = [False] * S, [ACTIVE] * S
    alphas = ALPHAS[:o["n_alpha"]]
    checked = kept = 0
    worst = 0.0
    for t in range(12):
        x0 = x.clone()
        _, b = sp.energy_grad(x0, c1, c2, 2, -1.0, c3=C3)
        inv = nw.pcg.set_blocks(sp.hess_diag(x0, c1, c2, 2, c3=C3), rel_floor=o["rel_floor"], want_inverse=True)
        d = torch.zeros_like(b, dtype=torch.float64)
        pair = [-1] * S
        for s in range(S):
            if status[s] != ACTIVE:
                continue
            sl = slice(vo[s], vo[s + 1])
            bs = b[sl].double().reshape(-1).cpu().numpy()
            if moved[s]:
                pair[s] = int(ring[s].push((x0[sl] - xp[sl]).double().reshape(-1).cpu().numpy(),
                                           (bp[sl] - b[sl]).double().reshape(-1).cpu().numpy()))
            H0 = _p_dense(inv, vo[s], vo[s + 1])
            ds = two_loop(bs, ring[s].pairs, H0)
            if not bs @ ds > 0 and ring[s].pairs:
                ring[s].pairs = []
                ds = H0 @ bs
            d[sl] = torch.from_numpy(ds.reshape(-1, 3)).cuda()
        d32 = d.float().contiguous()
        ls = sp.line_search(x0, d32, alphas, c1, c2, 2, c3=C3, per_sphere=True)
        r = nw.lbfgs_step(x, c1, c2, 2, c3=C3, **o)
        sd, ss = ls.sphere_delta[:, :, 0].cpu().numpy(), ls.sphere_max_step.cpu().numpy()
        ra, rk, rs = r.alpha.cpu().tolist(), r.k.cpu().tolist(), r.status.cpu().tolist()
        assert r.pair_kept.cpu().tolist() == pair, t
        for s in range(S):
            sl = slice(vo[s], vo[s + 1])
            if status[s] != ACTIVE:
                assert ra[s] == 0.0 and torch.equal(x[sl], x0[sl])
                continue
            bd = float((b[sl].double() * d[sl]).sum())
            assert abs(float(r.b_dot_d[s]) - bd) <= 1e-4 * abs(bd), (t, s)
            lim = f32(o["eta"]) * float(ss[s])
            ks, margin = -1, np.inf
            for k, a in enumerate(alphas):
                rhs = -f32(o["sigma"]) * a * bd
                margin = min(margin, abs(a - lim) / lim, abs(sd[s, k] - rhs) / (abs(sd[s, k]) + abs(rhs)))
                if bd > 0 and a < lim and sd[s, k] <= rhs:
                    ks = k
                    break
            if margin > 1e-3:
                checked += 1
                assert (rk[s], ra[s]) == (ks, alphas[ks] if ks >= 0 else 0.0), (t, s)
                exp_status = ACTIVE if ks >= 0 or ring[s].pairs else STALLED
                assert rs[s] == exp_status, (t, s)
                if ks >= 0:
                    dx = (x[sl].double() - (x0[sl].double() + ra[s] * d[sl])).abs().max().item()
                    bound = 1e-3 * ra[s] * d[sl].abs().max().item() + 2.0 ** -22 * x0[sl].abs().max().item()
                    worst = max(worst, dx / bound)
                    assert dx <= bound, (t, s, dx, bound)
        hc = r.history_cleared.cpu().tolist()
        for s in range(S):
            if hc[s]:
                ring[s].pairs = []
            kept += pair[s] == 1
        assert r.n_pairs.cpu().tolist() == [len(q.pairs) for q in ring], t
        moved, status = [a > 0 for a in ra], rs
        xp, bp = x0, b
    print(f"composition: {checked} sphere steps checked, {kept} pairs kept, worst x error {worst:.3f} of the bound")
    assert checked >= 24 and kept >= 12


def _quiet_convergence(ext, amips):
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    pk, x_np = _pack("mixed")
    flags = dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000, amips_coeff=C3 if amips else 0.0,
                 deterministic=True, newton_method="lbfgs")
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    x = torch.nn.Parameter(_cuda(x_np))
    it = 0

    def stats():
        st = E.sphere_stats(x, it)
        c1, c2 = E.coeff_scheduler(it)
        return c1 * st.smooth + c2 * st.barrier + E.amips_coeff * st.amips, st.n_inverted

    e_start, inv_start = stats()
    g0 = E.newton_step(x.detach().clone(), it, n_alpha=1, gtol=3e38).grad_norm       # |g_c| at the start (x untouched)
    E.device_newton.reset()
    quiet = torch.arange(pk.num_spheres, device="cuda") % 4 != 0
    gtol = 1e-3 * g0
    n = math.ceil(LBFGS_REF_STEPS[amips] * (1 + LBFGS_GPU_SLACK))
    acc = torch.zeros(pk.num_spheres, dtype=torch.float64, device="cuda")
    inv_prev, done = inv_start, None
    for t in range(n):
        r = E.newton_step(x, it, gtol=float(gtol[quiet].min()))
        assert (r.delta <= 0).all(), t
        acc += r.delta.double()
        e, inv = stats()
        err = (e - e_start - acc).abs()
        assert (err[quiet] <= 1e-4 * e_start.abs()[quiet]).all(), t
        assert (inv[quiet] <= inv_prev[quiet]).all(), t
        assert int((inv - inv_prev).clamp(min=0).max()) <= MAX_ROUNDING_FLIPS, t
        inv_prev = inv
        if done is None and bool((r.status[quiet] == N_CONVERGED).all()):
            done = t + 1
            break
    print(f"lbfgs amips={amips}: quiet spheres converged after {done} steps (allowed {n}); status {r.status.cpu().tolist()}; "
          f"inverted on the rough spheres {inv_start[~quiet].sum().item()} -> {inv[~quiet].sum().item()}")
    assert done is not None and (r.status[quiet] == N_CONVERGED).all()
    return E, x


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_convergence_mixed_pack_through_module(ext, amips):
    """The mixed 64 x 4096 pack through SmoothnessBarrierEnergy.newton_step with FLAGS.newton_method = "lbfgs": every
    quiet sphere's |g_c| falls by 1e3 (gtol = 1e-3 min |g_c(0)| over them, so each falls by at least that) within
    (1 + LBFGS_GPU_SLACK) times the model's step count; every step's energy change is <= 0 and, on the quiet spheres,
    agrees with a fresh sphere_stats launch; the quiet spheres' inverted-tet counts never grow, and no sphere gains more
    than MAX_ROUNDING_FLIPS in a step."""
    _quiet_convergence(ext, amips)


def _small_setup(ext, **kw):
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True, **kw)
    return pk, sp, DeviceNewton(sp), _cuda(x_np)


@pytest.mark.gpu
def test_proximal_zero_weight_is_plain_and_bad_weights_freeze(ext):
    """With every w_c = 0 ten proximal steps give bitwise the plain steps' x and records; on the shuffled mesh (500
    orphans) a NaN weight (sphere 0) and a negative one (sphere 1) freeze that sphere as STALLED without moving it,
    while sphere 2 steps and orphans stay put."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    pk, sp, nw, x0 = _small_setup(ext)
    c1, c2 = COEF
    y = _cuda(perturb(pk, sigma_rel=0.02, seed=5))
    w = torch.zeros(pk.num_spheres, dtype=torch.float32, device="cuda")
    runs = []
    for prox in (False, True):
        nw.reset()
        x = x0.clone()
        recs = [nw.lbfgs_step(x, c1, c2, 2, c3=C3, anchor=y if prox else None, weight=w if prox else None) for _ in range(10)]
        runs.append((x, _records(torch, recs)))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    V, T, xs_np = _shuffled_mesh()
    sp2 = _handle(ext, V, T, deterministic=True)
    sid_np, orph_np, S = _labels(V, T)
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    nw2 = DeviceNewton(sp2)
    xs0 = _cuda(xs_np)
    x = xs0.clone()
    ya = (xs0 + 0.01 * torch.randn_like(xs0)).contiguous()
    wb = torch.tensor([float("nan"), -1e-3, 1e-3], device="cuda")
    for t in range(6):
        r = nw2.lbfgs_step(x, c1, c2, 2, anchor=ya, weight=wb)
        assert r.status[:2].tolist() == [STALLED, STALLED] and r.alpha[:2].tolist() == [0.0, 0.0]
        assert (r.delta <= 0).all() and not torch.isnan(x).any()
        assert torch.equal(x[orph], xs0[orph])
    frozen = (sid < 2) & ~orph
    assert torch.equal(x[frozen], xs0[frozen]) and not torch.equal(x[(sid == 2) & ~orph], xs0[(sid == 2) & ~orph])


@pytest.mark.gpu
def test_orphans_fixed_and_energy_falls(ext):
    """The shuffled mesh (500 orphans): eight plain steps never move an orphan vertex and lower E on every sphere."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    V, T, x_np = _shuffled_mesh()
    sp = _handle(ext, V, T, deterministic=True)
    _, orph_np, _ = _labels(V, T)
    orph = torch.from_numpy(orph_np).cuda()
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    x0 = _cuda(x_np)
    x = x0.clone()
    e0 = sp.energy_grad_spheres(x0, c1, c2, 2, want_grad=False)[2]
    for _ in range(8):
        r = nw.lbfgs_step(x, c1, c2, 2)
        assert torch.equal(x[orph], x0[orph]) and (r.delta <= 0).all()
    e1 = sp.energy_grad_spheres(x, c1, c2, 2, want_grad=False)[2]
    assert ((c1 * e1.smooth + c2 * e1.barrier) < (c1 * e0.smooth + c2 * e0.barrier)).all()


@pytest.mark.gpu
def test_determinism_graph_and_independence(ext):
    """On the mixed 64 x 4096 pack (AMIPS on, proximal weights 1e-3 .. 1e-1 of the largest diagonal entry): ten steps
    twice and on another stream give bitwise the same x and records, plain and proximal; ten steps captured in one CUDA
    graph replay bitwise, also after new anchor and weight data is copied into the buffers; another start, anchor or
    weight for sphere 4 leaves every other sphere's trajectory bitwise unchanged."""
    torch = _torch()
    from _newton_model import _weights
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("mixed")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    S = pk.num_spheres
    sid = torch.from_numpy(np.repeat(np.arange(S), np.diff(pk.vert_offsets))).cuda()
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    N = 10
    x0 = _cuda(x_np)
    y0 = _cuda(perturb(pk, sigma_rel=0.02, seed=7))
    w0 = _weights(torch, sp.hess_diag(x0, c1, c2, 2, c3=C3), sid, torch.zeros_like(sid, dtype=torch.bool), S, [1e-3, 1e-2, 1e-1])

    def steps(x, y, w):
        return [nw.lbfgs_step(x, c1, c2, 2, c3=C3, anchor=y, weight=w) for _ in range(N)]

    def run(x_start, y=None, w=None):
        nw.reset()
        x = x_start.clone()
        res = steps(x, y, w)
        torch.cuda.synchronize()
        return x, _records(torch, res), res

    for y, w in ((None, None), (y0, w0)):
        xa, ra, res = run(x0, y, w)
        assert int(sum((r.pair_kept == 1).sum() for r in res)) > 0
        xb, rb, _ = run(x0, None if y is None else y.clone(), None if w is None else w.clone())
        assert torch.equal(xa, xb) and torch.equal(ra, rb)
        other = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(other):
            xc, rc, _ = run(x0, y, w)
        torch.cuda.synchronize()
        assert torch.equal(xa, xc) and torch.equal(ra, rc)
    yb, wb = y0.clone(), w0.clone()
    xg = x0.clone()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        nw.lbfgs_step(x0.clone(), c1, c2, 2, c3=C3, anchor=yb, weight=wb)
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        nw.reset()
        rg = _records(torch, steps(xg, yb, wb))
    y1 = _cuda(perturb(pk, sigma_rel=0.03, seed=8))
    w1 = (w0 * torch.linspace(0.5, 2.0, S, device="cuda")).contiguous()
    x1, r1, _ = run(x0, y1, w1)
    assert not torch.equal(x1, xa)
    for yv, wv, xe, re in ((y0, w0, xa, ra), (y1, w1, x1, r1), (y0, w0, xa, ra)):
        yb.copy_(yv)
        wb.copy_(wv)
        xg.copy_(x0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(xg, xe) and torch.equal(rg, re)
    vo, k = pk.vert_offsets, 4
    keep = torch.ones(len(x0), dtype=torch.bool, device="cuda")
    keep[vo[k]:vo[k + 1]] = False
    others = torch.arange(S, device="cuda") != k
    xs0, y2, w2 = x0.clone(), y0.clone(), w0.clone()
    xs0[vo[k]:vo[k + 1]] += 0.01 * torch.randn_like(xs0[vo[k]:vo[k + 1]])
    y2[vo[k]:vo[k + 1]] += 0.01 * torch.randn_like(y2[vo[k]:vo[k + 1]])
    w2[k] *= 3.0
    for xv, yv, wv, yr, wr in ((xs0, None, None, None, None), (x0, y2, w0, y0, w0), (x0, y0, w2, y0, w0)):
        nw.reset()
        xs = xv.clone()
        recs = steps(xs, yv, wv)
        nw.reset()
        xr = x0.clone()
        refs = steps(xr, yr, wr)
        assert torch.equal(xs[keep], xr[keep]) and not torch.equal(xs[~keep], xr[~keep])
        for p, q in zip(recs, refs):
            for f in p._fields:
                assert torch.equal(getattr(p, f)[others], getattr(q, f)[others]), f


@pytest.mark.gpu
def test_reset_equals_fresh_workspace(ext):
    """After five steps and reset, a step gives bitwise the x and record of a fresh workspace's first step; the
    workspace's device bytes follow the header's formula from the first step on."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    pk, sp, nw, x0 = _small_setup(ext)
    c1, c2 = COEF
    before = nw.device_bytes
    x = x0.clone()
    for _ in range(5):
        r = nw.lbfgs_step(x, c1, c2, 2, c3=C3)
    assert int(r.n_pairs.min()) > 0
    m, rows, S = LBFGS_OPTS["m"], len(pk.verts), pk.num_spheres
    assert nw.device_bytes - before == 24 * (m + 2) * rows + 8 * (m + 1) * S + 64 * S
    nw.reset()
    xa = x.clone()
    ra = nw.lbfgs_step(xa, c1, c2, 2, c3=C3)
    fresh = DeviceNewton(sp)
    xb = x.clone()
    rb = fresh.lbfgs_step(xb, c1, c2, 2, c3=C3)
    assert torch.equal(xa, xb) and torch.equal(_records(torch, [ra]), _records(torch, [rb]))
    assert (ra.pair_kept == -1).all() and (ra.n_pairs == 0).all()


@pytest.mark.gpu
def test_refusals(ext):
    """TSB_E_INVALID with nothing launched (x unchanged): options out of range, NaN or with a reserved word set; another
    m than the first call's; one of anchor and weight; anchor == x; c3 without AMIPS; a negative coefficient on a
    projected workspace; an SGS or coarse workspace; the first call under stream capture."""
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DeviceNewton, DevicePCG
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, deterministic=True)
    c1, c2 = COEF
    x = _cuda(x_np)
    nw = DeviceNewton(sp)
    # the first call allocates: refused inside a capture (which survives, allocating nothing), then made outside it
    nw0 = nw.device_bytes
    graph = torch.cuda.CUDAGraph()
    g = x.clone()
    with torch.cuda.graph(graph):
        g.add_(1.0)
        with pytest.raises(RuntimeError, match="capture"):
            nw.lbfgs_step(g, c1, c2, 2)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g, x + 1.0) and nw.device_bytes == nw0
    nw.lbfgs_step(x.clone(), c1, c2, 2)
    x0 = x.clone()
    bad = [dict(m=0), dict(m=17), dict(sigma=0.0), dict(sigma=1.0), dict(sigma=float("nan")), dict(eta=0.0), dict(eta=1.5),
           dict(n_alpha=0), dict(n_alpha=9), dict(rel_floor=-1.0), dict(gtol=float("nan")), dict(curv_eps=-1e-8),
           dict(curv_eps=float("inf")), dict(m=4)]
    for kw in bad:
        with pytest.raises(RuntimeError, match="code -1"):
            nw.lbfgs_step(x, c1, c2, 2, **kw)
    opt = nw.lbfgs_options()
    opt.reserved[3] = 1
    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=0.0)
    stream = nw._stream_ptr(x.device)
    assert _capi.lib.tsb_newton_lbfgs_step(nw._nw, x.data_ptr(), None, None, C.byref(terms), C.byref(opt), None, stream) == -1
    opt.reserved[3] = 0
    w = torch.ones(pk.num_spheres, device="cuda")
    y = x.clone()
    assert _capi.lib.tsb_newton_lbfgs_step(nw._nw, x.data_ptr(), y.data_ptr(), None, C.byref(terms), C.byref(opt), None, stream) == -1
    assert _capi.lib.tsb_newton_lbfgs_step(nw._nw, x.data_ptr(), None, w.data_ptr(), C.byref(terms), C.byref(opt), None, stream) == -1
    assert _capi.lib.tsb_newton_lbfgs_step(nw._nw, x.data_ptr(), x.data_ptr(), w.data_ptr(), C.byref(terms), C.byref(opt), None,
                                           stream) == -1
    assert _capi.lib.tsb_newton_lbfgs_step(nw._nw, x.data_ptr(), None, None, C.byref(terms), None, None, stream) == -1
    for t in (_capi.tsb_terms_t(c1=c1, c2=c2, order=3), _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=1e-4)):
        assert _capi.lib.tsb_newton_lbfgs_step(nw._nw, x.data_ptr(), None, None, C.byref(t), C.byref(opt), None, stream) == -1
    torch.cuda.synchronize()
    assert torch.equal(x, x0)
    nw_psd = DeviceNewton(sp, hessian="psd")
    with pytest.raises(RuntimeError, match="code -1"):
        nw_psd.lbfgs_step(x, -c1, c2, 2)
    for kw in (dict(precond="sgs"), dict(coarse="affine")):
        nwk = DeviceNewton(sp, pcg=DevicePCG(sp, **kw))
        with pytest.raises(RuntimeError, match="block Jacobi"):
            nwk.lbfgs_step(x, c1, c2, 2)
    torch.cuda.synchronize()
    assert torch.equal(x, x0)


@pytest.mark.gpu
def test_prox_step_and_minimize_through_module(ext):
    """SmoothnessBarrierEnergy.prox_step with FLAGS.newton_method = "lbfgs": after five steps the quiet spheres are
    still stepping with pairs in their histories (the rough sphere 0 may stall: where its inversion bound lies below
    eta 2^-7 no step size passes), and a restart re-activates every sphere and empties every history (the first step's
    records have no pair); DeviceNewton.minimize(method="lbfgs") matches lbfgs_step calls bitwise."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    pk, x_np = _pack("small")
    flags = dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000, deterministic=True,
                 newton_method="lbfgs")
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    x = torch.nn.Parameter(_cuda(x_np))
    y = x.detach().clone()
    r = E.prox_step(x, y, 0, 1e-3, n_steps=5)
    assert (r.status[1:] == ACTIVE).all() and (r.n_pairs[1:] > 0).all() and (r.delta <= 0).all()
    r1 = E.prox_step(x, x.detach().clone(), 0, 1e-3, n_steps=1)
    assert (r1.pair_kept == -1).all() and (r1.n_pairs[r1.alpha == 0] == 0).all() and (r1.grad_norm > 0).all()
    nw = E.device_newton
    c1, c2 = E.coeff_scheduler(0)
    xa, xb = x.detach().clone(), x.detach().clone()
    nw.reset()
    n, ra = nw.minimize(xa, 4, c1, c2, 2, method="lbfgs")
    nw.reset()
    for _ in range(4):
        rb = nw.lbfgs_step(xb, c1, c2, 2)
    assert n == 4 and torch.equal(xa, xb) and torch.equal(_records(torch, [ra]), _records(torch, [rb]))

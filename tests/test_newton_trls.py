"""The backtracking trust-region Newton step: tsb_newton_tr_step_ex with a tsb_newton_backtrack_t,
DeviceNewton.trls_step / minimize(method="trls") and SmoothnessBarrierEnergy with FLAGS.newton_method = "trls".

CPU: the trust-region rule with backtracking with known answers (full step, backtracked after a flip or a poor model, no
Armijo step, bd <= 0, STALLED, an unusable weight, the radius clamp).  GPU: bt == NULL is tsb_newton_tr_step bitwise,
and spheres that never backtrack follow the trust-region step's trajectory bitwise; bookkeeping and argument errors;
the module route.  What the backtracking step shares with the other Newton steps (the fp64 reference, plain, AMIPS on
and proximal, which pins the step counts; the step against its composition with every backtracked step's Armijo
decrease and inversion bound; determinism, graph replays and independence; handle variants, orphans and the projected
Hessian; convergence on the mixed 64 x 4096 pack) runs through the shared checks of _newton_checks."""
import ctypes as C

import numpy as np
import pytest

from _newton_checks import (check_composition, check_convergence, check_determinism, check_handle_variants,
                            check_reference)
from _newton_model import (ACTIVE, ALPHAS, BOUNDARY, C3, COEF, N_CONVERGED, STALLED, TRLS_OPTS, _cuda, _handle,  # noqa: F401
                           _pack, _records, _torch, decide_tr, ext, f32)
from tssplat_b200.mesh import perturb


# ---------------------------------------------------------------------------------------------------------------------
# the rule in numpy


# dphi(a) = -a + a^2 / 4 along d with bd = 1, dHd = 1/2 (a quadratic model that is exact): pred = 0.75, rho = 1
_DPHI = [-a + 0.25 * a * a for a in ALPHAS]
_B = dict(g=1.0, bd=1.0, dHd=0.5, dMd=0.64, pcg_status=BOUNDARY, dphi=_DPHI, ahat=np.inf)


def _rule(s, **kw):
    a = dict(_B, o=dict(TRLS_OPTS))
    a.update(kw)
    return decide_tr(s, **a)


def test_trls_rule_known_answers():
    # full step taken: rho = 1 on the boundary, Delta doubles, as the trust-region rule
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s) == (1.0, 1.0, 0.75, _DPHI[0]) and s == dict(radius=2.0, status=ACTIVE)
    # backtracked after a flip: eta alpha^ = 0.9 * 0.2 = 0.18, so 1/8 is the largest 2^-k below it (1/4 is not);
    # Delta = max(|d|_M / 8, Delta / 4) = max(0.1, 0.25), where the trust-region rule would cut it to 0.18 * 0.8 = 0.144
    s = dict(radius=1.0, status=ACTIVE)
    a, rho, pred, delta = _rule(s, ahat=np.float32(0.2))
    assert (a, rho, pred, delta) == (0.125, 1.0, 0.75, _DPHI[3]) and s == dict(radius=0.25, status=ACTIVE)
    s = dict(radius=0.2, status=ACTIVE)                                      # ... and |d|_M alpha when that is larger
    _rule(s, ahat=np.float32(0.2))
    assert s["radius"] == 0.1
    # backtracked after rho <= accept: the full step raises Phi, half of it satisfies Armijo; Delta = max(0.4, 0.25)
    dphi = [0.1, -0.3] + _DPHI[2:]
    s = dict(radius=1.0, status=ACTIVE)
    a, rho, _, delta = _rule(s, dphi=dphi)
    assert a == 0.5 and delta == -0.3 and abs(rho + 0.1 / 0.75) < 1e-15 and s == dict(radius=0.4, status=ACTIVE)
    # pred <= 0 (rho = 0): backtracking still runs on the Armijo test alone
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, dHd=3.0, dphi=dphi)[:3] == (0.5, 0.0, -0.5)
    # no Armijo step: every 2^-k raises Phi, or decreases it by less than sigma alpha bd -> the trust-region rejection
    for dp in ([0.1] * 8, [0.1] + [-f32(1e-4) * a * 0.5 for a in ALPHAS[1:]]):
        s = dict(radius=1.0, status=ACTIVE)
        assert _rule(s, dphi=dp)[0] == 0.0 and abs(s["radius"] - 0.2) < 1e-15 and s["status"] == ACTIVE
    # an Armijo step at 1/2 that is not below eta alpha^ (0.9 * 0.5 = 0.45): the next one, 1/4
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, dphi=dphi, ahat=np.float32(0.5))[0] == 0.25
    # n_alpha = 2 tries 1/2 only
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, ahat=np.float32(0.5), o=dict(TRLS_OPTS, n_alpha=2))[0] == 0.0 and abs(s["radius"] - 0.25) < 1e-15
    # bd <= 0: no backtracking, whatever the changes
    for bd in (0.0, -1.0):
        s = dict(radius=1.0, status=ACTIVE)
        assert _rule(s, bd=bd, dphi=dphi)[0] == 0.0 and abs(s["radius"] - 0.2) < 1e-15
    # STALLED below radius_min when nothing is taken; a backtracked step below it keeps going (and lifts the radius)
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, dphi=[0.1] * 8, o=dict(TRLS_OPTS, radius_min=0.3))[0] == 0.0 and s["status"] == STALLED
    assert _rule(s) == (0.0, 0.0, 0.0, 0.0) and s == dict(radius=0.2, status=STALLED)
    s = dict(radius=0.2, status=ACTIVE)
    assert _rule(s, ahat=np.float32(0.2), o=dict(TRLS_OPTS, radius_min=0.3))[0] == 0.125
    assert s == dict(radius=f32(0.3), status=ACTIVE)
    # the clamp from above: max(alpha |d|_M, Delta / 4) > radius_max
    s = dict(radius=8.0, status=ACTIVE)
    _rule(s, ahat=np.float32(0.2), o=dict(TRLS_OPTS, radius_max=1.5))
    assert s["radius"] == f32(1.5)
    # an unusable weight STALLS; CONVERGED
    for w in (float("nan"), float("inf"), -1.0):
        s = dict(radius=1.0, status=ACTIVE)
        assert _rule(s, w=w) == (0.0, 0.0, 0.0, 0.0) and s == dict(radius=1.0, status=STALLED)
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, g=f32(1e-3), o=dict(TRLS_OPTS, gtol=1e-3)) == (0.0, 0.0, 0.0, 0.0) and s["status"] == N_CONVERGED


# ---------------------------------------------------------------------------------------------------------------------
# GPU


def _raw_tr(torch, capi, nw, x, terms, opt, bt, S, ex=True):
    """tsb_newton_tr_step_ex (ex) or tsb_newton_tr_step on the current stream; the raw [S, 16] records."""
    rec = torch.zeros((S, 16), dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    if ex:
        rc = capi.lib.tsb_newton_tr_step_ex(nw._nw, x.data_ptr(), None, None, C.byref(terms), C.byref(opt),
                                            C.byref(bt) if bt is not None else None, rec.data_ptr(), st)
    else:
        rc = capi.lib.tsb_newton_tr_step(nw._nw, x.data_ptr(), None, None, C.byref(terms), C.byref(opt), rec.data_ptr(), st)
    assert rc == 0, nw._error(nw._nw)
    return rec


def _bits(torch, r, S):
    """[S, k] int32 view of every field of a NewtonTRStepResult."""
    return torch.cat([getattr(r, f).contiguous().view(torch.int32).reshape(S, -1) for f in r._fields], 1)


@pytest.mark.gpu
def test_trls_without_backtracking_is_tr(ext):
    """bt == NULL: tsb_newton_tr_step's x and records bitwise.  On the mixed 64 x 4096 pack, the trust-region and the
    backtracking step side by side, AMIPS off and on: every sphere whose full step was accepted at every step so far
    (or that converged) has a bitwise-identical trajectory and records, so the line search's alpha = 1 change does not
    depend on n_alpha."""
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("mixed")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    S = pk.num_spheres
    sid = torch.from_numpy(np.repeat(np.arange(S), np.diff(pk.vert_offsets))).cuda()
    c1, c2 = COEF
    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=0.0)
    na, nb = DeviceNewton(sp), DeviceNewton(sp)
    opt = na.tr_options(max_iter=10)
    xa, xb = _cuda(x_np), _cuda(x_np)
    for t in range(4):
        ra = _raw_tr(torch, _capi, na, xa, terms, opt, None, S, ex=False)
        rb = _raw_tr(torch, _capi, nb, xb, terms, opt, None, S)
        assert torch.equal(xa, xb) and torch.equal(ra, rb), t
    for c3 in (0.0, C3):
        ntr, nls = DeviceNewton(sp), DeviceNewton(sp)
        x_tr, x_ls = _cuda(x_np), _cuda(x_np)
        same = torch.ones(S, dtype=torch.bool, device="cuda")
        ever = torch.zeros(S, dtype=torch.bool, device="cuda")
        for t in range(12):
            a = ntr.tr_step(x_tr, c1, c2, 2, c3=c3, max_iter=10)
            b = nls.trls_step(x_ls, c1, c2, 2, c3=c3, max_iter=10)
            same &= (a.alpha == 1) | (a.status == N_CONVERGED)
            eq = (_bits(torch, a, S) == _bits(torch, b, S)).all(1)
            assert eq[same].all(), (c3, t)
            moved = torch.zeros(S, device="cuda").index_add_(0, sid, (x_tr != x_ls).any(1).float())
            assert (moved[same] == 0).all(), (c3, t)
            ever |= (b.alpha > 0) & (b.alpha < 1)
        print(f"c3={c3}: spheres on the trust-region trajectory throughout {int(same.sum())} of {S}, "
              f"spheres that backtracked {int(ever.sum())}")
        assert int(same.sum()) > 0 and int(ever.sum()) > 0


@pytest.mark.gpu
def test_trls_bookkeeping_and_argument_errors(ext):
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DeviceNewton, DevicePCG
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    ws = DevicePCG(sp)
    nw, ntr = DeviceNewton(sp, ws), DeviceNewton(sp, DevicePCG(sp))
    S = nw.n_spheres
    nw0 = nw.device_bytes
    c1, c2 = COEF
    x = _cuda(x_np)
    E = _capi.TSB_E_INVALID
    st = torch.cuda.current_stream().cuda_stream
    L = _capi.lib
    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=0.0)
    # the first step allocates: refused inside a capture (which survives), then made outside it
    graph = torch.cuda.CUDAGraph()
    g = x.clone()
    with torch.cuda.graph(graph):
        g.add_(1.0)
        with pytest.raises(RuntimeError, match="capture"):
            nw.trls_step(g, c1, c2, 2)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g, x + 1.0) and nw.device_bytes == nw0
    z = x.clone()
    o = nw.tr_options()
    for bad in (dict(n_alpha=1), dict(n_alpha=0), dict(n_alpha=9), dict(sigma=0.0), dict(sigma=0.5), dict(sigma=-1e-4),
                dict(sigma=float("nan")), dict(reserved=1)):
        bt = _capi.tsb_newton_backtrack_t(n_alpha=bad.get("n_alpha", 8), sigma=bad.get("sigma", 1e-4))
        if "reserved" in bad:
            bt.reserved[5] = 1
        assert L.tsb_newton_tr_step_ex(nw._nw, z.data_ptr(), None, None, C.byref(terms), C.byref(o), C.byref(bt), None, st) == E, bad
    bt = _capi.tsb_newton_backtrack_t(n_alpha=8, sigma=1e-4)
    for bad in (dict(max_iter=0), dict(radius_min=0.0), dict(accept=0.25), dict(eta=1.5)):       # the trust-region options' rules
        ob = nw.tr_options(**bad)
        assert L.tsb_newton_tr_step_ex(nw._nw, z.data_ptr(), None, None, C.byref(terms), C.byref(ob), C.byref(bt), None, st) == E, bad
    ob = nw.tr_options()
    ob.reserved[6] = 1
    assert L.tsb_newton_tr_step_ex(nw._nw, z.data_ptr(), None, None, C.byref(terms), C.byref(ob), C.byref(bt), None, st) == E
    y, w = x.clone(), torch.full((S,), 1e-3, device="cuda")
    for args in ((None, z.data_ptr(), None, None, C.byref(terms), C.byref(o)),
                 (nw._nw, None, None, None, C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), y.data_ptr(), None, C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), z.data_ptr(), w.data_ptr(), C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), None, None, C.byref(terms), None),
                 (nw._nw, z.data_ptr(), None, None, C.byref(_capi.tsb_terms_t(c1=c1, c2=c2, order=3)), C.byref(o))):
        assert L.tsb_newton_tr_step_ex(*args, C.byref(bt), None, st) == E
    with pytest.raises(TypeError):
        nw.trls_options(tau=1.0)
    with pytest.raises(TypeError):
        nw.tr_options(sigma=1e-4)
    with pytest.raises(ValueError):
        nw.minimize(z, 1, c1, c2, 2, method="cg")
    torch.cuda.synchronize()
    assert torch.equal(z, x) and nw.device_bytes == nw0
    # after the first step: exactly the trust-region step's device memory
    nw.trls_step(z, c1, c2, 2)
    ntr.tr_step(x.clone(), c1, c2, 2)
    assert nw.device_bytes == ntr.device_bytes > nw0
    nw.trls_step(z.clone(), c1, c2, 2, anchor=y, weight=w)
    ntr.tr_step(x.clone(), c1, c2, 2, anchor=y, weight=w)
    assert nw.device_bytes == ntr.device_bytes
    # later calls can be captured: a graph of one step replays the eager step bitwise
    nw.reset()
    xe = x.clone()
    re = _records(torch, [nw.trls_step(xe, c1, c2, 2, n_alpha=4)])
    xg = x.clone()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        nw.reset()
        rg = _records(torch, [nw.trls_step(xg, c1, c2, 2, n_alpha=4)])
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(xg, xe) and torch.equal(rg, re)


@pytest.mark.gpu
def test_module_trls_route(ext):
    """FLAGS.newton_method = "trls" routes newton_step and prox_step to the backtracking trust-region step."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    from tssplat_b200.newton import DeviceNewton, NewtonTRStepResult
    pk, x_np = _pack("small")
    flags = dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000, deterministic=True)
    it = 5
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, dict(flags, newton_method="trls"))
    xa = torch.nn.Parameter(_cuda(x_np))
    ra = E.newton_step(xa, it)
    E2 = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    nw = DeviceNewton(E2.tet_sp)
    c1, c2 = E2.coeff_scheduler(it)
    z = _cuda(x_np)
    rz = nw.trls_step(z, c1, c2, E2.order_at(it))
    assert isinstance(ra, NewtonTRStepResult) and torch.equal(z, xa.detach()) and torch.equal(ra.radius, rz.radius)
    y = _cuda(perturb(pk, sigma_rel=0.01, seed=5))
    r = E.prox_step(xa, y, it, 1e-2, n_steps=3, max_iter=15)
    assert isinstance(r, NewtonTRStepResult) and (r.alpha > 0).any()
    nw.reset()
    n, r2 = nw.minimize(z, 3, c1, c2, E2.order_at(it), anchor=y, weight=1e-2, method="trls", max_iter=15)
    assert n == 3 and torch.equal(z, xa.detach()) and torch.equal(r2.radius, r.radius)
    with pytest.raises(TypeError):
        E.newton_step(xa, it, tau=1.0)


# ---------------------------------------------------------------------------------------------------------------------
# the checks every Newton step shares (_newton_checks)


@pytest.mark.parametrize("kind", ["plain", "amips", "small", "large"])
def test_trls_reference_mixed_pack(kind):
    check_reference("trls", kind)


@pytest.mark.gpu
@pytest.mark.parametrize("prox", [False, True], ids=["plain", "prox"])
def test_trls_step_equals_its_composition(ext, prox):
    check_composition(ext, "trls", C3, prox)


@pytest.mark.gpu
def test_trls_determinism_graphs_and_independence(ext):
    check_determinism(ext, "trls")


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["w8", "global", "psd"])
def test_trls_handle_variants_and_orphans(ext, variant):
    check_handle_variants(ext, "trls", variant)


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_trls_convergence_mixed_pack(ext, amips):
    check_convergence(ext, "trls", amips)

"""compute-sanitizer target: one or two launches of every kernel variant and helper.
Usage: compute-sanitizer --tool memcheck|racecheck|synccheck python tools/sanitize_target.py [small|big]"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tssplat_b200 import tet_spheres_ext as ext  # noqa: E402
from tssplat_b200.mesh import make_pack, perturb, surface_vf  # noqa: E402
from tssplat_b200.optimizer import AdamUniform  # noqa: E402
from tssplat_b200.surface import SurfaceNormals  # noqa: E402

big = len(sys.argv) > 1 and sys.argv[1] == "big"
cases = [(3, 1024, {}), (3, 1024, {"warps_per_cta": 8}), (2, 1500, {"force_global": True}),
         (2, 1024, {"warps_per_cta": 8, "force_global": True}), (3, 1024, {"enable_amips": True})]
if big:      # persistent CTAs with several segments each: double-buffered staging, register prefetch, ring wrap-around
    cases += [(400, 4096, {}), (400, 4096, {"warps_per_cta": 8})]
for S, T, kw in cases:
    pack = make_pack(S, T, seed=3, unique=4)
    sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), **kw)
    for sig, order in ((0.02, 2), (0.35, 4)):
        x = torch.from_numpy(perturb(pack, sigma_rel=sig, seed=1)).cuda()
        e, g = sp.energy_grad(x, 2e-4, 3e-4, order, 0.7, c3=(1e-4 if kw.get("enable_amips") else 0.0))
        e2, _ = sp.energy_grad(x, 2e-4, 3e-4, order, 0.7, want_grad=False)
        torch.cuda.synchronize()
        print(S, T, kw, sig, order, "segments", sp.info["n_segments"], "E", float(e[0]), float(e2[0]), flush=True)
    if not big:
        xh = torch.from_numpy(perturb(pack, sigma_rel=0.02, seed=2)).pin_memory()
        gh, eh = torch.empty((pack.n, 3)).pin_memory(), torch.empty(3).pin_memory()
        for _ in range(3):
            ext.energy_grad_host(sp, xh, 2e-4, 3e-4, 2, 1.0, eh, gh)
        torch.cuda.synchronize()
if not big:
    pack = make_pack(2, 1024, seed=5)
    p = torch.nn.Parameter(torch.from_numpy(perturb(pack, sigma_rel=0.1, seed=1)).cuda())
    opt = AdamUniform([p], grad_limit=True, grad_limit_values=[0.01, 0.01], grad_limit_iters=[2], lr=0.1)
    for _ in range(3):
        p.grad = torch.randn_like(p)
        ext.grad_limit(p.grad, 0.5, 0.25)
        opt.step()
    sv, sf = surface_vf(pack.tets)
    sn = SurfaceNormals(sv, sf, pack.n, device="cuda")
    tv = p.detach().clone().requires_grad_(True)
    v_pos, v_nrm = sn(tv)
    (v_pos.sum() + (v_nrm * v_nrm).sum()).backward()
    torch.cuda.synchronize()
    print("helpers ok", float(tv.grad.abs().sum()))
    from tssplat_b200.mesh import surface_vf_gpu
    sv2, sf2 = surface_vf_gpu(pack.tets, pack.n)
    assert np.array_equal(sv, sv2) and np.array_equal(sf, sf2)
    print("surface extraction ok", len(sv2), len(sf2))
    # one proximal Newton step runs the whole Newton stack: gradient, diagonal blocks, the shifted block-Jacobi PCG,
    # the line search, the step's own kernels and the axpy, first in their proximal variants (one sphere with a NaN
    # weight), then the plain ones
    from tssplat_b200.newton import DeviceNewton
    pack = make_pack(3, 1024, seed=3, unique=4)
    sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), enable_amips=True, deterministic=True)
    nw = DeviceNewton(sp)
    x = torch.from_numpy(perturb(pack, sigma_rel=0.35, seed=1)).cuda()
    y = x.clone()
    w = torch.tensor([1e-3, 1.0, float("nan")], device="cuda")
    r = nw.step(x, 2e-4, 3e-4, 2, c3=1e-4, anchor=y, weight=w, max_iter=5)
    torch.cuda.synchronize()
    print("prox step ok", r.status.tolist(), r.alpha.tolist())
    nw.reset()                                         # and the plain step's kernels
    r = nw.step(x, 2e-4, 3e-4, 2, c3=1e-4, max_iter=5)
    torch.cuda.synchronize()
    print("newton step ok", r.status.tolist(), r.alpha.tolist())
    # one trust-region step, proximal then plain: the radius kernels, the trust-region solve's update and direction
    # kernels (shifted, then unshifted) and the decision kernels
    nw.reset()
    r = nw.tr_step(x, 2e-4, 3e-4, 2, c3=1e-4, anchor=y, weight=w, max_iter=5)
    torch.cuda.synchronize()
    print("prox tr step ok", r.status.tolist(), r.alpha.tolist(), r.pcg_status.tolist())
    r = nw.tr_step(x, 2e-4, 3e-4, 2, c3=1e-4, max_iter=5)
    torch.cuda.synchronize()
    print("tr step ok", r.status.tolist(), r.alpha.tolist(), r.pcg_status.tolist())
print("DONE")

"""Cost of one Newton-CG iteration, three ways on the SAME handle, timed in one process with CUDA events, alternating:
  hvp         bare tsb_hvp_ex (a CUDA graph of `--iters` launches),
  device pcg  tsb_pcg_solve with check_every = 0 and max_iter = `--iters`, preconditioner set, as a CUDA graph replay
              (the time includes the solve's two start-up kernels, amortised over the iterations),
  torch pcg   tssplat_b200.newton.pcg with rtol = 0 (it reads three scalars to the host per iteration, so it cannot be
              captured; its time is divided by the products it actually used, fewer than `--iters` when it stops at
              negative curvature).
The median over `--rounds` is reported in us per iteration.  Rows: 64 x 4096 and 1024 x 4096, benign (0.02 h) and
inverted (0.35 h), AMIPS off and on (c3 = 1e-4), on a deterministic handle (the gather follows every product).  In the
device solve a sphere that stops (negative curvature on the inverted rows) idles for the remaining iterations.

Then, on a 64 x 4096 pack in which every fourth sphere is perturbed at 0.35 h and the rest at 0.02 h: the products the
global newton.pcg needs to reach rtol against the per-sphere maximum and mean of the device solve.

Usage: python tools/time_pcg.py [--rounds 10] [--iters 20] [--out DIR]"""
import argparse
import ctypes as C
import json

import numpy as np
import torch

from _timing import TETS, capture, card, mixed_pack, p10_p90, timed, write_json
from tssplat_b200 import _capi
from tssplat_b200 import tet_spheres_ext as ext
from tssplat_b200.mesh import make_pack, perturb
from tssplat_b200.newton import DevicePCG, hess_blocks, pcg

CASES = [("64x4096 benign (0.02 h)", 64, 0.02), ("64x4096 inverted (0.35 h)", 64, 0.35),
         ("1024x4096 benign (0.02 h)", 1024, 0.02), ("1024x4096 inverted (0.35 h)", 1024, 0.35)]
C3 = 1e-4


def torch_blocks(ws, planes):
    """Sets the workspace's preconditioner and returns the same inverse blocks as [n, 3, 3] for newton.pcg, so that both
    solvers precondition identically (newton.block_jacobi's batched torch.linalg.eigh does not get through packs of
    this size reliably)."""
    q = ws.set_blocks(planes, want_inverse=True)
    return hess_blocks(torch.stack([q[:, :3], q[:, 3:]]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None, help="directory for time_pcg.json")
    args = ap.parse_args()
    dev = card()
    print(f"device: {dev}", flush=True)
    results = []
    K = args.iters
    for name, S, sig in CASES:
        pack = make_pack(S, TETS, seed=0, unique=8)
        x = torch.from_numpy(perturb(pack, sigma_rel=sig, seed=0)).cuda()
        c1, c2 = 2e-4 / S, 2e-4
        sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), enable_amips=True, deterministic=True)
        ws = DevicePCG(sp)
        d, hv = torch.empty_like(x), torch.empty_like(x)
        s = torch.cuda.Stream()
        for c3 in (0.0, C3):
            terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=c3)
            opt = _capi.tsb_pcg_options_t(max_iter=K, rtol=0.0, check_every=0)
            _, g = sp.energy_grad(x, c1, c2, 2, c3=c3)
            b = -g
            planes = sp.hess_diag(x, c1, c2, 2, c3=c3)
            P = torch_blocks(ws, planes)
            torch.cuda.synchronize()

            def hvp():
                return _capi.lib.tsb_hvp_ex(sp._h, x.data_ptr(), b.data_ptr(), C.byref(terms), 1.0, None, hv.data_ptr(), None,
                                            s.cuda_stream)

            def solve():
                return _capi.lib.tsb_pcg_solve(ws._s, x.data_ptr(), b.data_ptr(), C.byref(terms), C.byref(opt), d.data_ptr(),
                                               None, None, s.cuda_stream)

            g_hvp, g_solve = capture(hvp, s, K, 2 * K, "hvp"), capture(solve, s, 1, 2, "solve")
            torch_pcg = lambda: pcg(lambda p: sp.hvp(x, p, c1, c2, 2, c3=c3)[0], b, P, max_iter=K, rtol=0.0)
            torch_pcg()
            t = {"hvp": [], "device_pcg": [], "torch_pcg": []}
            for _ in range(args.rounds):                                  # alternating
                t["hvp"].append(timed(g_hvp.replay)[0] / K)
                t["device_pcg"].append(timed(g_solve.replay)[0] / K)
                us, ref = timed(torch_pcg)
                t["torch_pcg"].append(us / ref.n_hvp)
            r = {"case": name, "spheres": S, "sigma_rel": sig, "amips_c3": c3, "iters": K, "torch_pcg_products": ref.n_hvp,
                 "us_per_iteration": {k: float(np.median(v)) for k, v in t.items()},
                 "us_per_iteration_p10_p90": {k: p10_p90(v) for k, v in t.items()},
                 "workspace_bytes": ws.device_bytes, "device": dev}
            u = r["us_per_iteration"]
            print(f"{name:28s} c3={c3:<6g} hvp {u['hvp']:8.2f}  device pcg {u['device_pcg']:8.2f}  torch pcg {u['torch_pcg']:9.2f} "
                  f"us/iteration ({ref.n_hvp} torch products)", flush=True)
            results.append(r)
            del g_hvp, g_solve
        del ws, sp
        torch.cuda.empty_cache()

    # products to reach rtol: one Krylov space over all spheres against one per sphere
    S, rtol = 64, 1e-3
    pack, x_np, quiet = mixed_pack(S, 0, 0, 4)
    x = torch.from_numpy(x_np).cuda()
    c1, c2 = 2e-4 / S, 2e-4
    sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), enable_amips=True, deterministic=True)
    ws = DevicePCG(sp)
    for c3 in (0.0, C3):
        _, g = sp.energy_grad(x, c1, c2, 2, c3=c3)
        planes = sp.hess_diag(x, c1, c2, 2, c3=c3)
        ref = pcg(lambda p: sp.hvp(x, p, c1, c2, 2, c3=c3)[0], -g, torch_blocks(ws, planes), max_iter=2000, rtol=rtol)
        res = ws.solve(x, -g, c1, c2, 2, c3=c3, max_iter=2000, rtol=rtol, check_every=25)
        st, nh, rel = res.status.cpu().numpy(), res.n_hvp.cpu().numpy(), res.rel_residual.cpu().numpy()
        mixed = {"case": f"64x4096 mixed (every 4th sphere 0.35 h, rest 0.02 h), c3={c3:g}, rtol={rtol:g}",
                 "torch_pcg": {"products": ref.n_hvp, "converged": ref.converged, "negative_curvature": ref.negative_curvature,
                               "rel_residual": ref.rel_residual},
                 "device_pcg": {"iters_run": res.iters_run,
                                "status_counts": {n: int((st == k).sum()) for k, n in
                                                  enumerate(("maxiter", "converged", "negcurv", "negcurv_first", "zero_rhs"))},
                                "n_hvp_max": int(nh.max()), "n_hvp_mean": float(nh.mean()),
                                "quiet_spheres": int(quiet.sum()), "quiet_converged": int((st[quiet] == 1).sum()),
                                "quiet_n_hvp_max": int(nh[quiet].max()), "quiet_n_hvp_mean": float(nh[quiet].mean()),
                                "quiet_rel_residual_median": float(np.median(rel[quiet])),
                                "quiet_rel_residual_max": float(rel[quiet].max())},
                 "device": dev}
        print(json.dumps(mixed, indent=1), flush=True)
        results.append(mixed)
    write_json(args.out, "time_pcg.json", results)


if __name__ == "__main__":
    main()

"""Cost of one damped Newton step (tsb_newton_step) and its time to solution, timed with CUDA events in one process.

Step cost: a CUDA-graph replay of one step and of 10 steps, us per step, on 64 x 4096 and 1024 x 4096 packs (benign,
0.02 h), AMIPS off and on (c3 = 1e-4), max_iter 10 and 20, on a deterministic handle; and the same step split into its
public calls, each a CUDA-graph replay of its own: gradient (tsb_energy_grad_ex), diagonal (tsb_hess_diag), blocks
(tsb_pcg_set_blocks_ex), solve (tsb_pcg_solve_ex), line search (tsb_line_search) and axpy (tsb_sphere_axpy).  The step's
own small kernels (frozen-sphere mask and mu, b.d and |d|^2, decision) are the remainder: step minus the sum of the
phases.  Rounds alternate the arms; the median over `--rounds` is reported.

Time to solution on the mixed 64 x 4096 pack (every fourth sphere at 0.35 h, the rest at 0.02 h; c1 = 2e-4 / 64,
c2 = 2e-4): steps and summed step time until every quiet sphere's |g_c| has fallen by 1e3, for
  damped      DeviceNewton.step (gtol = 1e-3 times the smallest starting |g_c| of the quiet spheres),
  undamped    the INTEGRATION.md composition: newton_direction (max_iter 20, rtol 1e-2) plus a per-sphere Armijo
              choice from line_search(per_sphere=True) and DevicePCG.axpy,
  adam        tssplat_b200.optimizer.AdamUniform (lr 1e-3) on the geometry energy alone,
each up to `--max-steps` steps (Adam: `--adam-steps`), alternating the arms over `--tts-rounds` rounds.  The per-sphere
gradient norms between steps are not timed.

Usage: python tools/time_newton.py [--rounds 10] [--out DIR]"""
import argparse
import ctypes as C
import json

import numpy as np
import torch

from _timing import (TETS, alternate, capture, card, mixed_pack, p10_p90, sphere_gnorm, sphere_ids, steps_until, timed,
                     write_json)
from tssplat_b200 import _capi
from tssplat_b200 import tet_spheres_ext as ext
from tssplat_b200.mesh import make_pack, perturb
from tssplat_b200.newton import DeviceNewton
from tssplat_b200.optimizer import AdamUniform

C3 = 1e-4
ALPHAS = [2.0 ** -k for k in range(8)]


def step_cost(S, args, dev, results):
    pack = make_pack(S, TETS, seed=0, unique=8)
    x0 = torch.from_numpy(perturb(pack, sigma_rel=0.02, seed=0)).cuda()
    c1, c2 = 2e-4 / S, 2e-4
    sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), enable_amips=True, deterministic=True)
    nw = DeviceNewton(sp)
    ws = nw.pcg
    s = torch.cuda.Stream()
    x = x0.clone()
    b, d = torch.empty_like(x), torch.empty_like(x)
    planes = torch.empty((2, sp.n, 3), device="cuda")
    energy = torch.empty(4, device="cuda")
    shift = torch.full((ws.n_spheres,), 1e-3, device="cuda")
    alphas = torch.tensor(ALPHAS, device="cuda")
    aS = torch.full((ws.n_spheres,), 0.5, device="cuda")
    delta, sdelta, sstep = (torch.empty(n, device="cuda") for n in (32, ws.n_spheres * 32, ws.n_spheres))
    xo = torch.empty_like(x)
    for c3 in (0.0, C3):
        terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=c3)
        for K in (10, 20):
            opts = dict(max_iter=K, rtol=1e-2)
            nwo = nw.options(**opts)
            popt = _capi.tsb_pcg_options_t(max_iter=K, rtol=1e-2, check_every=0)
            st = s.cuda_stream
            L = _capi.lib

            def step():
                return L.tsb_newton_step(nw._nw, x.data_ptr(), C.byref(terms), C.byref(nwo), None, st)

            phases = {
                "gradient": lambda: L.tsb_energy_grad_ex(sp._h, x.data_ptr(), C.byref(terms), -1.0, None, energy.data_ptr(),
                                                         b.data_ptr(), st),
                "diagonal": lambda: L.tsb_hess_diag(sp._h, x.data_ptr(), C.byref(terms), 1.0, None, planes.data_ptr(), st),
                "blocks": lambda: L.tsb_pcg_set_blocks_ex(ws._s, planes.data_ptr(), 1e-6, shift.data_ptr(), None, st),
                "solve": lambda: L.tsb_pcg_solve_ex(ws._s, x.data_ptr(), b.data_ptr(), C.byref(terms), C.byref(popt),
                                                    shift.data_ptr(), d.data_ptr(), None, None, st),
                "line_search": lambda: L.tsb_line_search(sp._h, x.data_ptr(), d.data_ptr(), C.byref(terms), alphas.data_ptr(), 8,
                                                         delta.data_ptr(), None, sdelta.data_ptr(), sstep.data_ptr(), st),
                "axpy": lambda: L.tsb_sphere_axpy(ws._s, x.data_ptr(), aS.data_ptr(), d.data_ptr(), xo.data_ptr(), st),
            }
            nw.reset()
            graphs = {"step": capture(step, s, 1, 2, "step"), "10 steps": capture(step, s, 10, 20, "10 steps")}
            graphs.update({k: capture(f, s, 1, 2, k) for k, f in phases.items()})
            # alternating; x restarts from the same point every round
            t = alternate(graphs, args.rounds, before=lambda k: (x.copy_(x0), nw.reset()))
            del graphs
            t["10 steps"] = [us / 10 for us in t["10 steps"]]
            med = {k: float(np.median(v)) for k, v in t.items()}
            med["small kernels (step - phases)"] = med["step"] - sum(med[k] for k in phases)
            r = {"case": f"{S}x{TETS} benign (0.02 h)", "amips_c3": c3, "max_iter": K, "us": med,
                 "us_p10_p90": {k: p10_p90(v) for k, v in t.items()},
                 "newton_workspace_bytes": nw.device_bytes, "device": dev}
            print(f"{r['case']:26s} c3={c3:<6g} max_iter={K:<3d} " + "  ".join(f"{k} {v:.1f}" for k, v in med.items()), flush=True)
            results.append(r)
    del nw, ws, sp
    torch.cuda.empty_cache()


def time_to_solution(args, dev, results):
    S = 64
    pack, x_np, quiet = mixed_pack(S, 0, 0, 4)
    x0 = torch.from_numpy(x_np).cuda()
    c1, c2 = 2e-4 / S, 2e-4
    sid = sphere_ids(pack).cuda()
    quiet = torch.from_numpy(quiet).cuda()
    alphas = torch.tensor(ALPHAS, device="cuda")
    for c3 in (0.0, C3):
        sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), enable_amips=True, deterministic=True)
        nw = DeviceNewton(sp)
        g0 = sphere_gnorm(sp, x0, c1, c2, c3, sid, S)
        target = g0 / 1e3
        gtol = float(g0[quiet].min()) * 1e-3

        def damped(x):
            nw.step(x, c1, c2, 2, c3=c3, gtol=gtol)

        def undamped(x):
            b = -sp.energy_grad(x, c1, c2, 2, c3=c3)[1]
            nw.pcg.set_blocks(sp.hess_diag(x, c1, c2, 2, c3=c3))
            res = nw.pcg.solve(x, b, c1, c2, 2, c3=c3, max_iter=20, rtol=1e-2)
            ls = sp.line_search(x, res.d, alphas, c1, c2, 2, c3=c3, per_sphere=True)
            ok = (ls.sphere_delta[:, :, 0] <= -1e-4 * alphas[None, :] * res.b_dot_d[:, None]) & \
                 (alphas[None, :] < ls.sphere_max_step[:, None]) & (res.b_dot_d > 0)[:, None]
            nw.pcg.axpy(x, (ok * alphas[None, :]).max(dim=1).values, res.d, out=x)

        arms = {"damped": (damped, args.max_steps), "undamped": (undamped, args.max_steps)}
        out = {k: [] for k in arms}
        out["adam"] = []
        for _ in range(args.tts_rounds):
            for name, (fn, n_max) in arms.items():
                x = x0.clone()
                nw.reset()
                steps, total, done = steps_until(lambda: fn(x), lambda: bool(
                    (sphere_gnorm(sp, x, c1, c2, c3, sid, S)[quiet] <= target[quiet]).all()), n_max)
                out[name].append((steps if done else None, total))
            p = torch.nn.Parameter(x0.clone())
            opt = AdamUniform([p], lr=1e-3)
            total, steps, done = 0.0, 0, False
            best = None
            for steps in range(1, args.adam_steps + 1):
                def adam():
                    p.grad = sp.energy_grad(p.data, c1, c2, 2, c3=c3)[1]
                    opt.step()
                total += timed(adam)[0]
                if steps % 50 == 0 or steps == args.adam_steps:
                    ratio = sphere_gnorm(sp, p.data, c1, c2, c3, sid, S)[quiet] / g0[quiet]
                    best = float(ratio.max())
                    if best <= 1e-3:
                        done = True
                        break
            out["adam"].append((steps if done else None, total, best))
        r = {"case": f"64x{TETS} mixed, c3={c3:g}, |g_c| of every quiet sphere down by 1e3", "device": dev,
             "arms": {k: {"steps": v[0][0], "ms_median": float(np.median([q[1] for q in v])) / 1e3,
                          **({"worst_quiet_ratio_at_end": v[-1][2]} if k == "adam" else {})} for k, v in out.items()}}
        print(json.dumps(r, indent=1), flush=True)
        results.append(r)
        del nw, sp
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--tts-rounds", type=int, default=2)
    ap.add_argument("--max-steps", type=int, default=60)
    ap.add_argument("--adam-steps", type=int, default=2000)
    ap.add_argument("--sizes", default="64,1024")
    ap.add_argument("--out", default=None, help="directory for time_newton.json")
    args = ap.parse_args()
    dev = card()
    print(f"device: {dev}", flush=True)
    results = []
    for S in (int(v) for v in args.sizes.split(",")):
        step_cost(S, args, dev, results)
    time_to_solution(args, dev, results)
    write_json(args.out, "time_newton.json", results)


if __name__ == "__main__":
    main()

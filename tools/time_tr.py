"""Cost and time to solution of the trust-region Newton step (tsb_newton_tr_step) against the damped (LM) step
tsb_newton_step, and against LM over the projected Hessian, timed with CUDA events in one process.

Step cost: one CUDA graph per arm holding (copy the start into x, reset, one step), on 64 x 4096 and 1024 x 4096 packs
(benign, every sphere at 0.02 h; c1 = 2e-4 / S, c2 = 2e-4, order 2), AMIPS off and on (c3 = 1e-4), max_iter 10 and 20,
on a deterministic handle -- the setup of DESIGN.md section 5's step-cost table.  Arms lm10, lm20, tr10, tr20; rounds
alternate the arms, each round one replay; median, min and max over `--rounds` rounds, in us per step.  One eager step per
arm also reports its solve: mean products per sphere and the spheres per PCG status.  The SM clock (nvidia-smi clocks.sm)
is read while about half a second of the tr20 arm's replays is queued.

Time to solution: the mixed 64 x 4096 pack of tools/time_psd.py (every fourth sphere at 0.35 h, with inverted tets; the
rest at 0.02 h; c1 = 2e-4 / 64, c2 = 2e-4, AMIPS off and on), arms "lm" (DeviceNewton.step), "psd" (the same over the
projected Hessian) and "tr" (DeviceNewton.tr_step), gtol = 1e-3 times the smallest starting |g_c| of the quiet spheres:
steps and summed CUDA-event step time until every quiet sphere's |g_c| has fallen by 1e3 (the criterion of
time_newton.py's table), and until every sphere's has; and after `--steps` steps (always run in full) the worst rough
sphere's |g_c| / |g_c,0| and the per-sphere statuses.  `--tts-rounds` rounds alternating the arms, median time.  The
gradient norms between steps are not timed.  Also, for the first solve on that pack, the spheres per PCG status of the
exact solve and of the trust-region solve at the step's initial radius.

Usage: python tools/time_tr.py [--rounds 7] [--steps 40] [--tts-rounds 2] [--out DIR]"""
import argparse
import json

import numpy as np
import torch

from _timing import (TETS, alternate, capture, card, mixed_pack, sm_clock_under_load, sphere_gnorm, sphere_ids, summary,
                     timed, write_json)
from tssplat_b200 import tet_spheres_ext as ext
from tssplat_b200.mesh import make_pack, perturb
from tssplat_b200.newton import DeviceNewton

C3 = 1e-4


def step_cost(args, results):
    for S in (64, 1024):
        pk = make_pack(S, TETS, seed=0, unique=8)
        x0 = torch.from_numpy(perturb(pk, sigma_rel=0.02, seed=0)).cuda()
        sp = ext.TetSpheres(pk.verts.reshape(-1), pk.tets.reshape(-1), enable_amips=True, deterministic=True)
        nw = DeviceNewton(sp)
        c1, c2 = 2e-4 / S, 2e-4
        for c3 in (0.0, C3):
            xs = {k: x0.clone() for k in ("lm10", "lm20", "tr10", "tr20")}

            def arm(key):
                it = int(key[2:])

                def f():
                    xs[key].copy_(x0)
                    nw.reset()
                    if key.startswith("tr"):
                        nw.tr_step(xs[key], c1, c2, 2, c3=c3, max_iter=it)
                    else:
                        nw.step(xs[key], c1, c2, 2, c3=c3, max_iter=it)
                return f

            s = torch.cuda.Stream()
            fns = {k: arm(k) for k in xs}
            t = alternate({k: capture(f, s, 1, 3, k) for k, f in fns.items()}, args.rounds)
            t = {k: summary(v) for k, v in t.items()}
            solves = {}
            for k in ("lm20", "tr20"):
                x = x0.clone()
                nw.reset()
                r = (nw.tr_step if k.startswith("tr") else nw.step)(x, c1, c2, 2, c3=c3, max_iter=20)
                solves[k] = dict(mean_hvp=float(r.n_hvp.float().mean()), status=torch.bincount(r.pcg_status, minlength=7).tolist(),
                                 accepted=int((r.alpha > 0).sum()))
            g = capture(fns["tr20"], s, 1, 1)
            mhz = sm_clock_under_load(g, t["tr20"]["median"])
            del g
            r = dict(S=S, c3=c3, times_us=t, solves=solves, sm_mhz_under_load=mhz,
                     tr_over_lm={k: t["tr" + k]["median"] / t["lm" + k]["median"] for k in ("10", "20")})
            print(f"{S} x {TETS} c3={c3}: " + ", ".join(f"{k} {v['median']:.1f} us" for k, v in t.items()) +
                  f"; solves {solves}; SM clock {mhz} MHz", flush=True)
            results.append(r)
        del nw, sp
        torch.cuda.empty_cache()


def time_to_solution(args, dev, results):
    S = 64
    pack, x_np, quiet = mixed_pack(S, 0, 0, 4)
    x0 = torch.from_numpy(x_np).cuda()
    c1, c2 = 2e-4 / S, 2e-4
    sid = sphere_ids(pack).cuda()
    quiet = torch.from_numpy(quiet).cuda()
    for c3 in (0.0, C3):
        sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), enable_amips=True, deterministic=True)
        arms = {"lm": DeviceNewton(sp), "psd": DeviceNewton(sp, hessian="psd"), "tr": None}
        arms["tr"] = DeviceNewton(sp, arms["lm"].pcg)
        g0 = sphere_gnorm(sp, x0, c1, c2, c3, sid, S)
        target, gtol = g0 / 1e3, float(g0[quiet].min()) * 1e-3
        # the first solve: exact (max_iter 20, as the steps) against the trust-region solve at the step's first radius
        x = x0.clone()
        arms["tr"].reset()
        r0 = arms["tr"].tr_step(x, c1, c2, 2, c3=c3, gtol=gtol)
        x = x0.clone()
        arms["lm"].reset()
        l0 = arms["lm"].step(x, c1, c2, 2, c3=c3, gtol=gtol)
        first = dict(lm_status=torch.bincount(l0.pcg_status, minlength=7).tolist(), tr_status=torch.bincount(r0.pcg_status, minlength=7).tolist(),
                     lm_mean_hvp_quiet=float(l0.n_hvp[quiet].float().mean()), tr_mean_hvp_quiet=float(r0.n_hvp[quiet].float().mean()))
        out = {k: [] for k in arms}
        for _ in range(args.tts_rounds):
            for name, nw in arms.items():
                x = x0.clone()
                nw.reset()
                total, t_quiet, n_quiet, n_all, t_all = 0.0, None, None, None, None
                for step in range(1, args.steps + 1):
                    run = nw.tr_step if name == "tr" else nw.step
                    dt, last = timed(lambda: run(x, c1, c2, 2, c3=c3, gtol=gtol))
                    total += dt
                    ok = sphere_gnorm(sp, x, c1, c2, c3, sid, S) <= target
                    if n_quiet is None and bool(ok[quiet].all()):
                        n_quiet, t_quiet = step, total
                    if n_all is None and bool(ok.all()):
                        n_all, t_all = step, total
                ratio = sphere_gnorm(sp, x, c1, c2, c3, sid, S) / g0
                out[name].append((n_quiet, t_quiet, n_all, t_all, float(ratio[~quiet].max()),
                                  torch.bincount(last.status, minlength=3).tolist()))

        def med(v, i):
            q = [e[i] for e in v if e[i] is not None]
            return float(np.median(q)) / 1e3 if len(q) == len(v) else None

        r = {"case": f"64x{TETS} mixed, c3={c3:g}, time to |g_c| / 1e3, {args.steps} steps", "device": dev, "first_solve": first,
             "arms": {k: {"steps_quiet": v[0][0], "ms_quiet_median": med(v, 1), "steps_all": v[0][2], "ms_all_median": med(v, 3),
                          "worst_rough_ratio": v[0][4], "status_counts_active_converged_stalled": v[0][5]} for k, v in out.items()}}
        print(json.dumps(r, indent=1), flush=True)
        results.append(r)
        del arms, sp
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--tts-rounds", type=int, default=2)
    ap.add_argument("--no-cost", action="store_true", help="only time to solution")
    ap.add_argument("--no-tts", action="store_true", help="only the step cost")
    ap.add_argument("--out", default=None, help="directory for time_tr.json")
    args = ap.parse_args()
    dev = card()
    print(f"device: {dev}", flush=True)
    results = []
    if not args.no_cost:
        step_cost(args, results)
    if not args.no_tts:
        time_to_solution(args, dev, results)
    write_json(args.out, "time_tr.json", dict(device=dev, results=results))


if __name__ == "__main__":
    main()

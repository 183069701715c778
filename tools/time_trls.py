"""Cost and time to solution of the backtracking trust-region Newton step (tsb_newton_tr_step_ex with a
tsb_newton_backtrack_t, DeviceNewton.trls_step) against the trust-region step tsb_newton_tr_step, and the damped (LM)
step, timed with CUDA events in one process.

Step cost: the setup of tools/time_tr.py -- one CUDA graph per arm holding (copy the start into x, reset, one step), on
64 x 4096 and 1024 x 4096 packs (benign, every sphere at 0.02 h; c1 = 2e-4 / S, c2 = 2e-4, order 2), AMIPS off and on
(c3 = 1e-4), max_iter 10 and 20, on a deterministic handle.  Arms tr10, tr20, trls10, trls20; rounds alternate the
arms, each round one replay; median, min and max over `--rounds` rounds, in us per step.  The line search on its own:
one graph per arm of tsb_line_search with per-sphere outputs along the first trust-region direction, at 8 step sizes
(2^-k) and at 1 (alpha = 1), as the two steps call it.  The SM clock (nvidia-smi clocks.sm) is read while about half a
second of the trls20 arm's replays is queued.

Time to solution: the mixed 64 x 4096 pack of tools/time_tr.py (every fourth sphere at 0.35 h, with inverted tets; the
rest at 0.02 h; c1 = 2e-4 / 64, c2 = 2e-4, AMIPS off and on), arms "lm", "tr" and "trls", gtol = 1e-3 times the smallest
starting |g_c| of the quiet spheres: steps and summed CUDA-event step time until every quiet sphere's |g_c| has fallen by
1e3, and until every sphere's has; after `--steps` steps (always run in full) the worst rough sphere's |g_c| / |g_c,0|,
the per-sphere statuses, and how many of the rough spheres' steps were backtracked (0 < alpha < 1; LM: k > 0).
`--tts-rounds` rounds alternating the arms, median time.  The gradient norms between steps are not timed.

Usage: python tools/time_trls.py [--rounds 7] [--steps 40] [--tts-rounds 2] [--out DIR]"""
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
            xs = {k: x0.clone() for k in ("tr10", "tr20", "trls10", "trls20")}

            def arm(key):
                it = int(key.lstrip("trls"))
                run = nw.trls_step if key.startswith("trls") else nw.tr_step

                def f():
                    xs[key].copy_(x0)
                    nw.reset()
                    run(xs[key], c1, c2, 2, c3=c3, max_iter=it)
                return f

            s = torch.cuda.Stream()
            fns = {k: arm(k) for k in xs}
            t = alternate({k: capture(f, s, 1, 3, k) for k, f in fns.items()}, args.rounds)
            t = {k: summary(v) for k, v in t.items()}
            # the line search alone along the first trust-region direction, at 8 sizes and at 1
            d = torch.zeros_like(x0)
            nw.reset()
            xd = x0.clone()
            nw.tr_step(xd, c1, c2, 2, c3=c3, max_iter=20)
            d.copy_(xd - x0)
            a8 = torch.tensor([2.0 ** -k for k in range(8)], device="cuda")
            a1 = a8[:1].clone()

            def ls(alphas):
                def f():
                    sp.line_search(x0, d, alphas, c1, c2, 2, c3=c3, per_sphere=True)
                return f
            tl = alternate({k: capture(ls(a), s, 20, 3, k) for k, a in (("ls8", a8), ("ls1", a1))}, args.rounds, calls=20)
            tl = {k: summary(v) for k, v in tl.items()}
            g = capture(fns["trls20"], s, 1, 1)
            mhz = sm_clock_under_load(g, t["trls20"]["median"])
            del g
            r = dict(S=S, c3=c3, times_us=t, line_search_us=tl, sm_mhz_under_load=mhz,
                     trls_over_tr={k: t["trls" + k]["median"] / t["tr" + k]["median"] for k in ("10", "20")})
            print(f"{S} x {TETS} c3={c3}: " + ", ".join(f"{k} {v['median']:.1f} us" for k, v in {**t, **tl}.items()) +
                  f"; SM clock {mhz} MHz", flush=True)
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
        lm = DeviceNewton(sp)
        arms = {"lm": (lm, lm.step), "tr": None, "trls": None}
        tr = DeviceNewton(sp, lm.pcg)
        trls = DeviceNewton(sp, lm.pcg)
        arms["tr"], arms["trls"] = (tr, tr.tr_step), (trls, trls.trls_step)
        g0 = sphere_gnorm(sp, x0, c1, c2, c3, sid, S)
        target, gtol = g0 / 1e3, float(g0[quiet].min()) * 1e-3
        out = {k: [] for k in arms}
        for _ in range(args.tts_rounds):
            for name, (nw, run) in arms.items():
                x = x0.clone()
                nw.reset()
                total, t_quiet, n_quiet, n_all, t_all = 0.0, None, None, None, None
                back = torch.zeros(S, dtype=torch.int64, device="cuda")
                for step in range(1, args.steps + 1):
                    dt, last = timed(lambda: run(x, c1, c2, 2, c3=c3, gtol=gtol))
                    total += dt
                    back += ((last.k > 0) if name == "lm" else (last.alpha > 0) & (last.alpha < 1)).long()
                    ok = sphere_gnorm(sp, x, c1, c2, c3, sid, S) <= target
                    if n_quiet is None and bool(ok[quiet].all()):
                        n_quiet, t_quiet = step, total
                    if n_all is None and bool(ok.all()):
                        n_all, t_all = step, total
                ratio = sphere_gnorm(sp, x, c1, c2, c3, sid, S) / g0
                out[name].append((n_quiet, t_quiet, n_all, t_all, float(ratio[~quiet].max()),
                                  torch.bincount(last.status, minlength=3).tolist(), int(back[~quiet].sum()),
                                  float(ratio[~quiet].median())))

        def med(v, i):
            q = [e[i] for e in v if e[i] is not None]
            return float(np.median(q)) / 1e3 if len(q) == len(v) else None

        r = {"case": f"64x{TETS} mixed, c3={c3:g}, time to |g_c| / 1e3, {args.steps} steps", "device": dev,
             "arms": {k: {"steps_quiet": v[0][0], "ms_quiet_median": med(v, 1), "steps_all": v[0][2], "ms_all_median": med(v, 3),
                          "worst_rough_ratio": v[0][4], "median_rough_ratio": v[0][7],
                          "status_counts_active_converged_stalled": v[0][5], "rough_backtracked_steps": v[0][6]}
                      for k, v in out.items()}}
        print(json.dumps(r, indent=1), flush=True)
        results.append(r)
        del arms, lm, tr, trls, sp
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--tts-rounds", type=int, default=2)
    ap.add_argument("--no-cost", action="store_true", help="only time to solution")
    ap.add_argument("--no-tts", action="store_true", help="only the step cost")
    ap.add_argument("--out", default=None, help="directory for time_trls.json")
    args = ap.parse_args()
    dev = card()
    print(f"device: {dev}", flush=True)
    results = []
    if not args.no_cost:
        step_cost(args, results)
    if not args.no_tts:
        time_to_solution(args, dev, results)
    write_json(args.out, "time_trls.json", dict(device=dev, results=results))


if __name__ == "__main__":
    main()

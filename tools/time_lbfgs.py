"""The L-BFGS step (DeviceNewton.lbfgs_step) against the damped Newton step (DeviceNewton.step), timed with CUDA events in
one process.

Packs: "mixed" (every fourth sphere at 0.35 h, the rest at 0.02 h) of 64 x 4096 and 1024 x 4096 tets; c1 = 2e-4 / S,
c2 = 2e-4, order 2, AMIPS off and on (c3 = 1e-4); a deterministic handle; every step at its defaults
(NEWTON_LBFGS_DEFAULTS: m = 8; NEWTON_DEFAULTS: max_iter = 20).  Per pack and AMIPS setting, the two arms alternating
round by round (median, min and max over the rounds):
  step      us per step: one captured step replayed, on a workspace that has taken 10 steps (a full L-BFGS history)
  step/10   us per step of 10 captured steps (reset, then 10 steps from the start)
Time to solution (64 x 4096 mixed, AMIPS off and on): steps and summed step time (CUDA events per step) until every
quiet sphere's |g_c| has fallen by 1e3 (DESIGN.md's criterion), up to --max-steps.  The card, its power limit and its SM
clocks (maximum and current, read after the timed work) are read in the same process.

Usage: python tools/time_lbfgs.py [--rounds 5] [--max-steps 400] [--out DIR]"""
import argparse
import json

import torch

from _timing import alternate, capture, card, mixed_pack, sphere_gnorm, sphere_ids, steps_until, summary, write_json
from tssplat_b200 import tet_spheres_ext as ext
from tssplat_b200.newton import DeviceNewton

C3 = 1e-4
ARMS = {"lm": "step", "lbfgs": "lbfgs_step"}


def run_pack(S, amips, args):
    pk, x_np, quiet = mixed_pack(S, 1, 3, 4)
    sp = ext.TetSpheres(pk.verts.reshape(-1), pk.tets.reshape(-1), enable_amips=True, deterministic=True)
    c1, c2, c3 = 2e-4 / S, 2e-4, (C3 if amips else 0.0)
    x0 = torch.from_numpy(x_np).cuda()
    one, ten = {}, {}
    for arm, fn in ARMS.items():
        nw = DeviceNewton(sp)
        xs, xt = x0.clone(), x0.clone()
        for _ in range(10):
            getattr(nw, fn)(xs, c1, c2, 2, c3=c3)
        one[arm] = lambda nw=nw, xs=xs, fn=fn: getattr(nw, fn)(xs, c1, c2, 2, c3=c3)
        nw10 = DeviceNewton(sp, pcg=nw.pcg)

        def tens(nw=nw10, xt=xt, fn=fn):
            xt.copy_(x0)
            nw.reset()
            for _ in range(10):
                getattr(nw, fn)(xt, c1, c2, 2, c3=c3)
        ten[arm] = tens
    # each arm captured once (after one warm-up call: every first call's allocations), replayed once untimed, then 20
    # replays between two events per round, arms alternating within every round
    res = {}
    for key, fns, steps in (("step_us", one, 1), ("step_of_10_us", ten, 10)):
        s = torch.cuda.Stream()
        torch.cuda.synchronize()
        graphs = {k: capture(fn, s, 1, 1, k) for k, fn in fns.items()}
        res[key] = {k: summary(v) for k, v in alternate(graphs, args.rounds, reps=20, calls=steps, warmup=1).items()}
        del graphs
    return res, (sp, pk, x0, quiet, c1, c2, c3)


def time_to_solution(ctx, args):
    sp, pk, x0, quiet, c1, c2, c3 = ctx
    S = pk.num_spheres
    sid = sphere_ids(pk).cuda()
    q = torch.from_numpy(quiet).cuda()
    out = {}
    for arm, fn in ARMS.items():
        nw = DeviceNewton(sp)
        x = x0.clone()
        g0 = sphere_gnorm(sp, x, c1, c2, c3, sid, S)
        k, total, reached = steps_until(lambda: getattr(nw, fn)(x, c1, c2, 2, c3=c3), lambda: bool(
            (sphere_gnorm(sp, x, c1, c2, c3, sid, S)[q] <= 1e-3 * g0[q]).all()), args.max_steps)
        out[arm] = dict(steps=k, ms=total / 1e3, reached=reached)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--max-steps", type=int, default=400)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_lbfgs.py needs a CUDA device")
    result = {"packs": {}, "time_to_solution_64x4096": {}}
    for S in (64, 1024):
        for amips in (False, True):
            r, ctx = run_pack(S, amips, args)
            key = f"{S}x4096/amips={'on' if amips else 'off'}"
            result["packs"][key] = r
            print(json.dumps({key: r}), flush=True)
            if S == 64:
                t = time_to_solution(ctx, args)
                result["time_to_solution_64x4096"][f"amips={'on' if amips else 'off'}"] = t
                print(json.dumps({f"time to solution {key}": t}), flush=True)
    result["card"] = card("name,power.limit,clocks.max.sm,clocks.sm")
    print(json.dumps({"card": result["card"]}), flush=True)
    write_json(args.out, "time_lbfgs.json", result)


if __name__ == "__main__":
    main()

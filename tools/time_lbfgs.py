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
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from time_sgs import pack_x, sphere_gnorm  # noqa: E402
from tssplat_b200 import tet_spheres_ext as ext  # noqa: E402
from tssplat_b200.newton import DeviceNewton  # noqa: E402

C3 = 1e-4
ARMS = {"lm": "step", "lbfgs": "lbfgs_step"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def graph_us(fns, steps, rounds, reps=20):
    """{arm: median, min, max over rounds of us per step}: each arm's fn captured once in a CUDA graph, the graphs
    replayed reps times between two events, arms alternating within every round."""
    s = torch.cuda.Stream()
    graphs = {}
    torch.cuda.synchronize()
    for k, fn in fns.items():
        with torch.cuda.stream(s):
            fn()                                         # warm-up (and every first call's allocations) outside the capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            fn()
        graphs[k] = g
    for g in graphs.values():
        g.replay()
    torch.cuda.synchronize()
    out = {k: [] for k in fns}
    for _ in range(rounds):
        for k, g in graphs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                g.replay()
            b.record()
            b.synchronize()
            out[k].append(1e3 * a.elapsed_time(b) / (reps * steps))
    return {k: dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v))) for k, v in out.items()}


def run_pack(S, amips, args):
    pk, x_np, quiet = pack_x(S, "mixed")
    sp = ext.TetSpheres(pk.verts.astype(np.float32).reshape(-1), pk.tets.astype(np.int32).reshape(-1),
                        enable_amips=True, deterministic=True)
    c1, c2, c3 = 2e-4 / S, 2e-4, (C3 if amips else 0.0)
    x0 = torch.from_numpy(x_np.astype(np.float32)).cuda()
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
    return {"step_us": graph_us(one, 1, args.rounds), "step_of_10_us": graph_us(ten, 10, args.rounds)}, (sp, pk, x0, quiet, c1, c2, c3)


def time_to_solution(ctx, args):
    sp, pk, x0, quiet, c1, c2, c3 = ctx
    S = pk.num_spheres
    sid = torch.from_numpy(np.repeat(np.arange(S), np.diff(pk.vert_offsets))).cuda()
    keep = torch.ones(len(sid), dtype=torch.bool, device="cuda")
    q = torch.from_numpy(quiet).cuda()
    out = {}
    for arm, fn in ARMS.items():
        nw = DeviceNewton(sp)
        x = x0.clone()
        g0 = sphere_gnorm(sp, x, c1, c2, c3, sid, keep, S)
        total, k, reached = 0.0, 0, False
        while k < args.max_steps and not reached:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            getattr(nw, fn)(x, c1, c2, 2, c3=c3)
            b.record()
            b.synchronize()
            total += 1e3 * a.elapsed_time(b)
            k += 1
            reached = bool((sphere_gnorm(sp, x, c1, c2, c3, sid, keep, S)[q] <= 1e-3 * g0[q]).all())
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
    result["card"] = card()
    print(json.dumps({"card": result["card"]}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_lbfgs.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()

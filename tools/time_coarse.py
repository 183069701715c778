"""Affine coarse space (DevicePCG(coarse="affine")) against block Jacobi alone, timed with CUDA events in one process.

Packs: "mixed" (every fourth sphere at 0.35 h, the rest at 0.02 h) of 64 x 4096 and (--big) 1024 x 4096 tets; c1 = 2e-4 /
S, c2 = 2e-4, order 2, AMIPS off and on (c3 = 1e-4); a deterministic handle.  Per pack and AMIPS setting, Jacobi and
coarse alternating round by round (median, min and max µs over the rounds):
  products     mean Hessian-vector products to rtol = 1e-3 over the quiet spheres (max_iter 400): LM shift mu_c = 1e-3
               max (D_v)_ii (exact model) and unshifted PSD
  solve        us per tsb_pcg_solve with the LM shift at the steps' defaults (max_iter 20, rtol 1e-2, check_every 0)
  set_coarse   us per tsb_pcg_set_coarse (exact and PSD)
  step         us per DeviceNewton step (lm, psd) at the defaults, from the same x each time
Time to solution (64 x 4096 mixed, AMIPS on): steps and summed step time until every
quiet sphere's |g_c| has fallen by 1e3 (the criterion of DESIGN.md's LM and PSD tables), up to `--max-steps`.  The
card, its power limit and maximum SM clock are read in the same process.

Usage: python tools/time_coarse.py [--rounds 5] [--big] [--max-steps 60] [--out DIR]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from time_hvp import card  # noqa: E402
from time_sgs import pack_x, sphere_gnorm  # noqa: E402
from tssplat_b200 import tet_spheres_ext as ext  # noqa: E402
from tssplat_b200.newton import DeviceNewton, DevicePCG  # noqa: E402

C3 = 1e-4
METHODS = {"lm": ("exact", "step"), "psd": ("psd", "step")}   # the trust-region steps refuse a coarse workspace


def event_us(fns, rounds, reps=5):
    """{name: median, min, max over rounds of us per call}: every round times each fn in turn, reps calls between two
    CUDA events, so the arms share the machine's state"""
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    out = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                fn()
            b.record()
            b.synchronize()
            out[k].append(1e3 * a.elapsed_time(b) / reps)
    return {k: dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v))) for k, v in out.items()}


def run_pack(S, amips, args):
    pk, x_np, quiet = pack_x(S, "mixed")
    sp = ext.TetSpheres(pk.verts.astype(np.float32).reshape(-1), pk.tets.astype(np.int32).reshape(-1),
                        enable_amips=True, deterministic=True)
    c1, c2, c3 = 2e-4 / S, 2e-4, (C3 if amips else 0.0)
    x = torch.from_numpy(x_np.astype(np.float32)).cuda()
    q = torch.from_numpy(quiet).cuda()
    _, g = sp.energy_grad(x, c1, c2, 2, -1.0, c3=c3)
    b = g.reshape(-1, 3).contiguous()
    planes = sp.hess_diag(x, c1, c2, 2, c3=c3)
    sid = torch.from_numpy(np.repeat(np.arange(S), np.diff(pk.vert_offsets))).cuda()
    dmax = torch.zeros(S, dtype=torch.float32, device="cuda").index_reduce_(0, sid, planes[0].max(1).values, "amax",
                                                                           include_self=False)
    mu = (1e-3 * dmax).contiguous()       # the damped step's first shift, tau max (D_v)_ii per sphere
    res = {}
    for hessian in ("exact", "psd"):
        pj, pc = DevicePCG(sp, hessian=hessian), DevicePCG(sp, hessian=hessian, coarse="affine")
        sh = mu if hessian == "exact" else None
        pc.set_coarse(x, c1, c2, 2, c3=c3)
        for p in (pj, pc):
            p.set_blocks(planes, shift=sh)
        r = {name: dict(products=p.solve(x, b, c1, c2, 2, c3=c3, max_iter=400, rtol=1e-3, shift=sh).n_hvp[q].double().mean().item())
             for name, p in (("jacobi", pj), ("coarse", pc))}
        t = event_us({name: (lambda p=p: p.solve(x, b, c1, c2, 2, c3=c3, max_iter=20, rtol=1e-2, shift=sh))
                      for name, p in (("jacobi", pj), ("coarse", pc))}, args.rounds)
        for name in t:
            r[name]["solve_us"] = t[name]
        r["set_coarse_us"] = event_us({"coarse": lambda: pc.set_coarse(x, c1, c2, 2, c3=c3)}, args.rounds)["coarse"]
        res[hessian] = r
    steps = {}
    for m, (hessian, fn) in METHODS.items():
        arms = {}
        for name, coarse in (("jacobi", None), ("coarse", "affine")):
            nw = DeviceNewton(sp, hessian=hessian, coarse=coarse)
            xs = x.clone()

            def one(nw=nw, xs=xs):
                xs.copy_(x)
                nw.reset()
                getattr(nw, fn)(xs, c1, c2, 2, c3=c3)
            arms[name] = one
        steps[m] = event_us(arms, args.rounds)
    res["step_us"] = steps
    return res, (sp, pk, x, quiet, c1, c2, c3)


def time_to_solution(ctx, args):
    sp, pk, x0, quiet, c1, c2, c3 = ctx
    S = pk.num_spheres
    sid_np = np.repeat(np.arange(S), np.diff(pk.vert_offsets))
    keep = torch.ones(len(sid_np), dtype=torch.bool, device="cuda")
    sid = torch.from_numpy(sid_np).cuda()
    q = torch.from_numpy(quiet).cuda()
    out = {}
    for m, (hessian, fn) in METHODS.items():
        for name, coarse in (("jacobi", None), ("coarse", "affine")):
            nw = DeviceNewton(sp, hessian=hessian, coarse=coarse)
            x = x0.clone()
            g0 = sphere_gnorm(sp, x, c1, c2, c3, sid, keep, S)
            total, k = 0.0, 0
            while k < args.max_steps:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                getattr(nw, fn)(x, c1, c2, 2, c3=c3)
                b.record()
                b.synchronize()
                total += 1e3 * a.elapsed_time(b)
                k += 1
                if bool((sphere_gnorm(sp, x, c1, c2, c3, sid, keep, S)[q] <= 1e-3 * g0[q]).all()):
                    break
            out[f"{m}/{name}"] = dict(steps=k, us=total, reached=k < args.max_steps or
                                      bool((sphere_gnorm(sp, x, c1, c2, c3, sid, keep, S)[q] <= 1e-3 * g0[q]).all()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--big", action="store_true")
    ap.add_argument("--max-steps", type=int, default=60)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_coarse.py needs a CUDA device")
    result = {"card": card(), "packs": {}}
    ctx64 = None
    for S in ([64, 1024] if args.big else [64]):
        for amips in (False, True):
            r, ctx = run_pack(S, amips, args)
            result["packs"][f"{S}x4096/amips={'on' if amips else 'off'}"] = r
            print(json.dumps({f"{S}x4096 amips={amips}": r}), flush=True)
            if S == 64 and amips:
                ctx64 = ctx
    result["time_to_solution_64x4096_amips_on"] = time_to_solution(ctx64, args)
    print(json.dumps({"card": result["card"], "time_to_solution": result["time_to_solution_64x4096_amips_on"]}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_coarse.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()

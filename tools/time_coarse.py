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

import torch

from _timing import alternate, card, mixed_pack, sphere_gnorm, sphere_ids, steps_until, summary, write_json
from tssplat_b200 import tet_spheres_ext as ext
from tssplat_b200.newton import DeviceNewton, DevicePCG

C3 = 1e-4
METHODS = {"lm": ("exact", "step"), "psd": ("psd", "step")}   # the trust-region steps refuse a coarse workspace


def rounds_us(fns, rounds):
    """{name: median, min, max over rounds of us per call}: one untimed call of each fn, then every round times each fn in
    turn, 5 calls between two CUDA events, so the arms share the machine's state"""
    return {k: summary(v) for k, v in alternate(fns, rounds, reps=5, warmup=1).items()}


def run_pack(S, amips, args):
    pk, x_np, quiet = mixed_pack(S, 1, 3, 4)
    sp = ext.TetSpheres(pk.verts.reshape(-1), pk.tets.reshape(-1), enable_amips=True, deterministic=True)
    c1, c2, c3 = 2e-4 / S, 2e-4, (C3 if amips else 0.0)
    x = torch.from_numpy(x_np).cuda()
    q = torch.from_numpy(quiet).cuda()
    _, g = sp.energy_grad(x, c1, c2, 2, -1.0, c3=c3)
    b = g.reshape(-1, 3).contiguous()
    planes = sp.hess_diag(x, c1, c2, 2, c3=c3)
    sid = sphere_ids(pk).cuda()
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
        t = rounds_us({name: (lambda p=p: p.solve(x, b, c1, c2, 2, c3=c3, max_iter=20, rtol=1e-2, shift=sh))
                      for name, p in (("jacobi", pj), ("coarse", pc))}, args.rounds)
        for name in t:
            r[name]["solve_us"] = t[name]
        r["set_coarse_us"] = rounds_us({"coarse": lambda: pc.set_coarse(x, c1, c2, 2, c3=c3)}, args.rounds)["coarse"]
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
        steps[m] = rounds_us(arms, args.rounds)
    res["step_us"] = steps
    return res, (sp, pk, x, quiet, c1, c2, c3)


def time_to_solution(ctx, args):
    sp, pk, x0, quiet, c1, c2, c3 = ctx
    S = pk.num_spheres
    sid = sphere_ids(pk).cuda()
    q = torch.from_numpy(quiet).cuda()
    out = {}
    for m, (hessian, fn) in METHODS.items():
        for name, coarse in (("jacobi", None), ("coarse", "affine")):
            nw = DeviceNewton(sp, hessian=hessian, coarse=coarse)
            x = x0.clone()
            g0 = sphere_gnorm(sp, x, c1, c2, c3, sid, S)
            k, total, reached = steps_until(lambda: getattr(nw, fn)(x, c1, c2, 2, c3=c3), lambda: bool(
                (sphere_gnorm(sp, x, c1, c2, c3, sid, S)[q] <= 1e-3 * g0[q]).all()), args.max_steps)
            out[f"{m}/{name}"] = dict(steps=k, us=total, reached=reached)
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
    write_json(args.out, "time_coarse.json", result)


if __name__ == "__main__":
    main()

"""Symmetric Gauss-Seidel preconditioner (DevicePCG(precond="sgs")) against block Jacobi, timed with CUDA events in one
process.

Packs: 64 x 4096 and (--big) 1024 x 4096 tets, "benign" (every sphere at 0.02 h), "inverted" (every sphere at 0.35 h)
and "mixed" (every fourth sphere at 0.35 h, the rest at 0.02 h); c1 = 2e-4 / S, c2 = 2e-4, order 2, AMIPS off and on
(c3 = 1e-4); a deterministic handle.  Per pack and AMIPS setting:
  colours      the most colours of any sphere
  apply        us per tsb_pcg_apply_precond (one CUDA graph of `--launches` calls)
  iter         us per CG iteration: the slope of tsb_pcg_solve between max_iter 10 and 20 (rtol 0), both preconditioners
  set_matrix   us per tsb_pcg_set_matrix (the re-assembly an SGS Newton step adds)
  products     mean and max Hessian-vector products to rtol = 1e-3 over the spheres at 0.02 h (max_iter 400), unshifted
               and with the LM shift mu_c = 1e-3 max (D_v)_ii of the first damped step, both preconditioners
  step         us per DeviceNewton.step (max_iter 20, rtol 1e-2), both preconditioners
Graph arms are replayed alternately for `--rounds` rounds (median us).  Time to solution (mixed pack only): steps and
summed CUDA-event step time until every quiet sphere's |g_c| has fallen by 1e3 (the criterion of the LM, PSD and TR
tables), up to `--max-steps` steps, Jacobi and SGS alternating.  The card, its power limit and the SM clock under load
are read in the same process.

Usage: python tools/time_sgs.py [--rounds 5] [--launches 10] [--big] [--out DIR]"""
import argparse
import json

import numpy as np
import torch

from _timing import (TETS, alternate, capture, card, mixed_pack, sm_clock_under_load, sphere_gnorm, sphere_ids, steps_until,
                     write_json)
from tssplat_b200 import tet_spheres_ext as ext
from tssplat_b200.newton import DeviceNewton, DevicePCG

C3 = 1e-4
ROUGH_EVERY = {"benign": None, "inverted": 1, "mixed": 4}     # the spheres at 0.35 h: none, all, every fourth


def run_pack(S, kind, args, out):
    pk, x_np, quiet = mixed_pack(S, 1, 3, ROUGH_EVERY[kind])
    x = torch.from_numpy(x_np).cuda()
    c1, c2 = 2e-4 / S, 2e-4
    sp = ext.TetSpheres(pk.verts.reshape(-1), pk.tets.reshape(-1), enable_amips=True, deterministic=True)
    pj, ps = DevicePCG(sp), DevicePCG(sp, precond="sgs")
    s = torch.cuda.Stream()
    for c3 in (0.0, C3):
        key = f"{S}x{TETS} {kind} amips={'on' if c3 else 'off'}"
        res = dict(colours=ps.n_colors, device_bytes_sgs=ps.device_bytes, device_bytes_jacobi=pj.device_bytes,
                   hessian_bytes=ps.hessian_ws.device_bytes)
        _, g = sp.energy_grad(x, c1, c2, 2, -1.0, c3=c3)
        b = g.reshape(-1, 3).contiguous()
        with torch.cuda.stream(s):
            pj.set_blocks(sp.hess_diag(x, c1, c2, 2, c3=c3))
            planes = ps.set_matrix(x, c1, c2, 2, c3=c3)
            ps.set_blocks(planes)
        torch.cuda.synchronize()
        z = torch.zeros_like(b)
        planes_out = torch.empty_like(planes)

        def solve(p, k):
            return lambda: p.solve(x, b, c1, c2, 2, c3=c3, max_iter=k, rtol=0.0)

        fns = {"apply": lambda: ps.apply_precond(b, out=z),
               "set_matrix": lambda: ps.set_matrix(x, c1, c2, 2, c3=c3, out=planes_out),
               "jacobi10": solve(pj, 10), "jacobi20": solve(pj, 20), "sgs10": solve(ps, 10), "sgs20": solve(ps, 20)}
        with torch.cuda.stream(s):
            ps.set_blocks(planes)
        t = alternate({k: capture(f, s, args.launches, 3, k) for k, f in fns.items()}, args.rounds, calls=args.launches)
        med = {k: float(np.median(v)) for k, v in t.items()}
        res.update(apply_us=med["apply"], set_matrix_us=med["set_matrix"],
                   iter_us_jacobi=(med["jacobi20"] - med["jacobi10"]) / 10, iter_us_sgs=(med["sgs20"] - med["sgs10"]) / 10)
        # products to rtol 1e-3 on the quiet spheres, plain and LM-shifted
        mu = torch.full((pj.n_spheres,), 1e-3 * float(planes[0].max()), dtype=torch.float32, device="cuda")
        q = torch.from_numpy(quiet).cuda()
        for shifted in (False, True):
            sh = mu if shifted else None
            pj.set_blocks(sp.hess_diag(x, c1, c2, 2, c3=c3), shift=sh)
            ps.set_blocks(planes, shift=sh)
            for name, p in (("jacobi", pj), ("sgs", ps)):
                r = p.solve(x, b, c1, c2, 2, c3=c3, max_iter=400, rtol=1e-3, shift=sh)
                n = r.n_hvp[q].double()
                conv = int((r.status[q] == 1).sum())
                if len(n):
                    res[f"products_{'lm' if shifted else 'plain'}_{name}"] = dict(mean=float(n.mean()), max=int(n.max()),
                                                                                  converged=conv, of=int(q.sum()))
        # one damped step, both preconditioners, alternating graphs
        x0 = x.clone()
        arms = {}
        for name, p in (("jacobi", pj), ("sgs", ps)):
            nw = DeviceNewton(sp, p)
            xs = x0.clone()
            arms[name] = (nw, xs)
        o = dict(max_iter=20, rtol=1e-2)

        def step(name):
            nw, xs = arms[name]

            def f():
                xs.copy_(x0)
                nw.reset()
                nw.step(xs, c1, c2, 2, c3=c3, **o)
            return f

        t = alternate({f"step_{k}": capture(step(k), s, 1, 3, k) for k in ("jacobi", "sgs")}, args.rounds)
        res.update({k + "_us": float(np.median(v)) for k, v in t.items()})
        if kind == "mixed":
            res["tts"] = time_to_solution(sp, pk, x0, quiet, c1, c2, c3, {k: v[0] for k, v in arms.items()}, args)
        out[key] = res
        print(key, json.dumps(res), flush=True)
    del pj, ps


def time_to_solution(sp, pk, x0, quiet, c1, c2, c3, nws, args):
    S = len(quiet)
    sid = sphere_ids(pk).cuda()
    g0 = sphere_gnorm(sp, x0, c1, c2, c3, sid, S).cpu().numpy()
    o = dict(max_iter=20, rtol=1e-2, gtol=float(1e-3 * g0[quiet].min()))
    out = {k: dict(steps=[], ms=[]) for k in nws}
    for _ in range(args.tts_rounds):
        for name, nw in nws.items():          # alternating
            x = x0.clone()
            nw.reset()
            steps, us, done = steps_until(lambda: nw.step(x, c1, c2, 2, c3=c3, **o), lambda: bool(
                (sphere_gnorm(sp, x, c1, c2, c3, sid, S).cpu().numpy()[quiet] <= 1e-3 * g0[quiet]).all()), args.max_steps)
            out[name]["steps"].append(steps if done else None)
            out[name]["ms"].append(us / 1e3 if done else None)
    return {k: dict(steps=v["steps"][0], ms=float(np.median([m for m in v["ms"] if m is not None])) if all(v["ms"]) else None)
            for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--big", action="store_true")
    ap.add_argument("--tts-rounds", type=int, default=2)
    ap.add_argument("--max-steps", type=int, default=40)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_sgs.py measures on the GPU"
    out = {"card": card()}
    for S in ((64, 1024) if args.big else (64,)):
        for kind in ("benign", "inverted", "mixed"):
            run_pack(S, kind, args, out)
    # the SM clock while the last pack's Jacobi solve is replayed
    pk, x_np, _ = mixed_pack(64, 1, 3, ROUGH_EVERY["mixed"])
    sp = ext.TetSpheres(pk.verts.reshape(-1), pk.tets.reshape(-1), deterministic=True)
    p = DevicePCG(sp, precond="sgs")
    x = torch.from_numpy(x_np).cuda()
    p.set_blocks(p.set_matrix(x, 2e-4 / 64, 2e-4, 2))
    b = torch.ones_like(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = capture(lambda: p.solve(x, b, 2e-4 / 64, 2e-4, 2, max_iter=20, rtol=0.0), s, 1, 1)
    out["sm_clock_mhz_under_load"] = sm_clock_under_load(g, 500.0)
    print(json.dumps(out, indent=1))
    write_json(args.out, "time_sgs.json", out)


if __name__ == "__main__":
    main()

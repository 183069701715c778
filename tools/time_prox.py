"""Cost of the proximal Newton step (tsb_newton_prox_step) against the plain damped step, and a split training loop with
no renderer, timed with CUDA events in one process.

Cost: one CUDA graph per arm holding (copy the start into x, reset, one step), on 64 x 4096 and 1024 x 4096 packs
(benign, 0.02 h; c1 = 2e-4 / S, c2 = 2e-4), AMIPS off and on (c3 = 1e-4), max_iter 10, on a deterministic handle -- the
setup of DESIGN.md section 5's step-cost table.  The prox arm anchors at the start with w_c = 1e-2 for every sphere.
Rounds alternate the arms; each round times `--replays` replays; medians, minima and maxima over `--rounds` rounds.  The
SM clock (nvidia-smi clocks.sm) is read while about half a second of the prox arm's replays is queued on the GPU.  One
eager step per arm also reports its solve: mean products per sphere (n_hvp) and the spheres per PCG status.

Split loop: a synthetic data term 1/2 |x_s - t_s|^2 on the surface vertices of the 64 x 4096 pack, where t is the
surface at rest displaced by a seeded normal field of 0.3 h per coordinate.  Two loops of `--iters` iterations from the
same start, AdamUniform (lr 1e-3) in both:
  joint   AdamUniform on data + E (E: SmoothnessBarrierEnergy at it, the reference trainer's joint loss);
  split   AdamUniform on data alone, then y = x, SmoothnessBarrierEnergy.prox_step(x, y, it, w) (one step, max_iter 10).
Both loops first run one untimed round of `--warmup-iters` iterations (module loading, first-use allocations, the
energy handle's caches).  Reported: ms per iteration (host clock around a synchronised loop; `--loop-rounds` rounds, the
loop that goes first alternating) and, after the last round, the data term, E and the inverted-tet count.  Without a
renderer and image data this says nothing about reconstruction quality.

Usage: python tools/time_prox.py [--rounds 6] [--replays 5] [--iters 200] [--loop-rounds 5] [--out DIR]"""
import argparse
import json
import sys
import time

import numpy as np
import torch

from _timing import TETS, alternate, capture, card, sm_clock_under_load, summary, write_json
from tssplat_b200 import tet_spheres_ext as ext
from tssplat_b200.energies import SmoothnessBarrierEnergy
from tssplat_b200.mesh import make_pack, perturb, surface_vf
from tssplat_b200.newton import DeviceNewton
from tssplat_b200.optimizer import AdamUniform

C3 = 1e-4


def step_cost(S, args, results):
    pack = make_pack(S, TETS, seed=0, unique=8)
    x0 = torch.from_numpy(perturb(pack, sigma_rel=0.02, seed=0)).cuda()
    c1, c2 = 2e-4 / S, 2e-4
    sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), enable_amips=True, deterministic=True)
    nw = DeviceNewton(sp)
    x, y = x0.clone(), x0.clone()
    w = torch.full((nw.n_spheres,), 1e-2, device="cuda")
    s = torch.cuda.Stream()
    for c3 in (0.0, C3):
        arms = {"newton": dict(), "prox": dict(anchor=y, weight=w)}
        graphs = {}
        for name, kw in arms.items():
            def fn(kw=kw):
                x.copy_(x0)
                nw.reset()
                nw.step(x, c1, c2, 2, c3=c3, max_iter=10, **kw)
            graphs[name] = capture(fn, s, 1, 2, name)        # two warm-up calls: the first prox step allocates
        times = alternate(graphs, args.rounds, reps=args.replays, before=lambda k: graphs[k].replay())
        key = f"{S}x{TETS} c3={c3:g}"
        results["cost"][key] = {k: summary(v) for k, v in times.items()}
        r = results["cost"][key]
        clock = r["sm_mhz_under_load"] = sm_clock_under_load(graphs["prox"], r["prox"]["median"])
        for name, kw in arms.items():                 # what the solve did in one step of each arm
            x.copy_(x0)
            nw.reset()
            rec = nw.step(x, c1, c2, 2, c3=c3, max_iter=10, **kw)
            st = rec.pcg_status.cpu().numpy()
            r[name]["n_hvp_mean"] = float(rec.n_hvp.double().mean())
            r[name]["pcg_status_counts"] = {int(k): int((st == k).sum()) for k in np.unique(st)}
        print(f"{key}: newton {r['newton']['median']:.1f} us [{r['newton']['min']:.1f}, {r['newton']['max']:.1f}] "
              f"n_hvp {r['newton']['n_hvp_mean']:.2f} {r['newton']['pcg_status_counts']}, "
              f"prox {r['prox']['median']:.1f} us [{r['prox']['min']:.1f}, {r['prox']['max']:.1f}] "
              f"n_hvp {r['prox']['n_hvp_mean']:.2f} {r['prox']['pcg_status_counts']}; SM clock under load {clock} MHz", flush=True)
    del nw, sp
    torch.cuda.empty_cache()


def split_loop(args, results):
    pack = make_pack(64, TETS, seed=0, unique=8)
    x0 = torch.from_numpy(perturb(pack, sigma_rel=0.02, seed=0)).cuda()
    sv, _ = surface_vf(pack.tets)
    sv = torch.from_numpy(np.asarray(sv, np.int64)).cuda()
    V, T = pack.verts, pack.tets
    h = float(np.linalg.norm(V[T[:, 1]] - V[T[:, 0]], axis=1).mean())
    rng = np.random.default_rng(0)
    target = torch.from_numpy(V[sv.cpu().numpy()] + rng.normal(scale=0.3 * h, size=(len(sv), 3)).astype(np.float32)).cuda()
    flags = dict(smooth_eng_coeff=2e-4, barrier_coeff=2e-4, increase_order_iter=1000, deterministic=True)
    E = SmoothnessBarrierEnergy(V, T, flags)
    it = 0
    c1, c2 = E.coeff_scheduler(it)

    def data(p):
        return 0.5 * ((p[sv] - target) ** 2).sum()

    def run(kind, iters):
        p = torch.nn.Parameter(x0.clone())
        opt = AdamUniform([p], lr=1e-3)
        y = torch.empty_like(x0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(iters):
            opt.zero_grad(set_to_none=True)
            loss = data(p) + (E(p, it, c1, c2) if kind == "joint" else 0.0)
            loss.backward()
            opt.step()
            if kind == "split":
                y.copy_(p.data)
                E.prox_step(p, y, it, args.weight, max_iter=10)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3 / iters
        st = E.sphere_stats(p, it)
        energy = float((c1 * st.smooth + c2 * st.barrier).sum())
        return ms, dict(data=float(data(p.detach())), E=energy, inverted=int(st.n_inverted.sum()))

    times = {"joint": [], "split": []}
    for kind in times:                                # untimed warm-up of both loops
        run(kind, args.warmup_iters)
    final = {}
    for i in range(args.loop_rounds):
        for kind in (list(times) if i % 2 == 0 else list(times)[::-1]):
            ms, out = run(kind, args.iters)
            times[kind].append(ms)
            final[kind] = out
    st0 = E.sphere_stats(x0, it)
    results["split_loop"] = dict(iters=args.iters, rounds=args.loop_rounds, weight=args.weight, start=dict(
        data=float(data(x0)), E=float((c1 * st0.smooth + c2 * st0.barrier).sum()), inverted=int(st0.n_inverted.sum())),
        **{k: dict(ms_per_iter=summary(times[k]), **final[k]) for k in times})
    print(json.dumps(results["split_loop"], indent=1), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--replays", type=int, default=5)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--loop-rounds", type=int, default=5)
    ap.add_argument("--warmup-iters", type=int, default=20)
    ap.add_argument("--weight", type=float, default=1.0, help="w_c of the split loop's proximal step, every sphere")
    ap.add_argument("--out", default=None, help="directory for time_prox.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_prox.py needs a GPU")
    results = dict(card=card(), argv=sys.argv[1:], cost={})
    print(results["card"], flush=True)
    for S in (64, 1024):
        step_cost(S, args, results)
    split_loop(args, results)
    write_json(args.out, "time_prox.json", results)


if __name__ == "__main__":
    main()

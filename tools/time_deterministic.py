"""Cost of the deterministic gradient mode: default and deterministic handles of the same mesh and options, timed in
one process with CUDA events, alternating.  Each timed unit is a CUDA graph of `--launches` energy+gradient launches
(replayed `--rounds` times per handle); the median over rounds is reported in us per launch.

Usage: python tools/time_deterministic.py [--rounds 30] [--launches 50] [--out DIR]"""
import argparse

import numpy as np
import torch

from _timing import TETS, alternate, capture, card, p10_p90, write_json
from tssplat_b200 import tet_spheres_ext as ext
from tssplat_b200.mesh import make_pack, perturb

# (name, spheres, sigma relative to the edge length h, AMIPS coefficient)
CASES = [("64x4096 benign (0.02 h)", 64, 0.02, 0.0), ("64x4096 inverted (0.35 h)", 64, 0.35, 0.0),
         ("64x4096 AMIPS on (0.02 h)", 64, 0.02, 1e-4), ("1024x4096 benign (0.02 h)", 1024, 0.02, 0.0),
         ("1024x4096 AMIPS on (0.02 h)", 1024, 0.02, 1e-4)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for time_deterministic.json")
    args = ap.parse_args()
    dev = card()
    print(f"device: {dev}", flush=True)
    results = []
    for name, S, sig, c3 in CASES:
        pack = make_pack(S, TETS, seed=0, unique=8)
        kw = dict(enable_amips=c3 != 0.0)
        a = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), **kw)
        d = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), deterministic=True, **kw)
        assert a.info["grid"] == d.info["grid"]
        x = torch.from_numpy(perturb(pack, sigma_rel=sig, seed=0)).cuda()
        c1, c2 = 2e-4 / S, 2e-4
        ea, ga = a.energy_grad(x, c1, c2, 2, 1.0, c3=c3)
        ed, gd = d.energy_grad(x, c1, c2, 2, 1.0, c3=c3)
        torch.cuda.synchronize()
        rel = float((gd - ga).norm() / ga.norm())
        graphs = {k: capture(lambda h=h: h.energy_grad(x, c1, c2, 2, 1.0, c3=c3), None, args.launches, 3, k)
                  for k, h in (("default", a), ("deterministic", d))}
        times = alternate(graphs, args.rounds, calls=args.launches)
        r = {"case": name, "spheres": S, "tets": S * TETS, "sigma_rel": sig, "c3": c3, "barrier_energy": float(ea[2]),
             "grad_rel_diff": rel, "energies_bitwise_equal": bool(torch.equal(ea, ed)),
             "us_per_step": {k: float(np.median(v)) for k, v in times.items()},
             "us_per_step_p10_p90": {k: p10_p90(v) for k, v in times.items()},
             "device_bytes": {"default": a.info["device_bytes"], "deterministic": d.info["device_bytes"]}, "device": dev}
        us = r["us_per_step"]
        print(f"{name:30s} default {us['default']:8.2f} us  deterministic {us['deterministic']:8.2f} us "
              f"({us['deterministic'] / us['default'] - 1:+.1%})  device MB {a.info['device_bytes'] / 1e6:.0f} -> "
              f"{d.info['device_bytes'] / 1e6:.0f}  grad rel diff {rel:.1e}  barrier E {float(ea[2]):.3g}", flush=True)
        results.append(r)
        del graphs, a, d
        torch.cuda.empty_cache()
    write_json(args.out, "time_deterministic.json", results)


if __name__ == "__main__":
    main()

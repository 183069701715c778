"""Cost of the per-sphere statistics: the default fused launch (tsb_energy_grad_ex) and the statistics launch
(tsb_energy_grad_spheres: the SPH energy kernel plus the fold kernel) on the SAME handle, each with the gradient, timed
in one process with CUDA events, alternating.  Each timed unit is a CUDA graph of `--launches` launches (replayed
`--rounds` times per kind); the median over rounds is reported in us per step.

Usage: python tools/time_sphere_stats.py [--rounds 30] [--launches 50] [--out DIR]"""
import argparse
import ctypes as C

import numpy as np
import torch

from _timing import TETS, alternate, capture, card, p10_p90, write_json
from tssplat_b200 import _capi
from tssplat_b200 import tet_spheres_ext as ext
from tssplat_b200.mesh import make_pack, perturb

# (name, spheres, sigma relative to the edge length h)
CASES = [("64x4096 benign (0.02 h)", 64, 0.02), ("64x4096 inverted (0.35 h)", 64, 0.35), ("1024x4096 benign (0.02 h)", 1024, 0.02)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for time_sphere_stats.json")
    args = ap.parse_args()
    dev = card()
    print(f"device: {dev}", flush=True)
    results = []
    for name, S, sig in CASES:
        pack = make_pack(S, TETS, seed=0, unique=8)
        sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1))
        x = torch.from_numpy(perturb(pack, sigma_rel=sig, seed=0)).cuda()
        terms = _capi.tsb_terms_t(c1=2e-4 / S, c2=2e-4, order=2, c3=0.0)
        energy = torch.empty(4, device="cuda")
        grad = torch.empty_like(x)
        stats = torch.empty((sp.info["n_components"], 40), dtype=torch.uint8, device="cuda")
        s = torch.cuda.Stream()

        def default():
            return _capi.lib.tsb_energy_grad_ex(sp._h, x.data_ptr(), C.byref(terms), 1.0, None, energy.data_ptr(),
                                                grad.data_ptr(), s.cuda_stream)

        def spheres():
            return _capi.lib.tsb_energy_grad_spheres(sp._h, x.data_ptr(), C.byref(terms), 1.0, None, energy.data_ptr(),
                                                     grad.data_ptr(), stats.data_ptr(), s.cuda_stream)

        graphs = {k: capture(fn, s, args.launches, 3, k) for k, fn in (("default", default), ("spheres", spheres))}
        times = alternate(graphs, args.rounds, calls=args.launches)
        st = stats.view(-1)
        n_inv = int(st.view(-1, 40)[:, 28:32].contiguous().view(torch.int32).sum())
        r = {"case": name, "spheres": S, "tets": S * TETS, "sigma_rel": sig, "grid": sp.info["grid"],
             "inverted_tets": n_inv, "us_per_step": {k: float(np.median(v)) for k, v in times.items()},
             "us_per_step_p10_p90": {k: p10_p90(v) for k, v in times.items()},
             "device": dev}
        us = r["us_per_step"]
        print(f"{name:28s} default {us['default']:8.2f} us  spheres {us['spheres']:8.2f} us "
              f"({us['spheres'] / us['default'] - 1:+.1%})  inverted tets {n_inv}", flush=True)
        results.append(r)
        del graphs, sp
        torch.cuda.empty_cache()
    write_json(args.out, "time_sphere_stats.json", results)


if __name__ == "__main__":
    main()

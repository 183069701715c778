"""Cost of the Hessian-vector product: the default fused launch with the gradient (tsb_energy_grad) and tsb_hvp on the
SAME handle, timed in one process with CUDA events, alternating.  Each timed unit is a CUDA graph of `--launches`
launches (replayed `--rounds` times per kind); the median over rounds is reported in us per launch.

The AMIPS rows do the same with the AMIPS term on (c3 != 0, a handle created with enable_amips): tsb_energy_grad_ex
with the gradient against tsb_hvp_ex, on default and deterministic handles.

Usage: python tools/time_hvp.py [--rounds 30] [--launches 50] [--out DIR]"""
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
# AMIPS rows: (name, spheres, sigma, deterministic handle)
AMIPS_CASES = [("64x4096 AMIPS default", 64, 0.02, False), ("64x4096 AMIPS det", 64, 0.02, True),
               ("1024x4096 AMIPS default", 1024, 0.02, False), ("1024x4096 AMIPS det", 1024, 0.02, True)]
C3 = 1e-4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for time_hvp.json")
    args = ap.parse_args()
    dev = card()
    print(f"device: {dev}", flush=True)
    results = []
    runs = [(name, S, sig, None) for name, S, sig in CASES] + list(AMIPS_CASES)
    for name, S, sig, det in runs:
        amips = det is not None
        pack = make_pack(S, TETS, seed=0, unique=8)
        sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), enable_amips=amips, deterministic=bool(det))
        x = torch.from_numpy(perturb(pack, sigma_rel=sig, seed=0)).cuda()
        v = torch.randn(x.shape, generator=torch.Generator().manual_seed(1)).cuda()
        c1, c2 = 2e-4 / S, 2e-4
        terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=C3)
        energy = torch.empty(4, device="cuda")
        grad = torch.empty_like(x)
        hv = torch.empty_like(x)
        curv = torch.empty(4, device="cuda")
        s = torch.cuda.Stream()

        if amips:
            def gradient():
                return _capi.lib.tsb_energy_grad_ex(sp._h, x.data_ptr(), C.byref(terms), 1.0, None, energy.data_ptr(),
                                                    grad.data_ptr(), s.cuda_stream)

            def hvp():
                return _capi.lib.tsb_hvp_ex(sp._h, x.data_ptr(), v.data_ptr(), C.byref(terms), 1.0, None, hv.data_ptr(),
                                            curv.data_ptr(), s.cuda_stream)
        else:
            def gradient():
                return _capi.lib.tsb_energy_grad(sp._h, x.data_ptr(), c1, c2, 2, 1.0, None, energy.data_ptr(),
                                                 grad.data_ptr(), s.cuda_stream)

            def hvp():
                return _capi.lib.tsb_hvp(sp._h, x.data_ptr(), v.data_ptr(), c1, c2, 2, 1.0, None, hv.data_ptr(),
                                         curv.data_ptr(), s.cuda_stream)

        graphs = {k: capture(fn, s, args.launches, 3, k) for k, fn in (("gradient", gradient), ("hvp", hvp))}
        times = alternate(graphs, args.rounds, calls=args.launches)
        del graphs
        _, _, st = sp.energy_grad_spheres(x, c1, c2, 2, want_grad=False)
        n_inv = int(st.n_inverted.sum())
        r = {"case": name, "spheres": S, "tets": S * TETS, "sigma_rel": sig, "grid": sp.info["grid"],
             "amips_c3": C3 if amips else 0.0, "deterministic": bool(det),
             "inverted_tets": n_inv, "us_per_launch": {k: float(np.median(t)) for k, t in times.items()},
             "us_per_launch_p10_p90": {k: p10_p90(t) for k, t in times.items()},
             "device": dev}
        us = r["us_per_launch"]
        print(f"{name:28s} gradient {us['gradient']:8.2f} us  hvp {us['hvp']:8.2f} us "
              f"({us['hvp'] / us['gradient'] - 1:+.1%})  inverted tets {n_inv}", flush=True)
        results.append(r)
        del sp
        torch.cuda.empty_cache()
    write_json(args.out, "time_hvp.json", results)


if __name__ == "__main__":
    main()

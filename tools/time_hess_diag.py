"""Cost of the Hessian diagonal: tsb_hess_diag against a gradient launch on the SAME handle, timed in one process with
CUDA events, alternating.  Each timed unit is a CUDA graph of `--launches` calls (replayed `--rounds` times per kind); the
median over rounds is reported in us per call.  On a deterministic handle a call is two energy-kernel launches and two
gathers (one per output plane), a gradient one launch and one gather.

Rows: the workloads of time_line_search.py (64 x 4096 benign (0.02 h) and inverted (0.35 h), 1024 x 4096 benign), each with
AMIPS off and on (c3 = 1e-4), on default and deterministic handles.

Usage: python tools/time_hess_diag.py [--rounds 30] [--launches 50] [--out DIR]"""
import argparse
import ctypes as C

import numpy as np
import torch

from _timing import TETS, alternate, capture, card, p10_p90, write_json
from tssplat_b200 import _capi
from tssplat_b200 import tet_spheres_ext as ext
from tssplat_b200.mesh import make_pack, perturb
CASES = [("64x4096 benign (0.02 h)", 64, 0.02), ("64x4096 inverted (0.35 h)", 64, 0.35), ("1024x4096 benign (0.02 h)", 1024, 0.02)]
C3 = 1e-4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for time_hess_diag.json")
    args = ap.parse_args()
    dev = card()
    print(f"device: {dev}", flush=True)
    results = []
    for name, S, sig in CASES:
        pack = make_pack(S, TETS, seed=0, unique=8)
        x = torch.from_numpy(perturb(pack, sigma_rel=sig, seed=0)).cuda()
        c1, c2 = 2e-4 / S, 2e-4
        energy = torch.empty(4, device="cuda")
        grad = torch.empty_like(x)
        planes = torch.empty((2,) + tuple(x.shape), device="cuda")
        s = torch.cuda.Stream()
        for det in (False, True):
            sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), enable_amips=True, deterministic=det)
            for c3 in (0.0, C3):
                terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=c3)

                def gradient():
                    return _capi.lib.tsb_energy_grad_ex(sp._h, x.data_ptr(), C.byref(terms), 1.0, None, energy.data_ptr(),
                                                        grad.data_ptr(), s.cuda_stream)

                def hess_diag():
                    return _capi.lib.tsb_hess_diag(sp._h, x.data_ptr(), C.byref(terms), 1.0, None, planes.data_ptr(),
                                                   s.cuda_stream)

                fns = {"gradient": gradient, "hess_diag": hess_diag}
                times = alternate({k: capture(fn, s, args.launches, 3, k) for k, fn in fns.items()}, args.rounds,
                                  calls=args.launches)
                r = {"case": name, "spheres": S, "tets": S * TETS, "sigma_rel": sig, "amips_c3": c3, "deterministic": det,
                     "grid": sp.info["grid"], "us_per_call": {k: float(np.median(t)) for k, t in times.items()},
                     "us_per_call_p10_p90": {k: p10_p90(t) for k, t in times.items()},
                     "device": dev}
                us = r["us_per_call"]
                print(f"{name:28s} {'det' if det else 'default':7s} c3={c3:<6g} gradient {us['gradient']:8.2f}  "
                      f"hess_diag {us['hess_diag']:8.2f} us", flush=True)
                results.append(r)
            del sp
            torch.cuda.empty_cache()
    write_json(args.out, "time_hess_diag.json", results)


if __name__ == "__main__":
    main()

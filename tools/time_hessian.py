"""Cost of assembling the Hessian: tsb_hessian_assemble against tsb_hvp_ex and tsb_hess_diag on the SAME handle, timed in
one process with CUDA events over CUDA-graph replays, alternating (as time_hvp.py: median over rounds, us per call).
Also reports the values' bytes (36 per block) over the assembly time against the H100 SXM data sheet's 3.35 TB/s.

Rows: 64 x 4096 and 1024 x 4096, benign (0.02 h) and inverted (0.35 h) inputs, AMIPS off and on (c3 = 1e-4), exact and
PSD Hessians, on a default handle.

Usage: python tools/time_hessian.py [--rounds 20] [--launches 20] [--sizes 64,1024] [--out DIR]"""
import argparse
import ctypes as C

import numpy as np
import torch

from _timing import TETS, alternate, capture, card, p10_p90, write_json
from tssplat_b200 import _capi
from tssplat_b200 import tet_spheres_ext as ext
from tssplat_b200.hessian import DeviceHessian
from tssplat_b200.mesh import make_pack, perturb
from tssplat_b200.newton import DevicePCG
C3 = 1e-4
HBM = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--sizes", default="64,1024")
    ap.add_argument("--out", default=None, help="directory for time_hessian.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_hessian.py needs a CUDA device")
    dev = card()
    print(f"device: {dev}", flush=True)
    results = []
    for S in (int(v) for v in args.sizes.split(",")):
        pack = make_pack(S, TETS, seed=0, unique=8)
        sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), enable_amips=True)
        s = torch.cuda.Stream()
        for hessian in ("exact", "psd"):
            pcg = DevicePCG(sp, hessian=hessian)
            hs = DeviceHessian(pcg)
            vals = torch.empty((hs.nnzb, 3, 3), device="cuda")
            print(f"{S}x{TETS} {hessian}: nnzb {hs.nnzb}, values {36 * hs.nnzb / 1e6:.1f} MB, workspace "
                  f"{hs.device_bytes / 1e6:.1f} MB", flush=True)
            for sig in (0.02, 0.35):
                x = torch.from_numpy(perturb(pack, sigma_rel=sig, seed=0)).cuda()
                v = torch.randn_like(x)
                hv = torch.empty_like(x)
                planes = torch.empty((2,) + tuple(x.shape), device="cuda")
                c1, c2 = 2e-4 / S, 2e-4
                for c3 in (0.0, C3):
                    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=c3)
                    fns = {
                        "assemble": lambda: _capi.lib.tsb_hessian_assemble(hs._hs, x.data_ptr(), C.byref(terms), vals.data_ptr(),
                                                                           s.cuda_stream),
                        "hvp_ex": lambda: _capi.lib.tsb_hvp_ex(sp._h, x.data_ptr(), v.data_ptr(), C.byref(terms), 1.0, None,
                                                               hv.data_ptr(), None, s.cuda_stream),
                        "hess_diag": lambda: _capi.lib.tsb_hess_diag(sp._h, x.data_ptr(), C.byref(terms), 1.0, None,
                                                                     planes.data_ptr(), s.cuda_stream)}
                    times = alternate({k: capture(fn, s, args.launches, 3, k) for k, fn in fns.items()}, args.rounds,
                                      calls=args.launches)
                    us = {k: float(np.median(t)) for k, t in times.items()}
                    bw = 36 * hs.nnzb / (us["assemble"] * 1e-6)
                    r = {"spheres": S, "tets": S * TETS, "hessian": hessian, "sigma_rel": sig, "amips_c3": c3, "nnzb": hs.nnzb,
                         "us_per_call": us,
                         "us_per_call_p10_p90": {k: p10_p90(t) for k, t in times.items()},
                         "values_bytes_per_s": bw, "share_of_3_35_TBps": bw / HBM, "device": dev}
                    print(f"{S}x{TETS} {hessian:5s} sigma {sig:<5g} c3={c3:<6g} assemble {us['assemble']:9.1f}  hvp_ex "
                          f"{us['hvp_ex']:8.1f}  hess_diag {us['hess_diag']:8.1f} us   values {bw / 1e12:.2f} TB/s "
                          f"({100 * bw / HBM:.0f}% of 3.35)", flush=True)
                    results.append(r)
            del hs, pcg, vals
            torch.cuda.empty_cache()
        del sp
        torch.cuda.empty_cache()
    write_json(args.out, "time_hessian.json", results)


if __name__ == "__main__":
    main()

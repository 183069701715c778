"""Cost of the projected Hessian (tsb_pcg_hvp_psd, the PSD solve and the PSD Newton step) against the exact one, timed
with CUDA events in one process.

Packs: 64 x 4096 and 1024 x 4096 tets, "benign" (every sphere at 0.02 h) and "inverted" (every fourth sphere at 0.35 h,
with inverted tets); c1 = 2e-4 / S, c2 = 2e-4, order 2, AMIPS off and on (c3 = 1e-4); a deterministic handle.  Arms,
each one CUDA graph of `--launches` calls, replayed alternately for `--rounds` rounds (median, min, max in us per call):
  hvp_ex        tsb_hvp_ex
  hvp_psd       tsb_pcg_hvp_psd: the projection launch plus the projected product
  solve{10,20}  tsb_pcg_solve, unshifted, max_iter 10 and 20, exact and PSD workspaces: the slope over 10 iterations is
                the cost of one iteration (product and the three PCG kernels)
  step{10,20}   one tsb_newton_step (copy the start into x, reset, step) at max_iter 10 and 20, exact and PSD
  project       the projection launch alone: psd_project_kernel's mean duration over `--launches` tsb_pcg_hvp_psd calls
                under torch.profiler (CUDA activity; the kernel's own time, no launch gap)
The SM clock (nvidia-smi clocks.sm) is read while about half a second of the PSD step's replays is queued.

Time to solution (--tts): the mixed 64 x 4096 pack of tools/time_newton.py (every fourth sphere at 0.35 h, the rest at
0.02 h; c1 = 2e-4 / 64, c2 = 2e-4, AMIPS off and on), DeviceNewton.step with gtol = 1e-3 times the smallest starting
|g_c| of the quiet spheres, exact against PSD: steps and summed CUDA-event step time until every quiet sphere's |g_c| has
fallen by 1e3 (the criterion of time_newton.py's table), and until every sphere's has, up to `--max-steps` steps;
`--tts-rounds` rounds alternating the arms, median time.  The gradient norms between steps are not timed.

Usage: python tools/time_psd.py [--rounds 5] [--launches 10] [--big] [--tts] [--out DIR]"""
import argparse
import ctypes as C
import json

import numpy as np
import torch

from _timing import (TETS, alternate, capture, card, mixed_pack, sm_clock_under_load, sphere_gnorm, sphere_ids, summary,
                     timed, write_json)
from tssplat_b200 import _capi
from tssplat_b200 import tet_spheres_ext as ext
from tssplat_b200.newton import DeviceNewton, DevicePCG

C3 = 1e-4
ROUGH_EVERY = {"benign": None, "inverted": 4}      # "inverted": every fourth sphere at 0.35 h


def project_us(wp, x, v, terms, hv, curv, launches):
    """Mean device time of psd_project_kernel over `launches` tsb_pcg_hvp_psd calls, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    st = torch.cuda.current_stream().cuda_stream
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(launches):
            assert _capi.lib.tsb_pcg_hvp_psd(wp._s, x.data_ptr(), v.data_ptr(), C.byref(terms), hv.data_ptr(), curv.data_ptr(), st) == 0
        torch.cuda.synchronize()
    ts = [e.device_time for e in prof.events() if "psd_project_kernel" in e.name]
    return float(np.mean(ts)) if ts else None


def time_to_solution(args, dev, results):
    S = 64
    pack, x_np, quiet = mixed_pack(S, 0, 0, 4)
    x0 = torch.from_numpy(x_np).cuda()
    c1, c2 = 2e-4 / S, 2e-4
    sid = sphere_ids(pack).cuda()
    quiet = torch.from_numpy(quiet).cuda()
    for c3 in (0.0, C3):
        sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), enable_amips=True, deterministic=True)
        arms = {"exact": DeviceNewton(sp), "psd": DeviceNewton(sp, hessian="psd")}
        g0 = sphere_gnorm(sp, x0, c1, c2, c3, sid, S)
        target, gtol = g0 / 1e3, float(g0[quiet].min()) * 1e-3
        out = {k: [] for k in arms}
        for _ in range(args.tts_rounds):
            for name, nw in arms.items():
                x = x0.clone()
                nw.reset()
                total, t_quiet, n_quiet, n_all = 0.0, None, None, None
                for step in range(1, args.max_steps + 1):
                    total += timed(lambda: nw.step(x, c1, c2, 2, c3=c3, gtol=gtol))[0]
                    ok = sphere_gnorm(sp, x, c1, c2, c3, sid, S) <= target
                    if n_quiet is None and bool(ok[quiet].all()):
                        n_quiet, t_quiet = step, total
                    if bool(ok.all()):
                        n_all = step
                        break
                out[name].append((n_quiet, t_quiet, n_all, total,
                                  float((sphere_gnorm(sp, x, c1, c2, c3, sid, S) / g0)[~quiet].max())))
        r = {"case": f"64x{TETS} mixed, c3={c3:g}, time to |g_c| / 1e3", "device": dev,
             "arms": {k: {"steps_quiet": v[0][0], "ms_quiet_median": None if v[0][1] is None else float(np.median([q[1] for q in v])) / 1e3,
                          "steps_all": v[0][2], "ms_total_median": float(np.median([q[3] for q in v])) / 1e3,
                          "worst_rough_ratio_at_end": v[0][4]} for k, v in out.items()}}
        print(json.dumps(r, indent=1), flush=True)
        results.append(r)
        del arms, sp
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--big", action="store_true", help="also the 1024 x 4096 packs")
    ap.add_argument("--tts", action="store_true", help="also time to solution on the mixed 64 x 4096 pack")
    ap.add_argument("--tts-only", action="store_true", help="only time to solution")
    ap.add_argument("--max-steps", type=int, default=60)
    ap.add_argument("--tts-rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for time_psd.json")
    args = ap.parse_args()
    dev = card()
    print(f"device: {dev}", flush=True)
    L = _capi.lib
    results = []
    for S in (() if args.tts_only else (64, 1024) if args.big else (64,)):
        for kind in ("benign", "inverted"):
            pk, x_np, _ = mixed_pack(S, 1, 3, ROUGH_EVERY[kind])
            sp = ext.TetSpheres(pk.verts.reshape(-1), pk.tets.reshape(-1), enable_amips=True, deterministic=True)
            we, wp = DevicePCG(sp), DevicePCG(sp, hessian="psd")
            ne, npd = DeviceNewton(sp, we), DeviceNewton(sp, wp)
            x0 = torch.from_numpy(x_np).cuda()
            v = torch.randn_like(x0)
            hv, d = torch.empty_like(x0), torch.empty_like(x0)
            curv = torch.empty(4, device="cuda")
            for c3 in (0.0, C3):
                c1, c2 = 2e-4 / S, 2e-4
                terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=c3)
                _, b = sp.energy_grad(x0, c1, c2, 2, -1.0, c3=c3)
                for w in (we, wp):
                    w.set_blocks(sp.hess_diag(x0, c1, c2, 2, c3=c3))
                xs = {k: x0.clone() for k in ("e10", "e20", "p10", "p20")}
                s = torch.cuda.Stream()
                st = s.cuda_stream
                o10 = _capi.tsb_pcg_options_t(max_iter=10, rtol=0.0, check_every=0)
                o20 = _capi.tsb_pcg_options_t(max_iter=20, rtol=0.0, check_every=0)

                def step(nw, key, it):
                    def f():
                        xs[key].copy_(x0)
                        nw.reset()
                        nw.step(xs[key], c1, c2, 2, c3=c3, max_iter=it)
                    return f

                fns = {
                    "hvp_ex": lambda: L.tsb_hvp_ex(sp._h, x0.data_ptr(), v.data_ptr(), C.byref(terms), 1.0, None, hv.data_ptr(),
                                                   curv.data_ptr(), st),
                    "hvp_psd": lambda: L.tsb_pcg_hvp_psd(wp._s, x0.data_ptr(), v.data_ptr(), C.byref(terms), hv.data_ptr(),
                                                         curv.data_ptr(), st),
                    "solve10_exact": lambda: L.tsb_pcg_solve(we._s, x0.data_ptr(), b.data_ptr(), C.byref(terms), C.byref(o10),
                                                             d.data_ptr(), None, None, st),
                    "solve20_exact": lambda: L.tsb_pcg_solve(we._s, x0.data_ptr(), b.data_ptr(), C.byref(terms), C.byref(o20),
                                                             d.data_ptr(), None, None, st),
                    "solve10_psd": lambda: L.tsb_pcg_solve(wp._s, x0.data_ptr(), b.data_ptr(), C.byref(terms), C.byref(o10),
                                                           d.data_ptr(), None, None, st),
                    "solve20_psd": lambda: L.tsb_pcg_solve(wp._s, x0.data_ptr(), b.data_ptr(), C.byref(terms), C.byref(o20),
                                                           d.data_ptr(), None, None, st),
                }
                t = alternate({k: capture(f, s, args.launches, 3, k) for k, f in fns.items()}, args.rounds,
                              calls=args.launches)
                t = {k: summary(vv) for k, vv in t.items()}
                steps = {"step10_exact": step(ne, "e10", 10), "step20_exact": step(ne, "e20", 20),
                         "step10_psd": step(npd, "p10", 10), "step20_psd": step(npd, "p20", 20)}
                tv = alternate({k: capture(f, s, 1, 3, k) for k, f in steps.items()}, args.rounds)
                t.update({k: summary(vv) for k, vv in tv.items()})
                r = dict(S=S, kind=kind, c3=c3, times_us=t)
                iter_e = (t["solve20_exact"]["median"] - t["solve10_exact"]["median"]) / 10
                iter_p = (t["solve20_psd"]["median"] - t["solve10_psd"]["median"]) / 10
                r["iter_us"] = dict(exact=iter_e, psd=iter_p)
                r["psd_over_ex"] = t["hvp_psd"]["median"] / t["hvp_ex"]["median"]
                r["project_us"] = project_us(wp, x0, v, terms, hv, curv, args.launches)
                print(f"{S} x {TETS} {kind} c3={c3}: hvp_ex {t['hvp_ex']['median']:.1f} us, hvp_psd {t['hvp_psd']['median']:.1f} us "
                      f"({r['psd_over_ex']:.2f}x), projection alone {r['project_us']:.1f} us; solve iteration exact {iter_e:.1f} psd {iter_p:.1f} us; step10 exact "
                      f"{t['step10_exact']['median']:.1f} psd {t['step10_psd']['median']:.1f}; step20 exact "
                      f"{t['step20_exact']['median']:.1f} psd {t['step20_psd']['median']:.1f} us", flush=True)
                results.append(r)
            g = capture(step(npd, "p10", 10), s, 1, 1)
            results[-1]["sm_mhz_under_load"] = sm_clock_under_load(g, results[-1]["times_us"]["step10_psd"]["median"])
            print(f"SM clock under load {results[-1]['sm_mhz_under_load']} MHz", flush=True)
            del g, ne, npd, we, wp, sp
            torch.cuda.empty_cache()
    if args.tts or args.tts_only:
        time_to_solution(args, dev, results)
    write_json(args.out, "time_psd.json", dict(device=dev, results=results))


if __name__ == "__main__":
    main()

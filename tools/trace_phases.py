"""Phase timeline of the fused kernel from device-side stamps (profiling build, -DTSB_TRACE).

    python tools/trace_phases.py build          # here (no GPU): nvcc -> tssplat_b200/libtssplat_b200_trace.so
    python tools/trace_phases.py run [S ...]    # on the GPU box

Thread 0 of every CTA stamps clock64 at: 1 entry, 2 prologue done (first TMA chunk issued), 3 after
griddepcontrol.wait, 4 first component staged, 5 warp-0 rows of first segment done, 6 warp-0 tets done,
7 all segments done, 8 CTA energy barrier, 9 ticket atomic returned, 10 exit; 0/11 = globaltimer.  Lane 0 of warp w
stamps clock64 in slot 16 + w when its last chunk wait returns (the wait for the last chunk of its stream)."""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
TRACE_LIB = os.path.join(ROOT, "tssplat_b200", "libtssplat_b200_trace.so")
SLOTS = 32                    # tsb_kernels.cuh kTraceSlots: 16 phase stamps, then one per warp


def build():
    from tssplat_b200 import build as b
    cmd = [b._nvcc(), *b.NVCC_FLAGS, "-DTSB_TRACE", "-shared", "-o", TRACE_LIB, *[os.path.join(b.CSRC, s) for s in b.SOURCES]]
    env = dict(os.environ); env.pop("CC", None); env.pop("CXX", None)
    subprocess.run(cmd, check=True, env=env)
    print(TRACE_LIB)


def run(sizes):
    os.environ["TSSPLAT_B200_LIB"] = TRACE_LIB
    import numpy as np
    import torch
    from tssplat_b200 import _capi
    from tssplat_b200 import tet_spheres_ext as ext
    from tssplat_b200.mesh import make_pack, perturb
    lib = _capi.lib
    lib.tsb_trace_read.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    names = ["prologue", "gdc.wait", "stage0+sync", "rows(w0,seg0)", "tets(w0,seg0)", "rest of segs",
             "energy bar", "partial store", "tail(reducer)"]
    for S in sizes:
        for kw in ({}, {"warps_per_cta": 8, "ring_slots": 2}):
            pack = make_pack(S, 4096, seed=0, unique=8)
            sp = ext.TetSpheres(pack.verts.reshape(-1), pack.tets.reshape(-1), **kw)
            x = torch.from_numpy(perturb(pack, sigma_rel=0.02, seed=0)).cuda()
            energy = torch.zeros(3, device="cuda"); grad = torch.empty((pack.n, 3), device="cuda")
            st = torch.cuda.Stream()
            G = sp.info["grid"]
            with torch.cuda.stream(st):
                for _ in range(20):
                    lib.tsb_energy_grad(sp._h, x.data_ptr(), 2e-4 / S, 2e-4, 2, 1.0, None, energy.data_ptr(), grad.data_ptr(), st.cuda_stream)
                st.synchronize()
            tr = np.zeros((G, SLOTS), dtype=np.uint64)
            lib.tsb_trace_read(sp._h, tr.ctypes.data, tr.size)
            tr = tr.astype(np.int64)
            dur_ns = tr[:, 11].max() - tr[:, 0].min()
            d = np.diff(tr[:, 1:11], axis=1) / 1.965     # cycles -> ns at 1965 MHz
            print(f"S={S} {kw}: grid={G} kernel span {dur_ns} ns (first entry -> last exit); entry spread {tr[:, 0].max() - tr[:, 0].min()} ns; "
                  f"exit spread {tr[:, 11].max() - tr[:, 11].min()} ns; per-CTA total median {np.median(tr[:, 11] - tr[:, 0]):.0f} ns")
            for k, nm in enumerate(names[:d.shape[1]]):
                print(f"    {nm:18s} median {np.median(d[:, k]):8.0f} ns   max {d[:, k].max():8.0f} ns")
            inner = np.stack([tr[:, 12] - tr[:, 4], tr[:, 13] - tr[:, 12], tr[:, 14] - tr[:, 13], tr[:, 5] - tr[:, 14]], 1) / 1.965
            info = tr[:, 15]
            print("    inside rows(w0,seg0): begin-wait / seg setup loads / first RB / other RBs (median ns) = " +
                  " / ".join(f"{v:.0f}" for v in np.median(inner, 0)) +
                  f"; warp0 first RB len4 median {np.median(info & 0xFFFF):.0f}, RBs {np.median((info >> 16) & 0xFF):.0f}, tet cells {np.median((info >> 24) & 0xFF):.0f}")
            post = (tr[:, 9] - tr[:, 3]) / 1.965        # after griddepcontrol.wait -> partial stored
            try:                                         # correlate with the plan (host-side inspection library)
                sys.path.insert(0, os.path.join(ROOT, "tests"))
                from _helpers import build_host_plan
                pl = build_host_plan(pack.verts, pack.tets, nw=sp.info["warps_per_cta"], grid=G)
                NWp = pl["nw"]
                cells = pl["wdesc"].reshape(G, NWp, 2)[:, :, 1] // 768
                nseg = np.diff(pl["cta_seg"].reshape(G, 2), axis=1).ravel()
                ws_ = pl["wseg"].reshape(-1, NWp, 2)
                rbs = np.array([ws_[a:b, :, 0].sum() for a, b in pl["cta_seg"].reshape(G, 2)])
                # CTAs whose slowest warp has more cells than its ring holds: that warp waits on a ring refill
                big = cells.max(1) > 2 * 6
                busy = cells.sum(1) > 0
                wmax = cells.argmax(1)
                lw = tr[np.arange(G), 16 + wmax]
                last = np.where(lw > 0, (lw - tr[:, 3]) / 1.965, np.nan)    # its last chunk wait, after the gdc.wait
                for nm, m in (("slowest warp > 12 cells", big & busy), ("slowest warp <= 12 cells", ~big & busy)):
                    if m.any():
                        lm = last[m][np.isfinite(last[m])]      # empty when the warp's whole stream is one chunk
                        print(f"    {nm:25s}: {m.sum():3d} CTAs  post-wait median {np.median(post[m]):.0f} max {post[m].max():.0f} ns  " +
                              (f"last chunk wait of that warp median {np.median(lm):.0f} max {lm.max():.0f} ns after gdc.wait" if lm.size else "no chunk wait"))
                for k in sorted(set(nseg.tolist())):
                    m = nseg == k
                    print(f"    CTAs with {k} segment(s): {m.sum():3d}  post-wait mean {post[m].mean():.0f} ns  total cells {cells[m].sum(1).mean():.0f}  "
                          f"max warp cells {cells[m].max(1).mean():.1f}  row blocks {rbs[m].mean():.1f}  stage {d[m, 2].mean():.0f}  rows(w0,seg0) {d[m, 3].mean():.0f}  rest {d[m, 5].mean():.0f}")
            except Exception as ex:
                print("    (plan correlation unavailable:", ex, ")")
            pct = np.percentile(post, [0, 25, 50, 75, 90, 100])
            worst = int(np.argmax(post))
            print("    post-wait work per CTA (ns): min/25/50/75/90/max = " + "/".join(f"{v:.0f}" for v in pct) +
                  f"; slowest CTA {worst}: " + " ".join(f"{v:.0f}" for v in d[worst]))
            sys.stdout.flush()




def launch_floor():
    """Per-launch cost of a trivial kernel chain in a CUDA graph (the floor any one-launch step pays)."""
    import torch
    from tssplat_b200 import _capi
    lib = _capi.lib
    a = torch.zeros(1024, device="cuda"); b = torch.zeros(1024, device="cuda")
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(3):
            lib.tsb_scale(a.data_ptr(), 1024, 1.0, None, b.data_ptr(), st.cuda_stream)
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for _ in range(50):
                lib.tsb_scale(a.data_ptr(), 1024, 1.0, None, b.data_ptr(), st.cuda_stream)
        g.replay(); st.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(20):
            g.replay()
        e1.record(st); st.synchronize()
    print(f"trivial kernel chain in a graph: {e0.elapsed_time(e1) * 1e3 / 1000:.2f} us per launch")


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "build":
        build()
    else:
        run([int(a) for a in sys.argv[2:]] or [16, 64])
        launch_floor()

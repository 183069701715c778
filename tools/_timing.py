"""The harness the time_*.py scripts share: the card query, CUDA-event and CUDA-graph timers, the packs they measure on
and the per-sphere gradient norm of their time-to-solution loops.  Importing it puts the repository root on sys.path.

Each script passes its own warm-up count, calls per graph, replays per round, rounds and pack seeds: they differ between
scripts, and unifying them would change the state or the inputs a script times, and so the numbers DESIGN.md cites."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tssplat_b200.mesh import make_pack, perturb  # noqa: E402

TETS = 4096


def card(fields="name,power.limit,clocks.max.sm"):
    """The first GPU's `fields` as nvidia-smi prints them, or torch's device name where nvidia-smi cannot be run."""
    q = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def sm_clock():
    """The current SM clock in MHz (nvidia-smi clocks.sm), or None where it cannot be read."""
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"], capture_output=True, text=True)
    try:
        return int(q.stdout.strip().splitlines()[torch.cuda.current_device()])
    except (ValueError, IndexError):
        return None


def sm_clock_under_load(g, us_per_replay):
    """clocks.sm read while about 0.5 s of replays of the graph g is queued (enqueue, read, synchronise)."""
    for _ in range(max(1, int(5e5 / us_per_replay))):
        g.replay()
    mhz = sm_clock()
    torch.cuda.synchronize()
    return mhz


def summary(v):
    return dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v)))


def p10_p90(v):
    return [float(np.percentile(v, 10)), float(np.percentile(v, 90))]


def _check(rc, arm):
    """An int result is a C return code; anything else (None, a tensor, a record) is not checked."""
    if isinstance(rc, int) and rc != 0:
        raise RuntimeError(f"{arm}: returned {rc}")


def timed(fn):
    """(us, fn()): one CUDA event pair on the current stream around fn, synchronised on the second."""
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    out = fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) * 1e3, out


def capture(fn, stream, calls, warmup, arm="fn"):
    """A CUDA graph of `calls` calls of fn captured on `stream`, after `warmup` calls on it outside the capture
    (module loading, first-use allocations).  stream=None warms up on the current stream and captures on torch's."""
    with torch.cuda.stream(stream):
        for _ in range(warmup):
            _check(fn(), arm)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        for _ in range(calls):
            _check(fn(), arm)
    return g


def alternate(arms, rounds, reps=1, calls=1, before=None, warmup=0):
    """{arm: [us per call in each round]}.  First every arm runs `warmup` times untimed; then every round runs the arms
    in turn: before(arm) untimed and synchronised when given, then `reps` runs between two CUDA events, divided by
    reps * calls (the calls one run makes).  A CUDAGraph arm is replayed, any other is called."""
    runs = {k: (a.replay if isinstance(a, torch.cuda.CUDAGraph) else a) for k, a in arms.items()}
    for k, run in runs.items():
        for _ in range(warmup):
            _check(run(), k)
    if warmup:
        torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, run in runs.items():
            if before is not None:
                before(k)
                torch.cuda.synchronize()
            us, _ = timed(lambda: [_check(run(), k) for _ in range(reps)])
            times[k].append(us / (reps * calls))
    return times


def steps_until(step, reached, max_steps):
    """(steps, us, reached): calls step() up to max_steps times, each timed with one event pair, and after each call
    reached() untimed; stops at the first True.  us sums the steps' times."""
    total = 0.0
    for k in range(1, max_steps + 1):
        total += timed(step)[0]
        if reached():
            return k, total, True
    return max_steps, total, False


def mixed_pack(S, x_seed, rough_seed, rough_every):
    """(pack, x, quiet) on make_pack(S, 4096, seed=0, unique=8): x is the pack at 0.02 h (perturb seed x_seed) except
    the spheres k with k % rough_every == 0, which are at 0.35 h (perturb seed rough_seed); rough_every=None leaves every
    sphere at 0.02 h, 1 makes every sphere rough.  quiet marks the spheres at 0.02 h.  The scripts use two mixed
    64 x 4096 packs that differ only in the seeds, (0, 0) and (1, 3): tools/README.md lists which uses which."""
    pk = make_pack(S, TETS, seed=0, unique=8)
    x = perturb(pk, sigma_rel=0.02, seed=x_seed)
    quiet = np.ones(S, bool) if rough_every is None else np.arange(S) % rough_every != 0
    if not quiet.all():
        rough = perturb(pk, sigma_rel=0.35, seed=rough_seed)
        vo = pk.vert_offsets
        for k in np.flatnonzero(~quiet):
            x[vo[k]:vo[k + 1]] = rough[vo[k]:vo[k + 1]]
    return pk, x, quiet


def sphere_ids(pk):
    """The sphere of every vertex, int64 [n] on the CPU."""
    return torch.from_numpy(np.repeat(np.arange(pk.num_spheres), np.diff(pk.vert_offsets)))


def sphere_gnorm(sp, x, c1, c2, c3, sid, S):
    """fp64 |g_c| per sphere of the order-2 energy's gradient at x; sid from sphere_ids, on the device."""
    _, g = sp.energy_grad(x, c1, c2, 2, c3=c3)
    return torch.zeros(S, dtype=torch.float64, device="cuda").index_add_(0, sid, (g.double() ** 2).sum(1)).sqrt()


def write_json(out_dir, name, obj):
    """Writes obj to out_dir/name (indent 1); nothing when out_dir is None."""
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, name), "w") as f:
            json.dump(obj, f, indent=1)

"""Drop-in for the reference's ``tet_spheres_ext`` pybind11 module
(``tssplat_ext/tet_spheres/tet_spheres.cpp:225-266``): same names, same argument meaning.

    from tet_spheres import tet_spheres_ext        # energies/smooth_barrier.py:6, unchanged
    tet_sp = tet_spheres_ext.TetSpheres(v_flat, f_flat)
    e = tet_spheres_ext.forward(x, tet_sp, c1, c2, order)
    g = tet_spheres_ext.backward(grad_output, x, tet_sp, c1, c2, order)

Underneath: one sm_90a kernel launch through the C ABI (``include/tssplat_b200.h``) computes the
energy AND the gradient; ``backward`` only rescales the cached gradient by ``grad_output``.
PyTorch is used for device memory and the current stream, nothing else.

Deliberate differences from the reference (SURVEY.md section 2.4), all on error / sync behaviour:

* ``forward`` returns a 0-dim tensor on ``x``'s device instead of a CPU scalar
  (``tet_spheres_cuda.cu:194``) -- no host sync.  Set ``return_cpu_scalar = True`` for the
  reference's behaviour.
* bad constructor input raises ``RuntimeError`` instead of printing to stderr and returning a
  half-constructed object (``tet_spheres.cpp:240,249``).
* ``order`` outside {2,4} raises instead of silently returning zeros (``tet_spheres_cuda.cu:57-63``).
* ``grad_limit`` does what it was meant to (scale by the arg-max magnitude), silently.
* no module-import side effect (``pgo_init`` + "initializing" print, ``tet_spheres.cpp:14-30``).
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import _capi
from .mesh import load_veg

__all__ = ["TetSpheres", "SphereStats", "LineSearch", "forward", "backward", "hvp", "line_search", "hess_diag", "newton_step",
           "random_x",
           "grad_limit", "energy_grad_host"]

return_cpu_scalar = False
_limit_work = {}       # (device, stream) -> float32[4] scratch of grad_limit (caller-owned in the C ABI)
#: compute the gradient inside ``forward`` (one launch per iteration) when ``x.requires_grad``
fuse_backward_into_forward = True


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _stream_ptr(device) -> int:
    """cudaStream_t of torch's current stream on ``device`` (the raw query when torch exposes it: the public
    ``torch.cuda.current_stream`` costs several microseconds per call)."""
    if _raw_stream is not None:
        return int(_raw_stream(device.index if isinstance(device, torch.device) else int(device)))
    return int(torch.cuda.current_stream(device).cuda_stream)


class SphereStats(NamedTuple):
    """Geometry statistics per connected component (= tet-sphere), device tensors of length S = number of components,
    in the order of the components' lowest vertex ids (``tsb_sphere_stats_t`` in ``include/tssplat_b200.h``)."""
    smooth: torch.Tensor        # f64: 1/2 u^T M u over the sphere's rows (unweighted)
    barrier: torch.Tensor       # f64: sum of max(-J, 0)^order over its tets
    amips: torch.Tensor         # f64: AMIPS sum over its J > 0 tets (0 unless c3 != 0)
    min_J: torch.Tensor         # f32: smallest det F of its tets
    n_inverted: torch.Tensor    # i32: tets with J < 0
    n_tets: torch.Tensor        # i32
    first_vertex: torch.Tensor  # i32: lowest vertex id of the sphere


_STATS_BYTES = C.sizeof(_capi.tsb_sphere_stats_t)     # 40


class LineSearch(NamedTuple):
    """What ``TetSpheres.line_search`` returns, device tensors (``tsb_line_search`` in ``include/tssplat_b200.h``).
    K = number of step sizes, S = number of components (spheres, in the order of their lowest vertex ids)."""
    delta: torch.Tensor                        # f32 [K, 4]: (c1 ds + c2 db + c3 da, ds, db, da) = E(x + alpha_k d) - E(x)
    max_step: torch.Tensor                     # f32 []: first alpha in (0, max alphas] at which a tet inverts (+inf: none)
    sphere_delta: Optional[torch.Tensor]       # f32 [S, K, 4] per sphere, or None
    sphere_max_step: Optional[torch.Tensor]    # f32 [S] per sphere, or None


class TetSpheres:
    """State object (replaces ``struct TetSpheres``, ``tet_spheres.h:24-42``).

    ``TetSpheres(vertices, elements)``: ``vertices`` 1-D C-contiguous float32 of length 3n (REST
    positions), ``elements`` 1-D C-contiguous int32 of length 4*nele, 0-based
    (``tet_spheres.cpp:234-258``).  ``TetSpheres(filename)`` loads a ``.veg`` file
    (``tet_spheres.cpp:108-117``).

    ``deterministic=True``: the gradient is bitwise repeatable also with inverted tets and the AMIPS term (a second
    launch adds the tets' contributions in a fixed order; see ``tsb_energy_grad`` in the header).  Callers that set
    ``torch.use_deterministic_algorithms(True)`` should pass it: the flag is not followed automatically.
    """

    def __init__(self, vertices, elements=None, *, device=None, warps_per_cta: int = 0,
                 laplacian_scale: int = 0, force_global: bool = False, ring_slots: int = 0, enable_amips: bool = False,
                 deterministic: bool = False):
        self._h = None
        if isinstance(vertices, (str, bytes)) and elements is None:
            v, t = load_veg(vertices if isinstance(vertices, str) else vertices.decode())
            vertices = v.astype(np.float32).reshape(-1)
            elements = t.astype(np.int32).reshape(-1)
        if elements is None:
            raise RuntimeError("TetSpheres(vertices, elements): elements missing")
        vertices = np.asarray(vertices)
        elements = np.asarray(elements)
        if vertices.ndim != 1 or vertices.dtype != np.float32:
            raise RuntimeError(f"Wrong vertex type:{vertices.ndim},{vertices.dtype} (need 1-D float32)")
        if elements.ndim != 1 or elements.dtype != np.int32:
            raise RuntimeError(f"Wrong tet type:{elements.ndim},{elements.dtype} (need 1-D int32)")
        if vertices.size % 3 or elements.size % 4:
            raise RuntimeError("vertices must have 3n entries and elements 4*nele entries")
        vertices = np.ascontiguousarray(vertices)
        elements = np.ascontiguousarray(elements)
        if not torch.cuda.is_available():
            raise RuntimeError("tet_spheres_ext needs a CUDA device (H100); there is no CPU path")
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("tet_spheres_ext needs a CUDA device")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        torch.cuda.init()
        opt = _capi.tsb_options_t(warps_per_cta=int(warps_per_cta), laplacian_scale=int(laplacian_scale),
                                  ring_slots=int(ring_slots), force_global=int(bool(force_global)),
                                  enable_amips=int(bool(enable_amips)), deterministic=int(bool(deterministic)))
        h = C.c_void_p()
        rc = _capi.lib.tsb_create(vertices.ctypes.data, elements.ctypes.data, vertices.size // 3,
                                  elements.size // 4, C.byref(opt), self.device.index, C.byref(h))
        _capi.check(rc, None, "TetSpheres")
        self._h = h
        # copies of the mesh the handle was built from (flat float32 rest positions, flat int32 tets), so that a caller
        # changing its arrays later does not change what DevicePCG(hessian="psd") hands to tsb_pcg_enable_psd
        self.vertices, self.elements = vertices.copy(), elements.copy()
        info = _capi.tsb_info_t()
        _capi.check(_capi.lib.tsb_get_info(self._h, C.byref(info)), self._h, "TetSpheres")
        self.info = {k: getattr(info, k) for k, _ in _capi.tsb_info_t._fields_}
        self.n = int(info.n)
        self.nele = int(info.nele)
        self.n3 = 3 * self.n
        self.deterministic = bool(deterministic)
        self._cache_key = None
        self._cache_grad: Optional[torch.Tensor] = None
        # energies of the last 32 launches (a ring, so a loss tensor stays valid while it is being logged)
        self._energy_ring = torch.zeros((32, 4), dtype=torch.float32, device=self.device)
        self._ring_i = 0
        self._ring_ptr = self._energy_ring.data_ptr()
        self._ring3 = [self._energy_ring[i, :3] for i in range(32)]       # views made once, not per launch
        self._ring4 = [self._energy_ring[i] for i in range(32)]

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        ns, self._native = getattr(self, "_native", None), None
        if ns:
            try:
                ns[0].state_free(ns[1])
            except Exception:  # interpreter shutdown
                pass
        if h:
            try:
                _capi.lib.tsb_destroy(h)
            except Exception:  # interpreter shutdown
                pass

    def native_state(self):
        """(module, state) of the C++ autograd bridge for this handle, or None when it is not built
        (``tssplat_b200.native_autograd``)."""
        ns = getattr(self, "_native", None)
        if ns is None:
            from . import native_autograd
            mod = native_autograd.module()
            if mod is None:
                return None
            ns = self._native = (mod, mod.state_new(int(self._h.value), self.n, int(self.device.index)))
        return ns

    # ------------------------------------------------------------------------------------------
    def _check_x(self, x: torch.Tensor) -> torch.Tensor:
        if not isinstance(x, torch.Tensor) or x.dtype != torch.float32 or not x.is_cuda:
            raise RuntimeError("vertexPositions must be a float32 CUDA tensor")
        if x.device != self.device:
            raise RuntimeError(f"vertexPositions is on {x.device}, TetSpheres on {self.device}")
        if x.numel() != self.n3:
            raise RuntimeError(f"vertexPositions has {x.numel()} entries, expected {self.n3}")
        return x if x.is_contiguous() else x.contiguous()            # tet_spheres_cuda.cu:124

    def _gradH_arg(self, gradH):
        """gradH as the C ABI takes it: (host value, device pointer or None, tensor to keep alive until the launch is
        enqueued).  A CUDA tensor is read on the device (its first entry, as fp32); anything else is a host float."""
        if isinstance(gradH, torch.Tensor) and gradH.is_cuda:
            keep = gradH.detach().to(device=self.device, dtype=torch.float32).reshape(-1)[:1].contiguous()
            return 1.0, keep.data_ptr(), keep
        return float(gradH), None, None

    def energy_grad(self, x: torch.Tensor, c1: float, c2: float, order: int, gradH=1.0,
                    want_grad: bool = True, c3: float = 0.0):
        """The fused launch.  Returns (energy[3] = total/smooth/barrier on device, grad or None); with ``c3``
        (AMIPS coefficient, handle created with ``enable_amips=True``) the energy has a 4th entry, the AMIPS sum.
        The energy tensor is a slot of a 32-deep ring owned by the handle (no allocation per call)."""
        xc = self._check_x(x)
        i = self._ring_i
        self._ring_i = (i + 1) & 31
        energy = self._ring4[i] if c3 else self._ring3[i]
        e_ptr = self._ring_ptr + 16 * i
        grad = torch.empty((self.n, 3), dtype=torch.float32, device=self.device) if want_grad else None
        gh_val, gh_ptr, keep = self._gradH_arg(gradH)
        if c3:
            terms = _capi.tsb_terms_t(c1=float(c1), c2=float(c2), order=int(order), c3=float(c3))
            rc = _capi.lib.tsb_energy_grad_ex(self._h, xc.data_ptr(), C.byref(terms), gh_val, gh_ptr, e_ptr,
                                              grad.data_ptr() if want_grad else None, _stream_ptr(self.device))
        else:
            rc = _capi.lib.tsb_energy_grad(self._h, xc.data_ptr(), float(c1), float(c2), int(order), gh_val,
                                           gh_ptr, e_ptr, grad.data_ptr() if want_grad else None,
                                           _stream_ptr(self.device))
        if rc:
            _capi.check(rc, self._h, "tet_spheres_ext")
        del keep
        return energy, grad

    def energy_grad_spheres(self, x: torch.Tensor, c1: float, c2: float, order: int, gradH=1.0, want_grad: bool = True,
                            c3: float = 0.0):
        """``energy_grad`` plus per-sphere statistics (``tsb_energy_grad_spheres``): returns (energy[4] = total / smooth /
        barrier / AMIPS, grad or None, ``SphereStats``), all on the device, without a host sync.  Every call allocates
        fresh output tensors (this is a diagnostic call, not the training step).  The records of a sharded run
        (``ShardedEnergy``) cover the rank's own ``sphere_range`` and carry ``first_vertex`` in the rank's local
        numbering."""
        xc = self._check_x(x)
        S = int(self.info["n_components"])
        energy = torch.empty(4, dtype=torch.float32, device=self.device)
        grad = torch.empty((self.n, 3), dtype=torch.float32, device=self.device) if want_grad else None
        raw = torch.empty((S, _STATS_BYTES), dtype=torch.uint8, device=self.device)
        gh_val, gh_ptr, keep = self._gradH_arg(gradH)
        terms = _capi.tsb_terms_t(c1=float(c1), c2=float(c2), order=int(order), c3=float(c3))
        rc = _capi.lib.tsb_energy_grad_spheres(self._h, xc.data_ptr(), C.byref(terms), gh_val, gh_ptr, energy.data_ptr(),
                                               grad.data_ptr() if want_grad else None, raw.data_ptr(),
                                               _stream_ptr(self.device))
        if rc:
            _capi.check(rc, self._h, "tet_spheres_ext.energy_grad_spheres")
        del keep
        f = _capi.record_fields(raw, _capi.tsb_sphere_stats_t)
        return energy, grad, SphereStats(*(f[k] for k in SphereStats._fields))

    def hvp(self, x: torch.Tensor, v: torch.Tensor, c1: float, c2: float, order: int, gradH=1.0,
            want_curv: bool = False, c3: float = 0.0):
        """Hessian-vector product of ``c1 * smooth + c2 * barrier + c3 * amips`` at ``x`` along ``v``.  Returns
        (``gradH * H(x) v`` as [n,3], curvature or None), both on the device, no host sync.  The curvature is ``v^T H v``
        as [3] = (c1 vMv + c2 vHbv, vMv, vHbv), not scaled by ``gradH``; with ``c3`` (AMIPS coefficient, handle created
        with ``enable_amips=True``; ``tsb_hvp_ex``) it has a 4th entry, vHav, and its total includes ``c3 * vHav``, the
        same 3-vs-4 convention as ``energy_grad``.  ``c3 == 0`` is ``tsb_hvp``.  ``gradH`` may be a CUDA tensor (read
        on the device, like ``energy_grad``)."""
        xc = self._check_x(x)
        vc = self._check_x(v)
        hv = torch.empty((self.n, 3), dtype=torch.float32, device=self.device)
        curv = torch.empty(4 if c3 else 3, dtype=torch.float32, device=self.device) if want_curv else None
        gh_val, gh_ptr, keep = self._gradH_arg(gradH)
        if c3:
            terms = _capi.tsb_terms_t(c1=float(c1), c2=float(c2), order=int(order), c3=float(c3))
            rc = _capi.lib.tsb_hvp_ex(self._h, xc.data_ptr(), vc.data_ptr(), C.byref(terms), gh_val, gh_ptr, hv.data_ptr(),
                                      curv.data_ptr() if want_curv else None, _stream_ptr(self.device))
        else:
            rc = _capi.lib.tsb_hvp(self._h, xc.data_ptr(), vc.data_ptr(), float(c1), float(c2), int(order), gh_val,
                                   gh_ptr, hv.data_ptr(), curv.data_ptr() if want_curv else None, _stream_ptr(self.device))
        if rc:
            _capi.check(rc, self._h, "tet_spheres_ext.hvp")
        del keep
        return hv, curv

    def line_search(self, x: torch.Tensor, d: torch.Tensor, alphas, c1: float, c2: float, order: int, c3: float = 0.0,
                    per_sphere: bool = False) -> LineSearch:
        """Energy changes ``E(x + alpha_k d) - E(x)`` of ``c1 * smooth + c2 * barrier (+ c3 * amips)`` at up to 8 step
        sizes, per term, and the largest inversion-free step along ``d`` (``tsb_line_search``), in one pass over the plan
        and without a host sync.  ``alphas``: a sequence of floats, or a CUDA float32 tensor that is read on the device
        when the launch runs (so a captured CUDA graph can be replayed with new values written into it).  ``c3`` needs a
        handle created with ``enable_amips=True``.  ``per_sphere`` also returns each sphere's changes and step."""
        xc = self._check_x(x)
        dc = self._check_x(d)
        if isinstance(alphas, torch.Tensor):
            if not alphas.is_cuda or alphas.dtype != torch.float32 or alphas.device != self.device or not alphas.is_contiguous():
                raise RuntimeError("alphas must be a contiguous float32 tensor on the handle's device, or a sequence of floats")
            a = alphas.reshape(-1)
        else:
            a = torch.tensor([float(v) for v in alphas], dtype=torch.float32).to(self.device, non_blocking=True)
        K = int(a.numel())
        delta = torch.empty((K, 4), dtype=torch.float32, device=self.device)
        step = torch.empty((), dtype=torch.float32, device=self.device)
        S = int(self.info["n_components"])
        sd = torch.empty((S, K, 4), dtype=torch.float32, device=self.device) if per_sphere else None
        ss = torch.empty((S,), dtype=torch.float32, device=self.device) if per_sphere else None
        terms = _capi.tsb_terms_t(c1=float(c1), c2=float(c2), order=int(order), c3=float(c3))
        rc = _capi.lib.tsb_line_search(self._h, xc.data_ptr(), dc.data_ptr(), C.byref(terms), a.data_ptr(), K,
                                       delta.data_ptr(), step.data_ptr(), sd.data_ptr() if per_sphere else None,
                                       ss.data_ptr() if per_sphere else None, _stream_ptr(self.device))
        if rc:
            _capi.check(rc, self._h, "tet_spheres_ext.line_search")
        return LineSearch(delta, step, sd, ss)

    def hess_diag(self, x: torch.Tensor, c1: float, c2: float, order: int, c3: float = 0.0, gradH=1.0,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Per-vertex 3x3 diagonal blocks of the Hessian of ``c1 * smooth + c2 * barrier (+ c3 * amips)`` at ``x``
        (``tsb_hess_diag``), scaled by ``gradH``, as [2, n, 3] on the device without a host sync: ``[0]`` holds
        (H_xx, H_yy, H_zz) of each vertex, ``[1]`` (H_yz, H_xz, H_xy).  ``tssplat_b200.newton.hess_blocks`` turns them into
        [n, 3, 3] blocks.  ``c3`` needs a handle created with ``enable_amips=True``; ``gradH`` may be a CUDA tensor (read
        on the device).  ``out``: an optional contiguous float32 [2, n, 3] tensor on the handle's device to write into."""
        xc = self._check_x(x)
        if out is None:
            out = torch.empty((2, self.n, 3), dtype=torch.float32, device=self.device)
        elif (not isinstance(out, torch.Tensor) or out.dtype != torch.float32 or out.device != self.device
              or not out.is_contiguous() or out.numel() != 2 * self.n3):
            raise RuntimeError("out must be a contiguous float32 tensor of 2 * 3n entries on the handle's device")
        gh_val, gh_ptr, keep = self._gradH_arg(gradH)
        terms = _capi.tsb_terms_t(c1=float(c1), c2=float(c2), order=int(order), c3=float(c3))
        rc = _capi.lib.tsb_hess_diag(self._h, xc.data_ptr(), C.byref(terms), gh_val, gh_ptr, out.data_ptr(),
                                     _stream_ptr(self.device))
        if rc:
            _capi.check(rc, self._h, "tet_spheres_ext.hess_diag")
        del keep
        return out


def energy_grad_host(tet_sp: TetSpheres, x_host: torch.Tensor, c1: float, c2: float, order: int, gradH: float,
                     energy_host: torch.Tensor, grad_host: Optional[torch.Tensor]) -> None:
    """Host-buffer form of the fused launch (``tsb_energy_grad_host``): ``x_host`` [n,3] fp32 CPU
    (ideally pinned) in, ``energy_host`` [3] and ``grad_host`` [n,3] CPU out, asynchronous on the
    current stream -- synchronise the stream before reading the outputs."""
    for t in (x_host, energy_host) + ((grad_host,) if grad_host is not None else ()):
        if t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
            raise RuntimeError("energy_grad_host needs contiguous float32 CPU tensors")
    if x_host.numel() != tet_sp.n3 or energy_host.numel() < 3 or (grad_host is not None and grad_host.numel() != tet_sp.n3):
        raise RuntimeError("energy_grad_host: wrong buffer sizes")
    rc = _capi.lib.tsb_energy_grad_host(tet_sp._h, x_host.data_ptr(), float(c1), float(c2), int(order), float(gradH),
                                        energy_host.data_ptr(), grad_host.data_ptr() if grad_host is not None else None,
                                        _stream_ptr(tet_sp.device))
    _capi.check(rc, tet_sp._h, "tet_spheres_ext.energy_grad_host")


#: bumped by tssplat_b200.optimizer.AdamUniform.step: parameters updated through ``p.data`` do not bump
#: ``p._version``, so the fused-gradient cache keys on this counter too (ADVICE r1)
_mutation_epoch = 0


def note_parameters_changed() -> None:
    """Tell the fused-gradient cache that vertex positions were modified in place behind autograd's back."""
    global _mutation_epoch
    _mutation_epoch += 1
    from . import native_autograd
    mod = native_autograd.module()
    if mod is not None:
        mod.note_parameters_changed()


def _key(x: torch.Tensor, c1, c2, order):
    return (x.data_ptr(), x._version, _mutation_epoch, float(c1), float(c2), int(order))


def forward(vertexPositions: torch.Tensor, tet_sp: TetSpheres, c1: float, c2: float, order: int) -> torch.Tensor:
    """``E = c1 * 1/2 x^T G^T L^T L G x + c2 * sum_t max(-det F_t, 0)^order`` as a 0-dim tensor
    (``tet_spheres.cpp:208-211``, ``tet_spheres_cuda.cu:118-195``)."""
    want = bool(fuse_backward_into_forward and vertexPositions.requires_grad)
    energy, grad = tet_sp.energy_grad(vertexPositions, c1, c2, order, 1.0, want_grad=want)
    if want:
        tet_sp._cache_key, tet_sp._cache_grad = _key(vertexPositions, c1, c2, order), grad
    else:
        tet_sp._cache_key, tet_sp._cache_grad = None, None
    e = energy[0]
    return e.cpu() if return_cpu_scalar else e


def backward(gradH, vertexPositions: torch.Tensor, tet_sp: TetSpheres, c1: float, c2: float, order: int) -> torch.Tensor:
    """``gradH * dE/dx`` as a fresh tensor of ``x``'s shape on ``x``'s device
    (``tet_spheres.cpp:213-216``, ``tet_spheres_cuda.cu:197-263``).  Uses the gradient the fused forward
    launch already produced when ``x`` has not changed since (single use: a second backward recomputes)."""
    shape = vertexPositions.shape
    g = tet_sp._cache_grad
    if g is not None and tet_sp._cache_key == _key(vertexPositions, c1, c2, order):
        tet_sp._cache_key, tet_sp._cache_grad = None, None            # single use
        if isinstance(gradH, torch.Tensor) and gradH.is_cuda:
            keep = gradH if (gradH.dtype == torch.float32 and gradH.device == g.device) else gradH.detach().to(device=g.device, dtype=torch.float32)
            rc = _capi.lib.tsb_scale(g.data_ptr(), g.numel(), 1.0, keep.data_ptr(), g.data_ptr(), _stream_ptr(g.device))
            if rc:
                _capi.check(rc, None, "tet_spheres_ext.backward")
        else:
            gh = float(gradH)
            if gh != 1.0:
                rc = _capi.lib.tsb_scale(g.data_ptr(), g.numel(), gh, None, g.data_ptr(), _stream_ptr(g.device))
                if rc:
                    _capi.check(rc, None, "tet_spheres_ext.backward")
        out = g
    else:
        _, out = tet_sp.energy_grad(vertexPositions, c1, c2, order, gradH, want_grad=True)
    return out.reshape(shape)


def hvp(v: torch.Tensor, vertexPositions: torch.Tensor, tet_sp: TetSpheres, c1: float, c2: float, order: int,
        c3: float = 0.0) -> torch.Tensor:
    """``H(x) v`` of ``c1 * smooth + c2 * barrier (+ c3 * amips)`` as a fresh tensor of ``x``'s shape (argument order of
    ``backward``, with the direction in place of ``gradH``; ``c3`` as in ``TetSpheres.hvp``)."""
    hv, _ = tet_sp.hvp(vertexPositions, v, c1, c2, order, c3=c3)
    return hv.reshape(vertexPositions.shape)


def line_search(d: torch.Tensor, vertexPositions: torch.Tensor, tet_sp: TetSpheres, alphas, c1: float, c2: float,
                order: int, c3: float = 0.0, per_sphere: bool = False) -> LineSearch:
    """``TetSpheres.line_search`` in the argument order of ``hvp`` (direction first): the energy changes at ``alphas``
    along ``d`` and the largest inversion-free step."""
    return tet_sp.line_search(vertexPositions, d, alphas, c1, c2, order, c3=c3, per_sphere=per_sphere)


def hess_diag(vertexPositions: torch.Tensor, tet_sp: TetSpheres, c1: float, c2: float, order: int,
              c3: float = 0.0) -> torch.Tensor:
    """``TetSpheres.hess_diag`` in the argument order of ``forward``: the per-vertex 3x3 diagonal blocks of the Hessian
    as [2, n, 3] (diagonal entries, then (yz, xz, xy))."""
    return tet_sp.hess_diag(vertexPositions, c1, c2, order, c3=c3)


def newton_step(vertexPositions: torch.Tensor, newton, c1: float, c2: float, order: int, c3: float = 0.0, **opts):
    """``tssplat_b200.newton.DeviceNewton.step`` in the argument order of ``forward``, with the Newton workspace (created
    with ``DeviceNewton(tet_sp)``) in place of the handle: one damped Newton step per sphere, updating
    ``vertexPositions`` in place (``tsb_newton_step``)."""
    return newton.step(vertexPositions, c1, c2, order, c3=c3, **opts)


def random_x(tet_sp: TetSpheres) -> torch.Tensor:
    """``torch.rand({n, 3})`` on the CPU (``tet_spheres.cpp:218-221``)."""
    return torch.rand((tet_sp.n, 3))


def grad_limit(grad: torch.Tensor, s_threshold: float, s: float) -> None:
    """In place: if ``max|grad| > s_threshold`` scale ``grad`` so that its max magnitude is ``s``
    (the intent of ``tet_spheres_cuda.cu:265-303``)."""
    if not grad.is_cuda or grad.dtype != torch.float32 or not grad.is_contiguous():
        raise RuntimeError("grad_limit needs a contiguous float32 CUDA tensor")
    key = (grad.device.index, _stream_ptr(grad.device))
    work = _limit_work.get(key)
    if work is None:
        work = _limit_work[key] = torch.zeros(4, dtype=torch.float32, device=grad.device)
    rc = _capi.lib.tsb_grad_limit(grad.data_ptr(), grad.numel(), float(s_threshold), float(s), work.data_ptr(), key[1])
    _capi.check(rc, None, "tet_spheres_ext.grad_limit")

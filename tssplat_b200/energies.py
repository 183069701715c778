"""Host-side mirror of the reference's energy module (``energies/smooth_barrier.py``): same class
names, constructor arguments, scheduler and order switch, so ``geometry/tetmesh_geometry.py:155-189``
can use it unchanged.  The reference file itself also works as is once ``tet_spheres`` resolves to
this repo (its only other import, ``pypgo``, is unused by the module).

All arithmetic happens in the CUDA library behind ``tet_spheres_ext``; nothing here computes.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from tet_spheres import tet_spheres_ext
from . import _capi

__all__ = ["SmoothnessBarrierFunc", "SmoothnessBarrierFunc2", "SmoothnessBarrierAmipsFunc", "SmoothnessBarrierEnergy"]


#: route SmoothnessBarrierEnergy through the C++ autograd bridge when it has been built (same launches, same
#: semantics, no Python between autograd and the C ABI); False forces the Python Function below
use_native_autograd = True


class SmoothnessBarrierFunc(torch.autograd.Function):
    """autograd bridge (``energies/smooth_barrier.py:9-31``): forward returns the 0-dim energy,
    backward returns ``(dE/dx * grad_output, None, None, None, None)`` and short-circuits on a
    ``None`` grad_output."""

    @staticmethod
    def forward(ctx, x_cur, tet_sp, c1, c2, order):      # ctx-style like the reference's (no per-call signature binding)
        ctx.save_for_backward(x_cur)
        ctx.constants = (tet_sp, c1, c2, order)
        return tet_spheres_ext.forward(x_cur, tet_sp, c1, c2, order)

    @staticmethod
    def backward(ctx, grad_output):
        if grad_output is None:
            return (None,) * 5
        (x_cur,) = ctx.saved_tensors
        tet_sp, c1, c2, order = ctx.constants
        grad = tet_spheres_ext.backward(grad_output, x_cur, tet_sp, c1, c2, int(order))
        return grad, None, None, None, None


def _scaled_grad(tet_sp, grad, s, shape):
    """``s * grad`` as a fresh tensor of ``shape`` (``tsb_scale``; ``s`` may be a CUDA tensor, read on the device)."""
    out = torch.empty_like(grad)
    gh_val, gh_ptr, keep = tet_sp._gradH_arg(s)
    rc = _capi.lib.tsb_scale(grad.data_ptr(), grad.numel(), gh_val, gh_ptr, out.data_ptr(),
                             tet_spheres_ext._stream_ptr(grad.device))
    _capi.check(rc, None, "SmoothnessBarrierFunc2.backward")
    del keep
    return out.reshape(shape)


class _EnergyGrad(torch.autograd.Function):
    """``s * grad`` for the gradient ``grad`` = dE/dx at ``x`` that a forward launch produced, differentiable once more:
    given an upstream ``w`` its backward returns ``s * H(x) w`` for ``x`` (one ``tsb_hvp`` launch, gradH = s, or one
    ``tsb_hvp_ex`` with ``c3`` when the energy has the AMIPS term) and ``sum(grad * w)`` for ``s``.  A third derivative
    raises (``once_differentiable``)."""

    @staticmethod
    def forward(ctx, x, s, grad, tet_sp, c1, c2, order, c3=0.0):
        ctx.save_for_backward(x, s, grad)
        ctx.constants = (tet_sp, c1, c2, order, c3)
        return _scaled_grad(tet_sp, grad, s, x.shape)

    @staticmethod
    @once_differentiable
    def backward(ctx, w):
        x, s, grad = ctx.saved_tensors
        tet_sp, c1, c2, order, c3 = ctx.constants
        gx = gs = None
        if ctx.needs_input_grad[0]:
            gx, _ = tet_sp.hvp(x, w, c1, c2, order, gradH=s, c3=c3)
            gx = gx.reshape(x.shape)
        if ctx.needs_input_grad[1]:
            gs = (grad.reshape(-1) * w.reshape(-1)).sum().to(s.dtype).reshape(s.shape)
        return gx, gs, None, None, None, None, None, None


class SmoothnessBarrierFunc2(torch.autograd.Function):
    """``SmoothnessBarrierFunc`` made twice differentiable (``FLAGS.twice_differentiable``): its backward returns
    ``_EnergyGrad(x, grad_output)``, so ``torch.autograd.grad(E, x, create_graph=True)`` yields a gradient whose own
    backward is a Hessian-vector product of ``c1 * smooth + c2 * barrier``.  One fused launch in forward, as the
    default route; it does not use the fused-gradient cache."""

    @staticmethod
    def forward(ctx, x_cur, tet_sp, c1, c2, order):
        energy, grad = tet_sp.energy_grad(x_cur, c1, c2, order, 1.0, want_grad=bool(ctx.needs_input_grad[0]))
        ctx.save_for_backward(x_cur, grad)
        ctx.constants = (tet_sp, c1, c2, order)
        return energy[0]

    @staticmethod
    def backward(ctx, grad_output):
        if grad_output is None:
            return (None,) * 5
        x_cur, grad = ctx.saved_tensors
        tet_sp, c1, c2, order = ctx.constants
        return _EnergyGrad.apply(x_cur, grad_output, grad, tet_sp, c1, c2, int(order)), None, None, None, None


class SmoothnessBarrierAmipsFunc(torch.autograd.Function):
    """``c1 * smooth + c2 * barrier + c3 * amips`` (``FLAGS.amips_coeff``; the handle must be created with
    ``enable_amips=True``).  Forward is one fused launch (``tsb_energy_grad_ex``) that also produces the gradient;
    backward scales it by ``grad_output`` and does not relaunch.  With ``twice`` the gradient is an ``_EnergyGrad``,
    whose own backward is one ``tsb_hvp_ex`` with ``c3`` (all three terms); without it, as in ``SmoothnessBarrierFunc``,
    the gradient carries no graph."""

    @staticmethod
    def forward(ctx, x_cur, tet_sp, c1, c2, order, c3, twice):
        energy, grad = tet_sp.energy_grad(x_cur, c1, c2, order, 1.0, want_grad=bool(ctx.needs_input_grad[0]), c3=c3)
        ctx.save_for_backward(x_cur, grad)
        ctx.constants = (tet_sp, c1, c2, order, c3, twice)
        return energy[0]

    @staticmethod
    def backward(ctx, grad_output):
        if grad_output is None:
            return (None,) * 7
        x_cur, grad = ctx.saved_tensors
        tet_sp, c1, c2, order, c3, twice = ctx.constants
        if twice:
            gx = _EnergyGrad.apply(x_cur, grad_output, grad, tet_sp, c1, c2, int(order), float(c3))
        else:
            gx = _scaled_grad(tet_sp, grad, grad_output.detach(), x_cur.shape)
        return gx, None, None, None, None, None, None


class SmoothnessBarrierEnergy(torch.nn.Module):
    """``SmoothnessBarrierEnergy(tet_v, tet_f, FLAGS)`` (``energies/smooth_barrier.py:34-67``).

    ``tet_v``: numpy [n,3] REST positions; ``tet_f``: numpy [nele,4]; ``FLAGS``: mapping or object
    with ``smooth_eng_coeff``, ``barrier_coeff``, ``increase_order_iter`` (``config/gso.yaml:9-11``), and optionally
    ``deterministic`` (default False): a bitwise repeatable gradient (``TetSpheres(..., deterministic=True)``), and
    ``twice_differentiable`` (default False): ``forward`` goes through ``SmoothnessBarrierFunc2``, whose gradient can be
    differentiated once more (Hessian-vector products through autograd: ``create_graph=True``,
    ``torch.autograd.functional.vhp``), and ``amips_coeff`` (default 0): with a value > 0 the energy gains the AMIPS
    term, ``c1 * smooth + c2 * barrier + amips_coeff * amips``.  The coefficient is a constant (the scheduler's
    multiplier applies to the reference's two terms only); ``forward`` then goes through ``SmoothnessBarrierAmipsFunc``
    (one fused launch, twice differentiable under ``twice_differentiable``), and ``hvp`` and ``sphere_stats`` include
    the term.  With ``amips_coeff`` absent or 0 nothing changes.  ``newton_hessian`` (default ``"exact"``) selects the
    model of ``device_pcg``, which ``newton_direction``, ``newton_step`` and ``prox_step`` solve with: ``"psd"`` is the
    projected Hessian (``newton.DevicePCG``).  ``newton_precond`` (default ``"jacobi"``) selects that workspace's
    preconditioner: ``"sgs"`` is the multicolour block symmetric Gauss-Seidel preconditioner built from the assembled
    Hessian, which ``newton_direction``, ``newton_step``, ``prox_step`` and ``hessian`` then share.  ``newton_coarse``
    (default ``None``) set to ``"affine"`` adds the affine coarse space to that preconditioner (``newton.DevicePCG``).
    """

    #: the AMIPS coefficient; a class default, so that a module assembled without ``__init__`` (as ``bench.py`` does)
    #: keeps the route it had before the term existed
    amips_coeff = 0.0

    def __init__(self, tet_v, tet_f, FLAGS) -> None:
        super().__init__()
        v_flat = np.asarray(tet_v).flatten().astype(np.float32)
        f_flat = np.asarray(tet_f).flatten().astype(np.int32)
        self.FLAGS = SimpleNamespace(**FLAGS) if isinstance(FLAGS, dict) else FLAGS
        self.amips_coeff = float(getattr(self.FLAGS, "amips_coeff", 0.0) or 0.0)
        if not self.amips_coeff >= 0.0:
            raise ValueError(f"amips_coeff must be >= 0, got {self.amips_coeff}")
        kw = dict(enable_amips=True) if self.amips_coeff > 0 else {}
        self.tet_sp = tet_spheres_ext.TetSpheres(v_flat, f_flat, deterministic=bool(getattr(self.FLAGS, "deterministic", False)),
                                                 **kw)
        self.smooth_eng_func = SmoothnessBarrierFunc          # the reference instantiates it; .apply is static

    def coeff_scheduler(self, it):
        """Both coefficients times ``2 ** (4 |sin(min(it/2400 * pi, pi/2))|)`` in [1, 16]
        (``energies/smooth_barrier.py:47-58``)."""
        phase = min(it / 300.0 / 4 * 0.5 * math.pi, 0.5 * math.pi)
        multiplier = math.pow(2, abs(math.sin(phase)) * 4)
        return self.FLAGS.smooth_eng_coeff * multiplier, self.FLAGS.barrier_coeff * multiplier

    def order_at(self, it) -> int:
        return 4 if it > self.FLAGS.increase_order_iter else 2     # smooth_barrier.py:61-63

    def sphere_stats(self, x, it):
        """Per-sphere geometry statistics at ``x`` (``tet_spheres_ext.SphereStats`` of device tensors, no host sync):
        each sphere's smoothness and barrier terms (and AMIPS term with ``amips_coeff``), inverted-tet count and
        smallest det F, with the barrier order ``forward(x, it, ...)`` uses at ``it``.  An energy-only launch, outside
        autograd; it leaves the fused-gradient cache alone.  Meant to be logged every N iterations next to the loss."""
        c1, c2 = self.coeff_scheduler(it)
        _, _, stats = self.tet_sp.energy_grad_spheres(x.detach(), c1, c2, self.order_at(it), want_grad=False,
                                                      c3=self.amips_coeff)
        return stats

    def hvp(self, x, v, it):
        """``H(x) v`` of ``c1 * smooth + c2 * barrier (+ amips_coeff * amips)`` with the scheduler's coefficients and the
        barrier order at ``it`` (``tsb_hvp``, or ``tsb_hvp_ex`` with ``amips_coeff``), outside autograd, in ``x``'s
        shape."""
        c1, c2 = self.coeff_scheduler(it)
        hv, _ = self.tet_sp.hvp(x.detach(), v.detach(), c1, c2, self.order_at(it), c3=self.amips_coeff)
        return hv.reshape(x.shape)

    def line_search(self, x, d, it, alphas, per_sphere=False):
        """``E(x + alpha_k d) - E(x)`` of ``c1 * smooth + c2 * barrier (+ amips_coeff * amips)`` at the step sizes
        ``alphas`` and the largest inversion-free step along ``d`` (``tet_spheres_ext.LineSearch``), with the scheduler's
        coefficients and the barrier order at ``it``; outside autograd, no host sync."""
        c1, c2 = self.coeff_scheduler(it)
        return self.tet_sp.line_search(x.detach(), d.detach(), alphas, c1, c2, self.order_at(it), c3=self.amips_coeff,
                                       per_sphere=per_sphere)

    def hess_diag(self, x, it):
        """Per-vertex 3x3 diagonal blocks of the Hessian of ``c1 * smooth + c2 * barrier (+ amips_coeff * amips)`` with
        the scheduler's coefficients and the barrier order at ``it`` (``tsb_hess_diag``), as [2, n, 3] (see
        ``TetSpheres.hess_diag``); outside autograd, no host sync.  ``tssplat_b200.newton.block_jacobi`` makes a
        preconditioner of them."""
        c1, c2 = self.coeff_scheduler(it)
        return self.tet_sp.hess_diag(x.detach(), c1, c2, self.order_at(it), c3=self.amips_coeff)

    def hessian(self, x, it):
        """Block values [nnzb, 3, 3] of the Hessian of ``c1 * smooth + c2 * barrier (+ amips_coeff * amips)`` at ``x``,
        with the scheduler's coefficients and the barrier order at ``it``, in the model of ``device_pcg``
        (``FLAGS.newton_hessian``: exact or projected); the pattern is ``self.device_hessian``'s ``crow`` and ``col``
        (``tssplat_b200.hessian.DeviceHessian``, created on first use).  Outside autograd, no host sync."""
        from .hessian import DeviceHessian
        hs = getattr(self, "device_hessian", None)
        if hs is None:
            pcg = self._device_pcg()
            hs = self.device_hessian = pcg.hessian_ws or DeviceHessian(pcg)
        c1, c2 = self.coeff_scheduler(it)
        return hs.assemble(x.detach(), c1, c2, self.order_at(it), c3=self.amips_coeff)

    def _device_pcg(self):
        from .newton import DevicePCG
        pcg = getattr(self, "device_pcg", None)
        if pcg is None:
            pcg = self.device_pcg = DevicePCG(self.tet_sp, hessian=getattr(self.FLAGS, "newton_hessian", "exact") or "exact",
                                              precond=getattr(self.FLAGS, "newton_precond", "jacobi") or "jacobi",
                                              coarse=getattr(self.FLAGS, "newton_coarse", None) or None)
        return pcg

    def newton_direction(self, x, it, b=None, **solve_kw):
        """A Newton direction per sphere, on the device without a host sync: ``hess_diag`` -> block-Jacobi preconditioner
        -> ``tssplat_b200.newton.DevicePCG.solve`` of ``H(x) d = b`` with the scheduler's coefficients, the barrier order
        at ``it`` and ``amips_coeff``.  ``b=None`` takes ``b = -grad`` from one gradient launch.  ``solve_kw``:
        ``max_iter``, ``rtol``, ``check_every``.  Returns a ``DevicePCGResult`` (its ``b_dot_d`` is what a per-sphere
        Armijo test needs); the workspace, ``self.device_pcg`` (its ``axpy`` takes the per-sphere step), is created on
        first use."""
        pcg = self._device_pcg()
        c1, c2 = self.coeff_scheduler(it)
        order, xd = self.order_at(it), x.detach()
        if b is None:
            _, g = self.tet_sp.energy_grad(xd, c1, c2, order, -1.0, c3=self.amips_coeff)
            b = g.reshape(x.shape)
        if pcg.coarse is not None:
            pcg.set_coarse(xd, c1, c2, order, c3=self.amips_coeff)
        if pcg.precond == "sgs":    # the diagonal of the matrix the sweep uses
            pcg.set_blocks(pcg.set_matrix(xd, c1, c2, order, c3=self.amips_coeff))
        else:
            pcg.set_blocks(self.tet_sp.hess_diag(xd, c1, c2, order, c3=self.amips_coeff))
        return pcg.solve(xd, b.detach(), c1, c2, order, c3=self.amips_coeff, **solve_kw)

    def _device_newton(self):
        from .newton import DeviceNewton
        nw = getattr(self, "device_newton", None)
        if nw is None:
            nw = self.device_newton = DeviceNewton(self.tet_sp, self._device_pcg())
        return nw

    def newton_step(self, x, it, **opts):
        """One damped (Levenberg-Marquardt) Newton step per sphere of ``c1 * smooth + c2 * barrier (+ amips_coeff *
        amips)`` with the scheduler's coefficients and the barrier order at ``it``: ``tssplat_b200.newton.DeviceNewton``
        (``tsb_newton_step``), which updates ``x.data`` in place without a host read.  ``opts``: the fields of
        ``newton.NEWTON_DEFAULTS``.  The workspace, ``self.device_newton``, is created on first use (sharing
        ``self.device_pcg``); its ``reset()`` restarts every sphere.  Returns the ``NewtonStepResult``.
        ``FLAGS.newton_method = "tr"`` takes the trust-region step instead (``DeviceNewton.tr_step``; ``opts`` then the
        fields of ``newton.NEWTON_TR_DEFAULTS``; returns a ``NewtonTRStepResult``), ``"trls"`` the backtracking
        trust-region step (``DeviceNewton.trls_step``; the fields of ``newton.NEWTON_TRLS_DEFAULTS``), and ``"lbfgs"``
        the L-BFGS step (``DeviceNewton.lbfgs_step``; the fields of ``newton.NEWTON_LBFGS_DEFAULTS``; returns a
        ``NewtonLBFGSStepResult``)."""
        nw = self._device_newton()
        c1, c2 = self.coeff_scheduler(it)
        return nw._step(self._newton_method(), x.data, c1, c2, self.order_at(it), self.amips_coeff, None, None, opts)

    def _newton_method(self) -> str:
        from .newton import METHODS
        m = getattr(self.FLAGS, "newton_method", "lm") or "lm"
        if m not in METHODS:
            raise ValueError(f"FLAGS.newton_method must be one of {METHODS}, got {m!r}")
        return m

    def prox_step(self, x, y, it, weight, n_steps=1, restart=True, **opts):
        """The regulariser half of a split step: ``n_steps`` proximal Newton steps per sphere of
        ``E(x) + (w_c / 2) |x_c - y_c|^2``, ``E`` the energy of ``newton_step`` at ``it`` (scheduler coefficients,
        barrier order, ``amips_coeff``), anchored at ``y`` (typically ``x`` right after the optimiser's step on the data
        term, copied: ``y`` must not be ``x``).  ``weight``: a float for every sphere or a float32 CUDA tensor [S].
        Updates ``x.data`` in place with no host read (``tsb_newton_prox_step``) and returns the last
        ``NewtonStepResult``.  ``restart`` resets the workspace first: a new anchor is a new problem, and a sphere frozen
        on the old one must not stay frozen.  ``opts``: the fields of ``newton.NEWTON_DEFAULTS`` (of
        ``newton.NEWTON_TR_DEFAULTS`` with ``FLAGS.newton_method = "tr"``, which takes trust-region steps, and of
        ``newton.NEWTON_TRLS_DEFAULTS`` with ``"trls"``, which takes backtracking trust-region steps, and of
        ``newton.NEWTON_LBFGS_DEFAULTS`` with ``"lbfgs"``, which takes L-BFGS steps; the reset then also empties every
        sphere's L-BFGS history, which belongs to the old anchor)."""
        if n_steps < 1:
            raise ValueError("n_steps must be >= 1")
        nw = self._device_newton()
        if restart:
            nw.reset()
        c1, c2 = self.coeff_scheduler(it)
        _, res = nw.minimize(x.data, n_steps, c1, c2, self.order_at(it), c3=self.amips_coeff, anchor=y.detach(),
                             weight=weight, method=self._newton_method(), **opts)
        return res

    def forward(self, x, it, c1, c2):
        order = self.order_at(it)
        if self.amips_coeff > 0:
            return SmoothnessBarrierAmipsFunc.apply(x, self.tet_sp, c1, c2, order, self.amips_coeff,
                                                    bool(getattr(self.FLAGS, "twice_differentiable", False)))
        if getattr(self.FLAGS, "twice_differentiable", False):
            return SmoothnessBarrierFunc2.apply(x, self.tet_sp, c1, c2, order)
        if (use_native_autograd and self.smooth_eng_func is SmoothnessBarrierFunc and tet_spheres_ext.fuse_backward_into_forward
                and not tet_spheres_ext.return_cpu_scalar):
            ns = self.tet_sp.native_state()        # C++ torch::autograd::Function over the same C ABI (csrc/torch_binding.cpp)
            if ns is not None:
                return ns[0].energy(x, ns[1], float(c1), float(c2), order, self.tet_sp)
        return self.smooth_eng_func.apply(x, self.tet_sp, c1, c2, order)

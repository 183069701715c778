"""Block-Jacobi preconditioned truncated Newton-CG over the geometry energy's second-order calls.

``TetSpheres.hess_diag`` gives the per-vertex 3x3 diagonal blocks of the Hessian as two [n, 3] planes;
``block_jacobi`` turns them into an SPD preconditioner, and ``pcg`` runs truncated conjugate gradients over a
Hessian-vector product (``TetSpheres.hvp``), stopping at negative curvature.  Plain torch on the planes' device; the
Hessian itself is only ever touched through the CUDA library's launches.  INTEGRATION.md shows one Newton step built
from these and ``TetSpheres.line_search``.

``DevicePCG`` is the device-resident solver (``tsb_pcg_solve``): the same truncated PCG, but run independently on every
tet-sphere (the Hessian is block diagonal by sphere) with all scalars in device memory, so there is no host read inside
an iteration and the solve can be captured in a CUDA graph.  ``pcg`` below stays as the reference implementation.
With a per-sphere ``shift`` it solves ``(H + mu_c I) d = b`` (``tsb_pcg_solve_ex``).  ``DevicePCG(tet_sp, hessian="psd")``
multiplies by the projected Hessian instead (``tsb_pcg_enable_psd``): every tet's Hessian replaced by its positive
semidefinite projection, so the solve never stops at negative curvature from the tet terms.

``DeviceNewton`` joins the pieces into a minimiser (``tsb_newton_step``): one damped (Levenberg-Marquardt) Newton step per
sphere per call -- gradient, diagonal blocks, shifted solve, line search, step choice and damping update -- on one
stream without a host read.  Given an ``anchor`` y and per-sphere weights w, the step minimises the proximal objective
``E(x) + (w_c / 2) |x_c - y_c|^2`` instead (``tsb_newton_prox_step``): the regulariser half of a split training loop whose
data term keeps its first-order optimiser.  ``DeviceNewton.tr_step`` is the trust-region alternative
(``tsb_newton_tr_step``): no damping shift, a per-sphere radius in the preconditioner norm inside which the solve
(``DevicePCG.solve(..., radius=)``, ``tsb_pcg_solve_tr``) follows negative curvature to the boundary.
``DeviceNewton.trls_step`` (``tsb_newton_tr_step_ex``) is the same step, but one the trust-region rule rejects is
backtracked along ``2^-k`` with the Armijo test instead of being dropped whole.  ``DeviceNewton.lbfgs_step``
(``tsb_newton_lbfgs_step``) is the quasi-Newton alternative: a per-sphere L-BFGS direction from the gradients of earlier
steps with the block-Jacobi preconditioner as its initial inverse Hessian, and the damped step's line search; no
Hessian-vector products and no solve.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, NamedTuple, Optional, Union

import torch

__all__ = ["hess_blocks", "block_jacobi", "apply_blocks", "pcg", "PCGResult", "DevicePCG", "DevicePCGResult", "DeviceNewton",
           "NewtonStepResult", "NEWTON_DEFAULTS", "HESSIANS", "NewtonTRStepResult", "NEWTON_TR_DEFAULTS", "NEWTON_TRLS_DEFAULTS",
           "NEWTON_LBFGS_DEFAULTS", "NewtonLBFGSStepResult", "METHODS"]


def hess_blocks(planes: torch.Tensor) -> torch.Tensor:
    """[2, n, 3] planes of ``hess_diag`` ((H_xx, H_yy, H_zz), then (H_yz, H_xz, H_xy)) -> symmetric [n, 3, 3] blocks."""
    if planes.dim() != 3 or planes.shape[0] != 2 or planes.shape[2] != 3:
        raise ValueError(f"planes must have shape [2, n, 3], got {tuple(planes.shape)}")
    d, o = planes[0], planes[1]
    B = torch.diag_embed(d)
    B[:, 1, 2] = B[:, 2, 1] = o[:, 0]
    B[:, 0, 2] = B[:, 2, 0] = o[:, 1]
    B[:, 0, 1] = B[:, 1, 0] = o[:, 2]
    return B


def block_jacobi(planes: torch.Tensor, rel_floor: float = 1e-6) -> torch.Tensor:
    """SPD inverses of the diagonal blocks, [n, 3, 3]: each block's eigenvalues are clamped from below to
    ``rel_floor * lambda_max`` of that block before inverting, so indefinite blocks (AMIPS far from rest, or a barrier
    block's rank-1 null space) stay well conditioned; a block with ``lambda_max <= 0`` (a vertex no tet references, or
    one with only negative curvature) maps to 0, i.e. that vertex does not move."""
    B = hess_blocks(planes)
    lam, Q = torch.linalg.eigh(B)                      # ascending
    lmax = lam[:, 2]
    pos = lmax > 0
    lam_c = torch.where(pos[:, None], torch.maximum(lam, (rel_floor * lmax)[:, None]), torch.ones_like(lam))
    inv = (Q / lam_c[:, None, :]) @ Q.transpose(1, 2)
    return torch.where(pos[:, None, None], inv, torch.zeros_like(inv))


def apply_blocks(P: torch.Tensor, r: torch.Tensor) -> torch.Tensor:
    """Per-vertex product ``P_i r_i`` of [n, 3, 3] blocks and a vector of 3n entries, in ``r``'s shape."""
    return torch.einsum("nij,nj->ni", P, r.reshape(-1, 3)).reshape(r.shape)


class PCGResult(NamedTuple):
    x: torch.Tensor                 # the step, in b's shape
    n_hvp: int                      # Hessian-vector products used
    converged: bool                 # |r| <= rtol |b| reached
    negative_curvature: bool        # stopped at p^T H p <= 0
    rel_residual: float             # |r| / |b| of the returned step (1 when stopped at the first direction)


def _dot(a: torch.Tensor, b: torch.Tensor) -> float:
    return float(torch.dot(a.reshape(-1).double(), b.reshape(-1).double()))


def pcg(hvp_fn: Callable[[torch.Tensor], torch.Tensor], b: torch.Tensor,
        precond: Optional[Union[torch.Tensor, Callable[[torch.Tensor], torch.Tensor]]] = None, max_iter: int = 100,
        rtol: float = 1e-3) -> PCGResult:
    """Truncated (Steihaug) preconditioned CG for ``H x = b``: ``hvp_fn(p)`` returns ``H p`` in ``p``'s shape;
    ``precond`` is [n, 3, 3] blocks (``block_jacobi``), a callable ``r -> M^-1 r``, or None.  Stops when
    ``|r| <= rtol |b|``, after ``max_iter`` products, or at the first direction with ``p^T H p <= 0``: then it returns
    the iterate reached so far, or the preconditioned right-hand side ``M^-1 b`` if that happens at the first direction
    (a descent direction for ``b = -grad``, to be scaled by a line search).  Reads one scalar to the host per
    iteration."""
    if precond is None:
        apply = lambda r: r
    elif isinstance(precond, torch.Tensor):
        apply = lambda r: apply_blocks(precond, r)
    else:
        apply = precond
    x = torch.zeros_like(b)
    bnorm = float(b.double().norm())
    if bnorm == 0.0:
        return PCGResult(x, 0, True, False, 0.0)
    r = b.clone()
    z = apply(r)
    p = z.clone()
    rz = _dot(r, z)
    n = 0
    for _ in range(max_iter):
        Hp = hvp_fn(p)
        n += 1
        pHp = _dot(p, Hp)
        if not pHp > 0.0:
            if n == 1:
                return PCGResult(z, n, False, True, 1.0)
            return PCGResult(x, n, False, True, float(r.double().norm()) / bnorm)
        a = rz / pHp
        x = x + a * p
        r = r - a * Hp
        res = float(r.double().norm()) / bnorm
        if res <= rtol:
            return PCGResult(x, n, True, False, res)
        z = apply(r)
        rz_new = _dot(r, z)
        p = z + (rz_new / rz) * p
        rz = rz_new
    return PCGResult(x, n, False, False, float(r.double().norm()) / bnorm)


class DevicePCGResult(NamedTuple):
    """What ``DevicePCG.solve`` returns: device tensors, S = number of spheres in the order of their lowest vertex ids
    (``tsb_pcg_sphere_t`` in ``include/tssplat_b200.h``)."""
    d: torch.Tensor                 # f32 [n, 3]: the step of every sphere; 0 on vertices no tet references
    status: torch.Tensor            # i32 [S]: 0 max_iter, 1 converged, 2 negative curvature, 3 the same at the first
                                    # direction (d_c = P b_c), 4 zero right-hand side; with a radius also 5 stopped on
                                    # the boundary, 6 negative curvature followed to the boundary
    n_hvp: torch.Tensor             # i32 [S]: products in which the sphere was still active
    rel_residual: torch.Tensor      # f32 [S]: |r_c| / |b_c| of the returned step
    b_dot_d: torch.Tensor           # f32 [S]: b_c . d_c
    d_H_d: torch.Tensor             # f32 [S]: d_c^T H d_c as accumulated by CG
    iters_run: int                  # iterations enqueued (= max_iter with check_every = 0)


HESSIANS = ("exact", "psd")
#: preconditioners of ``DevicePCG``: block Jacobi, or multicolour block symmetric Gauss-Seidel from the assembled Hessian
PRECONDS = ("jacobi", "sgs")
#: coarse spaces of ``DevicePCG``: none, or the 9 linear affine motions of every sphere
COARSES = (None, "affine")


class DevicePCG:
    """Per-sphere block-Jacobi PCG workspace of one ``TetSpheres`` handle (``tsb_pcg_create``), which it keeps alive.
    Serves one stream at a time, like the handle.  ``hessian="psd"`` enables the projected Hessian on it
    (``tsb_pcg_enable_psd``, from the mesh the handle keeps): ``solve`` and every ``DeviceNewton`` step over this workspace
    then multiply by ``H+``, and ``hvp_psd`` is available.  ``precond="sgs"`` replaces block Jacobi by the multicolour
    block symmetric Gauss-Seidel preconditioner built from the assembled Hessian (``tsb_pcg_enable_sgs``): the workspace
    creates and owns a ``DeviceHessian`` in its mode (``hessian_ws``, usable while the workspace lives), ``set_matrix``
    assembles the matrix the sweep uses and returns its diagonal planes for ``set_blocks``, and ``apply_precond`` and
    ``colors`` are available.  ``coarse="affine"`` adds the affine coarse space on top of that preconditioner
    (``tsb_pcg_enable_coarse``): ``P + Z E+ Z^T`` with the sphere's 9 linear affine motions as ``Z`` and ``E+`` the
    pseudo-inverse of ``Z^T H Z`` (eigenvalues at or below ``coarse_floor * lambda_max`` dropped); ``set_coarse`` forms it at
    a point, ``set_blocks`` refactors it with its shift, ``coarse_matrix`` returns ``Z^T H Z`` and ``apply_precond`` applies
    the whole two-level preconditioner.  Creating it allocates, so not inside a CUDA graph capture."""

    def __init__(self, tet_sp, hessian: str = "exact", precond: str = "jacobi", coarse: Optional[str] = None,
                 coarse_floor: float = 1e-8):
        from . import _capi
        from .tet_spheres_ext import _stream_ptr
        self._capi, self._stream_ptr = _capi, _stream_ptr
        self._s = None
        if hessian not in HESSIANS:
            raise ValueError(f"hessian must be one of {HESSIANS}, got {hessian!r}")
        if precond not in PRECONDS:
            raise ValueError(f"precond must be one of {PRECONDS}, got {precond!r}")
        if hessian == "psd" and torch.cuda.is_current_stream_capturing():
            raise RuntimeError('DevicePCG(hessian="psd") allocates device memory and cannot be created during a CUDA graph capture')
        if precond == "sgs" and torch.cuda.is_current_stream_capturing():
            raise RuntimeError('DevicePCG(precond="sgs") allocates device memory and cannot be created during a CUDA graph capture')
        if coarse not in COARSES:
            raise ValueError(f"coarse must be one of {COARSES}, got {coarse!r}")
        if coarse is not None and torch.cuda.is_current_stream_capturing():
            raise RuntimeError('DevicePCG(coarse="affine") allocates device memory and cannot be created during a CUDA graph capture')
        self.tet_sp, self.hessian, self.precond, self.coarse = tet_sp, hessian, precond, coarse
        self.hessian_ws = None
        s = C.c_void_p()
        rc = _capi.lib.tsb_pcg_create(tet_sp._h, C.byref(s))
        if rc:
            raise RuntimeError(f"DevicePCG: {self._error(None)} (code {rc})")
        self._s = s
        self.n_spheres = int(tet_sp.info["n_components"])
        if hessian == "psd":
            rc = _capi.lib.tsb_pcg_enable_psd(s, tet_sp.vertices.ctypes.data, tet_sp.elements.ctypes.data, int(tet_sp.nele))
            self._check(rc, "__init__")
        if precond == "sgs":
            import weakref
            from .hessian import DeviceHessian
            self.hessian_ws = DeviceHessian(self)
            # the workspace owns its Hessian workspace; a weak link back keeps the pair out of a reference cycle, which
            # the garbage collector could otherwise free (cudaFree) in the middle of a later CUDA graph capture
            self.hessian_ws.pcg = weakref.proxy(self)
            self._check(_capi.lib.tsb_pcg_enable_sgs(s, self.hessian_ws._hs), "__init__")
        if coarse is not None:
            rc = _capi.lib.tsb_pcg_enable_coarse(s, tet_sp.vertices.ctypes.data, tet_sp.elements.ctypes.data, int(tet_sp.nele),
                                                 float(coarse_floor))
            self._check(rc, "__init__")
        self.device_bytes = int(_capi.lib.tsb_pcg_device_bytes(s))

    def __del__(self):
        s, self._s = getattr(self, "_s", None), None
        if s:
            try:
                self._capi.lib.tsb_pcg_destroy(s)
            except Exception:  # interpreter shutdown
                pass

    def _error(self, s) -> str:
        msg = self._capi.lib.tsb_pcg_last_error(s)
        return msg.decode("utf-8", "replace") if msg else ""

    def _check(self, rc: int, what: str) -> None:
        if rc:
            raise RuntimeError(f"DevicePCG.{what}: {self._error(self._s)} (code {rc})")

    def _f32(self, t: torch.Tensor, numel: int, name: str) -> torch.Tensor:
        if (not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.device != self.tet_sp.device
                or t.numel() != numel):
            raise RuntimeError(f"{name} must be a float32 tensor of {numel} entries on {self.tet_sp.device}")
        return t if t.is_contiguous() else t.contiguous()

    def _shift(self, shift, name: str = "shift") -> Optional[torch.Tensor]:
        """None, a Python float (every sphere), or a float32 CUDA tensor of one entry per sphere."""
        if shift is None:
            return None
        if isinstance(shift, torch.Tensor):
            return self._f32(shift, self.n_spheres, name)
        return torch.full((self.n_spheres,), float(shift), dtype=torch.float32, device=self.tet_sp.device)

    def set_blocks(self, planes: Optional[torch.Tensor] = None, rel_floor: float = 1e-6,
                   want_inverse: bool = False, shift=None) -> Optional[torch.Tensor]:
        """Preconditioner from the [2, n, 3] planes of ``hess_diag`` with ``block_jacobi``'s semantics, computed on the
        device (``tsb_pcg_set_blocks``); ``None`` is the identity.  ``want_inverse`` returns the inverse blocks as
        [n, 6] = (xx, yy, zz, yz, xz, xy).  ``shift``: per-sphere ``mu_c`` (a float32 CUDA tensor [S], or a float for
        every sphere); the blocks are then ``D_v + mu_c I`` (``tsb_pcg_set_blocks_ex``)."""
        n = self.tet_sp.n
        pc = None if planes is None else self._f32(planes, 6 * n, "planes")
        sh = self._shift(shift)
        inv = torch.empty((n, 6), dtype=torch.float32, device=self.tet_sp.device) if want_inverse else None
        rc = self._capi.lib.tsb_pcg_set_blocks_ex(self._s, pc.data_ptr() if pc is not None else None, float(rel_floor),
                                                  sh.data_ptr() if sh is not None else None,
                                                  inv.data_ptr() if want_inverse else None, self._stream_ptr(self.tet_sp.device))
        self._check(rc, "set_blocks")
        return inv

    def solve(self, x: torch.Tensor, b: torch.Tensor, c1: float, c2: float, order: int, c3: float = 0.0,
              max_iter: int = 100, rtol: float = 1e-3, check_every: int = 0, shift=None, radius=None) -> DevicePCGResult:
        """``H(x) d = b`` on every sphere by truncated PCG (``tsb_pcg_solve``), ``H`` the Hessian ``TetSpheres.hvp``
        multiplies by.  ``check_every = 0`` enqueues ``max_iter`` iterations without touching the host (and can be
        captured in a CUDA graph); ``k > 0`` reads the number of active spheres every ``k`` iterations and stops
        early.  ``shift`` (as in ``set_blocks``) solves ``(H + mu_c I) d = b`` instead (``tsb_pcg_solve_ex``); ``d_H_d``
        is then ``d^T (H + mu_c I) d``.  ``radius`` (a float for every sphere, or a float32 CUDA tensor [S] read on the
        device) keeps every sphere's step inside ``|d_c|_M <= radius_c`` in the preconditioner norm (``tsb_pcg_solve_tr``,
        Steihaug-Toint): negative curvature and a step that would leave the radius end on the boundary (status 6 and 5).
        ``radius=inf`` gives the bits of the call without it; the first call with a radius allocates, so it cannot be
        captured."""
        n3, dev = self.tet_sp.n3, self.tet_sp.device
        xc, bc = self._f32(x, n3, "x"), self._f32(b, n3, "b")
        sh = self._shift(shift)
        rad = self._shift(radius, "radius")
        d = torch.empty((self.tet_sp.n, 3), dtype=torch.float32, device=dev)
        raw = torch.empty((self.n_spheres, C.sizeof(self._capi.tsb_pcg_sphere_t)), dtype=torch.uint8, device=dev)
        terms = self._capi.tsb_terms_t(c1=float(c1), c2=float(c2), order=int(order), c3=float(c3))
        opt = self._capi.tsb_pcg_options_t(max_iter=int(max_iter), rtol=float(rtol), check_every=int(check_every))
        iters = C.c_int32(0)
        if rad is None:
            rc = self._capi.lib.tsb_pcg_solve_ex(self._s, xc.data_ptr(), bc.data_ptr(), C.byref(terms), C.byref(opt),
                                                 sh.data_ptr() if sh is not None else None, d.data_ptr(), raw.data_ptr(),
                                                 C.byref(iters), self._stream_ptr(dev))
        else:
            rc = self._capi.lib.tsb_pcg_solve_tr(self._s, xc.data_ptr(), bc.data_ptr(), C.byref(terms), C.byref(opt),
                                                 sh.data_ptr() if sh is not None else None, rad.data_ptr(), d.data_ptr(),
                                                 raw.data_ptr(), C.byref(iters), self._stream_ptr(dev))
        self._check(rc, "solve")
        f = self._capi.record_fields(raw, self._capi.tsb_pcg_sphere_t)
        return DevicePCGResult(d=d, iters_run=int(iters.value), **{k: f[k] for k in DevicePCGResult._fields if k in f})

    def _need_sgs(self, what: str) -> None:
        if self.precond != "sgs":
            raise RuntimeError(f'DevicePCG.{what} needs a workspace created with precond="sgs"')

    def set_matrix(self, x: torch.Tensor, c1: float, c2: float, order: int, c3: float = 0.0,
                   out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Assembles the Hessian at ``x`` (exact, or projected with ``hessian="psd"``) into the workspace's matrix, from
        which the symmetric Gauss-Seidel sweep reads its off-diagonal blocks (``tsb_pcg_set_matrix``), and returns its
        diagonal blocks as ``hess_diag``'s [2, n, 3] planes, to hand to ``set_blocks`` (with or without a shift).
        ``out``: a contiguous float32 tensor of 6n entries, overwritten and returned (then capturable)."""
        self._need_sgs("set_matrix")
        n, dev = self.tet_sp.n, self.tet_sp.device
        xc = self._f32(x, self.tet_sp.n3, "x")
        if out is None:
            out = torch.empty((2, n, 3), dtype=torch.float32, device=dev)
        elif self._f32(out, 6 * n, "out") is not out:
            raise RuntimeError("out must be contiguous")
        terms = self._capi.tsb_terms_t(c1=float(c1), c2=float(c2), order=int(order), c3=float(c3))
        rc = self._capi.lib.tsb_pcg_set_matrix(self._s, xc.data_ptr(), C.byref(terms), out.data_ptr(), self._stream_ptr(dev))
        self._check(rc, "set_matrix")
        return out

    def apply_precond(self, r: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``M^-1 r`` on every sphere with the symmetric Gauss-Seidel preconditioner of the last ``set_matrix`` and
        ``set_blocks`` (``tsb_pcg_apply_precond``), in ``r``'s shape.  Vertices no tet references are 0 in a new tensor and
        left as they are in ``out`` (not ``r``): a contiguous float32 tensor of 3n entries, returned (then no allocation).  On a ``coarse`` workspace it is
        the two-level ``P r + Z E+ Z^T r`` (``P`` block Jacobi or the sweep) at the last ``set_coarse`` and ``set_blocks``."""
        if self.precond != "sgs" and self.coarse is None:
            raise RuntimeError('DevicePCG.apply_precond needs a workspace created with precond="sgs" or coarse="affine"')
        n3 = self.tet_sp.n3
        rc_ = self._f32(r, n3, "r")
        if out is None:
            out = torch.zeros_like(rc_)
        elif self._f32(out, n3, "out") is not out:
            raise RuntimeError("out must be contiguous")
        rc = self._capi.lib.tsb_pcg_apply_precond(self._s, rc_.data_ptr(), out.data_ptr(), self._stream_ptr(self.tet_sp.device))
        self._check(rc, "apply_precond")
        return out.reshape(r.shape)

    def _need_coarse(self, what: str) -> None:
        if self.coarse is None:
            raise RuntimeError(f'DevicePCG.{what} needs a workspace created with coarse="affine"')

    def set_coarse(self, x: torch.Tensor, c1: float, c2: float, order: int, c3: float = 0.0) -> None:
        """Forms every sphere's coarse matrix ``Z^T H Z`` at ``x`` (exact, or projected with ``hessian="psd"``) and its
        unshifted pseudo-inverse (``tsb_pcg_set_coarse``); a following ``set_blocks`` with a shift refactors it with
        ``shift_c (S_c (x) I3)``.  No host sync, no allocation: capturable."""
        self._need_coarse("set_coarse")
        xc = self._f32(x, self.tet_sp.n3, "x")
        terms = self._capi.tsb_terms_t(c1=float(c1), c2=float(c2), order=int(order), c3=float(c3))
        rc = self._capi.lib.tsb_pcg_set_coarse(self._s, xc.data_ptr(), C.byref(terms), self._stream_ptr(self.tet_sp.device))
        self._check(rc, "set_coarse")

    def coarse_matrix(self) -> torch.Tensor:
        """float64 [S, 9, 9]: every sphere's unshifted ``Z^T H Z`` of the last ``set_coarse``, coarse unknowns the 3 x 3
        matrix ``A`` row-major (``tsb_pcg_coarse_matrix``; synchronises the device)."""
        self._need_coarse("coarse_matrix")
        out = torch.empty((self.n_spheres, 9, 9), dtype=torch.float64, device=self.tet_sp.device)
        torch.cuda.synchronize(self.tet_sp.device)
        self._check(self._capi.lib.tsb_pcg_coarse_matrix(self._s, out.data_ptr()), "coarse_matrix")
        return out

    @property
    def colors(self) -> torch.Tensor:
        """int32 [n]: the colour of every vertex in the sweep's order (-1 for vertices no tet references)."""
        self._need_sgs("colors")
        out = torch.empty(self.tet_sp.n, dtype=torch.int32, device=self.tet_sp.device)
        torch.cuda.synchronize(self.tet_sp.device)
        self._check(self._capi.lib.tsb_pcg_sgs_colors(self._s, out.data_ptr(), None), "colors")
        return out

    @property
    def n_colors(self) -> int:
        """The most colours any sphere uses."""
        self._need_sgs("n_colors")
        k = C.c_int32(0)
        self._check(self._capi.lib.tsb_pcg_sgs_colors(self._s, None, C.byref(k)), "n_colors")
        return int(k.value)

    def hvp_psd(self, x: torch.Tensor, v: torch.Tensor, c1: float, c2: float, order: int, c3: float = 0.0):
        """``H+(x) v`` of ``c1 * smooth + c2 * barrier (+ c3 * amips)`` with every tet's Hessian projected to PSD at ``x``
        (``tsb_pcg_hvp_psd``; needs ``hessian="psd"``), in ``v``'s shape, and the curvature record, a float32 CUDA
        tensor ``[c1 vMv + c2 vHb+v + c3 vHa+v, vMv, vHb+v, vHa+v]``.  Coefficients must be >= 0.  No host sync."""
        if self.hessian != "psd":
            raise RuntimeError('DevicePCG.hvp_psd needs a workspace created with hessian="psd"')
        n3, dev = self.tet_sp.n3, self.tet_sp.device
        xc, vc = self._f32(x, n3, "x"), self._f32(v, n3, "v")
        hv = torch.empty_like(vc)
        curv = torch.empty(4, dtype=torch.float32, device=dev)
        terms = self._capi.tsb_terms_t(c1=float(c1), c2=float(c2), order=int(order), c3=float(c3))
        rc = self._capi.lib.tsb_pcg_hvp_psd(self._s, xc.data_ptr(), vc.data_ptr(), C.byref(terms), hv.data_ptr(), curv.data_ptr(),
                                            self._stream_ptr(dev))
        self._check(rc, "hvp_psd")
        return hv.reshape(v.shape), curv

    def axpy(self, x: torch.Tensor, a_sphere: torch.Tensor, d: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``x + a_sphere[sphere of v] * d`` per vertex (``tsb_sphere_axpy``), in ``x``'s shape; vertices no tet
        references are copied.  ``out`` may be ``x`` (in place)."""
        n3 = self.tet_sp.n3
        xc, dc, ac = self._f32(x, n3, "x"), self._f32(d, n3, "d"), self._f32(a_sphere, self.n_spheres, "a_sphere")
        if out is None:
            out = torch.empty_like(xc)
        elif self._f32(out, n3, "out") is not out:
            raise RuntimeError("out must be contiguous")
        rc = self._capi.lib.tsb_sphere_axpy(self._s, xc.data_ptr(), ac.data_ptr(), dc.data_ptr(), out.data_ptr(),
                                            self._stream_ptr(self.tet_sp.device))
        self._check(rc, "axpy")
        return out


#: options of ``DeviceNewton.step`` (``tsb_newton_options_t``)
NEWTON_DEFAULTS = dict(max_iter=20, rtol=1e-2, rel_floor=1e-6, tau=1e-3, mu_min=1e-12, mu_max=1e12, gtol=0.0, sigma=1e-4,
                       eta=0.9, n_alpha=8)


class NewtonStepResult(NamedTuple):
    """What ``DeviceNewton.step`` returns: device tensors [S], spheres in the order of their lowest vertex ids
    (``tsb_newton_sphere_t`` in ``include/tssplat_b200.h``)."""
    grad_norm: torch.Tensor         # f32: |grad_c| before the step (0 once the sphere is frozen)
    alpha: torch.Tensor             # f32: step taken (0: none)
    k: torch.Tensor                 # i32: index of the step size 2^-k taken, -1 when none
    delta: torch.Tensor             # f32: E_c(x + alpha d) - E_c(x) of the step taken (0 if none)
    mu: torch.Tensor                # f64: damping after the update
    rho: torch.Tensor               # f64: gain ratio of the full step (0 when no decision ran)
    pcg_status: torch.Tensor        # i32: TSB_PCG_* of the damped solve
    n_hvp: torch.Tensor             # i32: products in which the sphere was active
    b_dot_d: torch.Tensor           # f32: b_c . d_c, b = -grad
    status: torch.Tensor            # i32: 0 active, 1 converged, 2 stalled (both frozen)
    first_vertex: torch.Tensor      # i32: lowest vertex id of the sphere


#: options of ``DeviceNewton.tr_step`` (``tsb_newton_tr_options_t``)
NEWTON_TR_DEFAULTS = dict(max_iter=20, rtol=1e-2, rel_floor=1e-6, gtol=0.0, radius_init=1.0, radius_min=1e-12,
                          radius_max=1e12, accept=1e-4, eta=0.9)

#: options of ``DeviceNewton.trls_step``: ``NEWTON_TR_DEFAULTS`` and the backtracking (``tsb_newton_backtrack_t``)
NEWTON_TRLS_DEFAULTS = dict(NEWTON_TR_DEFAULTS, n_alpha=8, sigma=1e-4)


class NewtonTRStepResult(NamedTuple):
    """What ``DeviceNewton.tr_step`` returns: device tensors [S], spheres in the order of their lowest vertex ids
    (``tsb_newton_tr_sphere_t`` in ``include/tssplat_b200.h``)."""
    grad_norm: torch.Tensor         # f32: |grad_c| before the step (0 once the sphere is frozen)
    alpha: torch.Tensor             # f32: 1 when the step was taken, else 0 (trls_step: the fraction 2^-k taken, or 0)
    delta: torch.Tensor             # f32: objective change of the step taken (0 if none)
    radius: torch.Tensor            # f64: trust radius after the update (preconditioner norm)
    rho: torch.Tensor               # f64: gain ratio -delta(1) / pred (0 when pred <= 0 or no decision ran)
    pred: torch.Tensor              # f32: model decrease b.d - d^T H d / 2
    d_norm: torch.Tensor            # f32: |d_c|_M of the solve's step
    pcg_status: torch.Tensor        # i32: TSB_PCG_* of the trust-region solve
    n_hvp: torch.Tensor             # i32: products in which the sphere was active
    b_dot_d: torch.Tensor           # f32: b_c . d_c, b = -grad
    status: torch.Tensor            # i32: 0 active, 1 converged, 2 stalled (both frozen)
    first_vertex: torch.Tensor      # i32: lowest vertex id of the sphere


#: options of ``DeviceNewton.lbfgs_step`` (``tsb_newton_lbfgs_options_t``)
NEWTON_LBFGS_DEFAULTS = dict(m=8, sigma=1e-4, eta=0.9, n_alpha=8, rel_floor=1e-6, gtol=0.0, curv_eps=1e-8)


class NewtonLBFGSStepResult(NamedTuple):
    """What ``DeviceNewton.lbfgs_step`` returns: device tensors [S], spheres in the order of their lowest vertex ids
    (``tsb_newton_lbfgs_sphere_t`` in ``include/tssplat_b200.h``)."""
    grad_norm: torch.Tensor         # f32: |grad_c| before the step (0 once the sphere is frozen)
    alpha: torch.Tensor             # f32: step taken (0: none)
    k: torch.Tensor                 # i32: index of the step size 2^-k taken, -1 when none
    delta: torch.Tensor             # f32: objective change of the step taken (0 if none)
    b_dot_d: torch.Tensor           # f32: b_c . d_c, b = -grad
    d_norm: torch.Tensor            # f32: |d_c|
    n_pairs: torch.Tensor           # i32: (s, y) pairs held after the step
    pair_kept: torch.Tensor         # i32: -1 no pair this step, 0 rejected by the curvature test, 1 kept
    history_cleared: torch.Tensor   # i32: 1 when the history was cleared this step
    status: torch.Tensor            # i32: 0 active, 1 converged, 2 stalled (both frozen)
    first_vertex: torch.Tensor      # i32: lowest vertex id of the sphere


class _Method(NamedTuple):
    defaults: dict                  # the options and their defaults
    what: str                       # what an unknown option's error calls them
    structs: tuple                  # the C entry's option structs (names in _capi), filled by field name from the options
    entry: str                      # the C entry (anchor and weight may be null unless ``plain`` takes that case)
    plain: Optional[str]            # the C entry without anchor and weight, if another
    record: str                     # the record struct
    result: type
    name: str                       # the DeviceNewton method


_STEPS = {
    "lm": _Method(NEWTON_DEFAULTS, "Newton", ("tsb_newton_options_t",), "tsb_newton_prox_step", "tsb_newton_step",
                  "tsb_newton_sphere_t", NewtonStepResult, "step"),
    "tr": _Method(NEWTON_TR_DEFAULTS, "trust-region", ("tsb_newton_tr_options_t",), "tsb_newton_tr_step", None,
                  "tsb_newton_tr_sphere_t", NewtonTRStepResult, "tr_step"),
    "trls": _Method(NEWTON_TRLS_DEFAULTS, "backtracking trust-region", ("tsb_newton_tr_options_t", "tsb_newton_backtrack_t"),
                    "tsb_newton_tr_step_ex", None, "tsb_newton_tr_sphere_t", NewtonTRStepResult, "trls_step"),
    "lbfgs": _Method(NEWTON_LBFGS_DEFAULTS, "L-BFGS", ("tsb_newton_lbfgs_options_t",), "tsb_newton_lbfgs_step", None,
                     "tsb_newton_lbfgs_sphere_t", NewtonLBFGSStepResult, "lbfgs_step"),
}

#: the steps of ``DeviceNewton.minimize``: Levenberg-Marquardt (``step``), trust region (``tr_step``), backtracking
#: trust region (``trls_step``) or L-BFGS (``lbfgs_step``)
METHODS = tuple(_STEPS)


class DeviceNewton:
    """Damped Newton workspace (``tsb_newton_create``) of one ``TetSpheres`` handle: reuses ``pcg`` (a ``DevicePCG`` of
    the same handle) or creates one, and keeps it alive.  Every sphere runs its own Levenberg-Marquardt iteration;
    ``reset`` starts them all again.  Serves one stream at a time, like the handle.  ``hessian``: the solve's model,
    ``"exact"`` or ``"psd"`` (the projected Hessian, see ``DevicePCG``); ``None`` takes ``pcg``'s, or ``"exact"`` when a
    workspace is created.  A given ``pcg`` of another mode is an error.  ``precond`` follows the same rules: ``"jacobi"``
    or ``"sgs"`` (see ``DevicePCG``); on an SGS workspace every step assembles the Hessian and takes its preconditioner
    diagonal from it.  ``coarse``: ``None`` or ``"affine"`` (see ``DevicePCG``), taken from ``pcg`` when one is given (a
    different value is an error); on a coarse workspace every damped and proximal step forms the coarse matrix at its
    point, and ``tr_step`` / ``trls_step`` are refused (``tsb_newton_tr_step``: the two-level norm is near-singular along
    the coarse modes and the trust-region steps stall).  ``lbfgs_step`` takes block Jacobi alone as its initial inverse
    Hessian, so it is refused on an SGS or coarse workspace."""

    def __init__(self, tet_sp, pcg: Optional[DevicePCG] = None, hessian: Optional[str] = None,
                 precond: Optional[str] = None, coarse: Optional[str] = None):
        from . import _capi
        from .tet_spheres_ext import _stream_ptr
        self._capi, self._stream_ptr = _capi, _stream_ptr
        self._nw = None
        if hessian is not None and hessian not in HESSIANS:
            raise ValueError(f"hessian must be one of {HESSIANS}, got {hessian!r}")
        if precond is not None and precond not in PRECONDS:
            raise ValueError(f"precond must be one of {PRECONDS}, got {precond!r}")
        if coarse not in COARSES:
            raise ValueError(f"coarse must be one of {COARSES}, got {coarse!r}")
        if pcg is None:
            pcg = DevicePCG(tet_sp, hessian=hessian or "exact", precond=precond or "jacobi", coarse=coarse)
        elif pcg.tet_sp is not tet_sp:
            raise RuntimeError("DeviceNewton: pcg belongs to another handle")
        elif hessian is not None and pcg.hessian != hessian:
            raise RuntimeError(f"DeviceNewton: hessian={hessian!r} but pcg was created with hessian={pcg.hessian!r}")
        elif precond is not None and pcg.precond != precond:
            raise RuntimeError(f"DeviceNewton: precond={precond!r} but pcg was created with precond={pcg.precond!r}")
        elif coarse is not None and pcg.coarse != coarse:
            raise RuntimeError(f"DeviceNewton: coarse={coarse!r} but pcg was created with coarse={pcg.coarse!r}")
        self.hessian, self.precond, self.coarse = pcg.hessian, pcg.precond, pcg.coarse
        self.tet_sp, self.pcg, self.n_spheres = tet_sp, pcg, pcg.n_spheres
        nw = C.c_void_p()
        rc = _capi.lib.tsb_newton_create(pcg._s, C.byref(nw))
        if rc:
            raise RuntimeError(f"DeviceNewton: {self._error(None)} (code {rc})")
        self._nw = nw

    @property
    def device_bytes(self) -> int:
        """``tsb_newton_device_bytes``: grows by 8 bytes per chunk at the first proximal step, by 20 bytes per sphere
        at the first trust-region step and by the L-BFGS history at the first ``lbfgs_step``."""
        return int(self._capi.lib.tsb_newton_device_bytes(self._nw))

    def __del__(self):
        nw, self._nw = getattr(self, "_nw", None), None
        if nw:
            try:
                self._capi.lib.tsb_newton_destroy(nw)
            except Exception:  # interpreter shutdown
                pass

    def _error(self, nw) -> str:
        msg = self._capi.lib.tsb_newton_last_error(nw)
        return msg.decode("utf-8", "replace") if msg else ""

    def _check(self, rc: int, what: str) -> None:
        if rc:
            raise RuntimeError(f"DeviceNewton.{what}: {self._error(self._nw)} (code {rc})")

    def reset(self) -> None:
        """Every sphere ACTIVE again, its damping (and trust radius) re-initialised at the next step and its L-BFGS
        history emptied."""
        self._check(self._capi.lib.tsb_newton_reset(self._nw, self._stream_ptr(self.tet_sp.device)), "reset")

    def _options(self, method: str, opts: dict) -> list:
        """The option structs of ``method``'s C entry from its defaults updated with ``opts``."""
        m = _STEPS[method]
        bad = set(opts) - set(m.defaults)
        if bad:
            raise TypeError(f"unknown {m.what} options: {sorted(bad)}")
        o = {**m.defaults, **opts}
        structs = [getattr(self._capi, name) for name in m.structs]
        return [S(**{k: (int(o[k]) if t is C.c_int32 else float(o[k])) for k, t in S._fields_ if k in o}) for S in structs]

    def options(self, **opts):
        """``tsb_newton_options_t`` from ``NEWTON_DEFAULTS`` updated with ``opts``."""
        return self._options("lm", opts)[0]

    def tr_options(self, **opts):
        """``tsb_newton_tr_options_t`` from ``NEWTON_TR_DEFAULTS`` updated with ``opts``."""
        return self._options("tr", opts)[0]

    def trls_options(self, **opts):
        """(``tsb_newton_tr_options_t``, ``tsb_newton_backtrack_t``) from ``NEWTON_TRLS_DEFAULTS`` updated with ``opts``."""
        return tuple(self._options("trls", opts))

    def lbfgs_options(self, **opts):
        """``tsb_newton_lbfgs_options_t`` from ``NEWTON_LBFGS_DEFAULTS`` updated with ``opts``."""
        return self._options("lbfgs", opts)[0]

    def _x_anchor(self, x, anchor, weight):
        """Checks x (updated in place) and the proximal pair; returns the weight tensor or None."""
        xc = self.pcg._f32(x, self.tet_sp.n3, "x")
        if xc is not x:
            raise RuntimeError("x must be contiguous (it is updated in place)")
        if anchor is None and weight is not None:
            raise RuntimeError("weight needs an anchor")
        if anchor is None:
            return None
        if weight is None:
            raise RuntimeError("an anchor needs a weight (a float or a float32 CUDA tensor of one entry per sphere)")
        if self.pcg._f32(anchor, self.tet_sp.n3, "anchor") is not anchor:
            raise RuntimeError("anchor must be contiguous")
        if anchor.data_ptr() == x.data_ptr():
            raise RuntimeError("anchor must not be x (x is updated in place while the anchor is read)")
        return self.pcg._shift(weight, "weight")

    def _step(self, method: str, x, c1, c2, order, c3, anchor, weight, opts: dict):
        """One step of ``method`` (a key of ``_STEPS``): the runner of ``step``, ``tr_step`` and ``trls_step``."""
        m = _STEPS[method]
        opt = self._options(method, opts)
        w = self._x_anchor(x, anchor, weight)
        rec = getattr(self._capi, m.record)
        raw = torch.empty((self.n_spheres, C.sizeof(rec)), dtype=torch.uint8, device=self.tet_sp.device)
        terms = self._capi.tsb_terms_t(c1=float(c1), c2=float(c2), order=int(order), c3=float(c3))
        args = (C.byref(terms), *(C.byref(o) for o in opt), raw.data_ptr(), self._stream_ptr(self.tet_sp.device))
        if anchor is None and m.plain:
            rc = getattr(self._capi.lib, m.plain)(self._nw, x.data_ptr(), *args)
        else:
            rc = getattr(self._capi.lib, m.entry)(self._nw, x.data_ptr(), anchor.data_ptr() if anchor is not None else None,
                                                  w.data_ptr() if w is not None else None, *args)
        self._check(rc, m.name)
        f = self._capi.record_fields(raw, rec)
        return m.result(*(f[k] for k in m.result._fields))

    def lbfgs_step(self, x: torch.Tensor, c1: float, c2: float, order: int, c3: float = 0.0,
                   anchor: Optional[torch.Tensor] = None, weight=None, **opts) -> NewtonLBFGSStepResult:
        """One L-BFGS step (``tsb_newton_lbfgs_step``) of ``c1 * smooth + c2 * barrier (+ c3 * amips)`` on every sphere,
        or of the proximal objective with ``anchor`` and ``weight`` as in ``step``; ``x`` is updated in place without a
        host read.  Each sphere keeps up to ``m`` pairs ``(s, y)`` of its own earlier steps (a pair is kept when
        ``s.y > curv_eps |s| |y|``); the direction is the two-loop recursion with the block-Jacobi preconditioner at
        ``x`` as the initial inverse Hessian, and the step is the largest ``2^-k`` with the damped step's Armijo test
        below the inversion bound.  No step clears the sphere's history, and no step from an empty history stalls it.
        ``opts``: the fields of ``NEWTON_LBFGS_DEFAULTS``; ``m`` is fixed by the first call.  ``reset`` empties every
        history.  The first call on a workspace allocates, so it cannot be captured in a CUDA graph; later ones can."""
        return self._step("lbfgs", x, c1, c2, order, c3, anchor, weight, opts)

    def trls_step(self, x: torch.Tensor, c1: float, c2: float, order: int, c3: float = 0.0,
                  anchor: Optional[torch.Tensor] = None, weight=None, **opts) -> NewtonTRStepResult:
        """One backtracking trust-region Newton step (``tsb_newton_tr_step_ex``): ``tr_step``, except that a step the
        trust-region rule rejects (it would invert a tet, or the model predicted the change poorly) is backtracked to the
        largest ``2^-k``, ``1 <= k < n_alpha``, below the inversion bound with the Armijo decrease
        ``dPhi <= -sigma 2^-k b.d``; the radius then becomes ``max(2^-k |d|_M, radius / 4)``, clamped.  The result's
        ``alpha`` is the fraction taken (1, ``2^-k`` or 0).  ``opts``: the fields of ``NEWTON_TRLS_DEFAULTS``.  The first
        call on a workspace allocates (as ``tr_step``'s), so it cannot be captured in a CUDA graph; later ones can."""
        return self._step("trls", x, c1, c2, order, c3, anchor, weight, opts)

    def tr_step(self, x: torch.Tensor, c1: float, c2: float, order: int, c3: float = 0.0,
                anchor: Optional[torch.Tensor] = None, weight=None, **opts) -> NewtonTRStepResult:
        """One trust-region Newton step (``tsb_newton_tr_step``) of ``c1 * smooth + c2 * barrier (+ c3 * amips)`` on every
        sphere, or of the proximal objective with ``anchor`` and ``weight`` as in ``step``; ``x`` is updated in place
        without a host read.  Each sphere keeps a radius in the preconditioner norm: the solve stays inside it (following
        negative curvature to its boundary), the step is taken whole or not at all, and the gain ratio grows or shrinks
        the radius.  ``opts``: the fields of ``NEWTON_TR_DEFAULTS``.  The first call on a workspace allocates, so it
        cannot be captured in a CUDA graph; later ones can."""
        return self._step("tr", x, c1, c2, order, c3, anchor, weight, opts)

    def step(self, x: torch.Tensor, c1: float, c2: float, order: int, c3: float = 0.0, anchor: Optional[torch.Tensor] = None,
             weight=None, **opts) -> NewtonStepResult:
        """One damped Newton step of ``c1 * smooth + c2 * barrier (+ c3 * amips)`` on every sphere, updating ``x`` (a
        contiguous float32 CUDA tensor of 3n entries) in place, without a host read (capturable in a CUDA graph).
        ``opts``: the fields of ``NEWTON_DEFAULTS``.

        With an ``anchor`` y (a contiguous float32 tensor of 3n entries on the handle's device, not ``x`` itself) the
        step is one of the proximal objective ``E(x) + (w_c / 2) |x_c - y_c|^2`` per sphere (``tsb_newton_prox_step``);
        ``weight`` is then required: a float for every sphere, or a float32 CUDA tensor [S] read on the device.  The
        records' ``grad_norm``, ``delta`` and ``b_dot_d`` are then those of the proximal objective, and a sphere whose
        weight is NaN, infinite or negative is frozen (STALLED) without moving.  A linear term ``q . x`` folds into the
        anchor: pass ``y = x0 - q / w``."""
        return self._step("lm", x, c1, c2, order, c3, anchor, weight, opts)

    def minimize(self, x: torch.Tensor, n_steps: int, c1: float, c2: float, order: int, c3: float = 0.0,
                 check_every: int = 0, anchor: Optional[torch.Tensor] = None, weight=None, method: str = "lm", **opts):
        """Up to ``n_steps`` calls of ``step`` (``method="lm"``), ``tr_step`` (``method="tr"``, ``opts`` then the fields
        of ``NEWTON_TR_DEFAULTS``), ``trls_step`` (``method="trls"``, the fields of ``NEWTON_TRLS_DEFAULTS``) or
        ``lbfgs_step`` (``method="lbfgs"``, the fields of ``NEWTON_LBFGS_DEFAULTS``); returns
        (steps run, the last result).  ``check_every = 0`` never touches the host
        (capturable); ``k > 0`` reads one integer, the number of spheres still active, every ``k`` steps and stops when
        it is 0 (refused while the stream is being captured).  ``anchor`` and ``weight``: the proximal step of
        ``step``."""
        if method not in METHODS:
            raise ValueError(f"method must be one of {METHODS}, got {method!r}")
        if check_every < 0 or n_steps < 0:
            raise ValueError("n_steps and check_every must be >= 0")
        if check_every > 0 and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("DeviceNewton.minimize: check_every > 0 reads the host and cannot be captured in a CUDA "
                               "graph: use check_every = 0")
        if anchor is not None and weight is not None and not isinstance(weight, torch.Tensor):
            weight = self.pcg._shift(weight, "weight")         # one tensor for every step
        res = None
        for i in range(n_steps):
            res = self._step(method, x, c1, c2, order, c3, anchor, weight, opts)
            if check_every > 0 and (i + 1) % check_every == 0 and i + 1 < n_steps:
                if int((res.status == 0).sum()) == 0:
                    return i + 1, res
        return n_steps, res

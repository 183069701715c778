"""Block-Jacobi preconditioned truncated Newton-CG over the geometry energy's second-order calls.

``TetSpheres.hess_diag`` gives the per-vertex 3x3 diagonal blocks of the Hessian as two [n, 3] planes;
``block_jacobi`` turns them into an SPD preconditioner, and ``pcg`` runs truncated conjugate gradients over a
Hessian-vector product (``TetSpheres.hvp``), stopping at negative curvature.  Plain torch on the planes' device; the
Hessian itself is only ever touched through the CUDA library's launches.  INTEGRATION.md shows one Newton step built
from these and ``TetSpheres.line_search``.
"""
from __future__ import annotations

from typing import Callable, NamedTuple, Optional, Union

import torch

__all__ = ["hess_blocks", "block_jacobi", "apply_blocks", "pcg", "PCGResult"]


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

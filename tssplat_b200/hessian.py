"""The geometry energy's Hessian as a sparse matrix: 3x3 block-CSR over all vertices (``tsb_hessian_create``,
``tsb_hessian_assemble``).

``DeviceHessian(pcg)`` assembles the matrix a ``newton.DevicePCG`` workspace's solve multiplies by: the exact Hessian of
``c1 * smooth + c2 * barrier (+ c3 * amips)``, or with ``DevicePCG(..., hessian="psd")`` the one whose tet blocks are
projected to PSD.  The layout is what ``torch.sparse_bsr_tensor`` and ``scipy.sparse.bsr_matrix`` take: ``crow`` int32
[n + 1], ``col`` int32 [nnzb] (ascending inside a row), values float32 [nnzb, 3, 3], both triangles stored, no block
between two spheres, empty rows for vertices no tet references.  Use it for a sparse direct solve, a stronger
preconditioner, or a look at one sphere's spectrum (``sphere``).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

__all__ = ["DeviceHessian"]


class DeviceHessian:
    """Hessian workspace beside a ``DevicePCG`` (which it keeps alive), in the mode of that workspace (``hessian``, when
    given, must be that mode).  Creating it builds
    the block pattern on the host and allocates (``device_bytes``), so not inside a CUDA graph capture; ``assemble`` with
    ``out`` has no host read and no allocation and can be captured."""

    def __init__(self, pcg, hessian: Optional[str] = None):
        from . import _capi
        from .tet_spheres_ext import _stream_ptr
        self._capi, self._stream_ptr = _capi, _stream_ptr
        self._hs = None
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("DeviceHessian allocates device memory and cannot be created during a CUDA graph capture")
        if hessian is not None and hessian != pcg.hessian:
            raise RuntimeError(f"DeviceHessian: hessian={hessian!r} but pcg was created with hessian={pcg.hessian!r}")
        tet_sp = pcg.tet_sp
        self.pcg, self.tet_sp, self.hessian = pcg, tet_sp, pcg.hessian
        hs = C.c_void_p()
        rc = _capi.lib.tsb_hessian_create(pcg._s, tet_sp.vertices.ctypes.data, tet_sp.elements.ctypes.data,
                                          int(tet_sp.nele), C.byref(hs))
        if rc:
            raise RuntimeError(f"DeviceHessian: {self._error(None)} (code {rc})")
        self._hs = hs
        nnzb = C.c_int64(0)
        self._check(_capi.lib.tsb_hessian_pattern(hs, C.byref(nnzb), None, None, None), "__init__")
        self.nnzb = int(nnzb.value)
        dev = tet_sp.device
        self.crow = torch.empty(tet_sp.n + 1, dtype=torch.int32, device=dev)
        self.col = torch.empty(self.nnzb, dtype=torch.int32, device=dev)
        self._check(_capi.lib.tsb_hessian_pattern(hs, None, self.crow.data_ptr(), self.col.data_ptr(), self._stream_ptr(dev)),
                    "__init__")
        self.device_bytes = int(_capi.lib.tsb_hessian_device_bytes(hs))
        self._host = None

    def __del__(self):
        hs, self._hs = getattr(self, "_hs", None), None
        if hs:
            try:
                self._capi.lib.tsb_hessian_destroy(hs)
            except Exception:  # interpreter shutdown
                pass

    def _error(self, hs) -> str:
        msg = self._capi.lib.tsb_hessian_last_error(hs)
        return msg.decode("utf-8", "replace") if msg else ""

    def _check(self, rc: int, what: str) -> None:
        if rc:
            raise RuntimeError(f"DeviceHessian.{what}: {self._error(self._hs)} (code {rc})")

    def assemble(self, x: torch.Tensor, c1: float, c2: float, order: int, c3: float = 0.0,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Block values [nnzb, 3, 3] of the Hessian at ``x`` (a float32 tensor of 3n entries on the handle's device), with
        ``tsb_hvp_ex``'s rules for the terms (and coefficients >= 0 in PSD mode).  ``out``: a contiguous float32 tensor of
        9 nnzb entries, fully overwritten and returned (then no allocation: capturable)."""
        xc = self.pcg._f32(x, self.tet_sp.n3, "x")
        if out is None:
            out = torch.empty((self.nnzb, 3, 3), dtype=torch.float32, device=self.tet_sp.device)
        elif self.pcg._f32(out, 9 * self.nnzb, "out") is not out:
            raise RuntimeError("out must be contiguous")
        terms = self._capi.tsb_terms_t(c1=float(c1), c2=float(c2), order=int(order), c3=float(c3))
        rc = self._capi.lib.tsb_hessian_assemble(self._hs, xc.data_ptr(), C.byref(terms), out.data_ptr(),
                                                 self._stream_ptr(self.tet_sp.device))
        self._check(rc, "assemble")
        return out

    def matrix(self, x: torch.Tensor, c1: float, c2: float, order: int, c3: float = 0.0) -> torch.Tensor:
        """``assemble`` as a ``torch.sparse_bsr_tensor`` of size [3n, 3n]."""
        v = self.assemble(x, c1, c2, order, c3=c3)
        n3 = self.tet_sp.n3
        return torch.sparse_bsr_tensor(self.crow, self.col, v, size=(n3, n3))

    def sphere_vertices(self, c: int) -> np.ndarray:
        """Vertex ids of sphere ``c`` (spheres in the order of their lowest vertex id, as everywhere in the library),
        ascending: the local numbering of ``sphere``."""
        if self._host is None:
            import scipy.sparse as sp
            from scipy.sparse.csgraph import connected_components
            crow, col = self.crow.cpu().numpy(), self.col.cpu().numpy()
            n = len(crow) - 1
            g = sp.csr_matrix((np.ones(len(col), np.int8), col, crow), shape=(n, n))
            _, lab = connected_components(g, directed=False)
            used = np.diff(crow) > 0
            first = {}
            for v in np.nonzero(used)[0]:
                first.setdefault(int(lab[v]), int(v))
            order = sorted(first, key=first.get)
            self._host = (crow, col, [np.nonzero((lab == L) & used)[0] for L in order])
        return self._host[2][c]

    def sphere(self, values: torch.Tensor, c: int):
        """Sphere ``c``'s block of ``values`` (from ``assemble``) as a ``scipy.sparse.bsr_matrix`` in the sphere's local
        numbering (``sphere_vertices``).  A host copy, for inspection and tests."""
        import scipy.sparse as sp
        verts = self.sphere_vertices(c)
        crow, col, _ = self._host
        local = np.full(len(crow) - 1, -1, np.int64)
        local[verts] = np.arange(len(verts))
        rows = [np.arange(crow[v], crow[v + 1]) for v in verts]
        idx = np.concatenate(rows)
        lcrow = np.concatenate([[0], np.cumsum([len(r) for r in rows])])
        vals = values.reshape(-1, 3, 3)[torch.from_numpy(idx).to(values.device)].cpu().numpy()
        return sp.bsr_matrix((vals, local[col[idx]], lcrow), shape=(3 * len(verts), 3 * len(verts)))

"""Generates tests/golden/surface_edge_fixtures.npz from REFERENCE-HELD code imported from a checkout of the reference
(gmh14/tssplat); the tests read only the committed fixture:

* geometry/mesh_utils.py:5-35          get_surface_vf          -> surface vertex ids + surface triangles
* geometry/tetmesh_geometry.py:39-66   _compute_vertex_normal  -> vertex normals (its function body, executed)

on the small edge meshes of tests/test_surface_rows.py: a sphere squashed in z by 1e-3, two spheres scaled to sit 10x
above and 10x below the 1e-20 degenerate-normal threshold, a duplicated tet with faces shared by three and four tets,
tets that repeat a vertex (degenerate (a, a, b) faces), and a hand-made surface (shuffled order, an entry no face uses,
an (a, a, b) face) whose normals alone are pinned.  Per mesh: tets (extraction meshes), x, surface_vid, surface_f,
v_nrm.  The repeated-vertex mesh has extraction only: its surface vertices whose every face is degenerate get a normal
from fp32 rounding noise (cross(e, e) under FMA is not 0), where the fp64 restatement falls back to (0, 0, 1).

No mesh has exactly three surface faces: the reference calls torch.cross without dim, which on a [3, 3] input
crosses along dim 0.

    python tests/golden/make_surface_fixtures.py <reference checkout>
"""
import ast
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
REF = None      # the reference checkout (first command-line argument)


def _load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _reference_normal_fn():
    import torch.nn.functional as F_
    src = open(os.path.join(REF, "geometry/tetmesh_geometry.py")).read()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "TetMeshGeometryForwardData")
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "_compute_vertex_normal")
    ns = {"torch": torch, "F": F_, "dot": lambda a, b: torch.sum(a * b, -1, keepdim=True)}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "ref:_compute_vertex_normal", "exec"), ns)
    return ns["_compute_vertex_normal"]


def main():
    import test_surface_rows as tsr
    mu = _load("ref_mesh_utils", "geometry/mesh_utils.py")
    normals = _reference_normal_fn()
    rng = np.random.default_rng(17)

    meshes = {"squashed": (tsr._sphere()[1], tsr.surface_case("squashed")[0])}
    for name, factor in (("thresh_above", 10.0), ("thresh_below", 0.1)):
        meshes[name] = tsr.threshold_sphere(factor)
    for name, T in (("shared_faces", tsr.shared_face_tets()), ("repeated_vertex", tsr.repeated_vertex_tets())):
        meshes[name] = (T, rng.normal(size=(int(T.max()) + 1, 3)).astype(np.float32))

    out = {}
    for name, (T, x) in meshes.items():
        sv, sf = mu.get_surface_vf(np.asarray(T, np.int64))
        out[name + "/tets"] = np.asarray(T, np.int32)
        out[name + "/x"] = np.asarray(x, np.float32)
        out[name + "/surface_vid"] = np.asarray(sv, np.int64)
        out[name + "/surface_f"] = np.asarray(sf, np.int64).reshape(-1, 3)
    x, sv, sf = tsr.handmade_surface()
    out["handmade/x"], out["handmade/surface_vid"], out["handmade/surface_f"] = x, sv.astype(np.int64), sf.astype(np.int64)

    for name in ["squashed", "thresh_above", "thresh_below", "shared_faces", "handmade"]:
        x, sv, sf = out[name + "/x"], out[name + "/surface_vid"], out[name + "/surface_f"]
        assert len(sf) != 3, name
        obj = types.SimpleNamespace(v_pos=torch.from_numpy(x)[torch.from_numpy(sv)], t_pos_idx=torch.from_numpy(sf))
        out[name + "/v_nrm"] = normals(obj).numpy()
    np.savez_compressed(os.path.join(HERE, "surface_edge_fixtures.npz"), **out)
    print("wrote", os.path.join(HERE, "surface_edge_fixtures.npz"), {k: np.asarray(v).shape for k, v in out.items()})


if __name__ == "__main__":
    REF = sys.argv[1]
    main()

"""tools/_timing.py, the harness of the tools/time_*.py scripts, on the CPU: its pack builder reproduces both mixed
64 x 4096 packs the scripts measured on, its sphere ids are the mesh's connected components, and every script imports
without running."""
import glob
import importlib
import os
import sys

import numpy as np
import pytest

pytest.importorskip("torch")

from _newton_model import _pack
from tssplat_b200.mesh import connected_components, make_pack, perturb

TOOLS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools")
if TOOLS not in sys.path:
    sys.path.insert(0, TOOLS)
import _timing  # noqa: E402

# time_surface_extract.py is a script body, not a module: it measures on import
SCRIPTS = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(TOOLS, "time_*.py"))
                 if not p.endswith("time_surface_extract.py"))


@pytest.fixture(scope="module")
def packs():
    """The two mixed packs: seeds (1, 3), as tests/_newton_model.py, and (0, 0), as time_newton.py and time_tr.py."""
    return {seeds: _timing.mixed_pack(64, *seeds, 4) for seeds in ((1, 3), (0, 0))}


def test_mixed_pack_seeds_1_3_is_the_newton_model_pack(packs):
    pk, x, quiet = packs[1, 3]
    ref_pk, ref_x = _pack("mixed")
    assert np.array_equal(pk.tets, ref_pk.tets) and np.array_equal(pk.verts, ref_pk.verts)
    assert x.dtype == ref_x.dtype and np.array_equal(x, ref_x)
    assert np.array_equal(quiet, np.arange(64) % 4 != 0)


def test_mixed_pack_seeds_0_0_is_the_inline_construction(packs):
    pk, x, quiet = packs[0, 0]
    ref = make_pack(64, 4096, seed=0, unique=8)
    x_np, rough = perturb(ref, sigma_rel=0.02, seed=0), perturb(ref, sigma_rel=0.35, seed=0)
    vo = ref.vert_offsets
    for k in range(0, 64, 4):
        x_np[vo[k]:vo[k + 1]] = rough[vo[k]:vo[k + 1]]
    assert np.array_equal(pk.tets, ref.tets) and np.array_equal(pk.verts, ref.verts)
    assert x.dtype == x_np.dtype and np.array_equal(x, x_np)
    assert np.array_equal(quiet, np.arange(64) % 4 != 0)


def test_rough_every_none_and_one():
    pk, benign, quiet = _timing.mixed_pack(4, 1, 3, None)
    assert quiet.all() and np.array_equal(benign, perturb(pk, sigma_rel=0.02, seed=1))
    _, inverted, quiet = _timing.mixed_pack(4, 1, 3, 1)
    assert not quiet.any() and np.array_equal(inverted, perturb(pk, sigma_rel=0.35, seed=3))


@pytest.mark.parametrize("seeds", [(1, 3), (0, 0)])
def test_sphere_ids_are_the_connected_components(packs, seeds):
    pk = packs[seeds][0]
    lab = connected_components(len(pk.verts), pk.tets)
    used = np.zeros(len(pk.verts), bool)
    used[np.unique(pk.tets)] = True
    assert used.all()
    sid = _timing.sphere_ids(pk).numpy()
    assert sid.dtype == np.int64 and np.array_equal(sid, np.searchsorted(np.unique(lab[used]), lab[used]))


@pytest.mark.parametrize("name", SCRIPTS)
def test_script_imports_without_running(name, monkeypatch):
    monkeypatch.setattr(sys, "argv", [name, "--help"])
    mod = importlib.import_module(name)
    assert callable(mod.main)
    assert not any(m.startswith("time_") for m in _imported_modules(mod)), f"{name} imports another time_*.py"


def _imported_modules(mod):
    import ast
    tree = ast.parse(open(mod.__file__).read())
    for n in ast.walk(tree):
        if isinstance(n, ast.ImportFrom) and n.module:
            yield n.module
        elif isinstance(n, ast.Import):
            yield from (a.name for a in n.names)

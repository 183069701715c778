"""``_capi.record_fields``: the per-field views of the C ABI's per-sphere record structs, checked on the CPU against the
ctypes records they were filled from and against the fixed column tables the Python front ends used to decode them with."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from tssplat_b200 import _capi

S = 5


def _records(struct):
    """S records of `struct` with a distinct value in every scalar field of every record, and array fields set to -7."""
    recs = (struct * S)()
    for s in range(S):
        for k, (name, ctype) in enumerate(struct._fields_):
            if issubclass(ctype, C.Array):
                for j in range(len(getattr(recs[s], name))):
                    getattr(recs[s], name)[j] = -7
            elif ctype in (C.c_float, C.c_double):
                setattr(recs[s], name, 100.0 * s + k + 0.25)
            else:
                setattr(recs[s], name, 100 * s + k + 1)
    raw = torch.from_numpy(np.frombuffer(bytes(recs), dtype=np.uint8).reshape(S, C.sizeof(struct)).copy())
    return recs, raw


# The column tables DevicePCG.solve, DeviceNewton.step, the trust-region steps and TetSpheres.energy_grad_spheres decoded
# the records with before record_fields: field -> (byte slice of the record, dtype, column of that view)
OLD_TABLES = {
    _capi.tsb_pcg_sphere_t: dict(status=((0, 32), torch.int32, 4), n_hvp=((0, 32), torch.int32, 3),
                                 rel_residual=((0, 32), torch.float32, 0), b_dot_d=((0, 32), torch.float32, 1),
                                 d_H_d=((0, 32), torch.float32, 2)),
    _capi.tsb_newton_sphere_t: dict(grad_norm=((16, 32), torch.float32, 0), alpha=((16, 32), torch.float32, 1),
                                    k=((0, 64), torch.int32, 8), delta=((16, 32), torch.float32, 2),
                                    mu=((0, 16), torch.float64, 0), rho=((0, 16), torch.float64, 1),
                                    pcg_status=((0, 64), torch.int32, 9), n_hvp=((0, 64), torch.int32, 10),
                                    b_dot_d=((16, 32), torch.float32, 3), status=((0, 64), torch.int32, 11),
                                    first_vertex=((0, 64), torch.int32, 12)),
    _capi.tsb_newton_tr_sphere_t: dict(grad_norm=((16, 40), torch.float32, 0), alpha=((16, 40), torch.float32, 1),
                                       delta=((16, 40), torch.float32, 2), radius=((0, 16), torch.float64, 0),
                                       rho=((0, 16), torch.float64, 1), pred=((16, 40), torch.float32, 4),
                                       d_norm=((16, 40), torch.float32, 5), pcg_status=((0, 64), torch.int32, 10),
                                       n_hvp=((0, 64), torch.int32, 11), b_dot_d=((16, 40), torch.float32, 3),
                                       status=((0, 64), torch.int32, 12), first_vertex=((0, 64), torch.int32, 13)),
    _capi.tsb_sphere_stats_t: dict(smooth=((0, 24), torch.float64, 0), barrier=((0, 24), torch.float64, 1),
                                   amips=((0, 24), torch.float64, 2), min_J=((24, 28), torch.float32, 0),
                                   n_inverted=((28, 40), torch.int32, 0), n_tets=((28, 40), torch.int32, 1),
                                   first_vertex=((28, 40), torch.int32, 2)),
}
DTYPES = {C.c_float: torch.float32, C.c_double: torch.float64, C.c_int32: torch.int32}


@pytest.mark.parametrize("struct", list(OLD_TABLES), ids=lambda t: t.__name__)
def test_record_fields_match_ctypes_and_the_old_tables(struct):
    recs, raw = _records(struct)
    f = _capi.record_fields(raw, struct)
    scalars = [(n, t) for n, t in struct._fields_ if not issubclass(t, C.Array)]
    assert list(f) == [n for n, _ in scalars]
    for name, ctype in scalars:
        v = f[name]
        assert v.shape == (S,) and v.dtype == DTYPES[ctype], name
        assert v.untyped_storage().data_ptr() == raw.untyped_storage().data_ptr(), name      # a view, not a copy
        assert v.tolist() == [getattr(recs[s], name) for s in range(S)], name
    for name, ((a, b), dtype, col) in OLD_TABLES[struct].items():
        assert torch.equal(f[name], raw[:, a:b].view(dtype)[:, col]), name
    # every field the front ends return is decoded
    assert set(OLD_TABLES[struct]) <= set(f)

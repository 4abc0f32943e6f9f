"""Engine.debug_linear (the gs_debug_linear test hook of the Ridge / ElasticNet pipeline) against a ctypes stand-in for the
library: the arguments it hands over, the two-call protocol (sizes first, then buffers of exactly those sizes) and the
arrays it returns.  No GPU."""
import numpy as np

from spark_sklearn_b200.engine import Engine, GsLinearDebug

SIZES = dict(n_blocks=6, n_plain=3, n_groups=2, n_sys=6, n_rows=10)


class _FakeLib:
    """Records gs_debug_linear calls; answers the sizes-only call with SIZES and fills the buffers of the second call"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            rec = args[-1]._obj
            self.calls.append((name, args[:-1], rec.sizes_only))
            if rec.sizes_only:
                for k, v in SIZES.items():
                    setattr(rec, k, v)
            else:
                rec.cg_iterations = 17
                rows = np.ctypeslib.as_array(ctypes_cast(rec.rows, np.int32), (10,))
                rows[:] = np.arange(10)[::-1]
                np.ctypeslib.as_array(ctypes_cast(rec.block_start, np.int32), (4,))[:] = [0, 3, 7, 10]
            return 0
        return f


def ctypes_cast(addr, dtype):
    import ctypes
    return ctypes.cast(addr, ctypes.POINTER(np.ctypeslib.as_ctypes_type(dtype)))


def _engine(d=5):
    eng = Engine.__new__(Engine)
    eng._L, eng._h = _FakeLib(), None
    eng.n, eng.d, eng.n_splits = 10, d, 2
    return eng


def test_debug_linear_ridge_arguments_and_shapes():
    eng = _engine()
    out = eng.debug_linear([0.5, 1.0, 2.0], fit_intercept=False)
    (n1, a1, s1), (n2, a2, s2) = eng._L.calls
    assert n1 == n2 == "gs_debug_linear" and (s1, s2) == (1, 0)
    assert a1[1:3] == (0, 3) and a1[4] is None and a1[5] == 0 and a1[8] == 0         # ridge, 3 candidates, no l1_ratio
    d, D = 5, 7
    want = dict(shift=(d + 1,), block_shift=(3, d + 1), ystat=(3, 2), G=(6, D, D), T=(D, D), Tw=(D, D), A=(2, d, d),
                rhs=(2, d), means=(2, d + 3), coef=(2, 3, d), qk=(2, 3), qt=(2, 3), scores=(2, 3, 2), test_block=(2,),
                train_block=(2,))
    for k, shape in want.items():
        assert out[k].shape == shape, k
    assert out["A"].dtype == np.float32 and out["G"].dtype == np.float64 and out["test_block"].dtype == np.int32
    assert "n_iter" not in out and "gap" not in out
    assert out["cg_iterations"] == 17 and out["weighted_copies"]
    assert [list(b) for b in out["blocks"]] == [[9, 8, 7], [6, 5, 4, 3], [2, 1, 0]]


def test_debug_linear_enet_and_refit():
    eng = _engine()
    out = eng.debug_linear(0.1, l1_ratio=0.5, tol=1e-6, max_iter=3, refit=True)
    (_, a, _), _ = eng._L.calls
    assert a[1:3] == (1, 1) and a[6:9] == (1e-6, 3, 1)
    assert out["n_iter"].shape == (2, 1) and out["gap"].shape == (2, 1)
    assert "scores" not in out and "qk" not in out                       # a refit is not scored
    assert {f for f, _ in GsLinearDebug._fields_} >= set(out) - {"blocks", "weighted_copies", "cg_iterations"}

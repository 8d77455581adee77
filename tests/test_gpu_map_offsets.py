"""mb200_map on column views that start 0..3 rows into their buffer, across whole tiles and a ragged tail.

Views shifted by an even number of 8-byte rows stay 16-byte aligned and take the vector path; odd shifts take the
scalar path.  Both must give what numpy gives, bit for bit, for 8-byte and 1-byte (bool) operands.
"""
import numpy as np
import pytest

N = 3 * 4096 + 777  # three full 4096-row tiles and a tail
W = 3


def _run(op, dtype_code, ins, out_dtype, shift, s0=None, s1=None):
    import torch

    from modin_b200 import _lib

    lib = _lib.load()
    dev = torch.device("cuda:0")
    bufs = [[torch.from_numpy(np.concatenate([np.zeros(shift, x.dtype), x])).to(dev) for x in cols] for cols in ins]
    outs = [torch.zeros(N + shift, dtype=out_dtype, device=dev) for _ in range(W)]

    def ptrs(ts):
        return _lib.ptr_array([t.data_ptr() + shift * t.element_size() for t in ts])

    args = [ptrs(b) for b in bufs] + [None] * (3 - len(bufs))
    a0 = _lib.u64_array(s0) if s0 is not None else None
    a1 = _lib.u64_array(s1) if s1 is not None else None
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.mb200_map(_lib.OP[op], dtype_code, W, args[0], args[1], args[2], ptrs(outs), N, a0, a1, st))
    torch.cuda.synchronize()
    return [o.cpu().numpy()[shift:] for o in outs]


def _f64_cols(seed):
    rng = np.random.default_rng(seed)
    cols = [rng.standard_normal(N) * 1e3 for _ in range(W)]
    cols[0][::97] = np.nan
    return cols


def _assert_same_f64(got, want):
    """Bit-identical, except that any NaN matches any NaN (the device does not keep NaN payloads)."""
    same = (got.view(np.uint64) == want.view(np.uint64)) | (np.isnan(got) & np.isnan(want))
    assert same.all(), f"{int((~same).sum())} of {len(same)} values differ"


def _bits(vals):
    return [int(np.array(v, dtype=np.float64).view(np.uint64)) for v in vals]


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0, 1, 2, 3])
def test_f64_affine_and_fma3(shift):
    import torch

    from modin_b200 import _lib

    a, b, c = _f64_cols(1), _f64_cols(2), _f64_cols(3)
    got = _run("affine", _lib.F64, [a], torch.float64, shift, _bits([1.25, -3.0, 0.1]),
               _bits([0.5, 7.0, -2.5]))  # fmt: skip
    for j, (s, t) in enumerate(zip([1.25, -3.0, 0.1], [0.5, 7.0, -2.5])):
        _assert_same_f64(got[j], a[j] * s + t)
    got = _run("fma3", _lib.F64, [a, b, c], torch.float64, shift)
    for j in range(W):
        _assert_same_f64(got[j], a[j] * b[j] + c[j])


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0, 1, 2, 3])
def test_f64_predicate_to_bool(shift):
    import torch

    from modin_b200 import _lib

    a = _f64_cols(4)
    got = _run("gt_s", _lib.F64, [a], torch.uint8, shift, _bits([0.0, 10.0, -10.0]))
    for j, s in enumerate([0.0, 10.0, -10.0]):
        np.testing.assert_array_equal(got[j], (a[j] > s).astype(np.uint8))


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0, 1, 2, 3])
def test_i64_add(shift):
    import torch

    from modin_b200 import _lib

    rng = np.random.default_rng(5)
    a = [rng.integers(-(2**62), 2**62, N) for _ in range(W)]
    b = [rng.integers(-(2**62), 2**62, N) for _ in range(W)]
    got = _run("add", _lib.I64, [a, b], torch.int64, shift)
    for j in range(W):
        np.testing.assert_array_equal(got[j], a[j] + b[j])


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0, 1, 2, 3])
def test_bool_and_and_widen(shift):
    import torch

    from modin_b200 import _lib

    rng = np.random.default_rng(6)
    p = [rng.integers(0, 2, N).astype(np.uint8) for _ in range(W)]
    q = [rng.integers(0, 2, N).astype(np.uint8) for _ in range(W)]
    got = _run("and", _lib.U8, [p, q], torch.uint8, shift)
    for j in range(W):
        np.testing.assert_array_equal(got[j], p[j] & q[j])
    got = _run("copy", _lib.U8, [p], torch.int64, shift)
    for j in range(W):
        np.testing.assert_array_equal(got[j], p[j].astype(np.int64))

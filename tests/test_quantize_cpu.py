"""CPU: the quantizer restatement (tests/quantize_ref.py) on hand cases, the quantizer headers as plain C with the ctypes
mirrors' sizes, and the parameter defaults.  No GPU compute calls."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import quantize_ref as Q

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include")


def test_lroundf_rounds_half_away_from_zero():
    f = np.array([0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 0.49999997, -0.49999997, 126.5, -127.5], np.float32)
    assert Q.lroundf(f).tolist() == [1, 2, 3, -1, -2, -3, 0, 0, 127, -128]


def test_transform_half_way_values_round_away_from_zero():
    # lo = -128, hi = 127: scale 1, offset 0, so the code is lroundf(x) itself
    x = np.array([[-127.5, -0.5, 0.5, 1.5, 126.5, 2.25]], np.float32)
    assert Q.scalar_transform(x, -128.0, 127.0).tolist() == [[-128, -1, 1, 2, 127, 2]]


def test_transform_at_the_range_ends_and_nan():
    x = np.array([[-1.0, 1.0, -2.0, 2.0, np.nan, 0.0]], np.float32)
    assert Q.scalar_transform(x, -1.0, 1.0).tolist() == [[-128, 127, -128, 127, -128, -1]]  # 0: lroundf(-0.5)
    lo, hi, scale, offset = Q.scalar_map(-1.0, 1.0, np.float32)
    assert scale == 127.5 and offset == -0.5


def test_equal_range_ends():
    x = np.array([[3.0, 2.0, 4.0, np.nan]], np.float16)
    assert Q.scalar_transform(x, 3.0, 3.0).tolist() == [[-128, -128, 127, -128]]
    lo, hi, scale, offset = Q.scalar_map(3.0, 3.0, np.float16)
    assert scale == 1.0 and offset == -131.0
    assert Q.scalar_inverse(np.array([[-128, 0, 127]], np.int8), 3.0, 3.0).tolist() == [[3.0, 131.0, 258.0]]


def test_range_ends_are_rounded_to_the_data_type():
    lo, hi, _, _ = Q.scalar_map(0.1, 1e10, np.float16)
    assert lo.dtype == np.float16 and float(lo) == float(np.float16(0.1)) and np.isinf(hi)


@pytest.mark.parametrize("S,q,expect", [(1, 0.99, (0, 0)), (1, 1.0, (0, 0)), (2, 0.99, (0, 1)), (2, 0.5, (0, 1)),
                                        (3, 0.99, (0, 2)), (3, 0.3, (1, 1)), (1000, 1.0, (0, 999)), (1000, 0.99, (4, 995)), (200, 0.99, (0, 199))])
def test_quantile_positions(S, q, expect):
    # q is the params struct's float32: 0.99f is 0.99000000953..., so (0.5 + 0.5 q) * 1000 lies just above 995
    assert Q.quantile_positions(S, q) == expect


def test_scalar_train_on_a_whole_sample():
    x = np.arange(1, 201, dtype=np.float32).reshape(20, 10)
    assert Q.scalar_train(x, 0.99) == (1.0, 200.0)  # p = ceil(199.000001) - 1
    assert Q.scalar_train(x, 0.9) == (11.0, 190.0)
    assert Q.scalar_train(x, 1.0) == (1.0, 200.0)


@pytest.mark.parametrize("n,ratio,s", [(100001, 0.1, 9999), (100021, 0.1, 10001), (100000, 0.1, 9999), (10, 0.1, 1), (11, 1.0, 11), (12, 1.0, 11),
                                       (1, 1.0, 1), (2, 1.0, 1), (7, 0.5, 3), (3, 0.01, 1), (1 << 25 | 1, 1.0, (1 << 25) - 1), (1 << 26 | 5, 1.0, 1 << 26 | 5)])
def test_median_sample_size(n, ratio, s):
    got = Q.median_sample_size(n, ratio)
    assert got == s and got % 2 == 1 and got <= n


def test_pack_is_lsb_first_and_strict():
    x = np.array([[1, 0, -1, 2, 0, 0, 0, 0, 5], [np.nan, 1, 1, 1, 1, 1, 1, 1, 0]], np.float32)
    assert Q.pack(x).tolist() == [[0b00001001, 1], [0b11111110, 0]]
    t = np.array([1, 0, 0, 1, 0, 0, 0, 0, 4], np.float32)
    assert Q.pack(x, t).tolist() == [[0b00001000, 1], [0b11110110, 0]]


def test_mean_and_median_thresholds():
    x = np.array([[1, 4], [2, 4], [3, 5], [6, 9]], np.float32)
    assert Q.thresholds(x, "mean").tolist() == [3.0, 5.5]
    assert Q.thresholds(x[:3], "sampling_median", 1.0).tolist() == [2.0, 4.0]
    assert Q.thresholds(x, "zero") is None


def test_inverse_table():
    codes = np.arange(-128, 128, dtype=np.int8)[None, :]
    v = Q.scalar_inverse(codes, -1.0, 1.0, np.float64)
    assert v[0, 0] == -1.0 and v[0, -1] == 1.0
    assert (Q.scalar_transform(v.astype(np.float64), -1.0, 1.0) == codes).all()


def test_headers_compile_as_plain_c_and_sizes_match_the_binding():
    src = r'''
#include <stdio.h>
#include <cuvs/core/all.h>
#include <cuvs/preprocessing/quantize/binary.h>
#include <cuvs/preprocessing/quantize/scalar.h>
int main(void) {
  printf("%zu %zu %zu %zu %d %d %d\n", sizeof(struct cuvsScalarQuantizerParams), sizeof(cuvsScalarQuantizer),
         sizeof(struct cuvsBinaryQuantizerParams), sizeof(cuvsBinaryQuantizer), (int)ZERO, (int)MEAN, (int)SAMPLING_MEDIAN);
  return 0;
}
'''
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "q.c")
        open(c, "w").write(src)
        exe = os.path.join(td, "q")
        subprocess.run(["/usr/bin/gcc", "-std=c11", "-Wall", "-Werror", "-I", INC, "-I", "/usr/local/cuda/include", c, "-o", exe],
                       check=True)
        got = list(map(int, subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()))
    from cuvs_b200 import _capi
    from cuvs_b200.preprocessing.quantize import binary, scalar
    assert got == [C.sizeof(scalar._ParamsC), C.sizeof(scalar._QuantizerC), C.sizeof(binary._ParamsC), C.sizeof(_capi.index_handle),
                   0, 1, 2]


def test_param_defaults():
    from cuvs_b200.preprocessing.quantize import binary, scalar
    assert scalar.QuantizerParams().quantile == pytest.approx(0.99, abs=1e-7)
    p = binary.QuantizerParams()
    assert p.threshold == "mean" and p.sampling_ratio == pytest.approx(0.1, abs=1e-8)
    q = scalar.Quantizer()
    assert (q.min, q.max) == (0.0, 0.0)
    with pytest.raises(ValueError):
        binary.QuantizerParams(threshold="median")

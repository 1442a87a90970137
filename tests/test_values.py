"""Host-side rule behind the FP32 copy of an FP64 operator's values (b200_values_fit_f32): the
operator qualifies only when every value has the same bits after double -> float -> double, so
the streaming passes that read the copy widen each value back to the very same double."""
import struct

import numpy as np
import pytest

import amgcl_b200 as ab


def one(x):
    return np.array([x], dtype=np.float64)


def from_bits(u):
    return struct.unpack("<d", struct.pack("<Q", u))[0]


EXACT = {
    "+0": 0.0,
    "-0": -0.0,
    "+1": 1.0,
    "-1": -1.0,
    "6": 6.0,
    "smallest float subnormal 2^-149": 2.0 ** -149,
    "FLT_MAX 2^127 (2 - 2^-23)": 2.0 ** 127 * (2.0 - 2.0 ** -23),
    "+inf": float("inf"),
    "-inf": float("-inf"),
    "quiet NaN with a float payload": from_bits(0x7FF8000000000000),
}

INEXACT = {
    "0.1": 0.1,
    "1/3": 1.0 / 3.0,
    "2^-150 (rounds to 0)": 2.0 ** -150,
    "1e39 (overflows)": 1e39,
    "double subnormal": 5e-324,
    "NaN whose low payload bits are lost": from_bits(0x7FF8000000000001),
    "signalling NaN (quietened)": from_bits(0x7FF0000000000001),
}


@pytest.mark.parametrize("name", list(EXACT))
def test_exact_values_qualify(name):
    assert ab.values_fit_f32(one(EXACT[name]))


@pytest.mark.parametrize("name", list(INEXACT))
def test_inexact_values_do_not_qualify(name):
    assert not ab.values_fit_f32(one(INEXACT[name]))


@pytest.mark.parametrize("name", list(INEXACT))
def test_one_inexact_value_among_a_million_exact_ones_fails_the_operator(name):
    rng = np.random.default_rng(len(name))
    val = rng.choice(np.array([6.0, -1.0, 0.5, -0.25, 2.0 ** -149, 3.0 * 2.0 ** 100]), size=1_000_000)
    assert ab.values_fit_f32(val)
    for pos in (0, 123457, val.size - 1):
        v = val.copy()
        v[pos] = INEXACT[name]
        assert not ab.values_fit_f32(v)


def test_poisson_operator_and_float_assembled_data_qualify():
    _, _, val, _ = ab.poisson3d(16)
    assert set(np.unique(val)) <= {6.0, -1.0}
    assert ab.values_fit_f32(val)
    rng = np.random.default_rng(5)
    assert ab.values_fit_f32(rng.standard_normal(100_000).astype(np.float32).astype(np.float64))
    assert not ab.values_fit_f32(rng.standard_normal(100_000))


def test_empty_input_qualifies():
    assert ab.values_fit_f32(np.zeros(0))

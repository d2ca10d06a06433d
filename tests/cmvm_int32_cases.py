"""Seeded CMVM inputs at the int32 limit of the CSD step, shared by the golden script and the tests that read its answers.

The CSD step centres each matrix (power-of-two column then row normalisation), converts the centred values to int32 and
takes ``N = ceil(log2(1.5 * max|x|))`` digits.  The family sits on both sides of every width boundary and beyond the int32
range:

- ``edge*``  a centred maximum just below / just above N = 31 (715 827 882.67) and N = 32 (1 431 655 765.33), and the
  largest float32 below 2^31, with both signs.  The large value shares its column and its row with odd values, so the
  centring cannot scale it down.  Float32 holds none of the exact boundaries, so the neighbours on each side are used.
- ``wide31*`` several 31-bit values in one matrix, and 31- and 32-bit values next to small ones.
- ``over*``  centred values of exactly +-2^31, 2^33 and 2^40 among small values in the same row and column: the float ->
  int32 conversion is out of range there.
- ``normal*`` unquantized float32 weights: ``standard_normal`` and ``standard_normal * 2^k``, k in [-12, 12], and a
  matrix whose entries span several powers of two.
- ``nonfinite*`` one +inf, -inf or NaN in an otherwise ordinary integer matrix.  The reference solves all of them.

``INTS`` holds int32 vectors for ``int_arr_to_csd``: INT_MIN, INT_MAX and the values next to each width boundary.
"""

import numpy as np

METHODS = ['mc', 'wmc', 'mc-dc', 'mc-pdc', 'wmc-dc', 'wmc-pdc', 'dummy']
# (decompose_dc, search_all_decompose_dc) of the full solves; every one but -2 runs the distance kernel
SOLVES = [(-2, False), (-1, False), (0, False), (1, False), (-1, True)]
KD_DCS = (-2, -1, 0, 1)

# float32 neighbours of the width boundaries: N = 30 | 31 at 2^30 / 1.5, N = 31 | 32 at 2^31 / 1.5, and 2^31 - 128
EDGE_VALUES = [715827840.0, 715827904.0, 1431655680.0, 1431655808.0, 2147483520.0]


def _f32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64).astype(np.float32))


def _small(rng, n_in, n_out, bits=6):
    """Odd-heavy small integers: every row and column keeps LSB 0 under the centring."""
    W = rng.integers(-(2 ** (bits - 1)), 2 ** (bits - 1), size=(n_in, n_out)).astype(np.float64)
    W[W == 0] = 1.0
    W[:, 0] = 2 * rng.integers(-8, 8, size=n_in) + 1
    W[0, :] = 2 * rng.integers(-8, 8, size=n_out) + 1
    return W


def matrices():
    """name -> float32 matrix, in a fixed order."""
    out = {}
    for v in EDGE_VALUES:
        tag = int(v)
        for s, sn in ((1.0, 'p'), (-1.0, 'n')):
            out[f'edge{tag}{sn}_2x2'] = _f32([[1.0, 3.0], [s * v, 5.0]])
        rng = np.random.default_rng(tag % 1000)
        W = _small(rng, 5, 4)
        W[2, 1] = v
        W[4, 3] = -v
        out[f'edge{tag}_both_5x4'] = _f32(W)
    rng = np.random.default_rng(31)
    W = _small(rng, 3, 3)
    W[0, 1], W[1, 2], W[2, 0] = 1431655680.0, -1073741824.0 - 64.0, 1000000000.0
    out['wide31_3x3'] = _f32(W)
    W = _small(rng, 6, 7)
    for i, j, v in ((1, 1, 1073741824.0), (2, 3, -1073741824.0), (3, 5, 2147483520.0), (5, 2, -1431655808.0), (4, 6, 715827904.0)):
        W[i, j] = v
    out['wide32_mixed_6x7'] = _f32(W)
    out['over_2p31_33'] = _f32([[1.0, 1.0], [2.0**31, 1.0], [3.0, 2.0**33]])
    out['over_neg2p31_3x2'] = _f32([[1.0, 1.0], [-(2.0**31), 1.0], [3.0, 5.0]])
    W = _small(np.random.default_rng(40), 5, 6)
    W[1, 2], W[3, 4], W[4, 0] = 2.0**40, -(2.0**33), 2.0**31
    out['over_mixed_5x6'] = _f32(W)
    out['normal_8x6'] = _f32(np.random.default_rng(0).standard_normal((8, 6)))
    for seed in range(6):
        rng = np.random.default_rng(100 + seed)
        n_in, n_out = int(rng.integers(2, 13)), int(rng.integers(2, 13))
        k = int(rng.integers(-12, 13))
        out[f'normal_s{seed}_{n_in}x{n_out}_k{k}'] = _f32(rng.standard_normal((n_in, n_out)) * 2.0**k)
    rng = np.random.default_rng(200)
    out['normal_span_7x5'] = _f32(rng.standard_normal((7, 5)) * 2.0 ** rng.integers(-4, 5, size=(7, 5)))
    out['normal_16x16'] = _f32(np.random.default_rng(201).standard_normal((16, 16)))
    for name, bad, pos in (('pinf', np.inf, (1, 2)), ('ninf', -np.inf, (0, 0)), ('nan', np.nan, (2, 3))):
        W = np.random.default_rng(300).integers(-64, 64, size=(5, 4)).astype(np.float64)
        W[pos] = bad
        out[f'nonfinite_{name}_5x4'] = _f32(W)
    return out


INT_MIN, INT_MAX = -(2**31), 2**31 - 1


def ints():
    """name -> int32 vector for int_arr_to_csd."""
    small = [0, 1, -1, 3, -5, 7, 100, -77]
    out = {
        'int_min': [INT_MIN, 1, -3, 5],
        'int_max': [INT_MAX, 1, -3, 5],
        'int_min_max': [INT_MIN, INT_MAX, 0, -1],
        'int_min_only': [INT_MIN, INT_MIN],
        'below2p31': [2**31 - 128, -(2**31 - 128), 1, 2],
        # the width is taken from float(max|x|): 1 431 655 765 and 715 827 882 round up across their boundaries
        'x1431655766': [1431655766, -1431655766, 3, -9],
        'x1431655765': [1431655765, -1431655765, 3, -9],
        'n31': [1431655680, -1431655680, 3, -9],
        'x715827883': [715827883, -715827883, 1, 6],
        'x715827882': [715827882, -715827882, 1, 6],
        'n30': [715827840, -715827840, 1, 6],
        'pow30': [2**30, -(2**30), 1, -1],
        'mixed': [2**30 + 1, -(2**31 - 1), 1500000000, 800000000, *small],
    }
    rng = np.random.default_rng(500)
    out['random32'] = [*rng.integers(INT_MIN, INT_MAX, size=12, endpoint=True).tolist(), *small]
    out['random31'] = [*rng.integers(-(2**30), 2**30, size=12).tolist(), *small]
    return {k: np.asarray(v, dtype=np.int32) for k, v in out.items()}

"""Table functions of the lookup-activation tests (module-level, so fronts that use them pickle) and a numeric
fixed-point quantizer that stands in for the ``quantizers`` package the tracer's ``_quantize`` calls.  TEST
INFRASTRUCTURE."""
import numpy as np


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def odd_cube(x):
    """An odd function that is not monotone on [-2, 2]: x**3 / 4 - x."""
    return x**3 / 4 - x


def get_fixed_quantizer_np(round_mode='TRN', overflow_mode='WRAP'):
    """``quantizers.fixed_point.fixed_point_ops_np.get_fixed_quantizer_np``: TRN / RND rounding to 2**-f, then WRAP
    (modulo 2**(k + i) into [-k * 2**i, 2**i)), SAT (clip to [-k * 2**i, 2**i - 2**-f]) or SAT_SYM (clip to
    [-k * (2**i - 2**-f), 2**i - 2**-f])."""

    def q(x, k, i, f):
        k, i, f = int(k), int(i), int(f)
        st = 2.0**-f
        y = np.floor(np.asarray(x, np.float64) / st + (0.5 if round_mode.upper() == 'RND' else 0.0)) * st
        hi = 2.0**i - st
        if overflow_mode.upper() == 'WRAP':
            return np.mod(y + k * 2.0**i, 2.0 ** (i + k)) - k * 2.0**i
        return np.clip(y, -k * (2.0**i if overflow_mode.upper() == 'SAT' else hi), hi)

    return q

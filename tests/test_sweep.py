"""solve_sweep without a device: argument checks on the host, the no-CPU-fallback error, and the front rule."""
import numpy as np
import pytest

W = np.arange(16, dtype=np.float32).reshape(4, 4)


def test_unknown_method_rejected_on_the_host():
    import da4ml_b200._binary as B

    for bad in (dict(method0='nope'), dict(method1='wmc-x'), dict(method0='dummy', method1='')):
        with pytest.raises(RuntimeError, match='Unknown method: '):
            B.solve_sweep(W, [dict(), bad])


def test_argument_checks():
    import da4ml_b200._binary as B

    with pytest.raises(ValueError, match='n_sets must be positive'):
        B.solve_sweep(W, [])
    with pytest.raises(ValueError, match='expected 4 qintervals'):
        B.solve_sweep(W, [dict()], qintervals=[(-1.0, 1.0, 1.0)] * 3)
    with pytest.raises(ValueError, match='expected 4 latencies'):
        B.solve_sweep(W, [dict()], latencies=[0.0] * 5)
    with pytest.raises(TypeError):
        B.solve_sweep(W.astype(np.float64), [dict()])
    for bad in (dict(adder_size=1), dict(offload_fn=None), dict(hard_dc=1, search_all=True)):
        with pytest.raises(TypeError, match='unsupported keys'):
            B.solve_sweep(W, [dict(), bad])


def test_no_cpu_fallback():
    import da4ml_b200._binary as B
    from da4ml_b200.cmvm import solve_sweep

    if B.device_info()['cuda_devices'] > 0:
        pytest.skip('a GPU is present')
    with pytest.raises(RuntimeError, match='no CUDA device'):
        solve_sweep(W, [dict(), dict(hard_dc=2, method0='mc')])


def front(cost, lat):
    import da4ml_b200._binary as B

    return B.sweep_front(np.asarray(cost, np.float32), np.asarray(lat, np.float32)).tolist()


def test_front_rule():
    assert front([], []) == []
    assert front([5.0], [3.0]) == [0]  # a single point
    assert front([2.0, 2.0, 2.0], [1.0, 1.0, 1.0]) == [0]  # all tied: the first
    assert front([4.0, 3.0, 3.0, 5.0], [2.0, 2.0, 2.0, 1.0]) == [1, 3]  # exact duplicates: the first of them
    assert front([4.0, 5.0, 3.0], [4.0, 5.0, 6.0]) == [0, 2]  # (5, 5) is strictly dominated by (4, 4)
    assert front([7.0, 7.0, 7.0], [3.0, 2.0, 4.0]) == [1]  # equal cost, lower latency dominates
    assert front([9.0, 8.0, 7.0], [1.0, 1.0, 1.0]) == [2]  # equal latency, lower cost dominates
    assert front([1.0, 2.0, 3.0], [3.0, 2.0, 1.0]) == [0, 1, 2]  # a trade-off curve
    with pytest.raises(ValueError):
        front([1.0, 2.0], [1.0])


def test_front_matches_the_definition_on_random_points():
    rng = np.random.default_rng(3)
    for n in (1, 2, 7, 40, 200):
        c = rng.integers(0, 6, n).astype(np.float32)
        l = rng.integers(0, 6, n).astype(np.float32)
        want = []
        for i in range(n):
            dom = any(c[j] <= c[i] and l[j] <= l[i] and (c[j] < c[i] or l[j] < l[i] or j < i) for j in range(n) if j != i)
            if not dom:
                want.append(i)
        assert front(c, l) == want

"""The DAIS interpreter on the GPU (da4ml_b200.dais): ``run_interp`` and ``DaisProgram`` equal the reference
interpreter's stored answers bit for bit on traced models, hand-written shift cases and seeded random programs, lookup
errors included; several chunks and 10^6 samples; CUDA tensors on non-default streams, also back to back without
synchronisation; and the adder-graph programs of the CMVM path."""
import dais_programs as G
import numpy as np
import pytest
from test_dais_interp import check_answer, named_programs
from test_dais_replay import cuda_replay_inputs, reference_run, run_key


@pytest.fixture(scope='module')
def stored():
    from test_oracle_cross import load_stored

    return load_stored('dais_programs.json.gz')


def _program_call(prog, x):
    from da4ml_b200.dais import DaisProgram

    with DaisProgram(prog) as p:
        return p(x)


@pytest.mark.gpu
def test_named_programs_equal_the_reference(cuda_binary, stored):
    from da4ml_b200.dais import run_interp

    for name, prog in named_programs(stored).items():
        for tag, x in G.stored_inputs(name, prog):
            for fn in (run_interp, _program_call):
                check_answer(stored[run_key(prog, x)], fn, prog, x, f'{name}/{tag}/{fn.__name__}')


@pytest.mark.gpu
def test_random_programs_equal_the_reference(cuda_binary, stored):
    from da4ml_b200.dais import run_interp

    for seed in G.RANDOM_SEEDS:
        prog, x = G.random_case(seed)
        for fn in (run_interp, _program_call):
            check_answer(stored[run_key(prog, x)], fn, prog, x, f'{seed}/{fn.__name__}')


@pytest.mark.gpu
def test_several_chunks_and_a_million_samples(cuda_binary, stored):
    from da4ml_b200.dais import DaisProgram, run_interp

    prog, x = G.random_program(**G.MULTI_CHUNK), G.multi_chunk_inputs()
    assert x.shape[0] > 2 * ((1 << 27) // G.MULTI_CHUNK['n_ops'])  # at least three chunks of samples
    assert not stored[run_key(prog, x)].startswith('error:')
    check_answer(stored[run_key(prog, x)], run_interp, prog, x, 'multi_chunk')
    prog = named_programs(stored)['traced_mlp']
    x = G.random_inputs(11, G.MILLION, int(prog[2]))
    with DaisProgram(prog) as p:
        check_answer(stored[run_key(prog, x)], lambda _, d: p(d), prog, x, 'million')


@pytest.mark.gpu
def test_lookup_out_of_bounds_names_the_first_failing_sample(cuda_binary, stored):
    from da4ml_b200.dais import DaisProgram, run_interp

    prog = named_programs(stored)['lookup_oob']
    (_, bad), (_, ok) = G.stored_inputs('lookup_oob', prog)
    want = stored[run_key(prog, bad)]
    assert want.startswith('error:Logic lookup index out of bounds')
    with DaisProgram(prog) as p:
        for _ in range(2):  # the program and the library stay usable after the error
            with pytest.raises(RuntimeError) as e:
                p(bad)
            assert str(e.value) == want[len('error:') :]
            assert np.array_equal(p(ok).view(np.uint64), stored[run_key(prog, ok)])
    with pytest.raises(RuntimeError, match='Logic lookup index out of bounds'):
        run_interp(prog, bad)
    # a program run in chunks of 2048 samples whose first failing lookup is at sample 4100, in the third chunk
    import torch

    prog, x = G.lookup_oob_program(0, pad=G.OOB_PAD), G.late_lookup_failure_inputs()
    assert G.OOB_FIRST_FAILING >= 2 * ((1 << 27) // int(prog[4]))
    want = stored[run_key(prog, x)]
    with DaisProgram(prog) as p:
        for data in (x, torch.from_numpy(x).cuda()):
            with pytest.raises(RuntimeError) as e:
                p(data)
            assert str(e.value) == want[len('error:') :]
        assert p(x[: G.OOB_FIRST_FAILING]).shape == (G.OOB_FIRST_FAILING, 3)
    good = named_programs(stored)['traced_lookup']
    (_, x), = G.stored_inputs('traced_lookup', good)
    check_answer(stored[run_key(good, x)], run_interp, good, x, 'after the error')


@pytest.mark.gpu
def test_cuda_tensor_on_a_side_stream_equals_the_numpy_path(cuda_binary, stored):
    import torch

    from da4ml_b200.dais import DaisProgram

    for name in ('traced_mlp', 'traced_msb_mux', 'traced_product'):
        prog = named_programs(stored)[name]
        (_, x), = G.stored_inputs(name, prog)
        with DaisProgram(prog) as p:
            want = p(x)
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                xt = torch.from_numpy(x).to('cuda', non_blocking=False)
                yt = p(xt)
                assert yt.is_cuda and yt.dtype == torch.float64 and tuple(yt.shape) == want.shape
            s.synchronize()
            assert np.array_equal(yt.cpu().numpy().view(np.uint64), want.view(np.uint64)), name


@pytest.mark.gpu
def test_back_to_back_runs_on_several_streams(cuda_binary, stored):
    """Runs on different streams share the library's scratch buffer and return before their kernels finish: queued back
    to back with no synchronisation in between (two side streams, the library's stream, two threads), every result
    still equals the reference's."""
    import threading

    import torch

    from da4ml_b200.dais import DaisProgram

    reps = 2000  # ~5*10^5 samples per run: the kernels of one run are still in flight when the next is queued
    cases = {}
    for name in ('traced_dense_relu', 'traced_msb_mux', 'traced_product', 'traced_bits'):
        prog = named_programs(stored)[name]
        (_, x), = G.stored_inputs(name, prog)
        cases[name] = (DaisProgram(prog), np.tile(x, (reps, 1)), np.tile(stored[run_key(prog, x)], (reps, 1)))
    try:
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        xs = {k: torch.from_numpy(x).cuda() for k, (_, x, _) in cases.items()}
        torch.cuda.synchronize()
        got = {}
        for k, s in zip(('traced_dense_relu', 'traced_msb_mux'), streams):
            with torch.cuda.stream(s):
                got[k] = cases[k][0](xs[k])
        got['traced_product'] = cases['traced_product'][0](cases['traced_product'][1])  # host arrays, the library's stream
        for k, s in zip(('traced_dense_relu', 'traced_msb_mux'), streams):
            s.synchronize()
            assert np.array_equal(got[k].cpu().numpy().view(np.uint64), cases[k][2]), k
        assert np.array_equal(got['traced_product'].view(np.uint64), cases['traced_product'][2])

        results, errors = {}, []

        def worker(k, s):
            try:
                with torch.cuda.stream(s):
                    y = cases[k][0](xs[k])
                s.synchronize()
                results[k] = y.cpu().numpy()
            except Exception as e:  # (reported below)
                errors.append(e)

        threads = [threading.Thread(target=worker, args=(k, s)) for k, s in zip(('traced_bits', 'traced_msb_mux'), streams)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
        for k, y in results.items():
            assert np.array_equal(y.view(np.uint64), cases[k][2]), k
    finally:
        for p, _, _ in cases.values():
            p.close()


@pytest.mark.gpu
def test_run_interp_equals_the_reference_on_adder_graphs(cuda_binary):
    """The CMVM path's golden adder graphs, including inputs that wrap, against the reference interpreter's stored
    outputs (tests/golden/dais_reference.json.gz)."""
    from test_oracle_cross import load_stored

    from da4ml_b200.dais import run_interp

    want = load_stored('dais_reference.json.gz')
    for tag, sol, x in cuda_replay_inputs():
        prog = sol.to_binary()
        assert np.array_equal(run_interp(prog, x).view(np.uint64), reference_run(want, prog, x).view(np.uint64)), tag

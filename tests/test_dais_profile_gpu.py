"""Profiling DAIS programs on the GPU (``DaisProgram.dump`` / ``profile``): the reference interpreter's value of every op
(tests/golden/dais_op_values.json.gz) through numpy inputs and CUDA tensors on a side stream; several chunks of samples;
10^6 samples against merged slices; lookup errors; runs, dumps and profiles queued back to back on several streams; and
the declared types of a CMVM adder graph."""
import dais_programs as G
import numpy as np
import pytest
from test_dais_interp import named_programs
from test_dais_profile import case_program, check_against_stored, harness_dump, harness_profile, harness_stats, load_op_values
from test_dais_replay import run_key


@pytest.fixture(scope='module')
def stored():
    from test_oracle_cross import load_stored

    return load_stored('dais_programs.json.gz')


def _same_profile(a, b, tag=''):
    assert a.n_samples == b.n_samples, tag
    for k in ('min', 'max', 'bits_or'):
        assert np.array_equal(getattr(a, k), getattr(b, k)), (tag, k)


@pytest.mark.gpu
def test_dump_and_profile_equal_the_reference_values(cuda_binary):
    import torch

    from da4ml_b200.dais import DaisProgram

    s = torch.cuda.Stream()
    for case, want in load_op_values().items():
        prog, x = case_program(case)
        with DaisProgram(prog) as p:
            if 'error' in want:
                for fn in (p.dump, p.profile):
                    for data in (x, torch.from_numpy(x).cuda()):
                        with pytest.raises(RuntimeError) as e:
                            fn(data)
                        assert str(e.value) == want['error'], case
                continue
            codes, prof = p.dump(x), p.profile(x)
            stats = np.stack([prof.min, prof.max, prof.bits_or], 1)
            check_against_stored(want, codes, stats, prog, case)
            assert prof.n_samples == len(x) and np.array_equal(stats, harness_stats(prog, x)), case
            with torch.cuda.stream(s):
                xt = torch.from_numpy(x).to('cuda')
                ct = p.dump(xt)
                assert ct.is_cuda and ct.dtype == torch.int64 and tuple(ct.shape) == codes.shape
                pt = p.profile(xt)
            s.synchronize()
            assert np.array_equal(ct.cpu().numpy(), codes), case
            _same_profile(pt, prof, case)
            sel = np.array([p.n_ops - 1, 0, p.n_ops // 2, 0])  # any order, repeats allowed
            assert np.array_equal(p.dump(x, sel), codes[:, sel]), case


@pytest.mark.gpu
def test_several_chunks(cuda_binary):
    """The 65 536-op program runs in chunks of 2048 samples: the profile folds all three, and a dump of a selection
    is stitched across them."""
    import torch

    from da4ml_b200.dais import DaisProgram

    prog, x = G.random_program(**G.MULTI_CHUNK), G.multi_chunk_inputs()
    assert x.shape[0] > 2 * ((1 << 27) // G.MULTI_CHUNK['n_ops'])
    want = harness_profile(prog, x[:1700])
    for a, b in ((1700, 2100), (2100, 4500), (4500, len(x))):
        want = want.merge(harness_profile(prog, x[a:b]))
    rng = np.random.default_rng(5)
    sel = np.concatenate([[0, 65535, 65535, 7], rng.integers(0, 65536, 300)])
    with DaisProgram(prog) as p:
        _same_profile(p.profile(x), want, 'multi_chunk')
        assert np.array_equal(p.dump(x, sel), harness_dump(prog, x, sel))
        assert np.array_equal(p.dump(torch.from_numpy(x).cuda(), sel).cpu().numpy(), harness_dump(prog, x, sel))


@pytest.mark.gpu
def test_a_million_samples(cuda_binary, stored):
    import torch

    from da4ml_b200.dais import DaisProgram

    prog = named_programs(stored)['traced_mlp']
    x = G.random_inputs(11, G.MILLION, int(prog[2]))
    with DaisProgram(prog) as p:
        xt = torch.from_numpy(x).cuda()
        whole = p.profile(xt)
        cut = np.linspace(0, G.MILLION, 9).astype(int)
        merged = p.profile(xt[cut[0] : cut[1]])
        for a, b in zip(cut[1:-1], cut[2:]):
            merged = merged.merge(p.profile(xt[a:b]))
        _same_profile(whole, merged, 'million')
        _same_profile(p.profile(x[:20000]), harness_profile(prog, x[:20000]), 'first 20 000')
        assert whole.n_samples == G.MILLION


@pytest.mark.gpu
def test_lookup_failure_in_a_later_chunk(cuda_binary, stored):
    import torch

    from da4ml_b200.dais import DaisProgram

    prog, x = G.lookup_oob_program(0, pad=G.OOB_PAD), G.late_lookup_failure_inputs()
    want = stored[run_key(prog, x)]
    assert want.startswith('error:Logic lookup index out of bounds')
    ok = x[: G.OOB_FIRST_FAILING]
    sel = np.array([5, 3, 4, 6, 65542])
    with DaisProgram(prog) as p:
        for fn in (p.profile, p.dump):
            for data in (x, torch.from_numpy(x).cuda()):
                with pytest.raises(RuntimeError) as e:
                    fn(data)
                assert str(e.value) == want[len('error:') :]
                assert np.array_equal(p.dump(ok[-300:], sel), harness_dump(prog, ok[-300:], sel))  # the next call succeeds
        assert p.profile(ok).n_samples == len(ok)
        assert np.array_equal(p.dump(ok, sel), harness_dump(prog, ok, sel))


@pytest.mark.gpu
def test_back_to_back_with_runs_on_several_streams(cuda_binary, stored):
    """Dumps and profiles share the scratch with runs: queued back to back on two streams with no synchronisation in
    between, each result equals what it gives alone."""
    import torch

    from da4ml_b200.dais import DaisProgram

    reps = 2000
    progs, xs, alone = {}, {}, {}
    for name in ('traced_dense_relu', 'traced_msb_mux', 'traced_product'):
        prog = named_programs(stored)[name]
        (_, x), = G.stored_inputs(name, prog)
        progs[name] = DaisProgram(prog)
        xs[name] = torch.from_numpy(np.tile(x, (reps, 1))).cuda()
        xh = xs[name].cpu().numpy()
        alone[name] = (progs[name](xh), progs[name].dump(xh), progs[name].profile(xh))
    try:
        a, b = torch.cuda.Stream(), torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(a):
            y0 = progs['traced_dense_relu'](xs['traced_dense_relu'])
        with torch.cuda.stream(b):
            d1 = progs['traced_msb_mux'].dump(xs['traced_msb_mux'])
        with torch.cuda.stream(a):
            d0 = progs['traced_dense_relu'].dump(xs['traced_dense_relu'])
        with torch.cuda.stream(b):
            y2 = progs['traced_product'](xs['traced_product'])
            p2 = progs['traced_product'].profile(xs['traced_product'])
        with torch.cuda.stream(a):
            p1 = progs['traced_msb_mux'].profile(xs['traced_msb_mux'])
        a.synchronize()
        b.synchronize()
        assert np.array_equal(y0.cpu().numpy().view(np.uint64), alone['traced_dense_relu'][0].view(np.uint64))
        assert np.array_equal(d0.cpu().numpy(), alone['traced_dense_relu'][1])
        assert np.array_equal(d1.cpu().numpy(), alone['traced_msb_mux'][1])
        assert np.array_equal(y2.cpu().numpy().view(np.uint64), alone['traced_product'][0].view(np.uint64))
        _same_profile(p1, alone['traced_msb_mux'][2])
        _same_profile(p2, alone['traced_product'][2])
    finally:
        for p in progs.values():
            p.close()


@pytest.mark.gpu
def test_adder_graph_stays_inside_its_declared_types(cuda_binary):
    """An adder graph of the CMVM solver, fed inputs drawn from its declared input intervals: no op leaves its declared
    type, and the observed types are no wider than the declared ones."""
    import da4ml_b200._binary as B
    from da4ml_b200.dais import DaisProgram

    rng = np.random.default_rng(3)
    W = rng.integers(-128, 128, size=(24, 20)).astype(np.float32)
    raw = B.solve_raw(W)
    prog = raw.to_binary()[0]
    st = raw.stages[0]
    ops_i, ops_f = np.asarray(st['ops_i']).reshape(-1, 4), np.asarray(st['ops_f'], np.float64).reshape(-1, 5)
    q = np.zeros((W.shape[0], 3))
    q[ops_i[ops_i[:, 2] == -1, 0]] = ops_f[ops_i[:, 2] == -1, :3]  # (min, max, step) of each input's op
    n = 20000
    steps = np.round((q[:, 1] - q[:, 0]) / q[:, 2]).astype(np.int64)
    x = q[:, 0] + q[:, 2] * rng.integers(0, steps + 1, size=(n, len(q)))
    x[0], x[1] = q[:, 0], q[:, 1]  # both ends of every interval
    x = x * np.ldexp(1.0, -np.asarray(st['inp_shifts'], np.int64))[None, :]  # the op reads x * 2^inp_shift
    with DaisProgram(prog) as p:
        prof = p.profile(x)
        assert not prof.overflow.any()
        live = prof.bits_or != 0
        assert live.sum() > p.n_ops // 2
        assert (prof.observed_kif[live] <= prof.kif[live]).all()
        assert np.array_equal(prof.observed_kif[~live], np.zeros((int((~live).sum()), 3)))

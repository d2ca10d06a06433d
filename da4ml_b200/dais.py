"""The DAIS interpreter on the GPU: drop-in for the reference's native ``dais_bin.run_interp``
(reference dais/bindings.cc:102-131 -> DAISInterpreter.cc), for every DAIS program -- all opcodes and lookup tables.

``run_interp(bin_logic, data)`` runs a program once.  ``DaisProgram(words)`` parses and validates a program once and
runs it on many batches, from numpy arrays or float64 CUDA tensors (no host copy).  Results are bit-for-bit those of
the reference interpreter; errors raise ``RuntimeError`` with its messages.  ``DaisProgram.dump`` returns the
intermediate values (int64 codes) of chosen ops, and ``DaisProgram.profile`` per-op ranges of all codes as an
``OpProfile`` (observed types, overflow of the declared types, merging of batches).
"""

from __future__ import annotations

import ctypes as C

import numpy as np

from . import _binary as B

_L = B._L


def _words(bin_logic) -> np.ndarray:
    return np.ascontiguousarray(np.ravel(bin_logic), dtype=np.int32)


class DaisProgram:
    """A DAIS program (int32 words of ``CombLogic.to_binary``) loaded into the library once: parsed and checked on the
    host at construction, uploaded to a device on first use there, released by ``close()`` (or on leaving a ``with``
    block, or when garbage-collected)."""

    def __init__(self, words):
        w = _words(words)
        h = B._vp()
        B._check(_L.da4ml_dais_program_load(w.ctypes.data_as(B._i32p), w.size, C.byref(h)))
        self._h = h
        info = np.zeros(6, np.int64)
        B._check(_L.da4ml_dais_program_info(h, B._ip(info)))
        self.n_in, self.n_out, self.n_ops, self.n_tables, self.n_levels, self.max_width = (int(v) for v in info)
        o = 6 + self.n_in + 3 * self.n_out
        # declared (k, i, f) = (is_signed, integers, fractionals) of every op: words 5..7 of its 8
        self.kif = w[o : o + 8 * self.n_ops].reshape(self.n_ops, 8)[:, 5:8].astype(np.int64)
        self.kif.flags.writeable = False

    def close(self):
        h, self._h = getattr(self, '_h', None), None
        if h:
            _L.da4ml_dais_program_free(h)

    def __del__(self):
        self.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _handle(self):
        if not self._h:
            raise RuntimeError('DaisProgram is closed')
        return self._h

    def __call__(self, x):
        """Outputs ``[n_samples, n_out]`` float64 for inputs ``[n_samples, n_in]`` (any shape; n_samples = size // n_in
        as in the reference).  A numpy input gives a numpy result.  A float64 CUDA ``torch.Tensor`` gives a CUDA
        tensor, computed in place on the tensor's device and current stream."""
        if type(x).__module__.startswith('torch'):
            return self._run_tensor(x)
        return self._run_host(np.asarray(x, dtype=np.float64))

    def _n_samples(self, size: int) -> int:
        # as the reference: n_samples = size / n_in, a trailing partial row is ignored
        if self.n_in == 0:
            if size:
                raise RuntimeError('a program without inputs cannot take input data')
            return 0
        return size // self.n_in

    def _run_host(self, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x.reshape(-1))
        n = self._n_samples(x.size)
        x = x[: n * self.n_in]
        out = np.zeros((n, self.n_out), np.float64)
        B._check(_L.da4ml_dais_program_run(self._handle(), x.ctypes.data, n, out.ctypes.data, 0))
        return out

    def _run_tensor(self, x):
        import torch

        if not x.is_cuda or x.dtype != torch.float64:
            raise TypeError('a tensor input must be a float64 CUDA tensor')
        x = x.contiguous().view(-1)
        n = self._n_samples(x.numel())
        out = torch.empty((n, self.n_out), dtype=torch.float64, device=x.device)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        with torch.cuda.device(x.device):  # (the stream travels with the call: the library's own stream is left alone)
            B._check(_L.da4ml_dais_program_run_stream(self._handle(), x.data_ptr(), n, out.data_ptr(), 1, B._vp(stream)))
        return out

    # ---- profiling: the op codes (int64 values in the interpreter; real value = code * 2^-f, f = kif[:, 2]) ----------
    def _tensor_input(self, x):
        import torch

        if not x.is_cuda or x.dtype != torch.float64:
            raise TypeError('a tensor input must be a float64 CUDA tensor')
        x = x.contiguous().view(-1)
        return x, self._n_samples(x.numel()), torch.cuda.current_stream(x.device).cuda_stream

    def dump(self, x, ops=None):
        """Codes ``[n_samples, len(ops)]`` int64 of the ops ``ops`` (default: all, in program order; repeats allowed)
        for inputs ``x``, as the interpreter computes them (an input op holds its quantised, wrapped code).  A numpy
        input gives numpy.  A float64 CUDA tensor gives an int64 CUDA tensor, computed on the tensor's current stream;
        the call returns without waiting unless the program has lookups."""
        sel = np.arange(self.n_ops, dtype=np.int64) if ops is None else np.asarray(ops, dtype=np.int64).reshape(-1)
        bad = np.flatnonzero((sel < 0) | (sel >= self.n_ops))
        if bad.size:
            k = int(bad[0])
            raise ValueError(f'dump: op id {int(sel[k])} at position {k} is out of range [0, {self.n_ops})')
        sel = np.ascontiguousarray(sel, dtype=np.int32)
        if type(x).__module__.startswith('torch'):
            import torch

            x, n, stream = self._tensor_input(x)
            out = torch.empty((n, sel.size), dtype=torch.int64, device=x.device)
            with torch.cuda.device(x.device):
                B._check(_L.da4ml_dais_program_dump(self._handle(), x.data_ptr(), n, sel.ctypes.data, sel.size, out.data_ptr(), 1, B._vp(stream)))
            return out
        x = np.ascontiguousarray(np.asarray(x, dtype=np.float64).reshape(-1))
        n = self._n_samples(x.size)
        out = np.zeros((n, sel.size), np.int64)
        B._check(_L.da4ml_dais_program_dump(self._handle(), x.ctypes.data, n, sel.ctypes.data, sel.size, out.ctypes.data, 0, None))
        return out

    def profile(self, x) -> OpProfile:
        """Per-op ``min``, ``max`` and bitwise OR of the codes over all samples of ``x`` (numpy, or a float64 CUDA tensor
        read on its current stream).  Always synchronises."""
        stats = np.zeros((self.n_ops, 3), np.int64)
        if type(x).__module__.startswith('torch'):
            import torch

            x, n, stream = self._tensor_input(x)
            with torch.cuda.device(x.device):
                B._check(_L.da4ml_dais_program_profile(self._handle(), x.data_ptr(), n, 1, B._vp(stream), stats.ctypes.data))
        else:
            x = np.ascontiguousarray(np.asarray(x, dtype=np.float64).reshape(-1))
            n = self._n_samples(x.size)
            B._check(_L.da4ml_dais_program_profile(self._handle(), x.ctypes.data, n, 0, None, stats.ctypes.data))
        return OpProfile(n, stats[:, 0], stats[:, 1], stats[:, 2], self.kif)


class OpProfile:
    """Statistics of every op's codes over ``n_samples`` samples: ``min``, ``max`` (signed) and ``bits_or`` (bitwise OR),
    int64 ``[n_ops]``, with the declared ``kif`` ``[n_ops, 3]``.  Zero samples give ``INT64_MAX``, ``INT64_MIN``, 0."""

    def __init__(self, n_samples: int, min, max, bits_or, kif):
        self.n_samples = int(n_samples)
        self.min = np.asarray(min, dtype=np.int64)
        self.max = np.asarray(max, dtype=np.int64)
        self.bits_or = np.asarray(bits_or, dtype=np.int64)
        self.kif = np.asarray(kif, dtype=np.int64).reshape(-1, 3)

    @property
    def observed_kif(self) -> np.ndarray:
        """``[n_ops, 3]`` (k, i, f) of the smallest type holding every observed code: with ``t`` the trailing zeros of
        ``bits_or``, ``f - t`` fractional bits, signed if ``min < 0``, and the integer bits that hold
        ``[min >> t, max >> t]``; (0, 0, 0) for an op that is always 0.  Equals ``types.minimal_kif_array`` of
        ``(min * 2^-f, max * 2^-f, 2^(t - f))``, computed exactly."""
        out = np.zeros((len(self.min), 3), np.int64)
        for j, (mn, mx, bo, f) in enumerate(zip(self.min.tolist(), self.max.tolist(), self.bits_or.tolist(), self.kif[:, 2].tolist())):
            if bo == 0:
                continue
            t = (bo & -bo).bit_length() - 1  # trailing zeros (Python's & is two's complement for negative ints too)
            bits = (mx >> t).bit_length() if mx >= 0 else 0
            if mn < 0:
                bits = max(bits, (-(mn >> t) - 1).bit_length())
            out[j] = (int(mn < 0), bits - (f - t), f - t)
        return out

    @property
    def overflow(self) -> np.ndarray:
        """``[n_ops]`` bool: an observed code lies outside the declared type's code range (``[-2^(w-1), 2^(w-1) - 1]``
        signed, ``[0, 2^w - 1]`` unsigned, ``{0}`` for ``w = k + i + f <= 0``)."""
        out = np.zeros(len(self.min), bool)
        for j, (mn, mx, (k, i, f)) in enumerate(zip(self.min.tolist(), self.max.tolist(), self.kif.tolist())):
            if mn > mx:  # no samples
                continue
            k = int(k != 0)
            w = min(k + i + f, 65)  # (from 64 bits on, every int64 of the right sign fits)
            lo, hi = (0, 0) if w <= 0 else (-(1 << (w - 1)), (1 << (w - 1)) - 1) if k else (0, (1 << w) - 1)
            out[j] = mn < lo or mx > hi
        return out

    def merge(self, other: OpProfile) -> OpProfile:
        """The profile of both sample sets together."""
        if self.kif.shape != other.kif.shape or not np.array_equal(self.kif, other.kif):
            raise ValueError('merge: the profiles are of different programs')
        return OpProfile(self.n_samples + other.n_samples, np.minimum(self.min, other.min), np.maximum(self.max, other.max), self.bits_or | other.bits_or, self.kif)


def run_interp(bin_logic, data, n_threads: int = 1) -> np.ndarray:
    """``dais_bin.run_interp`` (reference dais/bindings.cc:102-131): run a DAIS program on ``data`` (float64, read as
    rows of n_in) and return float64 ``[n_samples, n_out]``.  Runs on the current CUDA device; ``n_threads`` is
    accepted for signature compatibility and ignored."""
    w = _words(bin_logic)
    if w.size < 4:
        raise RuntimeError('Invalid binary logic data')
    if w[0] != 1:
        raise RuntimeError(f'DAIS version mismatch: expected version 1, got version {int(w[0])}')
    x = np.asarray(data, dtype=np.float64)
    if x.size == 0 or (w.size > 2 and w[2] > 0 and x.size < w[2]):  # no samples: the reference loads nothing
        return np.zeros((0, max(int(w[3]), 0)), np.float64)
    with DaisProgram(w) as prog:
        return prog(x)


__all__ = ['DaisProgram', 'OpProfile', 'run_interp']

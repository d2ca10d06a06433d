"""The DAIS interpreter on the GPU: drop-in for the reference's native ``dais_bin.run_interp``
(reference dais/bindings.cc:102-131 -> DAISInterpreter.cc), for every DAIS program -- all opcodes and lookup tables.

``run_interp(bin_logic, data)`` runs a program once.  ``DaisProgram(words)`` parses and validates a program once and
runs it on many batches, from numpy arrays or float64 CUDA tensors (no host copy).  Results are bit-for-bit those of
the reference interpreter; errors raise ``RuntimeError`` with its messages.
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


__all__ = ['DaisProgram', 'run_interp']

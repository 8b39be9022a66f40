"""Host tables of the Bluestein transforms of csrc/bluestein.cuh, shared by the RSS loss (loss.py: all n bins of an
n-point DFT) and the key-shifted mel (mel.py: the first K bins of an n'-point DFT).

Layout (floats): [0, 4) caller-defined scalars; the window (n floats) at 4; the chirp exp(+i pi (m^2 mod 2n) / n)
(n complex) at chirp_off(n); FFT_M(h) / M (M complex) at hspec_off(n), h the chirp on [0, n_out) and mirrored on
(M - n, M).  Chirp and filter spectrum are computed in float64 from the integer m^2 mod 2n and rounded once.
"""
import threading

import numpy as np
import torch

WIN_OFF = 4


def size(n, n_out):
    """the transform size for bins [0, n_out) of an n-point DFT: the smallest of 1024 / 2048 / 4096 that is
    >= n + n_out - 1 (the cyclic convolution then does not wrap onto those bins)"""
    need = int(n) + int(n_out) - 1
    for M in (1024, 2048, 4096):
        if M >= need:
            return M
    raise ValueError("no Bluestein size for n=%d with %d bins (n + bins - 1 > 4096)" % (n, n_out))


def chirp_off(n):
    return WIN_OFF + ((int(n) + 3) & ~3)


def hspec_off(n):
    return chirp_off(n) + 2 * int(n)


def table_floats(n, n_out):
    return hspec_off(n) + 2 * size(n, n_out)


def table_host(n, n_out, window, head=()):
    """float32 table for bins [0, n_out) of an n-point DFT: ``head`` (at most 4 floats) at 0, ``window`` (n values,
    stored as given) at WIN_OFF, the chirp and FFT_M(h) / M"""
    n, n_out = int(n), int(n_out)
    M = size(n, n_out)
    m = np.arange(n, dtype=np.int64)
    chirp = np.exp(1j * np.pi * ((m * m) % (2 * n)).astype(np.float64) / n)
    h = np.zeros(M, np.complex128)
    h[:n_out] = chirp[:n_out]
    h[M - n + 1:] = chirp[1:][::-1]
    hspec = np.fft.fft(h) / M
    t = np.zeros(table_floats(n, n_out), np.float32)
    t[:len(head)] = head
    t[WIN_OFF:WIN_OFF + n] = np.asarray(window, np.float32)
    t[chirp_off(n):chirp_off(n) + 2 * n] = chirp.astype(np.complex64).view(np.float32)
    t[hspec_off(n):hspec_off(n) + 2 * M] = hspec.astype(np.complex64).view(np.float32)
    return t


class TableCache:
    """build(n) -> float32 numpy table, uploaded once per (n, device) and kept; ``tables`` maps (n, device index) to the
    device tensor"""

    def __init__(self, build):
        self.build = build
        self.tables = {}
        self._lock = threading.Lock()

    def get(self, n, device):
        key = (int(n), torch.device(device).index)
        with self._lock:
            t = self.tables.get(key)
            if t is None:
                t = torch.from_numpy(self.build(n)).to(device)
                # built once per device and then read from whatever stream the caller is on: make it visible to all of them
                torch.cuda.current_stream().synchronize()
                self.tables[key] = t
        return t

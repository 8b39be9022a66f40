"""Generate tests/golden/rss_*.npz: the reference's OWN ddsp/loss.py RSSLoss under autograd, on CPU:

    DDSP_REFERENCE_ROOT=<DDSP-SVC checkout> python tests/golden/make_golden_rss_loss.py [case names; default: all]

For each case ``RSSLoss(256, 2048, n_scale)(x_pred, x_true).backward()`` with x_pred requiring grad; the .npz stores
x_pred, x_true, the scales, the loss, dL/dx_pred and input checksums.  Seeded cases draw their scales with the
reference's own torch.randint after torch.manual_seed(seed); pinned cases replace that draw by the listed sizes.

Cases: a seeded 4-scale draw on B=2 x 24 hops of audio-like signals; every transform size and both parities
(256 .. 2047, primes 1031 and 2039); a ragged length (not a multiple of n or of 4); one row with x_pred == x_true;
silent stretches in both signals (S = eps, |X| = 0); and a float16 x_true (the reference is fed its exact upcast).
The tests import ``CASES`` / ``build_inputs`` from this module and only read the stored files.
"""
import os
import sys
from collections import OrderedDict
from unittest import mock

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HERE = os.path.dirname(os.path.abspath(__file__))
FFT_MIN, FFT_MAX = 256, 2048

# name: (seed, B, T, scales: int n_scale (seeded draw) or a tuple of pinned sizes, kind)
CASES = OrderedDict([
    ("rss_seeded_b2_h24", (1, 2, 24 * 512, 4, "audio")),
    ("rss_pinned_all_sizes", (2, 2, 3 * 2047 + 9, (256, 300, 512, 513, 1024, 1025, 1031, 2039, 2047), "audio")),
    ("rss_ragged_t", (3, 3, 5003, (1031, 2047, 256, 513), "audio")),
    ("rss_equal_row", (4, 3, 6001, (300, 1025, 2039, 512), "equal_row")),
    ("rss_silence", (5, 2, 9000, (256, 513, 1024, 2047), "silence")),
    ("rss_fp16_true", (6, 2, 24 * 512, 4, "fp16")),
])


def path(name):
    return os.path.join(HERE, name + ".npz")


def audio_like(g, B, T, sr=44100):
    """harmonic tones with a slow f0 sweep, an envelope and a little noise: [B, T] float32"""
    t = torch.arange(T, dtype=torch.float64) / sr
    rows = []
    for _ in range(B):
        f0 = 110 + 300 * torch.rand((), generator=g, dtype=torch.float64)
        sweep = f0 * (1 + 0.1 * torch.sin(2 * np.pi * 1.5 * t))
        phase = 2 * np.pi * torch.cumsum(sweep, 0) / sr
        y = sum(torch.sin(k * phase) / k for k in range(1, 9))
        env = 0.5 + 0.5 * torch.sin(2 * np.pi * 3 * t + 6 * torch.rand((), generator=g, dtype=torch.float64))
        rows.append(0.2 * env * y + 0.01 * torch.randn(T, generator=g, dtype=torch.float64))
    return torch.stack(rows).float()


def build_inputs(name):
    """-> x_pred [B, T] float32, x_true [B, T] (float16 for the fp16 case), scales (n_scale or pinned tuple)"""
    seed, B, T, scales, kind = CASES[name]
    g = torch.Generator().manual_seed(seed)
    x_true = audio_like(g, B, T)
    x_pred = (0.8 * x_true + 0.05 * audio_like(g, B, T) + 0.005 * torch.randn(B, T, generator=g)).float()
    if kind == "equal_row":
        x_pred[1] = x_true[1]
    if kind == "silence":
        for a, b in ((0, 2100), (4000, 6500)):
            x_true[:, a:b] = 0.0
            x_pred[:, a:b] = 0.0
    if kind == "fp16":
        x_true = x_true.half()
    return x_pred, x_true, scales


def draw(name):
    """the scales of case ``name`` as the reference draws (or pins) them"""
    seed, _, _, scales, _ = CASES[name]
    if isinstance(scales, tuple):
        return torch.tensor(scales, dtype=torch.int64)
    torch.manual_seed(seed)
    return torch.randint(FFT_MIN, FFT_MAX, (scales,))


def checksums(x_pred, x_true):
    return {"sum_x_pred": float(x_pred.double().sum()), "abs_x_pred": float(x_pred.double().abs().sum()),
            "sum_x_true": float(x_true.double().sum()), "abs_x_true": float(x_true.double().abs().sum())}


def run_reference(name):
    from oracle import ref_loader
    ref_loader.load()                                          # stubs and sys.path of the reference checkout
    from ddsp.loss import RSSLoss
    x_pred, x_true, scales = build_inputs(name)
    n_ffts = draw(name)
    crit = RSSLoss(FFT_MIN, FFT_MAX, len(n_ffts), device="cpu")
    xp = x_pred.clone().requires_grad_(True)
    seed = CASES[name][0]
    torch.manual_seed(seed)
    if isinstance(scales, tuple):
        with mock.patch.object(torch, "randint", lambda *a, **k: n_ffts.clone()):
            loss = crit(xp, x_true.float())
    else:
        loss = crit(xp, x_true.float())                        # draws torch.randint itself, after manual_seed(seed)
    loss.backward()
    return x_pred, x_true, n_ffts, loss.detach(), xp.grad


def main():
    for name in sys.argv[1:] or CASES:
        x_pred, x_true, n_ffts, loss, grad = run_reference(name)
        np.savez_compressed(path(name), x_pred=x_pred.numpy(), x_true=x_true.numpy(), n_ffts=n_ffts.numpy(),
                            loss=loss.numpy(), grad=grad.numpy(), torch_version=np.array(torch.__version__),
                            **{k: np.float64(v) for k, v in checksums(x_pred, x_true).items()})
        print("%-22s n_ffts %-44s loss %.7f  |grad| max %.3e" % (name, n_ffts.tolist(), loss.item(),
                                                                 grad.abs().max()))


if __name__ == "__main__":
    main()

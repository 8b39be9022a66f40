"""Generate tests/golden/mel_grad_*.npz: the reference's OWN nsf_hifigan/nvSTFT.py STFT.get_mel under autograd, on CPU:

    python tests/golden/make_golden_mel_grad.py [case names; default: all]

For each case ``(get_mel(y) * cot).sum().backward()`` with a seeded cotangent ``cot`` of the mel's shape; the .npz stores
y, hop, cot, the mel and y.grad.  librosa / soundfile are stubbed as in make_golden_mel.py (oracle.mel.load_reference_stft).

Cases: the four shapes of make_golden_mel.py (same signals), and one training-shaped row (172 frames at hop 512, the
2 s crops of configs/reflow.yaml) with exactly silent stretches, where the clamp at clip_val is active.  The tests import
``CASES`` / ``build_inputs`` from this module and only read the stored files.
"""
import os
import sys
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import mel as om  # noqa: E402
from tests.golden import make_golden_mel as GM  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
SR, N_MELS, N_FFT, FMIN, FMAX = 44100, 128, 2048, 40, 16000

# name: (seed, B, T, hop, silent stretches [(start, stop), ...] zeroed in every row)
CASES = OrderedDict([("mel_grad" + name[3:], (seed, B, T, hop, ())) for name, (seed, B, T, hop) in GM.CASES.items()])
CASES["mel_grad_b1_f172_silence"] = (5, 1, 172 * 512, 512, ((0, 9000), (30000, 41000), (80000, 172 * 512)))


def path(name):
    return os.path.join(HERE, name + ".npz")


def n_frames(T, hop):
    pad_left = (N_FFT - hop) // 2
    pad_right = max((N_FFT - hop + 1) // 2, N_FFT - T - pad_left)
    return 1 + (T + pad_left + pad_right - N_FFT) // hop


def build_inputs(name):
    """y [B, T] float32, hop, cotangent [B, n_mels, n_frames] float32"""
    seed, B, T, hop, silent = CASES[name]
    y = GM.signal(seed, B, T)
    for a, b in silent:
        y[:, a:b] = 0.0
    cot = torch.randn(B, N_MELS, n_frames(T, hop), generator=torch.Generator().manual_seed(seed + 1000))
    return y, hop, cot


def run_reference(name):
    ref = om.load_reference_stft()
    y, hop, cot = build_inputs(name)
    st = ref.STFT(SR, N_MELS, N_FFT, N_FFT, hop, FMIN, FMAX)
    y = y.clone().requires_grad_(True)
    mel = st.get_mel(y)
    (mel * cot).sum().backward()
    return y.detach(), hop, cot, mel.detach(), y.grad


def main():
    for name in sys.argv[1:] or CASES:
        y, hop, cot, mel, grad = run_reference(name)
        np.savez_compressed(path(name), y=y.numpy(), hop=np.int64(hop), cot=cot.numpy(), mel=mel.numpy(),
                            grad=grad.numpy(), torch_version=np.array(torch.__version__))
        print("%-28s mel %s  clamped %d  |grad| max %.3e" % (name, tuple(mel.shape),
                                                               int((mel <= np.log(1e-5) + 1e-6).sum()), grad.abs().max()))


if __name__ == "__main__":
    main()

"""Generate tests/golden/keyshift_mel_*.npz with the reference's OWN nsf_hifigan/nvSTFT.py (build container only):

    python tests/golden/make_golden_keyshift_mel.py

STFT.get_mel(y, keyshift=k) in fp32 on the CPU, librosa and soundfile stubbed as in make_golden_mel.py.  The cases span
preprocess.py's U(-5, 5) pitch augmentation and the edges of the kernel: 768 bins then zero padding (keyshift -5,
n' = 1534), a prime transform length (+4.98, n' = 2731), the largest 4096-point Bluestein case (+7.02, n' = 3072), the
constant-padding branch, a ragged batch and hop 256.  (Not named mel_*.npz: those are keyshift-0 fixtures.)"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import mel as om  # noqa: E402
from tests.golden.make_golden_mel import signal  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = {   # name: (seed, B, T, hop, keyshift)
    "keyshift_mel_b1_m5": (11, 1, 512 * 20 + 77, 512, -5.0),
    "keyshift_mel_b1_m2p3": (12, 1, 512 * 15 + 10, 512, -2.3),
    "keyshift_mel_b1_p0p7": (13, 1, 512 * 13, 512, 0.7),
    "keyshift_mel_b1_p4p98_prime": (14, 1, 512 * 17 + 200, 512, 4.98),
    "keyshift_mel_b1_p7p02_edge": (15, 1, 512 * 12, 512, 7.02),
    "keyshift_mel_b1_short_constpad": (16, 1, 900, 512, 3.0),   # pad_right >= T: the 'constant' padding branch
    "keyshift_mel_b2_ragged": (17, 2, 512 * 9 + 333, 512, -4.1),
    "keyshift_mel_b1_hop256": (18, 1, 256 * 30, 256, 2.5),
}


def path(name):
    return os.path.join(HERE, name + ".npz")


def main():
    ref = om.load_reference_stft()
    for name, (seed, B, T, hop, keyshift) in CASES.items():
        st = ref.STFT(44100, 128, 2048, 2048, hop, 40, 16000)
        y = signal(seed, B, T)
        with torch.no_grad():
            mel = st.get_mel(y, keyshift=keyshift)
        n_fft = int(np.round(2048 * 2 ** (keyshift / 12)))
        np.savez_compressed(path(name), y=y.numpy(), hop=np.int64(hop), keyshift=np.float64(keyshift),
                            n_fft=np.int64(n_fft), mel=mel.numpy())
        print(name, n_fft, tuple(mel.shape), float(mel.min()), float(mel.max()))


if __name__ == "__main__":
    main()

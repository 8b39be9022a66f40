"""The restatement of the mel front end (oracle/mel.py) against the reference: fixtures produced by the reference's own
nvSTFT.py (tests/golden/mel_*.npz), its live code where present, and torchaudio's independent implementation of the
librosa / Slaney mel filterbank (librosa itself is an absent third-party dependency)."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import mel as om
from oracle import ref_loader

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = sorted(glob.glob(os.path.join(HERE, "golden", "mel_*.npz")))


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p)[:-4] for p in GOLD])
def test_restatement_reproduces_the_reference_fixtures(path):
    z = np.load(path)
    with torch.no_grad():
        got = om.get_mel(torch.from_numpy(z["y"]), hop_length=int(z["hop"])).numpy()
    assert got.shape == z["mel"].shape
    assert np.array_equal(got, z["mel"])


def test_filterbank_agrees_with_torchaudio_and_with_the_product_host_code():
    import torchaudio.functional as TF
    from ddsp_svc_b200 import mel as pm
    for sr, n_fft, n_mels, fmin, fmax in ((44100, 2048, 128, 40, 16000), (22050, 1024, 80, 20, 11025), (44100, 2048, 128, 0, None)):
        ours = om.librosa_mel(sr, n_fft, n_mels, fmin, fmax)
        ta = TF.melscale_fbanks(n_fft // 2 + 1, float(fmin), float(fmax or sr / 2), n_mels, sr, norm="slaney", mel_scale="slaney").T.numpy()
        assert ours.dtype == np.float32 and ours.shape == ta.shape
        assert np.abs(ours - ta).max() < 1e-5 * ours.max()
        prod = pm.mel_filterbank(sr, n_fft, n_mels, fmin, fmax)
        assert np.abs(prod - ours).max() < 1e-6 * ours.max()
        lohi = pm._support(prod)
        for m in range(n_mels):                      # the sparse form the kernel uses covers every non-zero weight
            assert not prod[m, :lohi[m, 0]].any() and not prod[m, lohi[m, 1]:].any()
        assert (ours.sum(1) > 0).all()


def test_restatement_equals_the_live_reference_code():
    """the reference's own STFT.get_mel on these inputs is stored in tests/golden/stft_live_reference.npz
    (tests/golden/make_golden_reference.py)"""
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stft_live_reference.npz"))
    g = torch.Generator().manual_seed(9)
    for i, (T, hop) in enumerate(((512 * 9 + 17, 512), (900, 512), (256 * 30, 256))):
        y = 0.2 * torch.randn(2, T, generator=g)
        with torch.no_grad():
            assert np.array_equal(om.get_mel(y, hop_length=hop).numpy(), gold["mel_%d" % i])

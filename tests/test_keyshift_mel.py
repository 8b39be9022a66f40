"""The key-shifted mel (STFT.get_mel with keyshift != 0; csrc/mel.cu's mel_keyshift_kernel) without a GPU: the oracle
against the reference's fixtures (tests/golden/keyshift_mel_*.npz), the float64 host tables against a direct DFT, the
kernel source executed on the CPU (tests/emu/host_emu.h) against the fixtures and under ThreadSanitizer, the C ABI's
argument checks, and patch_reference(vocoder=True).  The kernel itself runs on hardware in tests/test_gpu_keyshift_mel.py."""
import ctypes

import numpy as np
import pytest
import torch

import ddsp_svc_b200 as pkg
from ddsp_svc_b200 import _lib, bluestein
from ddsp_svc_b200 import loss as pl
from ddsp_svc_b200 import mel as pm
from oracle import mel as om
from oracle import ref_loader
from tests.emu_harness import abi_call, assert_race_free, shared, tsan
from tests.golden import make_golden_keyshift_mel as GK

# the keyshift-0 kernel's bounds in log-mel (tests/test_gpu_mel.py)
TOL_MAX, TOL_RMS = 2e-3, 5e-5


def _load(name):
    return np.load(GK.path(name))


@pytest.mark.parametrize("name", list(GK.CASES))
def test_oracle_reproduces_the_reference_fixtures(name):
    z = _load(name)
    assert int(z["n_fft"]) == pm.keyshift_n_fft(2048, float(z["keyshift"]))
    with torch.no_grad():
        got = om.get_mel(torch.from_numpy(z["y"]), hop_length=int(z["hop"]), keyshift=float(z["keyshift"])).numpy()
    assert got.shape == z["mel"].shape
    assert np.array_equal(got, z["mel"])


@pytest.mark.parametrize("n", [1534, 2048, 2731, 3072, 1021, 97])
def test_keyshift_table_is_a_bluestein_dft_of_the_first_bins(n):
    """prime, even and small n': chirp, filter spectrum and window reproduce a float64 DFT of the first K bins"""
    K = min(1025, n // 2 + 1)
    t = pm.keyshift_table_host(n)
    M = bluestein.size(n, K)
    assert t.dtype == np.float32 and t.size == _lib.lib().b2d_mel_keyshift_table_floats(n) == bluestein.table_floats(n, K)
    assert M >= n + K - 1 and (M == 1024 or M // 2 < n + K - 1)
    assert np.array_equal(t[4:4 + n], torch.hann_window(n).numpy())
    chirp = t[bluestein.chirp_off(n):bluestein.chirp_off(n) + 2 * n].view(np.complex64).astype(np.complex128)
    hspec = t[bluestein.hspec_off(n):bluestein.hspec_off(n) + 2 * M].view(np.complex64).astype(np.complex128)
    x = np.random.default_rng(n).standard_normal(n)
    u = np.zeros(M, np.complex128)
    u[:n] = x * np.conj(chirp)
    X = np.conj(chirp[:K]) * np.fft.ifft(np.fft.fft(u) * hspec * M)[:K]
    want = np.fft.fft(x)[:K]
    assert np.abs(X - want).max() < 1e-5 * np.abs(want).max()


def test_rss_tables_unchanged_by_the_shared_builder():
    """loss.table_host (all n bins) still builds the table of the RSS kernels: head c, window, the same Bluestein size"""
    for n in (256, 257, 1021, 2047):
        t = pl.table_host(n)
        w = torch.hann_window(n)
        assert t.size == _lib.lib().b2d_rss_table_floats(n) and pl.bluestein_size(n) == bluestein.size(n, n)
        assert t[0] == np.float32(w.pow(2.0).sum().sqrt().item()) and np.array_equal(t[4:4 + n], w.numpy())
        assert np.array_equal(t[4:], bluestein.table_host(n, n, w.numpy())[4:])


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = shared("emu_mel_keyshift.cpp", tmp_path_factory)
    basis = pm.mel_filterbank(44100, 2048, 128, 40, 16000)
    lohi = pm._support(basis)
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)

    def run(y, hop, n):
        y = np.ascontiguousarray(y, np.float32)
        table = pm.keyshift_table_host(n)
        nF = lib.emu_mel_keyshift_frames(y.shape[1], n, hop)
        assert nF == _lib.lib().b2d_mel_frames(y.shape[1], n, n, hop)
        out = np.full((y.shape[0], 128, nF), np.nan, np.float32)
        assert lib.emu_mel_keyshift(ptr(y), ptr(table), ptr(basis), ptr(lohi), y.shape[0], y.shape[1], n, hop, 128, 1e-5,
                                    ptr(out)) == 0
        return out
    return run


@pytest.mark.parametrize("name", list(GK.CASES))
def test_kernel_source_matches_the_reference_fixtures(emu, name):
    z = _load(name)
    got = emu(z["y"], int(z["hop"]), int(z["n_fft"]))
    assert got.shape == z["mel"].shape and np.isfinite(got).all()
    d = got.astype(np.float64) - z["mel"]
    assert np.abs(d).max() < TOL_MAX and np.sqrt((d ** 2).mean()) < TOL_RMS, (np.abs(d).max(), np.sqrt((d ** 2).mean()))


def test_kernel_source_has_no_shared_memory_race(tmp_path):
    assert_race_free(tsan("tsan_mel_keyshift.cpp", tmp_path))


def test_keyshift_abi_argument_errors_do_not_touch_the_device():
    _lib.build()
    L = _lib.lib()
    ok = dict(audio=16, table=16, mel_basis=16, filter_lohi=16, B=1, n_samples=8192, n_fft=1534, hop=512, n_mels=128,
              clip_val=1e-5, mel=16, stream=0)
    call = lambda **kw: abi_call("b2d_mel_spectrogram_keyshift", dict(ok, **kw))
    assert call(audio=0) == -1 and call(table=0) == -1 and call(mel=0) == -1 and call(filter_lohi=0) == -1  # NULL
    assert call(table=20) == -3                                                                              # ALIGN
    assert call(B=0) == -2 and call(B=70000) == -2 and call(n_samples=0) == -2 and call(hop=0) == -2        # SHAPE
    assert call(n_mels=0) == -2 and call(n_mels=129) == -2
    assert call(n_fft=3073) == -4 and call(n_fft=511) == -4 and call(n_fft=100, hop=256) == -4             # UNSUPPORTED
    assert b"mel_spectrogram_keyshift" in L.b2d_last_error()
    assert L.b2d_mel_keyshift_table_floats(0) == 0 and L.b2d_mel_keyshift_table_floats(3073) == 0


def test_get_mel_keyshift_refuses_before_any_launch():
    st = pm.STFT(44100, 128, 2048, 2048, 512, 40, 16000)
    y = torch.zeros(1, 4096)
    with pytest.raises(NotImplementedError, match=r"keyshift in about \(-24\.0[0-9], 7\.02\)"):
        st.get_mel_keyshift(y, 7.1)
    with pytest.raises(NotImplementedError):
        st.get_mel_keyshift(y, -25.0)
    with pytest.raises(NotImplementedError, match="no backward"):
        st.get_mel_keyshift(y.requires_grad_(), -5.0)
    with pytest.raises(ValueError, match="CUDA"):
        st.get_mel_keyshift(torch.zeros(1, 4096), -5.0)      # CPU tensor: no fallback
    with pytest.raises(NotImplementedError):
        pm.STFT(22050, 80, 1024, 1024, 256, 20, 11025).get_mel_keyshift(y.detach(), -5.0)


def test_vocoder_refuses_unknown_types_and_cpu_devices(tmp_path):
    with pytest.raises(ValueError, match="Unknown vocoder"):
        pkg.Vocoder("hifigan", str(tmp_path / "model.ckpt"))
    with pytest.raises(ValueError, match="CUDA"):
        pkg.Vocoder("nsf-hifigan", str(tmp_path / "model.ckpt"), device="cpu")


needs_reference = pytest.mark.skipif(not ref_loader.available(),
                                     reason="reference checkout not available (DDSP_REFERENCE_ROOT)")


def _vocoder_modules():
    """{name: module} of diffusion.vocoder / reflow.vocoder that import here (diffusion.vocoder imports librosa.sequence
    through diffusion.diffusion)"""
    import importlib
    om.load_reference_stft()                                 # librosa / soundfile stubs for nsf_hifigan.nvSTFT
    mods = {}
    for name in ("diffusion.vocoder", "reflow.vocoder"):
        try:
            mods[name] = importlib.import_module(name)
        except ImportError:
            pass
    return mods


@needs_reference
def test_default_patch_leaves_the_vocoder_alone():
    mods = _vocoder_modules()
    before = {name: m.Vocoder for name, m in mods.items()}
    saved = pkg.patch_reference()
    try:
        assert {name: m.Vocoder for name, m in mods.items()} == before and "vocoder" not in saved
    finally:
        pkg.unpatch_reference(saved)


@needs_reference
def test_vocoder_patch_and_unpatch():
    mods = _vocoder_modules()
    assert "reflow.vocoder" in mods
    before = {name: m.Vocoder for name, m in mods.items()}
    assert pkg.Vocoder not in before.values()
    saved = pkg.patch_reference(vocoder=True)
    try:
        for name in ("diffusion.vocoder", "reflow.vocoder"):
            if name in mods:
                assert mods[name].Vocoder is pkg.Vocoder and name not in saved.get("_not_patched", {})
            else:
                assert name in saved["_not_patched"]
    finally:
        pkg.unpatch_reference(saved)
    assert {name: m.Vocoder for name, m in mods.items()} == before

"""Race detection for kernels whose races a GPU run cannot see: their source is executed by the host emulator
(tests/emu/host_emu.h, one std::thread per CUDA thread, __syncthreads = std::barrier, a barrier per warp, cp.async
copies performed at their wait_group, a cluster barrier) under ThreadSanitizer.  All of these kernels have run on
hardware; a race that resolves the same way on every run passes a bit-identity check there, and here it is a reported
data race between those threads.  The `racy` control kernel proves the detector sees through the emulated barrier in
both directions."""
import pytest

from tests.emu_harness import assert_race_free, tsan


def test_detector_sees_a_missing_barrier_and_accepts_a_correct_one(tmp_path):
    bad = tsan("tsan_main.cpp", tmp_path, None, "racy")
    assert "ThreadSanitizer: data race" in bad.stderr and bad.returncode == 66
    assert_race_free(tsan("tsan_main.cpp", tmp_path, None, "ok"))


@pytest.mark.parametrize("define", ["TSAN_FIRFFT", "TSAN_CSFAST", "TSAN_SUPERFAST", "TSAN_LINATTN", "TSAN_HIFIGAN",
                                    "TSAN_RMVPE_CONV", "TSAN_RMVPE_GRU", "TSAN_RMVPE_MEL", "TSAN_HUBERT_ATTN",
                                    "TSAN_HUBERT_POSCONV", "TSAN_HUBERT_CONV0", "TSAN_HUBERT_LN"])
def test_kernel_source_has_no_shared_memory_race(tmp_path, define):
    assert_race_free(tsan("tsan_main.cpp", tmp_path, define))

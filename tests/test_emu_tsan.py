"""Race detection for the kernels that have not run on hardware yet: their source is executed by the host emulator
(tests/emu/host_emu.h, one std::thread per CUDA thread, __syncthreads = std::barrier) under ThreadSanitizer.  A missing
or misplaced __syncthreads around shared memory is a data race between those threads and gets reported; the `racy`
control kernel proves the detector sees through the emulated barrier in both directions."""
import pytest

from tests.emu_harness import assert_race_free, tsan


def test_detector_sees_a_missing_barrier_and_accepts_a_correct_one(tmp_path):
    bad = tsan("tsan_main.cpp", tmp_path, None, "racy")
    assert "ThreadSanitizer: data race" in bad.stderr and bad.returncode == 66
    assert_race_free(tsan("tsan_main.cpp", tmp_path, None, "ok"))


@pytest.mark.parametrize("define", ["TSAN_FIRFFT", "TSAN_CSFAST", "TSAN_SUPERFAST", "TSAN_LINATTN"])
def test_kernel_source_has_no_shared_memory_race(tmp_path, define):
    assert_race_free(tsan("tsan_main.cpp", tmp_path, define))

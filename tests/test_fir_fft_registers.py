"""ptxas report of csrc/ltv_fir_fft.cu compiled with the library's own flags: the 1024-point instantiations of the
FFT-domain FIR (one and two jobs, both complex-addition policies, taps from memory or spectra) keep everything in
registers -- no local-memory spill traffic competing with the shared-memory transforms."""
import os
import re
import shutil
import subprocess

import pytest

from ddsp_svc_b200 import _lib

NVCC = os.environ.get("NVCC") or shutil.which("nvcc")

pytestmark = pytest.mark.skipif(NVCC is None, reason="nvcc not available")


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ptxas") / "ltv_fir_fft.cubin")
    flags = [f for f in _lib.NVCC_FLAGS if f not in ("-shared",)]
    cmd = [NVCC] + flags + ["-Xptxas", "-v", "-cubin", "-o", out, os.path.join(_lib.CSRC, "ltv_fir_fft.cu")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    # kernel (mangled name) -> (spill store bytes, spill load bytes)
    report, kernel = {}, None
    for line in proc.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            kernel = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and kernel:
            report[kernel] = (int(m.group(1)), int(m.group(2)))
    return report


# ltv_fir_fft_kernel<N, NJ, PK, NBANK, SPEC> as it appears in the mangled name
# (the spectrum variant exists for two jobs only)
@pytest.mark.parametrize("pk", [0, 1])
@pytest.mark.parametrize("nj,spec", [(1, 0), (2, 0), (2, 1)])
def test_1024_point_instantiations_do_not_spill(ptxas_report, nj, pk, spec):
    pat = re.compile(r"ltv_fir_fft_kernelILi1024ELi%dELb%dELi0ELb%dE" % (nj, pk, spec))
    hits = {k: v for k, v in ptxas_report.items() if pat.search(k)}
    assert len(hits) == 1, sorted(ptxas_report)
    (name, spills), = hits.items()
    assert spills == (0, 0), (name, spills)

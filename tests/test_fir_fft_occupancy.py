"""Resources of the two-job 1024-point FFT-domain FIR (the Sins split path's all-pass + noise filters and mix, both
complex-addition policies, taps from memory): compiled with the library's own flags it asks for 4 resident CTAs per SM,
holds at most 128 registers with no spill and no stack frame, and its shared memory leaves room for 4 CTAs per SM on
an H100 (228 KB per SM, 1 KB reserved per CTA)."""
import os
import re
import shutil
import subprocess

import pytest

from ddsp_svc_b200 import _lib
from tests import emu_harness

NVCC = os.environ.get("NVCC") or shutil.which("nvcc")
SRC = os.path.join(_lib.CSRC, "ltv_fir_fft.cu")
HEADLINE = r"ltv_fir_fft_kernelILi1024ELi2ELb%dELi0ELb0E"

pytestmark = pytest.mark.skipif(NVCC is None, reason="nvcc not available")


def _flags():
    return [f for f in _lib.NVCC_FLAGS if f not in ("-shared",)]


@pytest.fixture(scope="module")
def ptxas(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ptxas") / "ltv_fir_fft.cubin")
    proc = subprocess.run([NVCC] + _flags() + ["-Xptxas", "-v", "-cubin", "-o", out, SRC], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    report, kernel = {}, None
    for line in proc.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            kernel = m.group(1)
            report[kernel] = {}
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and kernel:
            report[kernel].update(stack=int(m.group(1)), spill_st=int(m.group(2)), spill_ld=int(m.group(3)))
        m = re.search(r"Used (\d+) registers", line)
        if m and kernel:
            report[kernel]["regs"] = int(m.group(1))
    return report


@pytest.fixture(scope="module")
def ptx(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ptx") / "ltv_fir_fft.ptx")
    proc = subprocess.run([NVCC] + _flags() + ["-ptx", "-o", out, SRC], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    with open(out) as f:
        return f.read()


def _one(items, pk):
    pat = re.compile(HEADLINE % pk)
    hits = [k for k in items if pat.search(k)]
    assert len(hits) == 1, hits
    return hits[0]


@pytest.mark.parametrize("pk", [0, 1])
def test_headline_fits_128_registers_without_spilling(ptxas, pk):
    name = _one(ptxas, pk)
    r = ptxas[name]
    assert r["regs"] <= 128 and r["stack"] == 0 and r["spill_st"] == 0 and r["spill_ld"] == 0, (name, r)


@pytest.mark.parametrize("pk", [0, 1])
def test_headline_asks_for_four_ctas_per_sm(ptx, pk):
    entries = re.findall(r"\.entry\s+(\S+)\(.*?\)\s*((?:\.\w+[^\n{]*\n\s*)*)\{", ptx, re.S)
    name = _one([e[0] for e in entries], pk)
    directives = dict(entries)[name]
    assert re.search(r"\.maxntid\s+128,\s*1,\s*1", directives), directives
    assert re.search(r"\.minnctapersm\s+4\b", directives), directives


def test_headline_shared_memory_fits_four_ctas(tmp_path):
    emu_harness._need_gxx()
    src = tmp_path / "smem.cpp"
    src.write_text('#define B2D_HOST_EMU 1\n#include "%s"\n#include "%s"\n#include <cstdio>\n'
                   'int main() { std::printf("%%zu\\n", fir_fft_smem<1024, 2>()); }\n'
                   % (os.path.join(emu_harness.EMU, "host_emu.h"), SRC))
    exe = str(tmp_path / "smem")
    proc = subprocess.run(emu_harness.GXX + ["-O0", "-o", exe, str(src)], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    smem = int(subprocess.run([exe], capture_output=True, text=True, check=True).stdout)
    assert 4 * (smem + 1024) <= 228 * 1024, smem

"""Generate tests/golden/offline_diff_settings.json from the LIVE reference (build container only):

    DDSP_REFERENCE_ROOT=<DDSP-SVC checkout> python tests/golden/make_golden_offline_diff.py

The choices main_diff.py and batch_infer.py make before they run a diffusion model -- whether the external DDSP model
feeds the shallow diffusion, whether the input's mel does, k_step, the speedup, the method and the diffusion speaker --
are executed from the drivers' own source text (neither file can be imported here), with stub ``cmd`` / ``args`` and a
stub ``load_model`` that returns a DDSP config:

- main_diff.py: its lines from ``spk_id = torch.LongTensor(...)`` up to ``# forward and save the output``, with its own
  ``check_args``;
- batch_infer.py: its loader lines (``ddsp = None`` up to ``# load units encoder``, __main__) and then its infer()
  lines from ``spk_id = torch.LongTensor(...)`` up to ``with torch.no_grad():``, with its own ``check_args``.

The mode is then read as each driver's model call reads it: main_diff.py's loop takes the DDSP model if it is not None,
else input_mel if not None; batch_infer.py's infer() overwrites input_mel with the DDSP model's mel when it has one.

The grid: every model.type x k_step (None, below model.k_step_max, above it) x DDSP checkpoint (none, compatible, one
incompatible per checked field) x speedup / method ('auto' and given) x diff_spk_id ('auto' and given) x driver."""
import contextlib
import io
import itertools
import json
import os
import sys
import textwrap

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from tests.golden.make_golden_frontend import reference_function  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

DATA = {"sampling_rate": 44100, "block_size": 512, "encoder": "contentvec768l12"}
INFER = {"speedup": 10, "method": "dpm-solver"}
K_STEP_MAX = 100
SPK_ID = "2"
MODEL_TYPES = ("Diffusion", "DiffusionNew", "DiffusionFast")
K_STEPS = (None, "40", "150")
DDSPS = ("none", "compatible", "sampling_rate", "block_size", "encoder")   # a field name: that field differs
SAMPLERS = (("auto", "auto"), ("1", "ddim"), ("20", "unipc"))
DIFF_SPK_IDS = ("auto", "3")
BAD = {"sampling_rate": 48000, "block_size": 256, "encoder": "hubertsoft"}


class DotDict(dict):
    def __getattr__(self, key):
        val = self.get(key)
        return DotDict(val) if type(val) is dict else val


def lines(py_file, first, stop, after=None):
    """the statements of a reference file from the first line starting with ``first`` (searched after the line
    starting with ``after``) up to, not including, the next line starting with ``stop``; dedented"""
    src = open(os.path.join(ref_loader.REFERENCE_ROOT, py_file)).read().splitlines()
    begin = 0
    if after is not None:
        begin = [i for i, l in enumerate(src) if l.strip().startswith(after)][0] + 1
    a = [i for i in range(begin, len(src)) if src[i].strip().startswith(first)][0]
    b = [i for i in range(a + 1, len(src)) if src[i].strip().startswith(stop)][0]
    return compile(textwrap.dedent("\n".join(src[a:b])), py_file, "exec")


class Vocoder:
    def extract(self, audio, sample_rate, keyshift=0):
        return torch.zeros(1, 3, 2)


def namespace(py_file, cmd, args, ddsp_args):
    def load_model(path, device="cpu"):
        assert path == cmd.ddsp_ckpt
        return object(), ddsp_args
    return {"np": np, "torch": torch, "cmd": cmd, "args": args, "device": "cpu", "vocoder": Vocoder(),
            "audio": np.zeros(8, np.float32), "sample_rate": 44100, "spk_mix_dict": None, "load_model": load_model,
            "check_args": reference_function(py_file, "check_args")}


def outcome(ns):
    ddsp = ns["ddsp"] is not None
    return {"ddsp": ddsp, "input_mel": not ddsp and ns["input_mel"] is not None, "k_step": ns["k_step"],
            "infer_speedup": ns["infer_speedup"], "method": ns["method"],
            "diff_spk_id": int(ns["diff_spk_id"].reshape(-1)[0])}


def main():
    main_diff = lines("main_diff.py", "spk_id = torch.LongTensor(", "# forward and save the output")
    loader = lines("batch_infer.py", "ddsp = None", "# load units encoder",
                   after="model, vocoder, args = load_model_vocoder")
    infer = lines("batch_infer.py", "spk_id = torch.LongTensor(", "with torch.no_grad():")
    cases = []
    for kind, k_step, ddsp, (speedup, method), diff_spk_id, whole in itertools.product(
            MODEL_TYPES, K_STEPS, DDSPS, SAMPLERS, DIFF_SPK_IDS, (False, True)):
        cmd = DotDict(spk_id=SPK_ID, diff_spk_id=diff_spk_id, speedup=speedup, method=method, k_step=k_step,
                      ddsp_ckpt=None if ddsp == "none" else "ddsp/model.pt", spk_mix_dict="None")
        args = DotDict(data=dict(DATA), model={"type": kind, "k_step_max": K_STEP_MAX}, infer=dict(INFER))
        ddsp_args = DotDict(data=dict(DATA, **({ddsp: BAD[ddsp]} if ddsp in BAD else {})))
        ns = namespace("batch_infer.py" if whole else "main_diff.py", cmd, args, ddsp_args)
        with contextlib.redirect_stdout(io.StringIO()):
            if whole:
                exec(loader, ns)
                exec(infer, ns)
            else:
                exec(main_diff, ns)
        cases.append({"model_type": kind, "k_step": k_step, "ddsp": ddsp, "speedup": speedup, "method": method,
                      "diff_spk_id": diff_spk_id, "whole": whole, "want": outcome(ns)})
    out = {"data": DATA, "infer": INFER, "k_step_max": K_STEP_MAX, "spk_id": int(SPK_ID), "bad": BAD, "cases": cases}
    text = json.dumps(out, sort_keys=True)                               # one case per line
    with open(os.path.join(HERE, "offline_diff_settings.json"), "w") as f:
        f.write(text.replace(', {"ddsp"', ',\n{"ddsp"').replace('[{"ddsp"', '[\n{"ddsp"') + "\n")
    print(len(cases), "cases")


if __name__ == "__main__":
    main()

"""Generate tests/golden/offline_slicer.npz from the LIVE reference (build container only):

    DDSP_REFERENCE_ROOT=<DDSP-SVC checkout> python tests/golden/make_golden_offline.py

For every case of tests/offline_oracle.SLICER_CASES at 44.1 and 16 kHz (rebuilt from its seed; no audio is stored):

- the reference's ``Slicer`` (slicer.py) is imported and run.  librosa is not installed, so it gets a stub whose
  ``feature.rms`` is ``offline_oracle.rms64``: librosa >= 0.10's framing (center=True, zero padding) in float64;
- main.py's ``split`` and ``cross_fade`` are compiled from main.py's own source text (main.py itself cannot be
  imported), and its assembly lines (``silent_length = ...`` to ``current_length = ...``) are executed from that text
  on seeded segment outputs at an enhancer rate (48 kHz) other than the model's (44.1 kHz).

Stored per case: the rms, the Slicer's chunks, split()'s (start_frame, end_frame) list and the float64 assembly (or
the error main.py's cross_fade raises, for a case with one segment shorter than its overlap)."""
import os
import sys
import textwrap
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from tests import offline_oracle as oo  # noqa: E402
from tests.golden.make_golden_frontend import reference_function  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def install_librosa_stub():
    librosa = types.ModuleType("librosa")
    librosa.feature = types.SimpleNamespace(rms=lambda y, frame_length, hop_length: oo.rms64(y, frame_length,
                                                                                                hop_length))
    librosa.to_mono = lambda y: np.mean(y, axis=0)
    sys.modules["librosa"] = librosa
    try:
        import torchaudio  # noqa: F401
    except Exception:
        sys.modules["torchaudio"] = types.ModuleType("torchaudio")


def assembly_lines():
    """main.py's per-segment assembly statements, from its own text, as a function of (result, current_length,
    start_frame, seg_output, args, output_sample_rate)"""
    src = open(os.path.join(ref_loader.REFERENCE_ROOT, "main.py")).read().splitlines()
    first = [i for i, l in enumerate(src) if l.strip().startswith("silent_length = round(")][0]
    last = [i for i, l in enumerate(src) if l.strip().startswith("current_length = current_length")][0]
    body = textwrap.dedent("\n".join(src[first:last + 1]))
    code = ("def step(result, current_length, start_frame, seg_output, args, output_sample_rate):\n" +
            textwrap.indent(body, "    ") + "\n    return result, current_length\n")
    ns = {"np": np, "cross_fade": reference_function("main.py", "cross_fade")}
    exec(compile(code, "main.py", "exec"), ns)
    return ns["step"]


def main():
    install_librosa_stub()
    sys.dont_write_bytecode = True
    sys.path.insert(0, ref_loader.REFERENCE_ROOT)
    from slicer import Slicer
    split = reference_function("main.py", "split")
    split.__globals__["Slicer"] = Slicer
    step = assembly_lines()
    A = oo.ASSEMBLY
    args = types.SimpleNamespace(data=types.SimpleNamespace(block_size=A["block_size"], sampling_rate=A["model_sr"]))
    out = {}
    for sr in oo.SLICER_RATES:
        for name in sorted(oo.SLICER_CASES):
            key = "%s_%d" % (name, sr)
            audio = oo.slicer_case(name, sr)
            s = Slicer(sr=sr, threshold=-40, min_length=5000)
            out[key + "_rms"] = oo.rms64(audio, s.win_size, s.hop_size)[0]
            chunks = s.slice(audio)
            out[key + "_chunks"] = np.array([[int(t) for t in c["split_time"].split(",")] + [int(c["slice"])]
                                             for c in chunks.values()], dtype=np.int64)
            hop = oo.SPLIT_HOP[sr]
            segs = split(audio, sr, float(hop))
            frames = np.array([[a, a + seg.shape[0] // hop] for a, seg in segs], dtype=np.int64).reshape(-1, 2)
            out[key + "_split"] = frames
            if not len(frames):
                continue
            for short in (None, len(frames) - 1) if len(frames) > 1 else (None,):
                seed = 1000 * oo.SLICER_RATES.index(sr) + 10 * sorted(oo.SLICER_CASES).index(name) + (short is not None)
                outs = oo.assembly_segments(frames[:, 0], frames[:, 1], seed=seed, short=short, **A)
                result, current = np.zeros(0), 0
                tag = key + ("_assembly" if short is None else "_assembly_short")
                out[tag + "_seed"] = np.int64(seed)
                try:
                    for a, seg in zip(frames[:, 0], outs):
                        result, current = step(result, current, int(a), seg, args, A["out_sr"])
                    out[tag] = result
                except ValueError as e:
                    out[tag + "_error"] = np.array(str(e))
            print(key, len(chunks), frames.tolist())
    np.savez_compressed(os.path.join(HERE, "offline_slicer.npz"), **out)


if __name__ == "__main__":
    torch.manual_seed(0)
    main()

"""The internal side streams of the Sins and CombSub drivers (b2d_set_overlap).  Every overlap mode gives the bits of
mode 0, and a call captured into a CUDA graph replays to the bits of the eager call.  A driver that leaves one of its
side streams unjoined on the caller's stream makes the capture end with an error, so the capture checks the join on
every path: the split / fused / spectrum Sins variants, the staggered sub-batches, and the two side lanes a launch of
less than one wave of frames takes."""
import pytest
import torch

from ddsp_svc_b200 import ops, synthetic as syn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, P, B = 44100, 512, 3
MODES = (0, 1, 2, 3, -2)

# name: (synthesizer, b2d_set_sins_impl variant, control widths of the split map, explicit noise input)
CASES = {
    "sins_split": ("sins", "split", (64, 129, 129), False),
    "sins_fused": ("sins", "fused", (64, 129, 129), False),
    "sins_spectrum": ("sins", "spectrum", (64, 129, 129), True),
    "sins_unequal_taps": ("sins", "split", (64, 65, 129), True),
    "combsub_equal_taps": ("combsub", "auto", (129, 257, 129), False),
    "combsub_unequal_taps": ("combsub", "auto", (65, 257, 129), True),
}


def _frames(rows):
    # the Sins driver builds the two impulse responses of a launch of at most 64 frames per SM on two side streams
    if rows == "one_wave":
        return 40
    return torch.cuda.get_device_properties(DEV).multi_processor_count * 64 // B + 1


def _synth(synth, f0, fp, c, noise):
    if synth == "sins":
        return ops.sins_synth(f0, fp, c["amplitudes"], c["group_delay"], c["noise_magnitude"], P, SR, noise_in=noise,
                              seed=5, utterance_offset=2)
    return ops.combsub_synth(f0, fp, c["group_delay"], c["harmonic_magnitude"], c["noise_magnitude"], P, SR,
                             noise_in=noise, seed=5, utterance_offset=2)


@pytest.mark.parametrize("rows", ["one_wave", "many_waves"])
@pytest.mark.parametrize("case", list(CASES))
def test_overlap_modes_agree_and_capture_joins_every_side_stream(case, rows):
    synth, impl, widths, explicit = CASES[case]
    nF = _frames(rows)
    sm = (syn.sins_split_map if synth == "sins" else syn.combsub_split_map)(*widths)
    f0 = syn.make_f0(B, nF, SR, P, seed=31, unvoiced_fraction=0.1).to(DEV)
    c = syn.split_views(syn.make_ctrl(B, nF, sm, seed=32)[0].to(DEV), sm)
    noise = syn.uniform_noise(B, nF * P, 33).to(DEV) if explicit else None
    fp, _ = ops.phase_scan(f0, P, SR)
    base = None
    try:
        if synth == "sins":
            ops.set_sins_impl(impl)
        for mode in MODES:
            ops.set_overlap(mode)
            # the eager call is also the warm-up: it builds the DFT tables (which synchronise) and the side streams
            eager = _synth(synth, f0, fp, c, noise)
            base = eager if base is None else base
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                captured = _synth(synth, f0, fp, c, noise)
            graph.replay()
            torch.cuda.synchronize()
            for name, b, e, r in zip(("signal", "harmonic", "noise"), base, eager, captured):
                assert torch.equal(b, e), (mode, name, "eager differs from mode 0")
                assert torch.equal(e, r), (mode, name, "graph replay differs from the eager call")
    finally:
        ops.set_overlap(1)
        ops.set_sins_impl("auto")

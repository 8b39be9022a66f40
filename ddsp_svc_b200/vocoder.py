"""Drop-in synthesizer modules: same constructor arguments, buffers (state-dict keys) and
forward() contract as the reference's ddsp/vocoder.py classes, with the DSP executed by the
sm_90a kernels of libb200ddsp.so.

    signal, hidden, (harmonic, noise) = model(units_frames, f0_frames, volume_frames,
                                              spk_id=..., spk_mix_dict=..., initial_phase=..., infer=True)

``unit2ctrl`` (the small network that predicts the frame-rate controls, reference
ddsp/unit2control.py) is outside the accelerated path: pass your own module, or leave it None
to use the reference's Unit2Control when the reference package is importable (the
``patch_reference()`` drop-in scenario).

Two noise modes: by default white noise is generated inside the FIR kernel (Philox, seeded
from torch's CPU generator so ``torch.manual_seed`` makes runs reproducible); pass
``noise=tensor [B, T]`` to feed explicit samples (parity tests feed what the reference's
``rand_like`` drew).
"""
import torch

from . import ops


def _reference_unit2ctrl(n_unit, n_spk, split_map, **kw):
    """The control network: this package's own Unit2Control (same parameter tree as the reference's
    ddsp/unit2control.py, so its checkpoints load strictly; fused kernels + library GEMMs; trainable with the convolution-only decoder that
    CombSubSuperFast selects, and with the PCmer decoder of Sins, CombSub and CombSubFast when
    ``Unit2Control.pcmer_backward`` is set -- off by default, outputs detached)."""
    from .unit2control import Unit2Control
    return Unit2Control(n_unit, n_spk, split_map, **kw)


def _host_seed():
    # consumes torch's CPU generator (reproducible under torch.manual_seed), no device sync
    return int(torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).item())


def _check_shape(cls, ok, what):
    """Shapes the kernels do not cover fail when the model is BUILT (load_model / patch_reference time), not at the
    first forward after some kernels have already been launched."""
    if not ok:
        raise ValueError("%s: %s (every config the reference ships uses block_size 512)" % (cls, what))


class _SynthBase(torch.nn.Module):
    def _scalars(self):
        """sampling_rate / block_size live in 0-dim buffers (state-dict compatible with the
        reference, ddsp/vocoder.py:546-547); read them once, not on every call."""
        c = self.__dict__.get("_scalar_cache")
        if c is None:
            c = (int(self.sampling_rate.item()), int(self.block_size.item()))
            self.__dict__["_scalar_cache"] = c
        return c

    def _load_from_state_dict(self, *a, **k):
        super()._load_from_state_dict(*a, **k)
        self.__dict__["_scalar_cache"] = None


class Sins(_SynthBase):
    """Sinusoids additive synthesiser -- reference ddsp/vocoder.py:532-611."""

    def __init__(self, sampling_rate, block_size, n_harmonics, n_mag_allpass, n_mag_noise, n_unit=256, n_spk=1,
                 unit2ctrl=None):
        super().__init__()
        _check_shape("Sins", int(block_size) % 256 == 0 and 0 < int(block_size) <= 2048, "block_size %s must be a "
                     "multiple of 256 up to 2048" % (block_size,))
        _check_shape("Sins", 0 < int(n_harmonics) <= 512 and min(int(n_mag_allpass), int(n_mag_noise)) >= 2 and
                     max(int(n_mag_allpass), int(n_mag_noise)) <= 1025, "n_harmonics <= 512 and 2 <= n_mag <= 1025")
        self.register_buffer("sampling_rate", torch.tensor(sampling_rate))
        self.register_buffer("block_size", torch.tensor(block_size))
        split_map = {
            "amplitudes": n_harmonics,
            "group_delay": n_mag_allpass,
            "noise_magnitude": n_mag_noise,
        }
        self.unit2ctrl = unit2ctrl if unit2ctrl is not None else _reference_unit2ctrl(n_unit, n_spk, split_map)

    def forward(self, units_frames, f0_frames, volume_frames, spk_id=None, spk_mix_dict=None, initial_phase=None,
                infer=True, max_upsample_dim=32, noise=None, utterance_offset=0, signal_out=None):
        """units_frames B x n_frames x n_unit; f0_frames B x n_frames x 1; volume_frames B x n_frames x 1.
        ``max_upsample_dim`` only chunks the reference's temporaries and has no effect here.
        ``signal_out``: optional preallocated [B, T] destination of ``signal`` (may be peer-mapped memory).

        Trainable in the training phase: with ``infer=False`` (what the reference's solver.py calls) and a control
        from ``unit2ctrl`` that requires grad (grad mode on), signal, harmonic and noise are differentiable with
        respect to the three controls (CUDA backward, ops.sins_synth_backward) for block 512, n_mag <= 257 and up
        to 512 harmonics.  f0 is data, as in the reference's train.py: an f0 that requires grad is refused."""
        sr, block = self._scalars()
        if torch.is_grad_enabled() and isinstance(f0_frames, torch.Tensor) and f0_frames.requires_grad:
            raise NotImplementedError("Sins has no gradient with respect to f0_frames; pass f0 as data "
                                      "(f0_frames.detach()), as the reference's train.py does")
        frame_phase, phase_frames = ops.phase_scan(f0_frames, block, sr, initial_phase, infer)
        ctrls, hidden = self.unit2ctrl(units_frames, f0_frames, phase_frames, volume_frames, spk_id=spk_id,
                                       spk_mix_dict=spk_mix_dict)
        signal, harmonic, noise_out = ops.sins_synth(
            f0_frames, frame_phase, ctrls["amplitudes"], ctrls["group_delay"], ctrls["noise_magnitude"], block, sr,
            noise_in=noise, seed=0 if noise is not None else _host_seed(), utterance_offset=utterance_offset,
            infer=infer, signal_out=signal_out)
        return signal, hidden, (harmonic, noise_out)


class CombSub(_SynthBase):
    """Combtooth subtractive synthesiser (old version) -- reference ddsp/vocoder.py:788-862."""

    def __init__(self, sampling_rate, block_size, n_mag_allpass, n_mag_harmonic, n_mag_noise, n_unit=256, n_spk=1,
                 unit2ctrl=None):
        super().__init__()
        _check_shape("CombSub", int(block_size) % 256 == 0 and 0 < int(block_size) <= 2048, "block_size %s must be a "
                     "multiple of 256 up to 2048" % (block_size,))
        _check_shape("CombSub", min(int(n_mag_allpass), int(n_mag_harmonic), int(n_mag_noise)) >= 2 and
                     max(int(n_mag_allpass), int(n_mag_harmonic), int(n_mag_noise)) <= 1025, "2 <= n_mag <= 1025")
        self.register_buffer("sampling_rate", torch.tensor(sampling_rate))
        self.register_buffer("block_size", torch.tensor(block_size))
        split_map = {
            "group_delay": n_mag_allpass,
            "harmonic_magnitude": n_mag_harmonic,
            "noise_magnitude": n_mag_noise,
        }
        self.unit2ctrl = unit2ctrl if unit2ctrl is not None else _reference_unit2ctrl(n_unit, n_spk, split_map)

    def forward(self, units_frames, f0_frames, volume_frames, spk_id=None, spk_mix_dict=None, initial_phase=None,
                infer=True, noise=None, utterance_offset=0, signal_out=None, **kwargs):
        """units_frames B x n_frames x n_unit; f0_frames B x n_frames x 1; volume_frames B x n_frames x 1.
        ``signal_out``: optional preallocated [B, T] destination of ``signal`` (may be peer-mapped memory).

        Trainable in the training phase: with ``infer=False`` (what the reference's solver.py calls) and a control
        from ``unit2ctrl`` that requires grad (grad mode on), signal, harmonic and noise are differentiable with
        respect to the three controls (CUDA backward, ops.combsub_synth_backward) for block 512 and n_mag <= 513.
        f0 is data, as in the reference's train.py: an f0 that requires grad is refused."""
        sr, block = self._scalars()
        if torch.is_grad_enabled() and isinstance(f0_frames, torch.Tensor) and f0_frames.requires_grad:
            raise NotImplementedError("CombSub has no gradient with respect to f0_frames; pass f0 as data "
                                      "(f0_frames.detach()), as the reference's train.py does")
        frame_phase, phase_frames = ops.phase_scan(f0_frames, block, sr, initial_phase, infer)
        ctrls, hidden = self.unit2ctrl(units_frames, f0_frames, phase_frames, volume_frames, spk_id=spk_id,
                                       spk_mix_dict=spk_mix_dict)
        signal, harmonic, noise_out = ops.combsub_synth(
            f0_frames, frame_phase, ctrls["group_delay"], ctrls["harmonic_magnitude"], ctrls["noise_magnitude"],
            block, sr, noise_in=noise, seed=0 if noise is not None else _host_seed(),
            utterance_offset=utterance_offset, infer=infer, signal_out=signal_out)
        return signal, hidden, (harmonic, noise_out)


class CombSubSuperFast(_SynthBase):
    """Combtooth subtractive synthesiser (STFT-domain filtering; what configs/combsub.yaml
    selects) -- reference ddsp/vocoder.py:613-710.  Returns (signal, hidden, (signal, signal))
    with the same tensor three times, like the reference."""

    def __init__(self, sampling_rate, block_size, win_length, n_unit=256, n_spk=1, use_pitch_aug=False,
                 pcmer_norm=False, unit2ctrl=None):
        super().__init__()
        _check_shape("CombSubSuperFast", int(block_size) == 512 and int(win_length) == 2048,
                     "only block_size 512 / win_length 2048 (configs/combsub.yaml) is built, got %s / %s" % (block_size, win_length))
        self.register_buffer("sampling_rate", torch.tensor(sampling_rate))
        self.register_buffer("block_size", torch.tensor(block_size))
        self.register_buffer("win_length", torch.tensor(win_length))
        self.register_buffer("window", torch.hann_window(win_length))
        split_map = {
            "harmonic_magnitude": win_length // 2 + 1,
            "harmonic_phase": win_length // 2 + 1,
            "noise_magnitude": win_length // 2 + 1,
            "noise_phase": win_length // 2 + 1,
        }
        self.unit2ctrl = unit2ctrl if unit2ctrl is not None else _reference_unit2ctrl(
            n_unit, n_spk, split_map, use_pitch_aug=use_pitch_aug, use_naive_v2=True, use_conv_stack=True)

    def _scalars(self):
        c = self.__dict__.get("_scalar_cache")
        if c is None:
            c = (int(self.sampling_rate.item()), int(self.block_size.item()), int(self.win_length.item()))
            self.__dict__["_scalar_cache"] = c
        return c

    def forward(self, units_frames, f0_frames, volume_frames, spk_id=None, spk_mix_dict=None, aug_shift=None,
                initial_phase=None, infer=True, noise=None, utterance_offset=0, signal_out=None, **kwargs):
        """``initial_phase`` is accepted and ignored, like the reference (ddsp/vocoder.py:653-661).

        Trainable: when a control from ``unit2ctrl`` requires grad (and grad mode is on), ``signal`` is
        differentiable with respect to the four controls (CUDA backward, ops.superfast_synth_backward).
        f0 is data (reference train.py), so an f0 that requires grad is refused."""
        sr, block, win = self._scalars()
        if torch.is_grad_enabled() and isinstance(f0_frames, torch.Tensor) and f0_frames.requires_grad:
            raise NotImplementedError("CombSubSuperFast has no gradient with respect to f0_frames; pass f0 as data "
                                      "(f0_frames.detach()), as the reference's train.py does")
        ws, phase_frames = ops.superfast_scan(f0_frames, block, sr)
        ctrls, hidden = self.unit2ctrl(units_frames, f0_frames, phase_frames, volume_frames, spk_id=spk_id,
                                       spk_mix_dict=spk_mix_dict, aug_shift=aug_shift)
        if signal_out is not None and torch.is_grad_enabled() and any(v.requires_grad for v in ctrls.values()):
            raise ValueError("signal_out cannot be combined with controls that require grad; call under "
                             "torch.no_grad() or drop signal_out")
        signal = ops.superfast_synth(ws, ctrls["harmonic_magnitude"], ctrls["harmonic_phase"],
                                     ctrls["noise_magnitude"], ctrls["noise_phase"], block, win, noise_in=noise,
                                     seed=0 if noise is not None else _host_seed(),
                                     utterance_offset=utterance_offset, signal_out=signal_out)
        return signal, hidden, (signal, signal)


class CombSubFast(_SynthBase):
    """Combtooth subtractive synthesiser with 2*block sqrt-Hann frames (the variant the diffusion / reflow vocoders
    embed) -- reference ddsp/vocoder.py:712-786.  Returns (signal, hidden, (signal, signal)) like the reference.

    Parity: checked against the live-reference goldens (tests/test_gpu_combsubfast.py)."""

    def __init__(self, sampling_rate, block_size, n_unit=256, n_spk=1, use_pitch_aug=False, pcmer_norm=False,
                 unit2ctrl=None):
        super().__init__()
        _check_shape("CombSubFast", int(block_size) == 512, "only block_size 512 is built, got %s" % (block_size,))
        self.register_buffer("sampling_rate", torch.tensor(sampling_rate))
        self.register_buffer("block_size", torch.tensor(block_size))
        self.register_buffer("window", torch.sqrt(torch.hann_window(2 * block_size)))
        split_map = {
            "harmonic_magnitude": block_size + 1,
            "harmonic_phase": block_size + 1,
            "noise_magnitude": block_size + 1,
        }
        self.unit2ctrl = unit2ctrl if unit2ctrl is not None else _reference_unit2ctrl(
            n_unit, n_spk, split_map, use_pitch_aug=use_pitch_aug, pcmer_norm=pcmer_norm)

    def forward(self, units_frames, f0_frames, volume_frames, spk_id=None, spk_mix_dict=None, aug_shift=None,
                initial_phase=None, infer=True, noise=None, utterance_offset=0, **kwargs):
        """Trainable in the training phase: with ``infer=False`` (what the reference's diffusion/solver_new.py
        passes through vocoder.Unit2Wav) and a control from ``unit2ctrl`` that requires grad (grad mode on),
        ``signal`` is differentiable with respect to the three controls (CUDA backward,
        ops.combsubfast_filter_backward).  Under grad, ``infer=True`` is refused.  f0 is data, as in the
        reference's training loop: an f0 that requires grad is refused."""
        sr, block = self._scalars()
        if torch.is_grad_enabled() and isinstance(f0_frames, torch.Tensor) and f0_frames.requires_grad:
            raise NotImplementedError("CombSubFast has no gradient with respect to f0_frames; pass f0 as data "
                                      "(f0_frames.detach()), as the reference's training loop does")
        frame_phase, phase_frames = ops.phase_scan(f0_frames, block, sr, initial_phase, infer)
        ctrls, hidden = self.unit2ctrl(units_frames, f0_frames, phase_frames, volume_frames, spk_id=spk_id,
                                       spk_mix_dict=spk_mix_dict, aug_shift=aug_shift)
        if infer and torch.is_grad_enabled() and any(v.requires_grad for v in ctrls.values()):
            raise NotImplementedError(
                "CombSubFast is differentiable in the training phase only: call it with infer=False (what the "
                "reference's diffusion/solver_new.py does), or under torch.no_grad() for inference")
        comb = ops.comb_source(f0_frames, frame_phase, block, sr, infer)
        signal = ops.combsubfast_filter(comb, ctrls["harmonic_magnitude"], ctrls["harmonic_phase"],
                                        ctrls["noise_magnitude"], block, noise_in=noise,
                                        seed=0 if noise is not None else _host_seed(),
                                        utterance_offset=utterance_offset)
        return signal, hidden, (signal, signal)


class FixedControls(torch.nn.Module):
    """Stand-in for Unit2Control that returns preset raw controls: isolates the DSP path (the
    seam the parity tests and the benchmark use; reference ddsp/vocoder.py:578)."""

    def __init__(self, ctrls=None, hidden=None):
        super().__init__()
        self.ctrls, self.hidden = ctrls, hidden

    def forward(self, units, f0, phase, volume, **kw):
        self.last_phase_frames = phase
        return self.ctrls, self.hidden

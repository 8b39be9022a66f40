"""Thin tensor-level wrappers over the C ABI: PyTorch CUDA tensors in, PyTorch CUDA tensors out.

PyTorch is only the plumbing here (device memory from its caching allocator, the current
stream); all arithmetic happens in libb200ddsp.so.  Every function requires CUDA fp32 inputs
and raises otherwise -- there is no CPU path.
"""
import threading

import torch

from . import _lib

IR_ALLPASS, IR_MAG_HANN, IR_MAG_DYNAMIC = 0, 1, 2

# kernel launches issued through this module (bench.py reports it as gpu_launches)
_launches = 0
_tables = {}
_overlap_mode = 1   # mirrors the library's default (b2d_set_overlap)
_sins_impl = "auto"
_fir_impl = "auto"
_tables_lock = threading.Lock()


def set_fir_impl(impl):
    """'auto' (FFT-domain kernel for block size 512 and <= 1024 taps, else CUDA cores), 'cuda' (CUDA-core direct
    form), 'tc' (wgmma 3xTF32 kernel, block size 512), 'cuda8' (older scalar CUDA-core kernel) or 'fft'."""
    global _fir_impl
    _lib.check(_lib.lib().b2d_set_fir_impl({"auto": 0, "cuda": 1, "tc": 2, "cuda8": 3, "fft": 4}[impl]), "b2d_set_fir_impl")
    _fir_impl = impl


def set_ir_impl(impl):
    """'auto' (wgmma when supported), 'cuda' (CUDA-core kernel) or 'tc' (wgmma 3xTF32 kernel)."""
    _lib.check(_lib.lib().b2d_set_ir_impl({"auto": 0, "cuda": 1, "tc": 2}[impl]), "b2d_set_ir_impl")


def launches():
    return _launches


def _count(n):
    global _launches
    _launches += n


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _need_cuda_f32(name, t, dtype=torch.float32, local=True):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise ValueError("%s must be a CUDA tensor (the kernels have no CPU fallback)" % name)
    if t.dtype != dtype:
        raise ValueError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if local and t.device.index != torch.cuda.current_device():
        # the library launches on the calling thread's current device and on torch's current stream of it
        raise ValueError("%s lives on %s but the current CUDA device is %d; call torch.cuda.set_device(%d) "
                         "(one process per GPU) or wrap the call in torch.cuda.device(...)"
                         % (name, t.device, torch.cuda.current_device(), t.device.index))


def _need_frame_phase(frame_phase, B, nF):
    _need_cuda_f32("frame_phase", frame_phase, torch.float64)
    if tuple(frame_phase.shape) != (B, nF) or not frame_phase.is_contiguous():
        raise ValueError("frame_phase must be a contiguous [%d, %d] tensor (phase_scan of the same f0), got %s"
                         % (B, nF, tuple(frame_phase.shape)))


def _noise_rows(noise_in, B, T):
    """explicit noise samples for B utterances of T samples -> contiguous [B, T]"""
    _need_cuda_f32("noise_in", noise_in)
    if noise_in.numel() != B * T:
        raise ValueError("noise must hold B*T = %d*%d samples, got %s" % (B, T, tuple(noise_in.shape)))
    return noise_in.reshape(B, T).contiguous()


def _frames_2d(f0_frames):
    """[B, nF, 1] or [B, nF] -> contiguous [B, nF]."""
    _need_cuda_f32("f0_frames", f0_frames)
    f0 = f0_frames.squeeze(-1) if f0_frames.dim() == 3 else f0_frames
    if f0.dim() != 2:
        raise ValueError("f0_frames must be [B, n_frames, 1] or [B, n_frames]")
    return f0.contiguous()


def _ctrl_view(name, c, B, nF):
    """A raw control tensor [B, nF, C] that is a strided view of the dense Unit2Control output
    (torch.split, reference ddsp/unit2control.py:22): returns (tensor, frame stride)."""
    _need_cuda_f32(name, c)
    if c.dim() != 3 or c.shape[0] != B or c.shape[1] != nF:
        raise ValueError("Batch/frame size of %s %s does not match f0 (%d, %d)" % (name, tuple(c.shape), B, nF))
    if c.stride(2) != 1 or (B > 1 and c.stride(0) != nF * c.stride(1)) or c.stride(1) < c.shape[2]:
        c = c.contiguous()
    return c, c.stride(1)


def _same_stride(named, B, nF):
    """Views of one dense control tensor share a frame stride; otherwise densify."""
    views = [_ctrl_view(n, c, B, nF) for n, c in named]
    if len({s for _, s in views}) == 1:
        return [c for c, _ in views], views[0][1]
    dense = torch.cat([c.contiguous() for c, _ in views], dim=-1)
    parts = torch.split(dense, [c.shape[2] for c, _ in views], dim=-1)
    return list(parts), dense.stride(1)


def _signal_dest(signal_out, B, T, device):
    """where a synthesizer writes its [B, T] mixed signal: a new tensor, or the caller's ``signal_out``"""
    if signal_out is None:
        return torch.empty(B, T, dtype=torch.float32, device=device)
    _need_cuda_f32("signal_out", signal_out, local=False)        # may be peer-mapped memory of another GPU
    if tuple(signal_out.shape) != (B, T) or not signal_out.is_contiguous():
        raise ValueError("signal_out must be a contiguous [B, T] tensor")
    return signal_out


def _cotangent(name, g, B, T):
    """a cotangent of a [B, T] output, checked -> contiguous"""
    _need_cuda_f32(name, g)
    if tuple(g.shape) != (B, T):
        raise ValueError("%s must be [B, n_frames*block] = [%d, %d], got %s" % (name, B, T, tuple(g.shape)))
    return g.contiguous()


def _output_cotangents(grad_signal, grad_harmonic, grad_noise, B, T):
    """checked cotangents of (signal, harmonic, noise), None = zero"""
    named = (("grad_signal", grad_signal), ("grad_harmonic", grad_harmonic), ("grad_noise", grad_noise))
    return [None if g is None else _cotangent(name, g, B, T) for name, g in named]


def _grad_gate(synth, unsupported, f0_frames, ctrls, block, infer, signal_out):
    """True when a synthesizer call must be differentiable (a control requires grad and grad mode is on); raises
    when its backward does not cover the call.  ``unsupported``: the synthesizer's *_grad_unsupported, called with the
    block size and the controls' widths."""
    if not (torch.is_grad_enabled() and any(isinstance(c, torch.Tensor) and c.requires_grad for c in ctrls)):
        return False
    if infer:
        raise NotImplementedError("the %s backward covers the training phase only: call with infer=False (what the "
                                  "reference's solver.py does), or under torch.no_grad() for inference" % synth)
    if signal_out is not None:
        raise ValueError("signal_out cannot be used when the controls require grad (it may be peer-mapped memory "
                         "that autograd does not own)")
    if isinstance(f0_frames, torch.Tensor) and f0_frames.requires_grad:
        raise NotImplementedError("%s has no gradient with respect to f0_frames; pass f0 as data" % synth)
    why = unsupported(block, *(c.shape[-1] for c in ctrls))
    if why is not None:
        raise NotImplementedError("the %s backward does not cover %s" % (synth, why))
    return True


def dft_tables(n_mag, device):
    """Constant cos/sin matrices of the 2(n_mag-1)-point inverse real DFT, cached per device."""
    key = (int(n_mag), torch.device(device).index)
    with _tables_lock:
        t = _tables.get(key)
        if t is None:
            L = _lib.lib()
            nbytes = L.b2d_dft_tables_bytes(int(n_mag))
            if nbytes == 0:
                raise ValueError("n_mag=%d out of range" % n_mag)
            t = torch.empty(nbytes // 4, dtype=torch.float32, device=device)
            _lib.check(L.b2d_dft_tables(int(n_mag), t.data_ptr(), _stream()), "b2d_dft_tables")
            _count(2)
            # built once per device and then read from whatever stream the caller is on: make it visible to all of them
            torch.cuda.current_stream().synchronize()
            _tables[key] = t
    return t


def phase_scan(f0_frames, block, sampling_rate, initial_phase=None, infer=True):
    """-> (frame_phase fp64 [B, nF] unwrapped cycles, phase_frames fp32 [B, nF, 1] radians)."""
    f0 = _frames_2d(f0_frames)
    B, nF = f0.shape
    ip = None
    if initial_phase is not None:
        ip = initial_phase.to(device=f0.device, dtype=torch.float32).reshape(-1).contiguous()
        if ip.numel() == 1 and B > 1:
            ip = ip.expand(B).contiguous()
        if ip.numel() != B:
            raise ValueError("initial_phase must have one value per utterance")
    frame_phase = torch.empty(B, nF, dtype=torch.float64, device=f0.device)
    phase_frames = torch.empty(B, nF, 1, dtype=torch.float32, device=f0.device)
    rc = _lib.lib().b2d_phase_scan(f0.data_ptr(), _ptr(ip), B, nF, int(block), float(sampling_rate),
                                   0 if infer else 1, frame_phase.data_ptr(), phase_frames.data_ptr(), _stream())
    _lib.check(rc, "b2d_phase_scan")
    _count(1)
    return frame_phase, phase_frames


def sins_bank(f0_frames, frame_phase, c_amp, block, sampling_rate, infer=True):
    f0 = _frames_2d(f0_frames)
    B, nF = f0.shape
    _need_frame_phase(frame_phase, B, nF)
    c, stride = _ctrl_view("amplitudes", c_amp, B, nF)
    out = torch.empty(B, nF * block, dtype=torch.float32, device=f0.device)
    rc = _lib.lib().b2d_sins_bank(f0.data_ptr(), frame_phase.data_ptr(), c.data_ptr(), stride, B, nF, int(block),
                                  c.shape[2], float(sampling_rate), 0 if infer else 1, out.data_ptr(), _stream())
    _lib.check(rc, "b2d_sins_bank")
    _count(1)
    return out


def ir_build(c_raw, mode, sampling_rate, f0_frames=None):
    """raw control [B, nF, M] -> impulse responses [B, nF, 2(M-1)]."""
    _need_cuda_f32("control", c_raw)
    B, nF, M = c_raw.shape
    c, stride = _ctrl_view("control", c_raw, B, nF)
    f0 = _frames_2d(f0_frames) if f0_frames is not None else None
    ir = torch.empty(B, nF, 2 * (M - 1), dtype=torch.float32, device=c.device)
    tab = dft_tables(M, c.device)
    rc = _lib.lib().b2d_ir_build(c.data_ptr(), stride, int(mode), _ptr(f0), tab.data_ptr(), B, nF, M,
                                 float(sampling_rate), ir.data_ptr(), _stream())
    _lib.check(rc, "b2d_ir_build")
    _count(1)
    return ir


def ltv_fir(x, ir, block, seed=0, utterance_offset=0, generic=False):
    """Time-varying FIR of x [B, T] (or None = in-kernel uniform noise) with ir [B, nF, L]."""
    _need_cuda_f32("ir", ir)
    ir = ir.contiguous()
    B, nF, L = ir.shape
    if x is not None:
        _need_cuda_f32("x", x)
        if x.shape[0] != B:
            raise ValueError("Batch size of audio ({}) and impulse response ({}) must be the same."
                             .format(x.shape[0], B))
        if x.dim() != 2 or x.shape[1] != nF * int(block):
            raise ValueError("audio must be [B, n_frames*block] = [%d, %d], got %s (the reference derives the hop "
                             "from the lengths, ddsp/core.py:156; here block is explicit)" % (B, nF * int(block), tuple(x.shape)))
        x = x.contiguous()
    y = torch.empty(B, nF * block, dtype=torch.float32, device=ir.device)
    Lh = _lib.lib()
    if generic:
        rc = Lh.b2d_ltv_fir_generic(_ptr(x), ir.data_ptr(), L, y.data_ptr(), B, nF, int(block), _stream())
    else:
        rc = Lh.b2d_ltv_fir(_ptr(x), ir.data_ptr(), L, y.data_ptr(), 0, 0, 0, 0, 0, int(seed),
                            int(utterance_offset), B, nF, int(block), _stream())
    _lib.check(rc, "b2d_ltv_fir")
    _count(1)
    return y


SINS_GRAD_MAX_MAG, SINS_GRAD_MAX_HARMONICS = 257, 512


def sins_grad_unsupported(block, n_harmonics, n_mag_allpass, n_mag_noise):
    """None if sins_synth_backward covers the shape, else why not."""
    if int(block) != 512:
        return "block size %d (the backward is built for 512)" % block
    if max(n_mag_allpass, n_mag_noise) > SINS_GRAD_MAX_MAG:
        return "n_mag %d / %d (the backward is built for <= %d)" % (n_mag_allpass, n_mag_noise, SINS_GRAD_MAX_MAG)
    if n_harmonics > SINS_GRAD_MAX_HARMONICS:
        return "%d harmonics (the backward is built for <= %d)" % (n_harmonics, SINS_GRAD_MAX_HARMONICS)
    return None


def sins_synth(f0_frames, frame_phase, c_amp, c_group_delay, c_noise, block, sampling_rate, noise_in=None,
               seed=0, utterance_offset=0, infer=True, want_parts=True, signal_out=None):
    """Whole Sins DSP after Unit2Control -> (signal, harmonic, noise) [B, T] each.
    ``signal_out``: optional preallocated [B, T] fp32 CUDA tensor for the mixed signal; it may live in
    another GPU's memory (peer-mapped, see sharding.PeerGather): the FIR kernel then writes the
    waveform straight over NVLink.

    Differentiable with respect to the three controls when one of them requires grad (and grad mode is on), in the
    training phase (``infer=False``, frame_phase from phase_scan(..., infer=False)): the backward runs
    sins_synth_backward with the forward's workspace, noise and seed.  All three outputs are differentiable."""
    if _grad_gate("Sins", sins_grad_unsupported, f0_frames, (c_amp, c_group_delay, c_noise), block, infer, signal_out):
        if noise_in is not None:
            noise_in = noise_in.detach()
        return _SinsSynth.apply(f0_frames.detach(), frame_phase, int(block), float(sampling_rate), noise_in, int(seed),
                                int(utterance_offset), c_amp, c_group_delay, c_noise)
    return _sins_synth(f0_frames, frame_phase, c_amp, c_group_delay, c_noise, block, sampling_rate, noise_in, seed,
                       utterance_offset, infer, want_parts, signal_out)[:3]


def _sins_args(f0_frames, frame_phase, c_amp, c_group_delay, c_noise, block, noise_in):
    """checked (f0 [B, nF], controls sharing one frame stride, the stride, noise rows) of a Sins call"""
    f0 = _frames_2d(f0_frames)
    B, nF = f0.shape
    _need_frame_phase(frame_phase, B, nF)
    (ca, cg, cn), stride = _same_stride([("amplitudes", c_amp), ("group_delay", c_group_delay),
                                         ("noise_magnitude", c_noise)], B, nF)
    if noise_in is not None:
        noise_in = _noise_rows(noise_in, B, nF * int(block))
    return f0, ca, cg, cn, stride, noise_in


def sins_synth_backward(f0_frames, frame_phase, c_amp, c_group_delay, c_noise, ws, grad_signal, block, sampling_rate,
                        grad_harmonic=None, grad_noise=None, noise_in=None, seed=0, utterance_offset=0,
                        ws_has_sinusoids=True):
    """Gradient of sins_synth (infer=False) with respect to the three raw controls, for the cotangents of signal,
    harmonic and noise [B, T] (None = zero).  f0 / frame_phase / controls / noise_in / seed / utterance_offset must be
    those of the forward call and ``ws`` the workspace it filled (its impulse responses, and its sinusoids unless
    ``ws_has_sinusoids`` is False: the 'fused' variant does not store them and the bank is rerun).
    -> dense [B, nF, H + Ma + Mn]: amplitudes | group_delay | noise_magnitude (the split_to_dict layout)."""
    f0, ca, cg, cn, stride, noise_in = _sins_args(f0_frames, frame_phase, c_amp, c_group_delay, c_noise, block, noise_in)
    B, nF = f0.shape
    H, Ma, Mn = ca.shape[2], cg.shape[2], cn.shape[2]
    T = nF * int(block)
    L = _lib.lib()
    if not isinstance(ws, torch.Tensor) or not ws.is_cuda or ws.dtype != torch.uint8 or \
            ws.numel() < L.b2d_sins_workspace_bytes(B, nF, int(block), Ma, Mn):
        raise ValueError("ws must be the workspace sins_synth filled for the same shapes")
    cots = _output_cotangents(grad_signal, grad_harmonic, grad_noise, B, T)
    grad = torch.empty(B, nF, H + Ma + Mn, dtype=torch.float32, device=f0.device)
    bws_bytes = L.b2d_sins_synth_backward_workspace_bytes(B, nF, int(block))
    bws = torch.empty(bws_bytes, dtype=torch.uint8, device=f0.device)
    rc = L.b2d_sins_synth_backward(f0.data_ptr(), frame_phase.data_ptr(), ca.data_ptr(), cg.data_ptr(), cn.data_ptr(),
                                   stride, _ptr(noise_in), int(seed), int(utterance_offset), ws.data_ptr(),
                                   1 if ws_has_sinusoids else 0, _ptr(cots[0]), _ptr(cots[1]), _ptr(cots[2]), B, nF,
                                   int(block), H, Ma, Mn, float(sampling_rate), grad.data_ptr(), bws.data_ptr(),
                                   bws_bytes, _stream())
    _lib.check(rc, "b2d_sins_synth_backward")
    _count(2 if ws_has_sinusoids else 3)
    return grad


class _SinsSynth(torch.autograd.Function):
    """sins_synth (infer=False) with a CUDA backward.  Saves the forward's workspace (sinusoids | impulse responses),
    f0, frame_phase, the control views and the noise input; the backward regenerates the in-kernel noise from seed."""

    @staticmethod
    def forward(ctx, f0, frame_phase, block, sampling_rate, noise_in, seed, utterance_offset, c_amp, c_gd, c_nm):
        signal, harmonic, noise, ws = _sins_synth(f0, frame_phase, c_amp, c_gd, c_nm, block, sampling_rate, noise_in,
                                                  seed, utterance_offset, False, True, None)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(ws, f0, frame_phase, noise_in, c_amp, c_gd, c_nm)
        # the 'fused' variant evaluates the bank inside its FIR kernel and leaves the sinusoid slot unwritten
        ctx.cfg = (block, sampling_rate, seed, utterance_offset, _sins_impl != "fused")
        return signal, harmonic, noise

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_signal, grad_harmonic, grad_noise):
        ws, f0, frame_phase, noise_in, c_amp, c_gd, c_nm = ctx.saved_tensors
        block, sampling_rate, seed, utterance_offset, has_sinusoids = ctx.cfg
        grad = sins_synth_backward(f0, frame_phase, c_amp, c_gd, c_nm, ws, grad_signal, block, sampling_rate,
                                   grad_harmonic=grad_harmonic, grad_noise=grad_noise, noise_in=noise_in, seed=seed,
                                   utterance_offset=utterance_offset, ws_has_sinusoids=has_sinusoids)
        parts = torch.split(grad, [c_amp.shape[-1], c_gd.shape[-1], c_nm.shape[-1]], dim=-1)
        return (None,) * 7 + tuple(parts)


def _sins_synth(f0_frames, frame_phase, c_amp, c_group_delay, c_noise, block, sampling_rate, noise_in=None,
                seed=0, utterance_offset=0, infer=True, want_parts=True, signal_out=None):
    """-> (signal, harmonic, noise, workspace)"""
    f0, ca, cg, cn, s0, noise_in = _sins_args(f0_frames, frame_phase, c_amp, c_group_delay, c_noise, block, noise_in)
    B, nF = f0.shape
    H, Ma, Mn = ca.shape[2], cg.shape[2], cn.shape[2]
    dev = f0.device
    T = nF * block
    L = _lib.lib()
    ws_bytes = L.b2d_sins_workspace_bytes(B, nF, int(block), Ma, Mn)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    signal = _signal_dest(signal_out, B, T, dev)
    harmonic = torch.empty(B, T, dtype=torch.float32, device=dev) if want_parts else None
    noise = torch.empty(B, T, dtype=torch.float32, device=dev) if (want_parts or Ma != Mn) else None
    ta, tn = dft_tables(Ma, dev), dft_tables(Mn, dev)
    rc = L.b2d_sins_synth(f0.data_ptr(), frame_phase.data_ptr(), ca.data_ptr(), cg.data_ptr(), cn.data_ptr(), s0,
                          _ptr(noise_in), int(seed), int(utterance_offset), ta.data_ptr(), tn.data_ptr(), B, nF,
                          int(block), H, Ma, Mn, float(sampling_rate), 0 if infer else 1, signal.data_ptr(),
                          _ptr(harmonic), _ptr(noise), ws.data_ptr(), ws_bytes, _stream())
    _lib.check(rc, "b2d_sins_synth")
    fft_ok = int(block) == 512 and max(Ma, Mn) <= 257 and _fir_impl in ("auto", "fft")
    fused = _sins_impl == "fused" and Ma == Mn and fft_ok and H <= 128
    spectrum = _sins_impl == "spectrum" and fft_ok
    nsplit = max(1, min(abs(_overlap_mode), B)) if abs(_overlap_mode) >= 2 else 1
    _count(3 if fused else 5 if spectrum else 2 + nsplit * (2 if Ma == Mn else 3))
    return signal, harmonic, noise, ws


def sinegen(f0, upp, sampling_rate, dim, rand_ini, sine_amp=0.1, noise_std=0.003, voiced_threshold=0.0,
            noise_in=None, seed=0, utterance_offset=0):
    """f0 [B, nF] -> [B, nF*upp, dim]  (reference nsf_hifigan/models.py:150-165)."""
    _need_cuda_f32("f0", f0)
    if f0.dim() != 2:
        raise ValueError("f0 must be [B, n_frames]")
    f0 = f0.contiguous()
    B, nF = f0.shape
    rand_ini = rand_ini.to(device=f0.device, dtype=torch.float32).reshape(-1).contiguous()
    if rand_ini.numel() != dim:
        raise ValueError("rand_ini must have %d elements" % dim)
    if noise_in is not None:
        _need_cuda_f32("noise_in", noise_in)
        if tuple(noise_in.shape) != (B, nF * upp, dim):
            raise ValueError("noise_in must be [B, n_frames*upp, dim]")
        noise_in = noise_in.contiguous()
    out = torch.empty(B, nF * upp, dim, dtype=torch.float32, device=f0.device)
    ws = torch.empty(B, nF, dtype=torch.float32, device=f0.device)
    rc = _lib.lib().b2d_sinegen(f0.data_ptr(), rand_ini.data_ptr(), _ptr(noise_in), int(seed), int(utterance_offset),
                                B, nF, int(upp), int(dim), float(sampling_rate), float(sine_amp), float(noise_std),
                                float(voiced_threshold), ws.data_ptr(), out.data_ptr(), _stream())
    _lib.check(rc, "b2d_sinegen")
    _count(2)
    return out


def comb_source(f0_frames, frame_phase, block, sampling_rate, infer=True):
    f0 = _frames_2d(f0_frames)
    B, nF = f0.shape
    _need_frame_phase(frame_phase, B, nF)
    out = torch.empty(B, nF * block, dtype=torch.float32, device=f0.device)
    rc = _lib.lib().b2d_comb_source(f0.data_ptr(), frame_phase.data_ptr(), B, nF, int(block), float(sampling_rate),
                                    0 if infer else 1, out.data_ptr(), _stream())
    _lib.check(rc, "b2d_comb_source")
    _count(1)
    return out


COMBSUB_GRAD_MAX_MAG = 513


def combsub_grad_unsupported(block, n_mag_allpass, n_mag_harmonic, n_mag_noise):
    """None if combsub_synth_backward covers the shape, else why not."""
    if int(block) != 512:
        return "block size %d (the backward is built for 512)" % block
    if max(n_mag_allpass, n_mag_harmonic, n_mag_noise) > COMBSUB_GRAD_MAX_MAG:
        return "n_mag %d / %d / %d (the backward is built for <= %d)" % (n_mag_allpass, n_mag_harmonic, n_mag_noise,
                                                                        COMBSUB_GRAD_MAX_MAG)
    return None


def combsub_synth(f0_frames, frame_phase, c_group_delay, c_harmonic, c_noise, block, sampling_rate, noise_in=None,
                  seed=0, utterance_offset=0, infer=True, signal_out=None):
    """Whole old-CombSub DSP after Unit2Control -> (signal, harmonic, noise) [B, T] each.

    Differentiable with respect to the three controls when one of them requires grad (and grad mode is on), in the
    training phase (``infer=False``, frame_phase from phase_scan(..., infer=False)): the backward runs
    combsub_synth_backward with the forward's workspace, noise and seed.  All three outputs are differentiable."""
    if _grad_gate("CombSub", combsub_grad_unsupported, f0_frames, (c_group_delay, c_harmonic, c_noise), block, infer,
                  signal_out):
        if noise_in is not None:
            noise_in = noise_in.detach()
        return _CombSubSynth.apply(f0_frames.detach(), frame_phase, int(block), float(sampling_rate), noise_in,
                                   int(seed), int(utterance_offset), c_group_delay, c_harmonic, c_noise)
    return _combsub_synth(f0_frames, frame_phase, c_group_delay, c_harmonic, c_noise, block, sampling_rate, noise_in,
                          seed, utterance_offset, infer, signal_out)[:3]


def _combsub_synth(f0_frames, frame_phase, c_group_delay, c_harmonic, c_noise, block, sampling_rate, noise_in=None,
                   seed=0, utterance_offset=0, infer=True, signal_out=None):
    """-> (signal, harmonic, noise, workspace)"""
    f0 = _frames_2d(f0_frames)
    B, nF = f0.shape
    _need_frame_phase(frame_phase, B, nF)
    (cg, ch, cn), stride = _same_stride([("group_delay", c_group_delay), ("harmonic_magnitude", c_harmonic),
                                         ("noise_magnitude", c_noise)], B, nF)
    Ma, Mh, Mn = cg.shape[2], ch.shape[2], cn.shape[2]
    dev, T = f0.device, nF * block
    if noise_in is not None:
        noise_in = _noise_rows(noise_in, B, T)
    L = _lib.lib()
    ws_bytes = L.b2d_combsub_workspace_bytes(B, nF, int(block), Ma, Mh, Mn)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    signal = _signal_dest(signal_out, B, T, dev)
    harmonic, noise = (torch.empty(B, T, dtype=torch.float32, device=dev) for _ in range(2))
    rc = L.b2d_combsub_synth(f0.data_ptr(), frame_phase.data_ptr(), cg.data_ptr(), ch.data_ptr(), cn.data_ptr(),
                             stride, _ptr(noise_in), int(seed), int(utterance_offset), dft_tables(Ma, dev).data_ptr(),
                             dft_tables(Mh, dev).data_ptr(), dft_tables(Mn, dev).data_ptr(), B, nF, int(block), Ma,
                             Mh, Mn, float(sampling_rate), 0 if infer else 1, signal.data_ptr(), harmonic.data_ptr(),
                             noise.data_ptr(), ws.data_ptr(), ws_bytes, _stream())
    _lib.check(rc, "b2d_combsub_synth")
    _count(6 if Ma == Mn else 7)
    return signal, harmonic, noise, ws


def combsub_synth_backward(f0_frames, c_group_delay, c_harmonic, c_noise, ws, grad_signal, block, sampling_rate,
                           grad_harmonic=None, grad_noise=None, noise_in=None, seed=0, utterance_offset=0):
    """Gradient of combsub_synth (infer=False) with respect to the three raw controls, for the cotangents of signal,
    harmonic and noise [B, T] (None = zero).  f0 / controls / noise_in / seed / utterance_offset must be those of the
    forward call and ``ws`` the workspace it filled (its comb, all-passed comb and impulse responses).
    -> dense [B, nF, Ma + Mh + Mn]: group_delay | harmonic_magnitude | noise_magnitude (the split_to_dict layout)."""
    f0 = _frames_2d(f0_frames)
    B, nF = f0.shape
    (cg, ch, cn), stride = _same_stride([("group_delay", c_group_delay), ("harmonic_magnitude", c_harmonic),
                                         ("noise_magnitude", c_noise)], B, nF)
    Ma, Mh, Mn = cg.shape[2], ch.shape[2], cn.shape[2]
    T = nF * int(block)
    if noise_in is not None:
        noise_in = _noise_rows(noise_in, B, T)
    L = _lib.lib()
    if not isinstance(ws, torch.Tensor) or not ws.is_cuda or ws.dtype != torch.uint8 or \
            ws.numel() < L.b2d_combsub_workspace_bytes(B, nF, int(block), Ma, Mh, Mn):
        raise ValueError("ws must be the workspace combsub_synth filled for the same shapes")
    cots = _output_cotangents(grad_signal, grad_harmonic, grad_noise, B, T)
    grad = torch.empty(B, nF, Ma + Mh + Mn, dtype=torch.float32, device=f0.device)
    bws_bytes = L.b2d_combsub_synth_backward_workspace_bytes(B, nF, int(block))
    bws = torch.empty(bws_bytes, dtype=torch.uint8, device=f0.device)
    rc = L.b2d_combsub_synth_backward(f0.data_ptr(), cg.data_ptr(), ch.data_ptr(), cn.data_ptr(), stride,
                                      _ptr(noise_in), int(seed), int(utterance_offset), ws.data_ptr(), _ptr(cots[0]),
                                      _ptr(cots[1]), _ptr(cots[2]), B, nF, int(block), Ma, Mh, Mn,
                                      float(sampling_rate), grad.data_ptr(), bws.data_ptr(), bws_bytes, _stream())
    _lib.check(rc, "b2d_combsub_synth_backward")
    _count(2)
    return grad


class _CombSubSynth(torch.autograd.Function):
    """combsub_synth (infer=False) with a CUDA backward.  Saves the forward's workspace (comb | all-passed comb | noise
    | impulse responses), f0, the control views and the noise input; the backward regenerates the in-kernel noise from
    seed."""

    @staticmethod
    def forward(ctx, f0, frame_phase, block, sampling_rate, noise_in, seed, utterance_offset, c_gd, c_hm, c_nm):
        signal, harmonic, noise, ws = _combsub_synth(f0, frame_phase, c_gd, c_hm, c_nm, block, sampling_rate, noise_in,
                                                     seed, utterance_offset, False, None)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(ws, f0, noise_in, c_gd, c_hm, c_nm)
        ctx.cfg = (block, sampling_rate, seed, utterance_offset)
        return signal, harmonic, noise

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_signal, grad_harmonic, grad_noise):
        ws, f0, noise_in, c_gd, c_hm, c_nm = ctx.saved_tensors
        block, sampling_rate, seed, utterance_offset = ctx.cfg
        grad = combsub_synth_backward(f0, c_gd, c_hm, c_nm, ws, grad_signal, block, sampling_rate,
                                      grad_harmonic=grad_harmonic, grad_noise=grad_noise, noise_in=noise_in, seed=seed,
                                      utterance_offset=utterance_offset)
        parts = torch.split(grad, [c_gd.shape[-1], c_hm.shape[-1], c_nm.shape[-1]], dim=-1)
        return (None,) * 7 + tuple(parts)


def superfast_scan(f0_frames, block, sampling_rate):
    """-> (workspace tensor holding per-frame source parameters, phase_frames [B, nF, 1])."""
    f0 = _frames_2d(f0_frames)
    B, nF = f0.shape
    L = _lib.lib()
    ws = torch.empty(L.b2d_superfast_workspace_bytes(B, nF), dtype=torch.uint8, device=f0.device)
    phase_frames = torch.empty(B, nF, 1, dtype=torch.float32, device=f0.device)
    rc = L.b2d_superfast_scan(f0.data_ptr(), B, nF, int(block), float(sampling_rate), ws.data_ptr(),
                              phase_frames.data_ptr(), _stream())
    _lib.check(rc, "b2d_superfast_scan")
    _count(1)
    return ws, phase_frames


def superfast_synth(ws, c_hm, c_hp, c_nm, c_np, block, win_length, noise_in=None, seed=0, utterance_offset=0,
                    signal_out=None):
    """CombSubSuperFast after the frame scan: raw controls [B, nF, win_length/2+1] -> signal [B, nF*block].
    Differentiable with respect to the four controls when one of them requires grad (and grad mode is on):
    the backward runs superfast_synth_backward with the same workspace, noise and seed."""
    if torch.is_grad_enabled() and any(isinstance(c, torch.Tensor) and c.requires_grad for c in (c_hm, c_hp, c_nm, c_np)):
        if signal_out is not None:
            raise ValueError("signal_out cannot be used when the controls require grad (it may be peer-mapped memory "
                             "that autograd does not own)")
        if noise_in is not None:
            noise_in = noise_in.detach()
        return _SuperFastSynth.apply(ws, int(block), int(win_length), noise_in, int(seed), int(utterance_offset),
                                     c_hm, c_hp, c_nm, c_np)
    return _superfast_synth(ws, c_hm, c_hp, c_nm, c_np, block, win_length, noise_in, seed, utterance_offset,
                            signal_out)


def _superfast_args(ws, c_hm, c_hp, c_nm, c_np, block, win_length, noise_in):
    """checked (ws, controls, frame stride, noise rows, B, nF) of a superfast call"""
    if c_hm.dim() != 3:
        raise ValueError("controls must be [B, n_frames, win_length/2+1]")
    B, nF = c_hm.shape[0], c_hm.shape[1]
    if not isinstance(ws, torch.Tensor) or not ws.is_cuda or ws.dtype != torch.uint8 or \
            ws.numel() < _lib.lib().b2d_superfast_workspace_bytes(B, nF):
        raise ValueError("ws must be the workspace superfast_scan returned for the same (B, n_frames) = (%d, %d)" % (B, nF))
    ctrls, stride = _same_stride([("harmonic_magnitude", c_hm), ("harmonic_phase", c_hp),
                                  ("noise_magnitude", c_nm), ("noise_phase", c_np)], B, nF)
    if ctrls[0].shape[2] != win_length // 2 + 1:
        raise ValueError("controls must have win_length/2+1 = %d bins" % (win_length // 2 + 1))
    if noise_in is not None:
        noise_in = _noise_rows(noise_in, B, nF * block)
    return ctrls, stride, noise_in, B, nF


def superfast_synth_backward(ws, c_hm, c_hp, c_nm, c_np, grad_signal, block, win_length, noise_in=None, seed=0,
                             utterance_offset=0):
    """Gradient of superfast_synth with respect to the four raw controls, for dL/dsignal ``grad_signal`` [B, T].
    ws / controls / noise_in / seed / utterance_offset must be those of the forward call (the kernel recomputes the
    source spectra and regenerates the in-kernel noise).  -> dense [B, nF, 4*(win_length/2+1)]: harmonic_magnitude |
    harmonic_phase | noise_magnitude | noise_phase along the last axis (the split_to_dict layout)."""
    (hm, hp, nm, npz), stride, noise_in, B, nF = _superfast_args(ws, c_hm, c_hp, c_nm, c_np, block, win_length, noise_in)
    grad_signal = _cotangent("grad_signal", grad_signal, B, nF * block)
    grad = torch.empty(B, nF, 4 * (win_length // 2 + 1), dtype=torch.float32, device=hm.device)
    rc = _lib.lib().b2d_superfast_synth_backward(ws.data_ptr(), hm.data_ptr(), hp.data_ptr(), nm.data_ptr(),
                                                 npz.data_ptr(), stride, _ptr(noise_in), int(seed), int(utterance_offset),
                                                 grad_signal.data_ptr(), B, nF, int(block), int(win_length),
                                                 grad.data_ptr(), _stream())
    _lib.check(rc, "b2d_superfast_synth_backward")
    _count(1)
    return grad


class _SuperFastSynth(torch.autograd.Function):
    """superfast_synth with a CUDA backward.  Saves the scan workspace, the control views and the noise input (no
    spectra): the backward kernel recomputes the source spectra and regenerates the in-kernel noise from seed."""

    @staticmethod
    def forward(ctx, ws, block, win_length, noise_in, seed, utterance_offset, c_hm, c_hp, c_nm, c_np):
        signal = _superfast_synth(ws, c_hm, c_hp, c_nm, c_np, block, win_length, noise_in, seed, utterance_offset)
        ctx.save_for_backward(ws, noise_in, c_hm, c_hp, c_nm, c_np)
        ctx.cfg = (block, win_length, seed, utterance_offset)
        return signal

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_signal):
        ws, noise_in, c_hm, c_hp, c_nm, c_np = ctx.saved_tensors
        block, win_length, seed, utterance_offset = ctx.cfg
        grad = superfast_synth_backward(ws, c_hm, c_hp, c_nm, c_np, grad_signal, block, win_length, noise_in=noise_in,
                                        seed=seed, utterance_offset=utterance_offset)
        return (None,) * 6 + tuple(torch.split(grad, win_length // 2 + 1, dim=-1))


def _superfast_synth(ws, c_hm, c_hp, c_nm, c_np, block, win_length, noise_in=None, seed=0, utterance_offset=0,
                     signal_out=None):
    (hm, hp, nm, npz), stride, noise_in, B, nF = _superfast_args(ws, c_hm, c_hp, c_nm, c_np, block, win_length, noise_in)
    signal = _signal_dest(signal_out, B, nF * block, hm.device)
    rc = _lib.lib().b2d_superfast_synth(ws.data_ptr(), hm.data_ptr(), hp.data_ptr(), nm.data_ptr(), npz.data_ptr(),
                                        stride, _ptr(noise_in), int(seed), int(utterance_offset), B, nF, int(block),
                                        int(win_length), signal.data_ptr(), _stream())
    _lib.check(rc, "b2d_superfast_synth")
    _count(1)
    return signal


def source_module(f0, upp, sampling_rate, dim, rand_ini, linear_weight, linear_bias, sine_amp=0.1, noise_std=0.003,
                  voiced_threshold=0.0, noise_in=None, seed=0, utterance_offset=0):
    """SineGen + tanh(Linear(dim -> 1)) fused: f0 [B, nF] -> [B, nF*upp, 1]  (nsf_hifigan/models.py:201-204)."""
    _need_cuda_f32("f0", f0)
    f0 = f0.contiguous()
    B, nF = f0.shape
    rand_ini = rand_ini.to(device=f0.device, dtype=torch.float32).reshape(-1).contiguous()
    w = linear_weight.detach().to(device=f0.device, dtype=torch.float32).reshape(-1).contiguous()
    if rand_ini.numel() != dim or w.numel() != dim:
        raise ValueError("rand_ini and linear_weight must have %d elements" % dim)
    if noise_in is not None:
        _need_cuda_f32("noise_in", noise_in)
        if tuple(noise_in.shape) != (B, nF * upp, dim):
            raise ValueError("noise_in must be [B, n_frames*upp, dim]")
        noise_in = noise_in.contiguous()
    out = torch.empty(B, nF * upp, 1, dtype=torch.float32, device=f0.device)
    ws = torch.empty(B, nF, dtype=torch.float32, device=f0.device)
    rc = _lib.lib().b2d_source_module(f0.data_ptr(), rand_ini.data_ptr(), _ptr(noise_in), int(seed), int(utterance_offset),
                                      B, nF, int(upp), int(dim), float(sampling_rate), float(sine_amp), float(noise_std),
                                      float(voiced_threshold), w.data_ptr(), float(linear_bias), ws.data_ptr(),
                                      out.data_ptr(), _stream())
    _lib.check(rc, "b2d_source_module")
    _count(2)
    return out


def set_sinegen_impl(name):
    """'auto' | 'v1' (one sample per thread) | 'v2' (four per thread) | 'v2p' (four per thread, register pairs) | 'v2r7' (v2
    with Philox4x32-7 instead of -10 for the in-kernel noise)."""
    impl = {"auto": 0, "v1": 1, "v2": 2, "v2p": 3, "v2r7": 4}[name]
    _lib.check(_lib.lib().b2d_set_sinegen_impl(impl), "b2d_set_sinegen_impl")


def combsubfast_filter(comb, c_hm, c_hp, c_nm, block, noise_in=None, seed=0, utterance_offset=0):
    """CombSubFast after the source: comb [B, T] + raw controls [B, nF, block+1] -> signal [B, T]
    (reference ddsp/vocoder.py:758-784).
    Differentiable with respect to the three controls when one of them requires grad (and grad mode is on): the
    backward runs combsubfast_filter_backward with the same comb, noise and seed.  comb is data (no gradient)."""
    if torch.is_grad_enabled() and any(isinstance(c, torch.Tensor) and c.requires_grad for c in (c_hm, c_hp, c_nm)):
        if isinstance(comb, torch.Tensor) and comb.requires_grad:
            raise NotImplementedError("combsubfast_filter has no gradient with respect to comb; pass comb.detach()")
        if noise_in is not None:
            noise_in = noise_in.detach()
        return _CombSubFastFilter.apply(comb, noise_in, int(block), int(seed), int(utterance_offset), c_hm, c_hp, c_nm)
    return _combsubfast_filter(comb, c_hm, c_hp, c_nm, block, noise_in, seed, utterance_offset)


def combsubfast_filter_backward(comb, c_hm, c_hp, c_nm, grad_signal, block, noise_in=None, seed=0, utterance_offset=0):
    """Gradient of combsubfast_filter with respect to the three raw controls, for dL/dsignal ``grad_signal`` [B, T].
    comb / controls / noise_in / seed / utterance_offset must be those of the forward call (the kernel recomputes the
    source spectra and regenerates the in-kernel noise).  -> dense [B, nF, 3*(block+1)]: harmonic_magnitude |
    harmonic_phase | noise_magnitude along the last axis (the split_to_dict layout)."""
    comb, (hm, hp, nm), stride, noise_in, B, nF = _combsubfast_args(comb, c_hm, c_hp, c_nm, block, noise_in)
    grad_signal = _cotangent("grad_signal", grad_signal, B, nF * block)
    grad = torch.empty(B, nF, 3 * (block + 1), dtype=torch.float32, device=comb.device)
    rc = _lib.lib().b2d_combsubfast_filter_backward(comb.data_ptr(), hm.data_ptr(), hp.data_ptr(), nm.data_ptr(), stride,
                                                    _ptr(noise_in), int(seed), int(utterance_offset),
                                                    grad_signal.data_ptr(), B, nF, int(block), grad.data_ptr(), _stream())
    _lib.check(rc, "b2d_combsubfast_filter_backward")
    _count(1)
    return grad


class _CombSubFastFilter(torch.autograd.Function):
    """combsubfast_filter with a CUDA backward.  Saves the comb, the noise input and the control views (no spectra):
    the backward kernel recomputes the source spectra and regenerates the in-kernel noise from seed."""

    @staticmethod
    def forward(ctx, comb, noise_in, block, seed, utterance_offset, c_hm, c_hp, c_nm):
        signal = _combsubfast_filter(comb, c_hm, c_hp, c_nm, block, noise_in, seed, utterance_offset)
        ctx.save_for_backward(comb, noise_in, c_hm, c_hp, c_nm)
        ctx.cfg = (block, seed, utterance_offset)
        return signal

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_signal):
        comb, noise_in, c_hm, c_hp, c_nm = ctx.saved_tensors
        block, seed, utterance_offset = ctx.cfg
        grad = combsubfast_filter_backward(comb, c_hm, c_hp, c_nm, grad_signal, block, noise_in=noise_in, seed=seed,
                                           utterance_offset=utterance_offset)
        return (None,) * 5 + tuple(torch.split(grad, block + 1, dim=-1))


def _combsubfast_args(comb, c_hm, c_hp, c_nm, block, noise_in):
    """checked (comb, controls, frame stride, noise rows, B, nF) of a combsubfast call"""
    _need_cuda_f32("comb", comb)
    if comb.dim() != 2 or comb.shape[1] % int(block) != 0:
        raise ValueError("comb must be [B, n_frames*block] with block=%d, got %s" % (block, tuple(comb.shape)))
    B, T = comb.shape
    nF = T // block
    ctrls, stride = _same_stride([("harmonic_magnitude", c_hm), ("harmonic_phase", c_hp),
                                  ("noise_magnitude", c_nm)], B, nF)
    if ctrls[0].shape[2] != block + 1:
        raise ValueError("controls must have block_size+1 = %d bins" % (block + 1))
    if noise_in is not None:
        noise_in = _noise_rows(noise_in, B, T)
    return comb.contiguous(), ctrls, stride, noise_in, B, nF


def _combsubfast_filter(comb, c_hm, c_hp, c_nm, block, noise_in=None, seed=0, utterance_offset=0):
    comb, (hm, hp, nm), stride, noise_in, B, nF = _combsubfast_args(comb, c_hm, c_hp, c_nm, block, noise_in)
    signal = torch.empty(B, nF * block, dtype=torch.float32, device=comb.device)
    rc = _lib.lib().b2d_combsubfast_filter(comb.data_ptr(), hm.data_ptr(), hp.data_ptr(), nm.data_ptr(), stride,
                                           _ptr(noise_in), int(seed), int(utterance_offset), B, nF, int(block),
                                           signal.data_ptr(), _stream())
    _lib.check(rc, "b2d_combsubfast_filter")
    _count(1)
    return signal


def set_fft_arith(name):
    """'packed' (default) | 'scalar': instantiations of the FFT kernels (identical scalar additions on Hopper)."""
    _lib.check(_lib.lib().b2d_set_fft_arith({"scalar": 0, "packed": 1}[name]), "b2d_set_fft_arith")


def set_overlap(mode):
    """0 / False: every kernel of a synthesizer call in order on the current stream; 1 / True: impulse responses next to
    the bank on an internal side stream; k >= 2: additionally k staggered sub-batches on two streams (b200ddsp.h)."""
    global _overlap_mode
    _lib.check(_lib.lib().b2d_set_overlap(int(mode)), "b2d_set_overlap")
    _overlap_mode = int(mode)


def set_sins_impl(name):
    """'auto' (= 'split': separate bank kernel, measured fastest) | 'split' | 'fused' (bank inside the FFT-domain FIR kernel)
    | 'spectrum' (impulse-response spectra from their own kernel, read by the FIR kernel)."""
    global _sins_impl
    _lib.check(_lib.lib().b2d_set_sins_impl({"auto": 0, "split": 1, "fused": 2, "spectrum": 3}[name]), "b2d_set_sins_impl")
    _sins_impl = name


def hifigan_conv(x, w, bias, k, dilation, n_out, lrelu, residual=None, accum=None, div=1.0, up=0, source=None,
                 noise_w=None, noise_b=None, noise_stride=1, noise_pad=0, out=None):
    """One NSF-HiFiGAN convolution (b2d_hifigan_conv): x a [B, T, C_in] view with any strides -> out [B, T, n_out]
    = (conv(leaky_relu(x, 0.1) if lrelu else x) + bias (+ residual) (+ accum)) / div, or with up = u the polyphase
    transposed convolution -> [B, T u, n_out / u] plus the noise_convs term of ``source`` [B, T u noise_stride, 1].
    ``w`` is packed by hifigan.pack_conv / pack_transposed; ``out`` may be residual or accum."""
    _need_cuda_f32("x", x)
    B, T, Cin = x.shape
    for name, t in (("w", w), ("bias", bias), ("residual", residual), ("accum", accum), ("source", source),
                    ("noise_w", noise_w), ("noise_b", noise_b), ("out", out)):
        if t is not None:
            _need_cuda_f32(name, t)
            if not t.is_contiguous():
                raise ValueError("%s must be contiguous" % name)
    if w.numel() != 2 * k * Cin * n_out:
        raise ValueError("w must hold 2 k C_in N = %d floats, got %d" % (2 * k * Cin * n_out, w.numel()))
    shape = (B, T, n_out) if not up else (B, T * up, n_out // up)
    for name, t in (("residual", residual), ("accum", accum)):
        if t is not None and tuple(t.shape) != shape:
            raise ValueError("%s must be %s, got %s" % (name, shape, tuple(t.shape)))
    noise_k = 0
    if source is not None:
        if source.numel() != B * shape[1] * noise_stride:
            raise ValueError("source must hold B T_out noise_stride = %d samples" % (B * shape[1] * noise_stride))
        noise_k = noise_w.shape[-1]
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=x.device)
    elif tuple(out.shape) != shape:
        raise ValueError("out must be %s, got %s" % (shape, tuple(out.shape)))
    # the stride of a size-1 dimension is never followed; 0 keeps it from failing the kernel's alignment rule
    sb, st, sc = (0 if n == 1 else s for n, s in zip(x.shape, x.stride()))
    if sc == 1 and (x.data_ptr() % 16 or st % 4 or sb % 4):
        x = x.contiguous()
        sb, st, sc = T * Cin, Cin, 1
    rc = _lib.lib().b2d_hifigan_conv(x.data_ptr(), sb, st, sc, B, T, Cin, w.data_ptr(), bias.data_ptr(), int(k),
                                     int(dilation), int(n_out), int(bool(lrelu)), _ptr(residual), _ptr(accum),
                                     float(div), int(up), _ptr(source), _ptr(noise_w), _ptr(noise_b), int(noise_k),
                                     int(noise_stride), int(noise_pad), out.data_ptr(), _stream())
    _lib.check(rc, "b2d_hifigan_conv")
    _count(1)
    return out


def hifigan_post(x, w, bias):
    """tanh(Conv1d(C -> 1, 7, padding 3)(leaky_relu(x, 0.01)) + bias): x [B, T, C] token-major, w [7, C] tap-major,
    bias [1] on the device -> [B, 1, T] (b2d_hifigan_post)."""
    _need_cuda_f32("x", x)
    _need_cuda_f32("w", w)
    _need_cuda_f32("bias", bias)
    B, T, C = x.shape
    if not x.is_contiguous() or not w.is_contiguous() or w.numel() != 7 * C:
        raise ValueError("x must be a contiguous [B, T, C] tensor and w a contiguous [7, C] one")
    out = torch.empty(B, 1, T, dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().b2d_hifigan_post(x.data_ptr(), w.data_ptr(), bias.data_ptr(), B, T, C, out.data_ptr(),
                                           _stream()), "b2d_hifigan_post")
    _count(1)
    return out


def _rows(name, t, C):
    """a [..., C] channel slice of a channel-contiguous activation -> its pixel stride ld: element (..., c) of pixel
    index p (row-major over the leading dims) at p ld + c"""
    _need_cuda_f32(name, t)
    if t.shape[-1] != C or t.stride(-1) != 1:
        raise ValueError("%s must be a [..., %d] view with unit channel stride" % (name, C))
    lead = [d for d in range(t.dim() - 1) if t.shape[d] > 1]
    if not lead:
        return C
    inner = 1
    for d in range(lead[-1] + 1, t.dim() - 1):
        inner *= t.shape[d]
    ld = t.stride(lead[-1]) // inner
    for d in lead:
        span = 1
        for e in range(d + 1, t.dim() - 1):
            span *= t.shape[e]
        if t.stride(d) != ld * span:
            raise ValueError("%s must be dense apart from its channel slice" % name)
    return ld


def rmvpe_conv(x, w, bias, k, n_out, act=0, up=False, residual=None, out=None, n_valid=None):
    """One RMVPE convolution (b2d_rmvpe_conv): x a [B, T, F, C_in] channel slice -> out [B, T, F, n_valid] (or
    [B, 2T, 2F, n_out / 4] with up) = act(conv + bias) (+ residual); act 0 none, 1 relu, 2 sigmoid.  ``out`` and
    ``residual`` may be channel slices of wider buffers; ``w`` is packed by hifigan.pack_conv."""
    B, T, F, Cin = x.shape
    n_valid = n_out if n_valid is None else n_valid
    ldx = _rows("x", x, Cin)
    for name, t in (("w", w), ("bias", bias)):
        _need_cuda_f32(name, t)
    if w.numel() != 2 * k * k * Cin * n_out:
        raise ValueError("w must hold 2 k^2 C_in N = %d floats, got %d" % (2 * k * k * Cin * n_out, w.numel()))
    shape = (B, 2 * T, 2 * F, n_out // 4) if up else (B, T, F, n_valid)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=x.device)
    if tuple(out.shape) != shape:
        raise ValueError("out must be %s, got %s" % (shape, tuple(out.shape)))
    ldo = _rows("out", out, shape[-1])
    ldr = 0
    if residual is not None:
        if tuple(residual.shape) != shape:
            raise ValueError("residual must be %s, got %s" % (shape, tuple(residual.shape)))
        ldr = _rows("residual", residual, shape[-1])
    _lib.check(_lib.lib().b2d_rmvpe_conv(x.data_ptr(), ldx, B, T, F, Cin, w.data_ptr(), bias.data_ptr(), int(k),
                                         int(n_out), int(n_valid), int(act), int(bool(up)), _ptr(residual), ldr,
                                         out.data_ptr(), ldo, _stream()), "b2d_rmvpe_conv")
    _count(1)
    return out


def rmvpe_conv_small(x, w, bias, relu=False, in_scale=None, in_shift=None, head=False, out=None):
    """Direct fp32 convolution (b2d_rmvpe_conv_small): x a [B, T, F, C_in] view with any strides, w [C_out, C_in, k, k]
    (k 1 or 3, padding k // 2), optional input affine on the real pixels -> out [B, T, F, C_out] (a channel slice is
    fine), or with head [B, T, C_out F] (feature c F + f)."""
    _need_cuda_f32("x", x)
    _need_cuda_f32("w", w)
    B, T, F, Cin = x.shape
    Cout, k = w.shape[0], w.shape[-1]
    if tuple(w.shape) != (Cout, Cin, k, k) or not w.is_contiguous():
        raise ValueError("w must be a contiguous [C_out, %d, k, k] tensor" % Cin)
    for name, t in (("bias", bias), ("in_scale", in_scale), ("in_shift", in_shift)):
        if t is not None:
            _need_cuda_f32(name, t)
    shape = (B, T, Cout * F) if head else (B, T, F, Cout)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=x.device)
    if tuple(out.shape) != shape:
        raise ValueError("out must be %s, got %s" % (shape, tuple(out.shape)))
    if head:
        if not out.is_contiguous():
            raise ValueError("out must be contiguous")
        ldo = Cout
    else:
        ldo = _rows("out", out, Cout)
    s = x.stride()
    _lib.check(_lib.lib().b2d_rmvpe_conv_small(x.data_ptr(), s[0], s[1], s[2], s[3], B, T, F, Cin, _ptr(in_scale),
                                               _ptr(in_shift), w.data_ptr(), _ptr(bias), int(k), int(Cout),
                                               int(bool(relu)), int(bool(head)), out.data_ptr(), ldo, _stream()),
               "b2d_rmvpe_conv_small")
    _count(1)
    return out


def rmvpe_pool(x):
    """AvgPool2d(2) of a [B, T, F, C] channel slice -> a new [B, T / 2, F / 2, C] tensor (b2d_rmvpe_pool)"""
    B, T, F, C = x.shape
    ldx = _rows("x", x, C)
    out = torch.empty(B, T // 2, F // 2, C, dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().b2d_rmvpe_pool(x.data_ptr(), ldx, B, T, F, C, out.data_ptr(), _stream()), "b2d_rmvpe_pool")
    _count(1)
    return out


def rmvpe_gru(xg, w_hh, b_hh):
    """BiGRU(384 -> 256) recurrence (b2d_rmvpe_gru): xg [B, T, 1536] = W_ih x + b_ih of both directions, w_hh
    [2, 768, 256], b_hh [2, 768] -> [B, T, 512] = [forward | backward]"""
    for name, t in (("xg", xg), ("w_hh", w_hh), ("b_hh", b_hh)):
        _need_cuda_f32(name, t)
        if not t.is_contiguous():
            raise ValueError("%s must be contiguous" % name)
    B, T, G = xg.shape
    if G != 1536 or w_hh.numel() != 2 * 768 * 256 or b_hh.numel() != 2 * 768:
        raise ValueError("xg must be [B, T, 1536], w_hh [2, 768, 256], b_hh [2, 768]")
    out = torch.empty(B, T, 512, dtype=torch.float32, device=xg.device)
    _lib.check(_lib.lib().b2d_rmvpe_gru(xg.data_ptr(), w_hh.data_ptr(), b_hh.data_ptr(), B, T, out.data_ptr(),
                                        _stream()), "b2d_rmvpe_gru")
    _count(1)
    return out


def rmvpe_resample(x, table, new_freq, orig_freq, width, n_out):
    """x [B, N] -> [B, n_out] through the polyphase table [new_freq, taps] (b2d_rmvpe_resample)"""
    _need_cuda_f32("x", x)
    _need_cuda_f32("table", table)
    if x.dim() != 2 or not x.is_contiguous() or not table.is_contiguous() or table.shape[0] != new_freq:
        raise ValueError("x must be a contiguous [B, N] tensor and table a contiguous [new_freq, taps] one")
    B, N = x.shape
    out = torch.empty(B, n_out, dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().b2d_rmvpe_resample(x.data_ptr(), B, N, table.data_ptr(), int(new_freq), int(orig_freq),
                                             int(table.shape[1]), int(width), int(n_out), out.data_ptr(), _stream()),
               "b2d_rmvpe_resample")
    _count(1)
    return out


def rmvpe_mel(audio, window, basis, lohi, hop, t_pad):
    """audio [B, N] at 16 kHz -> log-mel [B, t_pad, 128] (frames past 1 + N // hop are zero) (b2d_rmvpe_mel)"""
    _need_cuda_f32("audio", audio)
    _need_cuda_f32("window", window)
    _need_cuda_f32("basis", basis)
    _need_cuda_f32("lohi", lohi, torch.int32)
    if audio.dim() != 2 or not audio.is_contiguous():
        raise ValueError("audio must be a contiguous [B, N] tensor")
    B, N = audio.shape
    out = torch.empty(B, t_pad, 128, dtype=torch.float32, device=audio.device)
    _lib.check(_lib.lib().b2d_rmvpe_mel(audio.data_ptr(), B, N, window.data_ptr(), basis.data_ptr(), lohi.data_ptr(),
                                        int(hop), 1 + N // hop, int(t_pad), out.data_ptr(), _stream()), "b2d_rmvpe_mel")
    _count(1)
    return out


def mel_keyshift(y, table, basis, lohi, n_fft, hop, clip_val):
    """y [B, T] -> key-shifted log-mel [B, n_mels, b2d_mel_frames(T, n_fft, n_fft, hop)] for the shifted transform length
    n_fft, through its Bluestein ``table`` (mel.keyshift_table_host) (b2d_mel_spectrogram_keyshift)"""
    _need_cuda_f32("y", y)
    _need_cuda_f32("table", table)
    _need_cuda_f32("basis", basis)
    _need_cuda_f32("lohi", lohi, torch.int32)
    if y.dim() != 2 or not y.is_contiguous() or basis.dim() != 2 or not basis.is_contiguous():
        raise ValueError("y must be a contiguous [B, T] tensor and basis a contiguous [n_mels, 1025] one")
    B, T = y.shape
    L = _lib.lib()
    n_frames = L.b2d_mel_frames(T, int(n_fft), int(n_fft), int(hop))
    if n_frames <= 0:
        raise ValueError("signal of %d samples is too short for one frame" % T)
    out = torch.empty(B, basis.shape[0], n_frames, dtype=torch.float32, device=y.device)
    _lib.check(L.b2d_mel_spectrogram_keyshift(y.data_ptr(), table.data_ptr(), basis.data_ptr(), lohi.data_ptr(), B, T,
                                              int(n_fft), int(hop), int(basis.shape[0]), float(clip_val), out.data_ptr(),
                                              _stream()), "b2d_mel_spectrogram_keyshift")
    _count(1)
    return out


def rmvpe_decode(salience, n_frames, thred):
    """salience [B, t_pad, 360] -> f0 [B, n_frames] in Hz, 0 where unvoiced (b2d_rmvpe_decode)"""
    _need_cuda_f32("salience", salience)
    if salience.dim() != 3 or salience.shape[-1] != 360 or not salience.is_contiguous():
        raise ValueError("salience must be a contiguous [B, T, 360] tensor")
    B, t_pad, _ = salience.shape
    out = torch.empty(B, n_frames, dtype=torch.float32, device=salience.device)
    _lib.check(_lib.lib().b2d_rmvpe_decode(salience.data_ptr(), B, t_pad, int(n_frames), float(thred), out.data_ptr(),
                                           _stream()), "b2d_rmvpe_decode")
    _count(1)
    return out


# ---- HuBERT / ContentVec units encoder (b2d_hubert_*) ------------------------------------------------------------------
def _contig(name, t, dtype=torch.float32):
    _need_cuda_f32(name, t, dtype)
    if not t.is_contiguous():
        raise ValueError("%s must be contiguous" % name)


def _operand(shape, device, split):
    """an output a library GEMM reads: (hi, lo) TF32 halves when split, else one fp32 tensor"""
    if split:
        return (torch.empty(shape, dtype=torch.float32, device=device),
                torch.empty(shape, dtype=torch.float32, device=device))
    return torch.empty(shape, dtype=torch.float32, device=device)


def _operand_ptrs(op):
    return (op[0].data_ptr(), op[1].data_ptr()) if isinstance(op, tuple) else (op.data_ptr(), 0)


def hubert_conv0(x, w, pad, La):
    """Conv1d(1 -> 512, 10, stride 5) of x [B, N] zero-padded by `pad` -> (y [B, La, 512], part [B, La / 64, 2, 512]
    fp64, L0) (b2d_hubert_conv0): y zero past the L0 valid frames, part the per-tile GroupNorm sums"""
    _contig("x", x)
    _contig("w", w)
    if x.dim() != 2 or w.numel() != 512 * 10:
        raise ValueError("x must be [B, N] and w [512, 1, 10]")
    B, N = x.shape
    y = torch.empty(B, La, 512, dtype=torch.float32, device=x.device)
    part = torch.empty(B, -(-La // 64), 2, 512, dtype=torch.float64, device=x.device)
    _lib.check(_lib.lib().b2d_hubert_conv0(x.data_ptr(), B, N, int(pad), w.data_ptr(), int(La), y.data_ptr(),
                                           part.data_ptr(), _stream()), "b2d_hubert_conv0")
    _count(1)
    return y, part, (N + 2 * pad - 10) // 5 + 1


def hubert_gn_finalize(part, L0, gamma, beta, eps=1e-5):
    """per-tile sums [B, n_tiles, 2, 512] -> GroupNorm(512, 512) (scale, shift) [B, 512] (b2d_hubert_gn_finalize)"""
    _contig("part", part, torch.float64)
    _contig("gamma", gamma)
    _contig("beta", beta)
    B, n_tiles = part.shape[:2]
    scale = torch.empty(B, 512, dtype=torch.float32, device=part.device)
    shift = torch.empty_like(scale)
    _lib.check(_lib.lib().b2d_hubert_gn_finalize(part.data_ptr(), B, n_tiles, int(L0), gamma.data_ptr(),
                                                 beta.data_ptr(), float(eps), scale.data_ptr(), shift.data_ptr(),
                                                 _stream()), "b2d_hubert_gn_finalize")
    _count(1)
    return scale, shift


def hubert_act(x, scale=None, shift=None, split=True):
    """GELU(x scale[b] + shift[b]) of x [B, L, C] (or [rows, C] without the affine) as a GEMM operand of the same
    shape (b2d_hubert_act)"""
    _contig("x", x)
    C = x.shape[-1]
    rows = x.numel() // C
    per_b = x.shape[1] if scale is not None else rows
    if scale is not None:
        _contig("scale", scale)
        _contig("shift", shift)
        if x.dim() != 3 or scale.shape != (x.shape[0], C) or shift.shape != scale.shape:
            raise ValueError("with an affine, x must be [B, L, C] and scale, shift [B, C]")
    out = _operand(x.shape, x.device, split)
    hi, lo = _operand_ptrs(out)
    _lib.check(_lib.lib().b2d_hubert_act(x.data_ptr(), rows, C, per_b, _ptr(scale), _ptr(shift), hi, lo, _stream()),
               "b2d_hubert_act")
    _count(1)
    return out


def hubert_ln(x, gamma, beta, T, y=None, gelu=False, eps=1e-5, h=None, operand=True, split=True):
    """LayerNorm(C) of rows of x [B, rows_per_b, C] (the first T of each utterance; x [B T, C] when rows_per_b = T)
    (+ y [B T, C]), GELU first when `gelu` -> (h [B T, C] or None, operand or None) (b2d_hubert_ln).  Pass h = x to
    normalize in place; h=False skips the fp32 output."""
    _contig("x", x)
    _contig("gamma", gamma)
    _contig("beta", beta)
    C = x.shape[-1]
    n_in = x.numel() // C
    B = x.shape[0] if x.dim() == 3 else n_in // T
    per_b = n_in // B
    rows = B * T
    if y is not None:
        _contig("y", y)
        if y.numel() != rows * C:
            raise ValueError("y must hold B T rows of %d" % C)
    if h is None:
        h = torch.empty(rows, C, dtype=torch.float32, device=x.device)
    elif h is False:
        h = None
    else:
        _contig("h", h)
    op = _operand((rows, C), x.device, split) if operand else None
    hi, lo = _operand_ptrs(op) if operand else (0, 0)
    _lib.check(_lib.lib().b2d_hubert_ln(x.data_ptr(), _ptr(y), rows, int(T), per_b, C, int(bool(gelu)),
                                        gamma.data_ptr(), beta.data_ptr(), float(eps), _ptr(h), hi, lo, _stream()),
               "b2d_hubert_ln")
    _count(1)
    return h, op


def hubert_posconv(x, w, bias, T):
    """GELU(grouped positional convolution + bias) of x [B T, 768] -> [B T, 768] (b2d_hubert_posconv); w the folded
    weight packed [16, 128, 48, 48]"""
    _contig("x", x)
    _contig("w", w)
    _contig("bias", bias)
    if x.shape[-1] != 768 or (x.numel() // 768) % T or w.numel() != 16 * 128 * 48 * 48:
        raise ValueError("x must be [B T, 768] and w [16, 128, 48, 48]")
    B = x.numel() // 768 // T
    y = torch.empty(B * T, 768, dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().b2d_hubert_posconv(x.data_ptr(), B, int(T), w.data_ptr(), bias.data_ptr(), y.data_ptr(),
                                             _stream()), "b2d_hubert_posconv")
    _count(1)
    return y


def hubert_attention(qkv, T, split=True):
    """12-head softmax attention of qkv [B T, 2304] -> the out-projection's operand [B T, 768] (b2d_hubert_attention)"""
    _contig("qkv", qkv)
    if qkv.shape[-1] != 2304 or (qkv.numel() // 2304) % T:
        raise ValueError("qkv must be [B T, 2304]")
    B = qkv.numel() // 2304 // T
    out = _operand((B * T, 768), qkv.device, split)
    hi, lo = _operand_ptrs(out)
    _lib.check(_lib.lib().b2d_hubert_attention(qkv.data_ptr(), B, int(T), hi, lo, _stream()), "b2d_hubert_attention")
    _count(1)
    return out


def hubert_align(units, ratio, n_frames):
    """units [B, T, C] -> [B, n_frames, C] at rows min(rint(float32(ratio) f), T - 1) (b2d_hubert_align)"""
    _contig("units", units)
    B, T, C = units.shape
    out = torch.empty(B, n_frames, C, dtype=torch.float32, device=units.device)
    _lib.check(_lib.lib().b2d_hubert_align(units.data_ptr(), B, T, C, float(ratio), int(n_frames), out.data_ptr(),
                                           _stream()), "b2d_hubert_align")
    _count(1)
    return out


def _need_vector(name, t, n=None):
    _need_cuda_f32(name, t)
    if t.dim() != 1 or not t.is_contiguous() or (n is not None and t.numel() < n):
        raise ValueError("%s must be a contiguous 1-D tensor%s, got %s"
                         % (name, "" if n is None else " of at least %d samples" % n, tuple(t.shape)))


def rt_f0_regrid(src, src_step, n_dst, dst_step, src_div=1.0, src_scale=1.0, rmvpe=False, pad=0, f0_min=0.0,
                 post_scale=1.0):
    """np.interp of src [n] from positions (src_step i) / src_div to positions dst_step j -> [n_dst] (b2d_rt_f0_regrid).
    rmvpe=False: src times src_scale first (Enhancer's real_factor).  rmvpe=True: F0_Extractor's 'rmvpe'
    post-processing with uv_interp, `pad` leading frames, the clamp to f0_min and the pitch factor post_scale."""
    _need_vector("src", src)
    n_src = src.numel()
    L = _lib.lib()
    out = torch.empty(int(n_dst), dtype=torch.float32, device=src.device)
    nbytes = L.b2d_rt_f0_regrid_workspace_bytes(n_src, int(n_dst))
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=src.device)
    _lib.check(L.b2d_rt_f0_regrid(src.data_ptr(), n_src, float(src_step), float(src_div), float(src_scale), int(n_dst),
                                  int(pad), float(dst_step), 1 if rmvpe else 0, float(f0_min), float(post_scale),
                                  out.data_ptr(), ws.data_ptr(), nbytes, _stream()), "b2d_rt_f0_regrid")
    _count(1)
    return out


def rt_sola(x, buf, search):
    """the SOLA shift of gui.py's callback -> int32 [1] on the device: the first s <= search maximising the normalised
    cross-correlation of x[s:][:crossfade] with buf [crossfade] (b2d_rt_sola)"""
    _need_vector("buf", buf)
    _need_vector("x", x, buf.numel() + int(search))
    shift = torch.empty(1, dtype=torch.int32, device=x.device)
    _lib.check(_lib.lib().b2d_rt_sola(x.data_ptr(), buf.data_ptr(), buf.numel(), int(search), shift.data_ptr(),
                                      _stream()), "b2d_rt_sola")
    _count(1)
    return shift


def rt_crossfade(x, shift, search, buf, fade_in, fade_out, block, phase_vocoder=False):
    """gui.py's crossfade at the device-side shift (int32 [1], <= search) -> (out [block], next_buf [crossfade]): the
    linear sin^2 fade or phase_vocoder over the first crossfade samples of x[shift:] (b2d_rt_crossfade)"""
    cf = buf.numel()
    _need_vector("buf", buf)
    _need_vector("fade_in", fade_in, cf)
    _need_vector("fade_out", fade_out, cf)
    _need_vector("x", x, int(search) + int(block) + cf)
    _need_cuda_f32("shift", shift, torch.int32)
    L = _lib.lib()
    out = torch.empty(int(block), dtype=torch.float32, device=x.device)
    next_buf = torch.empty(cf, dtype=torch.float32, device=x.device)
    nbytes = L.b2d_rt_crossfade_workspace_bytes(cf, int(bool(phase_vocoder)))
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=x.device)
    _lib.check(L.b2d_rt_crossfade(x.data_ptr(), shift.data_ptr(), buf.data_ptr(), fade_in.data_ptr(), fade_out.data_ptr(),
                                  int(block), cf, int(bool(phase_vocoder)), out.data_ptr(), next_buf.data_ptr(),
                                  ws.data_ptr(), nbytes, _stream()), "b2d_rt_crossfade")
    _count(2 if phase_vocoder else 1)
    return out, next_buf

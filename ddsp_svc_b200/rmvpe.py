"""Drop-in for the RMVPE pitch extractor (reference encoder/rmvpe/: ``E2E0`` model.py:36-60, ``RMVPE`` inference.py),
inference on the kernels of csrc/rmvpe.cu.

``E2E0(n_blocks, n_gru, kernel_size, ...)`` builds the reference's parameter tree (``unet.encoder`` / ``intermediate`` /
``tf`` / ``decoder``, ``cnn``, ``fc.0.gru``, ``fc.1``), including the TimbreFilter ``unet.tf`` that DeepUnet0 builds but
never runs, so a reference state dict maps key for key.  ``RMVPE(model_path)`` is the reference's extractor class:
``F0_Extractor('rmvpe')`` builds it once ``patch_reference(rmvpe=True)`` has rebound the name.

The path: resample to 16 kHz (torchaudio's polyphase sinc-Hann FIR, table restated here), log-mel (n_fft 1024, HTK mel
basis), the U-Net as 3xTF32 tensor-core convolutions with eval BatchNorm folded into them, the BiGRU (input projection
as a GEMM, the recurrence in one thread-block cluster per direction), Linear + sigmoid, and the local-average decode.
Weights are packed once per model and device (BatchNorm folded, TF32 hi/lo halves, the transposed convolutions in
polyphase form: about 0.72 GB for the published model) and re-packed only when a parameter changes, so a warm call
reads nothing back from the device.
"""
import math
import threading

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .hifigan import pack_conv
from .mel import _support, mel_filterbank

SAMPLE_RATE, N_CLASS, N_MELS, MEL_FMIN, MEL_FMAX, WINDOW_LENGTH = 16000, 360, 128, 30, 8000, 1024


# ---- the reference's parameter tree (deepunet.py, seq.py); the forward runs in E2E0.forward ----------------------------
class ConvBlockRes(nn.Module):
    def __init__(self, in_channels, out_channels, momentum=0.01):
        super().__init__()
        self.conv = nn.Sequential(
            nn.Conv2d(in_channels, out_channels, (3, 3), (1, 1), (1, 1), bias=False),
            nn.BatchNorm2d(out_channels, momentum=momentum), nn.ReLU(),
            nn.Conv2d(out_channels, out_channels, (3, 3), (1, 1), (1, 1), bias=False),
            nn.BatchNorm2d(out_channels, momentum=momentum), nn.ReLU())
        self.is_shortcut = in_channels != out_channels
        if self.is_shortcut:
            self.shortcut = nn.Conv2d(in_channels, out_channels, (1, 1))


class ResEncoderBlock(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, n_blocks=1, momentum=0.01):
        super().__init__()
        self.n_blocks = n_blocks
        self.conv = nn.ModuleList([ConvBlockRes(in_channels if i == 0 else out_channels, out_channels, momentum)
                                   for i in range(n_blocks)])
        self.kernel_size = kernel_size
        if kernel_size is not None:
            self.pool = nn.AvgPool2d(kernel_size=kernel_size)


class ResDecoderBlock(nn.Module):
    def __init__(self, in_channels, out_channels, stride, n_blocks=1, momentum=0.01):
        super().__init__()
        self.n_blocks = n_blocks
        self.conv1 = nn.Sequential(
            nn.ConvTranspose2d(in_channels, out_channels, (3, 3), stride, (1, 1), output_padding=(1, 1), bias=False),
            nn.BatchNorm2d(out_channels, momentum=momentum), nn.ReLU())
        self.conv2 = nn.ModuleList([ConvBlockRes(out_channels * 2 if i == 0 else out_channels, out_channels, momentum)
                                    for i in range(n_blocks)])


class Encoder(nn.Module):
    def __init__(self, in_channels, in_size, n_encoders, kernel_size, n_blocks, out_channels=16, momentum=0.01):
        super().__init__()
        self.n_encoders = n_encoders
        self.bn = nn.BatchNorm2d(in_channels, momentum=momentum)
        self.layers = nn.ModuleList()
        self.latent_channels = []
        for _ in range(n_encoders):
            self.layers.append(ResEncoderBlock(in_channels, out_channels, kernel_size, n_blocks, momentum=momentum))
            self.latent_channels.append([out_channels, in_size])
            in_channels, out_channels, in_size = out_channels, out_channels * 2, in_size // 2
        self.out_size, self.out_channel = in_size, out_channels


class Intermediate(nn.Module):
    def __init__(self, in_channels, out_channels, n_inters, n_blocks, momentum=0.01):
        super().__init__()
        self.n_inters = n_inters
        self.layers = nn.ModuleList([ResEncoderBlock(in_channels if i == 0 else out_channels, out_channels, None,
                                                     n_blocks, momentum) for i in range(n_inters)])


class Decoder(nn.Module):
    def __init__(self, in_channels, n_decoders, stride, n_blocks, momentum=0.01):
        super().__init__()
        self.n_decoders = n_decoders
        self.layers = nn.ModuleList()
        for _ in range(n_decoders):
            self.layers.append(ResDecoderBlock(in_channels, in_channels // 2, stride, n_blocks, momentum))
            in_channels //= 2


class TimbreFilter(nn.Module):
    def __init__(self, latent_rep_channels):
        super().__init__()
        self.layers = nn.ModuleList([ConvBlockRes(c, c) for c, _ in latent_rep_channels])


class DeepUnet0(nn.Module):
    def __init__(self, kernel_size, n_blocks, en_de_layers=5, inter_layers=4, in_channels=1, en_out_channels=16):
        super().__init__()
        self.encoder = Encoder(in_channels, N_MELS, en_de_layers, kernel_size, n_blocks, en_out_channels)
        self.intermediate = Intermediate(self.encoder.out_channel // 2, self.encoder.out_channel, inter_layers, n_blocks)
        self.tf = TimbreFilter(self.encoder.latent_channels)
        self.decoder = Decoder(self.encoder.out_channel, en_de_layers, kernel_size, n_blocks)


class BiGRU(nn.Module):
    def __init__(self, input_features, hidden_features, num_layers):
        super().__init__()
        self.gru = nn.GRU(input_features, hidden_features, num_layers=num_layers, batch_first=True, bidirectional=True)


def validate(n_blocks, n_gru, kernel_size, en_de_layers, inter_layers, in_channels, en_out_channels):
    """raise ValueError naming the field of a configuration the kernels do not implement"""
    if n_gru != 1:
        raise ValueError("n_gru: only one bidirectional GRU layer (1) is implemented, got %r" % (n_gru,))
    if tuple(kernel_size) != (2, 2):
        raise ValueError("kernel_size: only (2, 2) pooling / stride is implemented, got %r" % (kernel_size,))
    if in_channels != 1:
        raise ValueError("in_channels: only 1 (the mel spectrogram) is implemented, got %r" % (in_channels,))
    if en_out_channels <= 0 or en_out_channels % 16 or en_out_channels > 16:
        raise ValueError("en_out_channels: the first level's convolutions and `cnn` are implemented for 16 channels, "
                         "got %r" % (en_out_channels,))
    if n_blocks < 1:
        raise ValueError("n_blocks: at least 1, got %r" % (n_blocks,))
    if not 1 <= en_de_layers <= 7:
        raise ValueError("en_de_layers: 1 to 7 levels (the 128 mel bins halve at each), got %r" % (en_de_layers,))
    if inter_layers < 1:
        raise ValueError("inter_layers: at least 1, got %r" % (inter_layers,))


def fold_bn(w, bn):
    """weight [C_out, ...] and eval BatchNorm bn -> (w scaled per output channel, bias), in float64"""
    s = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
    return w.double() * s.view(-1, *([1] * (w.dim() - 1))), bn.bias.double() - bn.running_mean.double() * s


def bn_affine(bn):
    """eval BatchNorm bn as x scale + shift, float64"""
    s = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
    return s, bn.bias.double() - bn.running_mean.double() * s


# (output phase a, input offset d) -> tap of ConvTranspose2d(3, stride 2, padding 1, output_padding 1) along one axis:
# output 2m + a takes input m + d through tap 2 (m + d) - 1 + tap = 2m + a
_PHASE_TAP = {(0, 0): 1, (1, 0): 2, (1, 1): 0}


def polyphase2d(w):
    """ConvTranspose2d(C_in, C_out, 3, stride 2, padding 1, output_padding 1) weight [C_in, C_out, 3, 3] -> the
    equivalent 2x2 convolution weight [4 C_out, C_in, 2, 2] over input offsets {0, 1}^2: column r C_out + co, r = 2a + c,
    is output pixel (2t + a, 2f + c); the taps with no input (phase 0, offset 1) are zero"""
    C_in, C_out = w.shape[:2]
    out = w.new_zeros(2, 2, C_out, C_in, 2, 2)
    for (a, dt), kt in _PHASE_TAP.items():
        for (c, df), kf in _PHASE_TAP.items():
            out[a, c, :, :, dt, df] = w[:, :, kt, kf].t()
    return out.reshape(4 * C_out, C_in, 2, 2)


class E2E0(nn.Module):
    """E2E0(n_blocks, n_gru, kernel_size, en_de_layers=5, inter_layers=4, in_channels=1, en_out_channels=16): the
    reference's constructor and parameter tree (model.py:36-54).  forward(mel [B, 128, T] CUDA fp32, T a multiple of
    2^en_de_layers) -> salience [B, T, 360].  Inference only (eval BatchNorm, inert dropout)."""

    def __init__(self, n_blocks, n_gru, kernel_size, en_de_layers=5, inter_layers=4, in_channels=1, en_out_channels=16):
        super().__init__()
        validate(n_blocks, n_gru, kernel_size, en_de_layers, inter_layers, in_channels, en_out_channels)
        self.en_de_layers = en_de_layers
        self.unet = DeepUnet0(kernel_size, n_blocks, en_de_layers, inter_layers, in_channels, en_out_channels)
        self.cnn = nn.Conv2d(en_out_channels, 3, (3, 3), padding=(1, 1))
        self.fc = nn.Sequential(BiGRU(3 * N_MELS, 256, n_gru), nn.Linear(512, N_CLASS), nn.Dropout(0.25), nn.Sigmoid())

    # ---- weights in the kernels' layouts, rebuilt when a parameter or buffer changes ----
    def _pack(self):
        key = tuple((t.data_ptr(), t._version) for t in list(self.parameters()) + list(self.buffers()))
        c = self.__dict__.get("_packed")
        if c is not None and c[0] == key:
            return c[1]
        f32 = lambda t: t.detach().float().contiguous()
        with torch.no_grad():
            def tc(w, b):                                     # tensor-core convolution
                return dict(w=pack_conv(f32(w).reshape(w.shape[0], w.shape[1], -1)), b=f32(b), n=w.shape[0],
                            k=w.shape[-1])

            def block(m):
                w1, b1 = fold_bn(m.conv[0].weight, m.conv[1])
                w2, b2 = fold_bn(m.conv[3].weight, m.conv[4])
                cin = m.conv[0].in_channels
                d = dict(cin=cin, c2=tc(w2, b2))
                if cin == 1:                                   # the first convolution: direct fp32 (rv_conv_small)
                    d["c1"] = (f32(w1), f32(b1))
                    d["sc"] = (f32(m.shortcut.weight), f32(m.shortcut.bias))
                else:
                    d["c1"] = tc(w1, b1)
                    d["sc"] = tc(m.shortcut.weight, m.shortcut.bias) if m.is_shortcut else None
                return d

            unet = self.unet
            s, h = bn_affine(unet.encoder.bn)
            P = dict(in_scale=f32(s), in_shift=f32(h),
                     enc=[[block(m) for m in layer.conv] for layer in unet.encoder.layers],
                     inter=[[block(m) for m in layer.conv] for layer in unet.intermediate.layers], dec=[])
            for layer in unet.decoder.layers:
                wt, bt = fold_bn(layer.conv1[0].weight.transpose(0, 1), layer.conv1[1])   # [C_out, C_in, 3, 3]
                P["dec"].append(dict(up=tc(polyphase2d(wt.transpose(0, 1)), bt), blocks=[block(m) for m in layer.conv2]))
            P["cnn"] = (f32(self.cnn.weight), f32(self.cnn.bias))
            gru = self.fc[0].gru
            P["ih"] = tc(torch.cat([gru.weight_ih_l0, gru.weight_ih_l0_reverse])[:, :, None, None],
                         torch.cat([gru.bias_ih_l0, gru.bias_ih_l0_reverse]))
            P["whh"] = f32(torch.stack([gru.weight_hh_l0, gru.weight_hh_l0_reverse]))
            P["bhh"] = f32(torch.stack([gru.bias_hh_l0, gru.bias_hh_l0_reverse]))
            lin = self.fc[1]
            n_pad = -N_CLASS % 16                                  # 368 GEMM columns, 360 stored
            P["lin"] = tc(torch.cat([lin.weight, lin.weight.new_zeros(n_pad, 512)])[:, :, None, None],
                          torch.cat([lin.bias, lin.bias.new_zeros(n_pad)]))
        self.__dict__["_packed"] = (key, P)
        return P

    @staticmethod
    def _blocks(blocks, x, P, out_last=None):
        for j, d in enumerate(blocks):
            out = out_last if j == len(blocks) - 1 else None
            n = d["c2"]["n"]
            if d["cin"] == 1:
                y = ops.rmvpe_conv_small(x, d["c1"][0], d["c1"][1], relu=True, in_scale=P["in_scale"],
                                         in_shift=P["in_shift"])
                res = ops.rmvpe_conv_small(x, d["sc"][0], d["sc"][1], in_scale=P["in_scale"], in_shift=P["in_shift"])
            else:
                c1 = d["c1"]
                y = ops.rmvpe_conv(x, c1["w"], c1["b"], 3, n, act=1)
                sc = d["sc"]
                res = ops.rmvpe_conv(x, sc["w"], sc["b"], 1, n) if sc is not None else x
            c2 = d["c2"]
            x = ops.rmvpe_conv(y, c2["w"], c2["b"], 3, n, act=1, residual=res, out=out)
        return x

    def _salience(self, x):
        """x [B, T, 128, 1] (any strides: the log-mel) -> salience [B, T, 360]"""
        P = self._pack()
        B, T = x.shape[:2]
        cats = []
        for blocks in P["enc"]:
            n = blocks[-1]["c2"]["n"]
            cat = torch.empty(B, x.shape[1], x.shape[2], 2 * n, dtype=torch.float32, device=x.device)
            skip = self._blocks(blocks, x, P, out_last=cat[..., n:])   # the skip lands in the decoder's concat buffer
            cats.append(cat)
            x = ops.rmvpe_pool(skip)
        for blocks in P["inter"]:
            x = self._blocks(blocks, x, P)
        for dec, cat in zip(P["dec"], reversed(cats)):
            n = cat.shape[-1] // 2
            up = dec["up"]
            ops.rmvpe_conv(x, up["w"], up["b"], 2, 4 * n, act=1, up=True, out=cat[..., :n])
            x = self._blocks(dec["blocks"], cat, P)
        feat = ops.rmvpe_conv_small(x, P["cnn"][0], P["cnn"][1], head=True)          # [B, T, 3 128], c 128 + f
        ih = P["ih"]
        xg = ops.rmvpe_conv(feat.view(B, T, 1, 3 * N_MELS), ih["w"], ih["b"], 1, ih["n"])
        hid = ops.rmvpe_gru(xg.view(B, T, ih["n"]), P["whh"], P["bhh"])
        lin = P["lin"]
        sal = ops.rmvpe_conv(hid.view(B, T, 1, 512), lin["w"], lin["b"], 1, lin["n"], act=2, n_valid=N_CLASS)
        return sal.view(B, T, N_CLASS)

    def forward(self, mel):
        if not (isinstance(mel, torch.Tensor) and mel.is_cuda):
            raise ValueError("E2E0 runs on the CUDA kernels: mel must be a CUDA tensor")
        if mel.dim() != 3 or mel.shape[1] != N_MELS:
            raise ValueError("mel must be [B, %d, T], got %s" % (N_MELS, tuple(mel.shape)))
        if mel.shape[2] % (1 << self.en_de_layers):
            raise ValueError("the frame count must be a multiple of 2^en_de_layers = %d, got %d"
                             % (1 << self.en_de_layers, mel.shape[2]))
        if torch.is_grad_enabled() and self.training and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("the RMVPE network is inference-only; call it under torch.no_grad() or in eval() "
                                      "mode")
        with torch.no_grad():
            return self._salience(mel.float().transpose(1, 2).unsqueeze(-1))


# ---- host tables -------------------------------------------------------------------------------------------------------
def resample_table(orig_freq, new_freq=SAMPLE_RATE, lowpass_filter_width=128, rolloff=0.99):
    """torchaudio.transforms.Resample(orig_freq, new_freq, lowpass_filter_width=...).kernel restated (sinc_interp_hann,
    default dtype): -> (float32 [new / gcd, taps], width, orig / gcd, new / gcd)"""
    gcd = math.gcd(int(orig_freq), int(new_freq))
    orig, new = int(orig_freq) // gcd, int(new_freq) // gcd
    base = min(orig, new) * rolloff
    width = math.ceil(lowpass_filter_width * orig / base)
    idx = torch.arange(-width, width + orig, dtype=torch.float64)[None] / orig
    t = torch.arange(0, -new, -1)[:, None] / new + idx     # the phase offsets in the default dtype, as torchaudio has them
    t = (t * base).clamp(-lowpass_filter_width, lowpass_filter_width)
    window = torch.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    t = t * math.pi
    k = torch.where(t == 0, torch.tensor(1.0, dtype=t.dtype), t.sin() / t) * (window * (base / orig))
    return k.float().contiguous(), width, orig, new


def resampled_length(n, orig_freq, new_freq=SAMPLE_RATE):
    """ceil(new N / orig) with the rates divided by their gcd, as torchaudio crops"""
    gcd = math.gcd(int(orig_freq), int(new_freq))
    o, w = int(orig_freq) // gcd, int(new_freq) // gcd
    return -(-w * n // o)


class Resampler:
    """torchaudio Resample(orig_freq, new_freq, lowpass_filter_width=128) of CUDA [B, N] audio on the kernels
    (ops.rmvpe_resample), the polyphase table of each (orig_freq, device) built once: ``resampler(audio, orig_freq)``.
    ``tables`` maps (str(orig_freq), device) to (table, width, orig / gcd, new / gcd)."""

    def __init__(self, new_freq):
        self.new_freq = int(new_freq)
        self.tables = {}
        self._lock = threading.Lock()

    def __call__(self, audio, orig_freq):
        orig_freq = int(orig_freq)
        if orig_freq == self.new_freq:
            return audio
        key = (str(orig_freq), audio.device)
        with self._lock:
            tab = self.tables.get(key)
            if tab is None:
                k, width, orig, new = resample_table(orig_freq, self.new_freq)
                tab = self.tables[key] = (k.to(audio.device), width, orig, new)
        k, width, orig, new = tab
        return ops.rmvpe_resample(audio, k, new, orig, width, resampled_length(audio.shape[-1], orig_freq, self.new_freq))


def mel_basis():
    """spec.py's basis: librosa.filters.mel(sr=16000, n_fft=1024, n_mels=128, fmin=30, fmax=8000, htk=True)"""
    return mel_filterbank(SAMPLE_RATE, WINDOW_LENGTH, N_MELS, MEL_FMIN, MEL_FMAX, htk=True)


class RMVPE:
    """The reference's RMVPE (inference.py): RMVPE(model_path, hop_length=160) loads ``torch.load(model_path)['model']``
    into E2E0(4, 1, (2, 2)) with strict=False.  infer_from_audio(audio np.ndarray, sample_rate, device, thred,
    use_viterbi=False) -> f0 np.ndarray [n_frames] (hop_length samples at 16 kHz per frame).  infer_batch(audio [B, N]
    CUDA fp32, sample_rate, thred) -> f0 [B, n_frames] on the device, without syncs."""

    def __init__(self, model_path, hop_length=160):
        model = E2E0(4, 1, (2, 2))
        ckpt = torch.load(model_path, map_location="cpu")
        model.load_state_dict(ckpt["model"], strict=False)
        model.eval()
        self.model = model
        self.hop_length = hop_length
        self._lock = threading.Lock()
        self._tables = {}                                       # (rate or 'mel', device) -> device tables

    def _table(self, key, device, make):
        with self._lock:
            t = self._tables.get((key, device))
            if t is None:
                t = self._tables[(key, device)] = make()
            return t

    def _mel_tables(self, device):
        def make():
            basis = mel_basis()
            return (torch.hann_window(WINDOW_LENGTH, dtype=torch.float32).to(device),
                    torch.from_numpy(basis).to(device), torch.from_numpy(_support(basis)).to(device))
        return self._table("mel", device, make)

    def mel2hidden(self, mel):
        """mel [B, 128, n] -> salience [B, n, 360]: zero-padded to a multiple of 32 frames for the network, cropped"""
        with torch.no_grad():
            n = mel.shape[-1]
            pad = torch.zeros(*mel.shape[:-1], 32 * ((n - 1) // 32 + 1), dtype=torch.float32, device=mel.device)
            pad[..., :n] = mel
            return self.model(pad)[:, :n]

    def decode(self, hidden, thred=0.03, use_viterbi=False):
        """to_local_average_f0 of hidden [B, n, 360] -> np.ndarray (the batch dimension squeezed when B = 1)"""
        if use_viterbi:
            raise NotImplementedError("use_viterbi=True needs librosa.sequence.viterbi on the host; only the local "
                                      "average decode (use_viterbi=False) runs on the kernels")
        f0 = ops.rmvpe_decode(hidden.float().contiguous(), hidden.shape[1], thred)
        return f0.squeeze(0).cpu().numpy()

    def infer_batch(self, audio, sample_rate, thred=0.03):
        """audio [B, N] CUDA fp32 (equal-length clips at sample_rate) -> f0 [B, 1 + N16 // hop_length] (Hz, 0 where
        unvoiced) on the device, N16 the length at 16 kHz"""
        sal, n_frames = self.salience_batch(audio, sample_rate)
        return ops.rmvpe_decode(sal, n_frames, thred)

    def salience_batch(self, audio, sample_rate):
        """audio [B, N] CUDA fp32 -> (salience [B, T_pad, 360] of the frames padded to a multiple of 32, n_frames)"""
        if not (isinstance(audio, torch.Tensor) and audio.is_cuda):
            raise ValueError("RMVPE runs on the CUDA kernels: audio must be a CUDA tensor")
        if audio.dim() != 2:
            raise ValueError("audio must be [B, N], got %s" % (tuple(audio.shape),))
        sample_rate = int(sample_rate)
        if sample_rate <= 0:
            raise ValueError("sample_rate must be positive, got %r" % (sample_rate,))
        x = audio.float().contiguous()
        dev = x.device
        n16 = resampled_length(x.shape[1], sample_rate) if sample_rate != SAMPLE_RATE else x.shape[1]
        if n16 <= WINDOW_LENGTH // 2:
            raise ValueError("the audio at 16 kHz must be longer than %d samples (reflect padding of the STFT), got %d"
                             % (WINDOW_LENGTH // 2, n16))
        with torch.no_grad():
            if sample_rate != SAMPLE_RATE:
                def make():
                    k, width, orig, new = resample_table(sample_rate)
                    return k.to(dev), width, orig, new
                table, width, orig, new = self._table(sample_rate, dev, make)
                x = ops.rmvpe_resample(x, table, new, orig, width, n16)
            n_frames = 1 + n16 // self.hop_length
            t_pad = 32 * ((n_frames - 1) // 32 + 1)
            window, basis, lohi = self._mel_tables(dev)
            mel = ops.rmvpe_mel(x, window, basis, lohi, self.hop_length, t_pad)       # [B, t_pad, 128]
            if next(self.model.parameters()).device != dev:
                self.model.to(dev)                              # a warm call skips Module.to's walk over 700 tensors
            return self.model._salience(mel.unsqueeze(-1)), n_frames

    def infer_from_audio(self, audio, sample_rate=16000, device=None, thred=0.03, use_viterbi=False):
        if use_viterbi:
            raise NotImplementedError("use_viterbi=True needs librosa.sequence.viterbi on the host; only the local "
                                      "average decode (use_viterbi=False) runs on the kernels")
        device = torch.device("cuda" if device is None else device)
        if device.type != "cuda":
            raise ValueError("RMVPE runs on the CUDA kernels: device must be a CUDA device, got %s" % device)
        x = torch.from_numpy(np.asarray(audio)).float().unsqueeze(0).to(device)
        return self.infer_batch(x, sample_rate, thred).squeeze(0).cpu().numpy()

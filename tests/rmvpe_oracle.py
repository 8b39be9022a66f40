"""Plain-torch restatement of the RMVPE path (reference encoder/rmvpe/: inference.py:21-51, model.py:56-60,
deepunet.py, spec.py, utils.py:106-121) over the parameters of a ``ddsp_svc_b200.E2E0``, in any dtype and on any
device: float64 is the comparator of the GPU tests, fp32 on CUDA under torch's defaults (cuDNN TF32) is what the
reference runs and the eager arm of bench_rmvpe.py.  The host tables (resample taps, HTK mel basis) come from
ddsp_svc_b200.rmvpe; tests/test_oracle_rmvpe.py pins them against torchaudio."""
import torch
import torch.nn.functional as F

from ddsp_svc_b200 import rmvpe as R


def _bn(x, bn):
    return F.batch_norm(x, bn.running_mean.to(x), bn.running_var.to(x), bn.weight.to(x), bn.bias.to(x), False, 0.0,
                        bn.eps)


def _block(m, x):
    y = F.relu(_bn(F.conv2d(x, m.conv[0].weight.to(x), padding=1), m.conv[1]))
    y = F.relu(_bn(F.conv2d(y, m.conv[3].weight.to(x), padding=1), m.conv[4]))
    sc = F.conv2d(x, m.shortcut.weight.to(x), m.shortcut.bias.to(x)) if m.is_shortcut else x
    return y + sc


def salience(model, mel, dtype=torch.float64):
    """E2E0.forward: mel [B, 128, T] -> [B, T, 360] computed with model's parameters in dtype on mel's device"""
    x = mel.to(dtype).transpose(-1, -2).unsqueeze(1)
    u = model.unet
    x = _bn(x, u.encoder.bn)
    skips = []
    for layer in u.encoder.layers:
        for m in layer.conv:
            x = _block(m, x)
        skips.append(x)
        x = F.avg_pool2d(x, 2)
    for layer in u.intermediate.layers:
        for m in layer.conv:
            x = _block(m, x)
    for layer, skip in zip(u.decoder.layers, reversed(skips)):
        x = F.conv_transpose2d(x, layer.conv1[0].weight.to(x), stride=2, padding=1, output_padding=1)
        x = torch.cat((F.relu(_bn(x, layer.conv1[1])), skip), dim=1)
        for m in layer.conv2:
            x = _block(m, x)
    x = F.conv2d(x, model.cnn.weight.to(x), model.cnn.bias.to(x), padding=1)
    x = x.transpose(1, 2).flatten(-2)                     # [B, T, 3 128], feature c 128 + f
    g = model.fc[0].gru
    h = g(x)[0] if x.dtype == g.weight_ih_l0.dtype else gru(g, x)       # in the parameters' dtype: nn.GRU (cuDNN)
    return torch.sigmoid(F.linear(h, model.fc[1].weight.to(x), model.fc[1].bias.to(x)))


def gru(g, x):
    """bidirectional single-layer nn.GRU(batch_first) on x [B, T, I] as an explicit loop -> [B, T, 2 H]"""
    outs = []
    for sfx, rev in (("", False), ("_reverse", True)):
        w_ih, w_hh = getattr(g, "weight_ih_l0" + sfx).to(x), getattr(g, "weight_hh_l0" + sfx).to(x)
        b_ih, b_hh = getattr(g, "bias_ih_l0" + sfx).to(x), getattr(g, "bias_hh_l0" + sfx).to(x)
        xg = F.linear(x, w_ih, b_ih)
        H = w_hh.shape[1]
        h = x.new_zeros(x.shape[0], H)
        out = [None] * x.shape[1]
        for t in (reversed(range(x.shape[1])) if rev else range(x.shape[1])):
            hg = F.linear(h, w_hh, b_hh)
            r = torch.sigmoid(xg[:, t, :H] + hg[:, :H])
            z = torch.sigmoid(xg[:, t, H:2 * H] + hg[:, H:2 * H])
            n = torch.tanh(xg[:, t, 2 * H:] + r * hg[:, 2 * H:])
            h = (1 - z) * n + z * h
            out[t] = h
        outs.append(torch.stack(out, 1))
    return torch.cat(outs, -1)


def tables(sample_rate, dtype=torch.float64, device="cpu"):
    """the host tables of one sample rate on a device, built once as the reference builds them (Resample cached per
    rate, MelSpectrogram's basis in __init__, its window cached per device): resample (table, width, orig, new) or
    None at 16 kHz, the Hann window and the HTK mel basis"""
    rs = None
    if sample_rate != R.SAMPLE_RATE:
        table, width, orig, new = R.resample_table(sample_rate)
        rs = (table.to(device=device, dtype=dtype), width, orig, new)
    return dict(rate=sample_rate, resample=rs, window=torch.hann_window(R.WINDOW_LENGTH, dtype=dtype, device=device),
                basis=torch.from_numpy(R.mel_basis()).to(device=device, dtype=dtype))


def resample(audio, sample_rate, dtype=torch.float64, tabs=None):
    """torchaudio Resample(sample_rate, 16000, lowpass_filter_width=128) of audio [B, N]: conv1d with the table"""
    if sample_rate == R.SAMPLE_RATE:
        return audio.to(dtype)
    tabs = tabs or tables(sample_rate, dtype, audio.device)
    table, width, orig, new = tabs["resample"]
    n = audio.shape[-1]
    x = F.pad(audio.to(dtype), (width, width + orig))
    y = F.conv1d(x[:, None], table.to(x)[:, None], stride=orig)
    return y.transpose(1, 2).reshape(audio.shape[0], -1)[:, :R.resampled_length(n, sample_rate)]


def log_mel(audio16, hop_length=160, dtype=torch.float64, tabs=None):
    """spec.py MelSpectrogram(128, 16000, 1024, hop, None, 30, 8000).forward(audio, center=True) -> [B, 128, n]"""
    x = audio16.to(dtype)
    tabs = tabs or tables(R.SAMPLE_RATE, dtype, x.device)
    s = torch.stft(x, R.WINDOW_LENGTH, hop_length, R.WINDOW_LENGTH, tabs["window"].to(x), center=True,
                   return_complex=True)
    mag = torch.sqrt(s.real.pow(2) + s.imag.pow(2))
    return torch.log(torch.clamp(torch.matmul(tabs["basis"].to(x), mag), min=1e-5))


def mel2hidden(model, mel, dtype=torch.float64):
    n = mel.shape[-1]
    mel = F.pad(mel.to(dtype), (0, 32 * ((n - 1) // 32 + 1) - n))
    return salience(model, mel, dtype)[:, :n]


def decode(hidden, thred=0.03):
    """to_local_average_f0 without the final .cpu().numpy(): hidden [B, T, 360] -> f0 [B, T] (hidden's dtype)"""
    idx = torch.arange(R.N_CLASS, device=hidden.device)[None, None, :]
    cents_map = idx * 20 + 1997.3794084376191
    center = torch.argmax(hidden, dim=2, keepdim=True)
    mask = (idx >= torch.clip(center - 4, min=0)) & (idx < torch.clip(center + 5, max=R.N_CLASS))
    w = hidden * mask
    ps, ws = torch.sum(w * cents_map.to(hidden.dtype), dim=2), torch.sum(w, dim=2)
    f0 = 10 * 2 ** ((ps / (ws + (ws == 0))) / 1200)
    return f0 * ~(hidden.max(dim=2)[0] < thred)


def constructed_saliences():
    """[12, 360] saliences at the decode's edge cases"""
    g = torch.Generator().manual_seed(24)
    s = 0.2 * torch.rand(12, 360, generator=g)
    s[0, 100] = s[0, 103] = 0.9                              # a tie: the first index wins
    for i, c in enumerate((0, 1, 2, 3)):
        s[1 + i, c] = 0.95                                   # peaks at the low edge
    for i, c in enumerate((356, 357, 358, 359)):
        s[5 + i, c] = 0.95                                   # and at the high edge
    s[9] = 0.01 * torch.rand(360, generator=g)               # below the threshold
    s[10] = 0.01 * torch.rand(360, generator=g)
    s[10, 200] = 0.03                                        # exactly at the threshold: voiced
    s[11] = 0.0                                              # all zero: weight_sum 0
    return s


def infer(model, audio, sample_rate, hop_length=160, thred=0.03, dtype=torch.float64, tabs=None):
    """RMVPE.infer_from_audio on a batch audio [B, N] -> (f0 [B, n], salience [B, n, 360]); ``tabs`` (tables() of
    sample_rate, dtype and audio's device) keeps the host tables out of the call, as the reference keeps them"""
    tabs = tabs or tables(sample_rate, dtype, audio.device)
    mel = log_mel(resample(audio, sample_rate, dtype, tabs), hop_length, dtype, tabs)
    hidden = mel2hidden(model, mel, dtype)
    return decode(hidden, thred), hidden


def calibrate(model, seed=0, frames=64, batch=2):
    """Seeded weights leave BatchNorm at (mean 0, var 1), and the residual sums then grow through every block until
    the sigmoid saturates.  One train-mode forward of the reference's own modules with momentum=None (a cumulative
    average, here of one batch) on a seeded log-mel batch sets each BatchNorm to the statistics it sees; then eval()."""
    g = torch.Generator().manual_seed(seed)
    mel = torch.randn(batch, R.N_MELS, frames, generator=g, dtype=torch.float64) - 4.0
    model.double()
    bns = [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    for m in bns:
        m.reset_running_stats()
        m.momentum = None
    model.train()
    with torch.no_grad():
        x = mel.transpose(-1, -2).unsqueeze(1)
        u = model.unet
        x = u.encoder.bn(x)
        skips = []
        for layer in u.encoder.layers:
            for m in layer.conv:
                x = m.conv(x) + (m.shortcut(x) if m.is_shortcut else x)
            skips.append(x)
            x = F.avg_pool2d(x, 2)
        for layer in u.intermediate.layers:
            for m in layer.conv:
                x = m.conv(x) + (m.shortcut(x) if m.is_shortcut else x)
        for layer, skip in zip(u.decoder.layers, reversed(skips)):
            x = torch.cat((layer.conv1(x), skip), dim=1)
            for m in layer.conv2:
                x = m.conv(x) + (m.shortcut(x) if m.is_shortcut else x)
    for m in bns:
        m.momentum = 0.01
    model.eval()
    return model.float()


def seeded_model(n_blocks=4, en_de_layers=5, inter_layers=4, seed=0):
    """E2E0 with seeded weights (default init under torch.manual_seed) and calibrated BatchNorm statistics"""
    torch.manual_seed(seed)
    m = R.E2E0(n_blocks, 1, (2, 2), en_de_layers=en_de_layers, inter_layers=inter_layers)
    for bn in (x for x in m.modules() if isinstance(x, torch.nn.BatchNorm2d)):
        with torch.no_grad():
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.2, 0.2)
    return calibrate(m, seed + 1)

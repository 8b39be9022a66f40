"""Named, seeded input regimes for the synthesizers, and the references the regime tests compare against.

TEST INFRASTRUCTURE ONLY.  ``ddsp_svc_b200.synthetic`` draws one distribution (110-440 Hz with vibrato, magnitudes
N(-2, 0.5) / N(-3, 0.5), phase-like controls N(0, 0.3)): a benchmark workload.  The raw controls come out of an
unbounded Linear and the pitch out of a tracker, so the domain is wider; the regimes here name the corners of it where
the kernels' arithmetic changes character (range reduction of sin/cos, exp near overflow and underflow, tanh
saturation, sinc gain sr / f0, the Nyquist mask, the dynamic window's half width, unvoiced runs).

Pitch regimes   ``PITCH[name](B, nF, seed) -> f0_frames [B, nF, 1]`` fp32 Hz
  low           30-64 Hz per row with vibrato: dynamic window wider than the impulse response, comb gain sr / f0 ~ 1400
  high          1100-2000 Hz: most of 128 harmonics above Nyquist, a handful of window taps
  octave_jumps  a melody whose frames jump to 2f or f/2 at random frames (tracker octave errors)
  onsets        voiced / unvoiced RUNS of 1-40 frames that start and end unvoiced; row 1 wholly unvoiced; row 2
                alternating every frame
  glide         portamento of 2 octaves per second up and down between 110 and 440 Hz
  near_zero     a melody with voiced frames of 1e-3 .. 5 Hz mixed in (extractor garbage that is not exactly 0)

Control regimes ``CTRL[name](B, nF, split_map, seed) -> (dense [B, nF, n_out], views)``, the layout of
``synthetic.make_ctrl``; a control a regime does not name keeps make_ctrl's distribution
  trained       magnitudes with a spectral tilt across bins (-1 -> -9) plus N(0, 1.5), clipped to [-15, 4]; phase-like
                controls N(0, 1)
  phase_turns   phase-like controls = a per-frame linear ramp across bins reaching +-64 (a pure delay; exp(j pi p) then
                passes 30 turns) plus N(0, 4)
  saturated_gd  group_delay in +-[3, 30] with one sign for ~97 % of a frame's bins, so tanh is +-1 and the cumulative
                phase passes 700 rad; a synthesizer without an all-pass gets these values in its phase controls
  hot / cold    every magnitude control +4 / -20
  mixed_rows    row 0 cold, row 1 hot: a read across a row boundary is 1e10 wrong instead of 1 % wrong

Not covered: NaN, infinite or negative f0 and non-finite controls.  The reference's result there is an accident of
its operators, not a specification.
"""
import math
import zlib
from collections import OrderedDict

import numpy as np
import torch

from ddsp_svc_b200 import synthetic as syn
from oracle import closed_form as cf
from oracle import torch_port as tp

SR, P, WIN = 44100, 512, 2048
MAGNITUDES = ("amplitudes", "harmonic_magnitude", "noise_magnitude")
PHASES = ("group_delay", "harmonic_phase", "noise_phase")


def _gen(seed):
    return torch.Generator().manual_seed(int(seed))


def _vibrato(nF):
    k = torch.arange(nF, dtype=torch.float64)
    return 1.0 + 0.03 * torch.sin(2.0 * math.pi * 5.5 * k * P / SR)


def _melody(B, nF, g, lo=110.0, hi=440.0):
    u = torch.rand(B, generator=g, dtype=torch.float64)
    return (lo * (hi / lo) ** u)[:, None] * _vibrato(nF)[None, :]


def _frames(f0):
    return f0.to(torch.float32).unsqueeze(-1).contiguous()


# ------------------------------------------------------------------------------------------------ pitch
def low(B, nF, seed=0):
    return _frames(_melody(B, nF, _gen(seed), 31.0, 62.0))


def high(B, nF, seed=0):
    return _frames(_melody(B, nF, _gen(seed), 1135.0, 1940.0))


def octave_jumps(B, nF, seed=0):
    g = _gen(seed)
    f = _melody(B, nF, g)
    jump = torch.rand(B, nF, generator=g) < 0.2
    up = torch.rand(B, nF, generator=g) < 0.5
    jump[:, min(2, nF - 1)] = True
    return _frames(f * torch.where(jump, torch.where(up, 2.0, 0.5), 1.0).double())


def _runs(nF, g):
    """voiced mask of one row: runs of 1-40 frames, unvoiced first and last; the first voiced run is >= 20 frames
    when the row has room for it"""
    voiced = torch.zeros(nF, dtype=torch.bool)
    pos, state, first = 0, False, True
    while pos < nF:
        n = int(torch.randint(1, 41, (1,), generator=g))
        if state and first:
            n, first = (20 + n % 21 if nF >= 32 else n), False
        if not state and pos == 0:
            n = 1 + n % 4
        voiced[pos:pos + n] = state
        pos, state = pos + n, not state
    voiced[-1] = False
    return voiced


def onsets(B, nF, seed=0):
    g = _gen(seed)
    f = _melody(B, nF, g)
    for b in range(B):
        if b == 1:
            voiced = torch.zeros(nF, dtype=torch.bool)
        elif b == 2:
            voiced = torch.arange(nF) % 2 == 1
            voiced[-1] = False
        else:
            voiced = _runs(nF, g)
        f[b] = torch.where(voiced, f[b], torch.zeros((), dtype=torch.float64))
    return _frames(f)


def glide(B, nF, seed=0):
    g = _gen(seed)
    t = torch.arange(nF, dtype=torch.float64) * P / SR
    start = 4.0 * torch.rand(B, generator=g, dtype=torch.float64)
    pos = torch.remainder(start[:, None] + 2.0 * t[None, :], 4.0)          # 2 octaves per second
    return _frames(110.0 * 2.0 ** (2.0 - (pos - 2.0).abs()))


def near_zero(B, nF, seed=0):
    g = _gen(seed)
    f = _melody(B, nF, g)
    junk = 10.0 ** (-3.0 + (3.0 + math.log10(5.0)) * torch.rand(B, nF, generator=g, dtype=torch.float64))
    m = torch.rand(B, nF, generator=g) < 0.15
    m[0, min(1, nF - 1)] = True
    junk[0, min(1, nF - 1)] = 1e-3
    return _frames(torch.where(m, junk, f))


PITCH = OrderedDict((f.__name__, f) for f in (low, high, octave_jumps, onsets, glide, near_zero))


def check_pitch(name, f0):
    """the regime is what it says (raises AssertionError otherwise)"""
    f = f0[..., 0].double()
    assert f0.dtype == torch.float32 and f0.dim() == 3 and f0.shape[-1] == 1
    assert torch.isfinite(f).all() and (f >= 0).all()
    d = (f[:, 1:] - f[:, :-1]).abs()
    if name == "low":
        assert 30.0 <= f.min() and f.max() <= 64.0
    elif name == "high":
        assert 1100.0 <= f.min() and f.max() <= 2000.0
    elif name == "octave_jumps":
        ratio = f[:, 1:] / f[:, :-1]
        assert ((ratio > 1.8) | (ratio < 0.56)).any() and d.max() > 100.0
    elif name == "onsets":
        v = f > 0
        assert not v[:, 0].any() and not v[:, -1].any()
        longest, run = 0, 0
        for x in v[0].tolist():
            run = run + 1 if x else 0
            longest = max(longest, run)
        assert longest >= 20, longest
        assert not v[1].any()
        assert (v[2, 1:-1] != v[2, :-2]).all()
    elif name == "glide":
        octaves_per_s = (torch.log2(f[:, 1:] / f[:, :-1]).abs() * SR / P)
        assert 1.9 < octaves_per_s.median() < 2.1 and 110.0 <= f.min() and f.max() <= 440.0
    elif name == "near_zero":
        assert 0 < f.min() <= 1e-3 * 1.0001 and ((f > 0) & (f <= 5.0)).sum() >= 2 and f.max() > 100.0
    else:
        raise KeyError(name)


# ------------------------------------------------------------------------------------------------ controls
def _fill(B, nF, split_map, seed, fn):
    """make_ctrl's tensor with the splits ``fn(name, width, g)`` returns a value for overwritten"""
    dense, views = syn.make_ctrl(B, nF, split_map, seed=seed)
    g = _gen(seed + 17)
    for name, width in split_map.items():
        v = fn(name, width, g)
        if v is not None:
            views[name].copy_(v)
    return dense, views


def trained(B, nF, split_map, seed=0):
    def fn(name, width, g):
        if name in MAGNITUDES:
            tilt = torch.linspace(-1.0, -9.0, width)
            return (tilt + 1.5 * torch.randn(B, nF, width, generator=g)).clamp(-15.0, 4.0)
        return torch.randn(B, nF, width, generator=g)
    return _fill(B, nF, split_map, seed, fn)


def phase_turns(B, nF, split_map, seed=0):
    def fn(name, width, g):
        if name not in PHASES:
            return None
        top = 64.0 * (0.5 + 0.5 * torch.rand(B, nF, 1, generator=g))
        top = top * torch.where(torch.rand(B, nF, 1, generator=g) < 0.5, -1.0, 1.0)
        top[:, 0], top[:, -1] = 64.0, -64.0
        return top * torch.linspace(0.0, 1.0, width) + 4.0 * torch.randn(B, nF, width, generator=g)
    return _fill(B, nF, split_map, seed, fn)


def saturated_gd(B, nF, split_map, seed=0):
    targets = ("group_delay",) if "group_delay" in split_map else PHASES

    def fn(name, width, g):
        if name not in targets:
            return None
        frame_sign = torch.where(torch.rand(B, nF, 1, generator=g) < 0.5, -1.0, 1.0)
        flip = torch.where(torch.rand(B, nF, width, generator=g) < 0.97, 1.0, -1.0)
        return frame_sign * flip * (3.0 + 27.0 * torch.rand(B, nF, width, generator=g))
    return _fill(B, nF, split_map, seed, fn)


def _level(rows):
    def regime(B, nF, split_map, seed=0):
        def fn(name, width, g):
            if name not in MAGNITUDES:
                return None
            v = None
            for row, level in rows(B):
                if v is None:
                    v = syn.CTRL_STATS[name][0] + syn.CTRL_STATS[name][1] * torch.randn(B, nF, width, generator=g)
                v[row] = level
            return v
        return _fill(B, nF, split_map, seed, fn)
    return regime


hot = _level(lambda B: [(b, 4.0) for b in range(B)])
cold = _level(lambda B: [(b, -20.0) for b in range(B)])
mixed_rows = _level(lambda B: [(0, -20.0), (1, 4.0)])
CTRL = OrderedDict([("trained", trained), ("phase_turns", phase_turns), ("saturated_gd", saturated_gd),
                    ("hot", hot), ("cold", cold), ("mixed_rows", mixed_rows)])


def check_ctrl(name, views):
    """the regime is what it says (raises AssertionError otherwise)"""
    mags = [v for k, v in views.items() if k in MAGNITUDES]
    phases = [v for k, v in views.items() if k in PHASES]
    assert all(torch.isfinite(v).all() for v in views.values())
    if name == "trained":
        for v in mags:
            assert -15.0 <= v.min() and v.max() <= 4.0 and v.max() - v.min() > 12.0
            assert v[..., :8].mean() - v[..., -8:].mean() > 6.0            # the tilt
        assert all(0.9 < v.std() < 1.1 for v in phases)
    elif name == "phase_turns":
        assert phases and all(v.abs().max() / 2.0 > 30.0 for v in phases)  # exp(j pi p): p / 2 turns
    elif name == "saturated_gd":
        v = views["group_delay"] if "group_delay" in views else views["harmonic_phase"]
        assert 3.0 <= v.abs().min() and v.abs().max() <= 30.0
        assert (math.pi * torch.tanh(v.double())).cumsum(-1).abs().max() > 700.0
    elif name == "hot":
        assert all((v == 4.0).all() for v in mags)
    elif name == "cold":
        assert all((v == -20.0).all() for v in mags)
    elif name == "mixed_rows":
        assert all((v[0] == -20.0).all() and (v[1] == 4.0).all() for v in mags)
    else:
        raise KeyError(name)


# ------------------------------------------------------------------------------------------------ the table
SPLITS = OrderedDict([("sins", syn.sins_split_map()), ("combsub", syn.combsub_split_map()),
                      ("combsubfast", syn.combsubfast_split_map(P)), ("superfast", syn.superfast_split_map(WIN))])
HAS_PARTS = ("sins", "combsub")          # return (signal, harmonic, noise); the other two a signal only
HAS_INFER = ("sins", "combsub", "combsubfast")
# pairwise: every pitch regime twice, every control regime twice, the same pairs for every synthesizer
TABLE = [("low", "trained"), ("low", "saturated_gd"), ("high", "phase_turns"), ("high", "cold"),
         ("octave_jumps", "saturated_gd"), ("octave_jumps", "hot"), ("onsets", "mixed_rows"), ("onsets", "trained"),
         ("glide", "hot"), ("glide", "phase_turns"), ("near_zero", "cold"), ("near_zero", "mixed_rows")]
CASE_IDS = ["%s-%s" % pc for pc in TABLE]


def build(synth, pitch, ctrl, with_cotangents=False):
    """seeded inputs of one table entry: f0, dense controls + views, explicit noise (and cotangents)"""
    B, nF = (3, 48) if pitch == "onsets" else (2, 24)
    seed = zlib.crc32(("%s/%s/%s" % (synth, pitch, ctrl)).encode()) % (2 ** 31)
    f0 = PITCH[pitch](B, nF, seed)
    dense, views = CTRL[ctrl](B, nF, SPLITS[synth], seed + 1)
    g = _gen(seed + 2)
    T = nF * P
    # Sins / CombSub / CombSubFast draw uniform noise, CombSubSuperFast normal noise (ddsp/vocoder.py:603, :687)
    noise = torch.randn(B, T, generator=g) if synth == "superfast" else torch.rand(B, T, generator=g) * 2 - 1
    inp = {"synth": synth, "B": B, "nF": nF, "f0": f0, "dense": dense, "ctrls": views, "noise": noise}
    if with_cotangents:
        inp["cot"] = torch.randn(B, T, generator=g)
        if synth in HAS_PARTS:
            inp["cot_h"], inp["cot_n"] = torch.randn(B, T, generator=g), torch.randn(B, T, generator=g)
    return inp


# ------------------------------------------------------------------------------------------------ references
def _np(d):
    return {k: v.detach().numpy() for k, v in d.items()}


def truth_forward(inp):
    """float64 closed form: {'signal' (and 'harmonic', 'noise')} as numpy [B, T]"""
    s, f0, c, nz = inp["synth"], inp["f0"].numpy(), _np(inp["ctrls"]), inp["noise"].numpy()
    if s == "sins":
        return cf.sins(f0, c, SR, P, nz)
    if s == "combsub":
        return cf.combsub(f0, c, SR, P, nz)
    if s == "combsubfast":
        return cf.combsubfast(f0, c, SR, P, nz)
    return cf.superfast(f0, c, SR, P, WIN, nz)


def port_forward(inp, infer=True, ctrls=None):
    """the reference's own fp32 arithmetic (oracle.torch_port on the CPU): dict of torch tensors"""
    s, f0, nz = inp["synth"], inp["f0"], inp["noise"]
    c = inp["ctrls"] if ctrls is None else ctrls
    if s == "sins":
        return tp.sins_forward(f0, c, SR, P, noise=nz, infer=infer)
    if s == "combsub":
        return tp.combsub_forward(f0, c, SR, P, noise=nz, infer=infer)
    if s == "combsubfast":
        return tp.combsubfast_forward(f0, c, SR, P, noise=nz, infer=infer)
    return tp.superfast_forward(f0, c, SR, P, WIN, noise=nz)


def outputs_of(synth):
    return ("signal", "harmonic", "noise") if synth in HAS_PARTS else ("signal",)


def rms_rows(a):
    """[B, ...] -> per-row RMS, float64"""
    a = np.asarray(a, np.float64)
    return np.sqrt(np.mean(np.square(a.reshape(a.shape[0], -1)), axis=1))


def max_rows(a):
    a = np.asarray(a, np.float64)
    return np.abs(a.reshape(a.shape[0], -1)).max(axis=1)


def floor_rows(truth):
    """absolute RMS floor per row: the suite's 2e-6 gate at its signal RMS of 0.01, scaled up with the signal"""
    return 2e-6 * np.maximum(1.0, rms_rows(truth) / 0.01)


def forward_errors(got, ref32, truth):
    """per-row (rms, max) errors of ``got`` and of the fp32 reference against the float64 truth, and the floor"""
    got, ref32, truth = (np.asarray(a, np.float64) for a in (got, ref32, truth))
    return {"got_rms": rms_rows(got - truth), "ref_rms": rms_rows(ref32 - truth), "floor": floor_rows(truth),
            "got_max": max_rows(got - truth), "ref_max": max_rows(ref32 - truth), "truth_rms": rms_rows(truth)}


def within_budget(e, rms_factor, max_factor, crest=8.0):
    """err(got, truth) <= max(floor, factor * err(ref32, truth)) for every row, in RMS and (looser, the floor times
    ``crest``) in max-abs; returns the list of violations"""
    bad = []
    for b in range(len(e["floor"])):
        lim = max(e["floor"][b], rms_factor * e["ref_rms"][b])
        if not e["got_rms"][b] <= lim:
            bad.append(("rms", b, e["got_rms"][b], lim))
        lim = max(crest * e["floor"][b], max_factor * e["ref_max"][b])
        if not e["got_max"][b] <= lim:
            bad.append(("max", b, e["got_max"][b], lim))
    return bad


def summary(e):
    """worst row of each error, for tests.report.record"""
    return {"gpu_vs_truth": e["got_rms"].max(), "ref32_vs_truth": e["ref_rms"].max(), "floor": e["floor"].min(),
            "gpu_vs_truth_max": e["got_max"].max(), "ref32_vs_truth_max": e["ref_max"].max(),
            "truth_rms": e["truth_rms"].max(),
            "ratio": float(np.max(e["got_rms"] / np.maximum(e["floor"], e["ref_rms"])))}


def truth_grad(inp, only=None):
    """float64 closed-form gradient of sum(signal cot + harmonic cot_h + noise cot_n) with respect to the raw
    controls at the exact (float64) source; ``only``: 'harmonic' / 'noise' keeps that output's cotangent alone"""
    from tests import combsub_grad_closed_form as cg
    from tests import combsubfast_grad_closed_form as cfg
    from tests import sins_grad_closed_form as sg
    from tests import superfast_grad_closed_form as sfg
    s, f0, c, nz = inp["synth"], inp["f0"].numpy(), _np(inp["ctrls"]), inp["noise"].numpy()
    cot, cot_h, cot_n = cotangents(inp, only)
    npc = lambda t: None if t is None else t.numpy()
    if s == "sins":
        x32 = cf.phase_cycles(f0, SR, P).astype(np.float32)
        return sg.sins_grad(f0, c, x32, SR, P, nz, npc(cot), npc(cot_h), npc(cot_n), reference_rounding=False)
    if s == "combsub":
        return cg.combsub_grad(f0, c, truth_forward(inp)["comb"], SR, P, nz, npc(cot), npc(cot_h), npc(cot_n))
    if s == "combsubfast":
        return cfg.combsubfast_grad(truth_forward(inp)["comb"], c, P, nz, npc(cot))
    return sfg.superfast_grad(f0, c, SR, P, WIN, nz, npc(cot), comb=truth_forward(inp)["comb"])


def cotangents(inp, only=None):
    """(cot, cot_h, cot_n) of (signal, harmonic, noise); zero tensors where ``only`` switches an output off"""
    z = torch.zeros_like(inp["cot"])
    if inp["synth"] not in HAS_PARTS:
        return inp["cot"], None, None
    if only == "harmonic":
        return z, inp["cot_h"], z
    if only == "noise":
        return z, z, inp["cot_n"]
    return inp["cot"], inp["cot_h"], inp["cot_n"]


def objective(out, inp, only=None):
    cot, cot_h, cot_n = (None if t is None else t.to(out["signal"].device) for t in cotangents(inp, only))
    loss = (out["signal"] * cot).sum()
    if cot_h is not None:
        loss = loss + (out["harmonic"] * cot_h).sum() + (out["noise"] * cot_n).sum()
    return loss


def port_grad(inp, only=None):
    """torch autograd through oracle.torch_port in fp32 (training phase): {control: numpy [B, nF, C]}"""
    leaf = inp["dense"].clone().requires_grad_(True)
    split = SPLITS[inp["synth"]]
    objective(port_forward(inp, infer=False, ctrls=syn.split_views(leaf, split)), inp, only).backward()
    return _np(syn.split_views(leaf.grad, split))


GRAD_FLOOR = 1e-5                  # relative: 1.5 single-precision transforms per frame (the CombSubFast TIGHT bound)
GRAD_NEGLIGIBLE = 1e-12            # a group this far below the largest group is held to an absolute bound


def grad_errors(got, ref32, truth):
    """per control group and per ROW (so that a cold row is not hidden behind a hot one): relative L2 error of ``got``
    and of the fp32 reference against the float64 truth, as arrays over the rows.  Where the true gradient of a group
    is below GRAD_NEGLIGIBLE of the row's largest group the errors are absolute, in units of that largest group."""
    rows = lambda a: np.sqrt(np.sum(np.square(np.asarray(a, np.float64).reshape(len(a), -1)), axis=1))
    norm = {k: rows(truth[k]) for k in truth}
    top = np.maximum(np.max([norm[k] for k in truth], axis=0), 1e-300)
    out = {}
    for k in truth:
        relative = norm[k] > GRAD_NEGLIGIBLE * top
        scale = np.where(relative, norm[k], top)
        out[k] = {"got": rows(np.asarray(got[k], np.float64) - truth[k]) / scale,
                  "ref": rows(np.asarray(ref32[k], np.float64) - truth[k]) / scale, "norm": norm[k],
                  "relative": relative}
    return out


def grad_bound(e, factor):
    """per row: max(GRAD_FLOOR, factor x the fp32 reference's error), or the absolute bound"""
    return np.where(e["relative"], np.maximum(GRAD_FLOOR, factor * e["ref"]), GRAD_NEGLIGIBLE)

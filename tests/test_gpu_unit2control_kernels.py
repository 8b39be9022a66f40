"""Each CUDA entry point of the control network (csrc/unit2control.cu, csrc/linear_attention.cu) called on its own
through the C ABI and compared with a float64 restatement of the same formula, at the shapes where the kernels change
code path: T = 1 and 2, T on both sides of the 64-frame tiles, sizes past the grid-stride caps (taken from the device's
SM count), n % 4 != 0 tails, every feature count the kernels accept.  Kernel errors that a later LayerNorm absorbs or
the attention normaliser cancels show up here, where they do not at the module's output.

Error model.  u = 2^-24, the unit roundoff of fp32.  Each bound in the docstrings below counts the roundings of the
kernel's fp32 chain: an fp32 sum of n terms is within n u of their l1 norm, expf / rsqrtf are within 2 ulp (4 u) and
logf within 1 ulp (CUDA C Programming Guide, mathematical functions, without fast-math).  A bound is a worst case, not
a fit to measurements; the measured errors go to tests/report.record next to it.

Bitwise assertions are used where the kernels give a reason for identical bits: the TF32 split is integer arithmetic
on the bit pattern; every kernel except GroupNorm computes each row (token, utterance or (utterance, head)) from that
row's inputs alone, in an order that does not depend on the batch, so a row of a batch equals the same row run alone
and two identical calls give identical bits.  GroupNorm adds its per-CTA partial sums with fp64 atomics, in no fixed
order, and is held to 1 ulp instead."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from ddsp_svc_b200 import _lib
from tests import report
from tests import test_gpu_kernel_variants as V

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
F64 = torch.float64


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _call(name, *args):
    lib = _lib.lib()
    rc = getattr(lib, name)(*args, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, "%s -> %d: %s" % (name, rc, lib.b2d_last_error())
    torch.cuda.synchronize()


def _bits(t):
    return t.detach().cpu().contiguous().numpy().view(np.uint32)


def _assert_same_bits(a, b, what):
    ba, bb = _bits(a), _bits(b)
    bad = np.flatnonzero(ba.reshape(-1) != bb.reshape(-1))
    assert bad.size == 0, "%s: %d elements differ, first at flat index %d" % (what, bad.size, bad[0])


def _check(name, err, bound, **extra):
    """err, bound: float64 tensors of the same shape -> assert err <= bound everywhere; records the worst ratio."""
    assert torch.isfinite(err).all(), name
    ratio = (err / bound).max().item()
    report.record("u2c_kernels/" + name, max_err=err.max().item(), max_err_over_bound=ratio, **extra)
    assert ratio <= 1.0, "%s: error reaches %.3g x its bound" % (name, ratio)


# ---------------------------------------------------------------------------------------------------------------------
# b2d_split_tf32
# ---------------------------------------------------------------------------------------------------------------------
TF32_NAN = 0x7FFFE000
SPECIAL_BITS = [
    0x00000000, 0x80000000,                          # +-0
    0x00000001, 0x80000001, 0x00001000, 0x00003000,  # denormals: the smallest, and ties at the TF32 cut (even / odd)
    0x00401FFF, 0x807FFFFF,                          # denormals with all dropped bits set
    0x3F001000, 0x3F003000, 0x3F001001, 0xBF003000,  # 0.5 + 2^-12, 0.5 + 3 2^-12 (ties to even), just above a tie
    0x3FFFFFFF, 0x3F7FF000, 0xBFFFFFFF,              # all-ones mantissas whose rounding carries into the exponent
    0x7F800000, 0xFF800000,                          # +-inf
    0x7FC00000, 0x7FFFFFFF, 0xFFFFFFFF, 0x7F800001,  # NaNs: x86 default, the device's canonical NaN, payload in low bits
    0x7F7FE000, 0x7F7FEFFF,                          # the largest TF32 value, and the largest value rounding to it
    0x7F7FF000, 0x7F7FFFFF, 0xFF7FFFFF,              # (2 - 2^-11) 2^127 and above: hi rounds to inf
]


def split_model(x):
    """tests/test_gpu_kernel_variants.split_tf32 (round to nearest even on the 13 dropped bits, lo = split of x - hi),
    with the kernel's rules for non-finite inputs: a NaN gives the TF32 quiet NaN 0x7FFFE000 in both halves, +-inf gives
    (+-inf, +0).  A finite value at or above the overflow threshold (2 - 2^-11) 2^127 rounds to hi = +-inf, and
    lo = split(x - hi) = -+inf: hi + lo is NaN there.  That is what the kernel does, and what this model pins."""
    x = np.asarray(x, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        hi, lo = V.split_tf32(x)
    hb, lb = hi.view(np.uint32), lo.view(np.uint32)
    nan, inf = np.isnan(x), np.isinf(x)
    hb[nan] = TF32_NAN
    lb[nan] = TF32_NAN
    lb[inf] = 0
    return hi, lo


def _split_sizes():
    cap4 = 16 * _sms() * 256                          # float4 per launch before the grid-stride loop repeats
    return [1, 2, 3, 4, 5, 7, 1021, 4 * (2 * cap4 + 5) + 3]


@pytest.mark.parametrize("which", range(8))
def test_split_tf32_matches_the_bit_model(which):
    """hi and lo equal split_model bit for bit, at every size class: a lone tail (n < 4), a multiple of 4, float4 body +
    tail, and n past 16 SMs x 256 float4, where the grid-stride loop runs more than once, with a tail of 3.  The values
    are random bit patterns (every exponent, NaNs, infinities, denormals) and random normals, with SPECIAL_BITS written
    at the start and at the end, so they land both in the float4 body and in the scalar tail."""
    n = _split_sizes()[which]
    rng = np.random.default_rng(100 + which)
    bits = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    normal = rng.standard_normal(n).astype(np.float32).view(np.uint32)
    bits = np.where(np.arange(n) % 2 == 0, bits, normal)
    sp = np.array(SPECIAL_BITS, np.uint32)
    k = min(n, sp.size)
    bits[:k] = sp[:k]
    bits[n - k:] = sp[sp.size - k:]
    x = bits.view(np.float32)
    xt = torch.from_numpy(x).to(DEV)
    hi, lo = torch.empty_like(xt), torch.empty_like(xt)
    _call("b2d_split_tf32", xt.data_ptr(), hi.data_ptr(), lo.data_ptr(), n)
    want_hi, want_lo = split_model(x)
    bh, bl = _bits(hi), _bits(lo)
    bad = np.flatnonzero((bh != want_hi.view(np.uint32)) | (bl != want_lo.view(np.uint32)))
    report.record("u2c_kernels/split_tf32/n=%d" % n, mismatches=bad.size)
    assert bad.size == 0, "n = %d: %d mismatches, first x = 0x%08X -> (0x%08X, 0x%08X), want (0x%08X, 0x%08X)" % (
        n, bad.size, bits[bad[0]], bh[bad[0]], bl[bad[0]], want_hi.view(np.uint32)[bad[0]], want_lo.view(np.uint32)[bad[0]])


def test_split_tf32_pins_the_edge_values():
    """The values behind split_model's rules, spelled out: RNE ties go to even, a carry reaches the exponent, NaN stays
    NaN (the device's canonical NaN 0x7FFFFFFF included), inf splits into (inf, +0), and above the TF32 overflow
    threshold hi = inf, lo = -inf."""
    want = {0x3F001000: (0x3F000000, 0x39800000), 0x3F003000: (0x3F004000, 0xB9800000), 0x3FFFFFFF: (0x40000000, 0xB4000000),
            0x7FFFFFFF: (TF32_NAN, TF32_NAN), 0x7F800001: (TF32_NAN, TF32_NAN), 0xFF800000: (0xFF800000, 0),
            0x7F7FEFFF: (0x7F7FE000, 0x79800000), 0x7F7FF000: (0x7F800000, 0xFF800000), 0xFF7FFFFF: (0xFF800000, 0x7F800000)}
    x = np.array(list(want), np.uint32).view(np.float32)
    xt = torch.from_numpy(x).to(DEV)
    hi, lo = torch.empty_like(xt), torch.empty_like(xt)
    _call("b2d_split_tf32", xt.data_ptr(), hi.data_ptr(), lo.data_ptr(), x.size)
    got = list(zip(_bits(hi).tolist(), _bits(lo).tolist()))
    assert got == list(want.values())
    mh, ml = split_model(x)
    assert list(zip(mh.view(np.uint32).tolist(), ml.view(np.uint32).tolist())) == list(want.values())


# ---------------------------------------------------------------------------------------------------------------------
# b2d_u2c_embed
# ---------------------------------------------------------------------------------------------------------------------
def _embed_inputs(B, T, seed):
    g = np.random.default_rng(seed)
    n = B * T
    f0 = g.uniform(50.0, 1100.0, n)
    f0[::5] = 0.0                                     # unvoiced
    f0[1::7] = 1099.9
    phase = g.uniform(-math.pi, math.pi, n)
    phase[2::9], phase[3::9] = math.pi, -math.pi
    f32 = lambda a: torch.from_numpy(np.asarray(a, np.float32)).to(DEV)
    return dict(x=f32(g.standard_normal((n, 256))), f0=f32(f0), phase=f32(phase), volume=f32(g.uniform(0.0, 0.3, n)),
                emb=f32(g.standard_normal((7, 256)) * 0.5), spk=f32(g.standard_normal((B, 256))),
                aug=f32(np.linspace(-12.0, 12.0, B) + g.uniform(-1.0, 1.0, B)))


def _embed_run(I, B, T, spk_rows, with_aug):
    x = I["x"].clone()
    spk = 0 if spk_rows == 0 else I["spk"][:spk_rows].contiguous().data_ptr()
    _call("b2d_u2c_embed", x.data_ptr(), I["f0"].data_ptr(), I["phase"].data_ptr(), I["volume"].data_ptr(), I["emb"].data_ptr(),
          spk, max(spk_rows, 1), I["aug"].data_ptr() if with_aug else 0, B, T)
    return x


def _embed_check(B, T, spk_rows, with_aug, name, seed):
    """x + (w_f0 log(1 + f0/700) + b_f0) + (w_ph phase/pi + b_ph) + (w_vol vol + b_vol) + spk[b] + w_aug aug[b]/5.
    The fp32 chain has at most 16 roundings, each within u of the l1 norm of the terms; logf adds up to 4 u absolute
    (1 + f0/700 rounds twice, logf is within 1 ulp), hence bound = 16 u (l1 + 4 |w_f0|)."""
    I = _embed_inputs(B, T, seed)
    got = _embed_run(I, B, T, spk_rows, with_aug).to(F64)
    e = I["emb"].to(F64)
    col = lambda k: I[k].to(F64).reshape(-1, 1)
    b = torch.arange(B * T, device=DEV) // T
    terms = [I["x"].to(F64), e[0] * torch.log1p(col("f0") / 700.0), e[1], e[2] * (col("phase") / math.pi), e[3],
             e[4] * col("volume"), e[5]]
    if spk_rows:
        terms.append(I["spk"].to(F64)[b if spk_rows == B else torch.zeros_like(b)])
    if with_aug:
        terms.append(e[6] * (I["aug"].to(F64)[b].reshape(-1, 1) / 5.0))
    want = sum(terms)
    l1 = sum(t.abs() for t in terms) + 4.0 * e[0].abs()
    _check(name, (got - want).abs(), 16 * U * l1)


@pytest.mark.parametrize("with_aug", [False, True], ids=["noaug", "aug"])
@pytest.mark.parametrize("spk_rows", ["none", "one", "per_utt"])
@pytest.mark.parametrize("B,T", [(1, 1), (1, 7), (1, 150), (3, 1), (3, 7), (3, 150)])
def test_embed_against_float64(B, T, spk_rows, with_aug):
    rows = {"none": 0, "one": 1, "per_utt": B}[spk_rows]
    _embed_check(B, T, rows, with_aug, "embed/B=%d,T=%d,%s,aug=%d" % (B, T, spk_rows, with_aug), 10 + B * 1000 + T)


def test_embed_token_loop_past_the_grid():
    """The kernel launches min(B T, 8 SMs) CTAs and loops over the tokens: 3 (8 SMs + 2) tokens make every CTA run the
    loop three or four times."""
    B = 3
    T = 8 * _sms() + 2
    _embed_check(B, T, B, True, "embed/token_loop,B=%d,T=%d" % (B, T), 7)


# ---------------------------------------------------------------------------------------------------------------------
# b2d_u2c_groupnorm_lrelu
# ---------------------------------------------------------------------------------------------------------------------
SLOPE = float(np.float32(0.01))


def _gn_inputs(B, T, groups, seed):
    """x [B, T, 256]: (utterance, group) k = b + g cycles through a normal group, a group with mean / std = 1e3 and a
    constant group (only kinds reachable by the shape occur)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    cpg = 256 // groups
    x = torch.randn(B, T, 256, generator=g, device=DEV) * 0.7 + 0.3
    kind = torch.empty(B, groups, dtype=torch.long)
    for b in range(B):
        for q in range(groups):
            kind[b, q] = (b + q) % 3
            sl = x[b, :, q * cpg:(q + 1) * cpg]
            if kind[b, q] == 1:
                sl.mul_(0.25).add_(250.0)
            elif kind[b, q] == 2:
                sl.fill_(float(torch.randn(1, generator=g, device=DEV)))
    gamma = torch.randn(256, generator=g, device=DEV)
    beta = torch.randn(256, generator=g, device=DEV) * 0.5
    return x.contiguous(), gamma, beta, kind


def _gn_run(x, groups, gamma, beta):
    B, T, C = x.shape
    y = x.clone()
    stats = torch.empty(B * groups * 2, dtype=F64, device=DEV)
    _call("b2d_u2c_groupnorm_lrelu", y.data_ptr(), B, T, C, groups, gamma.data_ptr(), beta.data_ptr(), 1e-5, SLOPE, stats.data_ptr())
    return y


def _gn_ref(x, groups, gamma, beta):
    B, T, C = x.shape
    xg = x.to(F64).reshape(B, T, groups, C // groups)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    var = ((xg - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    y = ((xg - mean) / torch.sqrt(var + 1e-5)).reshape(B, T, C) * gamma.to(F64) + beta.to(F64)
    return torch.where(y >= 0, y, y * SLOPE)


@pytest.mark.parametrize("groups", [1, 4, 64, 256])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("T", [1, 2, 63, 64, 65, 127, 128, 129, 5168])
def test_groupnorm_lrelu_against_float64(T, B, groups):
    """Per (utterance, group), the largest error is at most 3x that of torch's fp32 group_norm + leaky_relu (CPU) on the
    same input, plus a floor of 6 u (|y| + |beta|) for groups where torch happens to be exact: the kernel's statistics
    are fp64, its apply step ((x - mean_hi) - mean_lo) rstd gamma + beta rounds five times in fp32.  The mean / std = 1e3
    groups test the fp64 E[x^2] - mean^2 and the two-float mean; a constant group must give exactly LeakyReLU(beta)."""
    x, gamma, beta, kind = _gn_inputs(B, T, groups, 1000 * groups + 10 * B + T)
    got = _gn_run(x, groups, gamma, beta).to(F64)
    want = _gn_ref(x, groups, gamma, beta)
    cpg = 256 // groups
    if B * cpg * T > 1:
        tx = F.leaky_relu(F.group_norm(x.cpu().transpose(1, 2), groups, gamma.cpu(), beta.cpu(), 1e-5), SLOPE).transpose(1, 2)
    else:                                             # torch refuses one value per group; that value normalises to 0
        tx, kind = want.float().cpu(), torch.full_like(kind, 2)
    grp = lambda t: t.reshape(B, T, groups, cpg).permute(0, 2, 1, 3).reshape(B, groups, -1)
    e_k = grp((got - want).abs()).amax(-1)
    e_t = grp((tx.to(F64).to(DEV) - want).abs()).amax(-1)
    floor = 6 * U * grp(want.abs() + beta.to(F64).abs()).amax(-1)
    bound = 3 * e_t + floor
    report.record("u2c_kernels/groupnorm/T=%d,B=%d,G=%d" % (T, B, groups), max_err=e_k.max().item(),
                  torch_fp32_max_err=e_t.max().item(), max_err_over_bound=(e_k / bound).max().item(),
                  large_mean_err=e_k[(kind == 1).to(DEV)].max().item() if (kind == 1).any() else 0.0)
    assert (e_k <= bound).all(), (e_k / bound).max().item()
    beta_f = beta.cpu().numpy()
    lrelu_beta = torch.from_numpy(np.where(beta_f >= 0, beta_f, beta_f * np.float32(SLOPE)).astype(np.float32))
    for b in range(B):
        for q in range(groups):
            if kind[b, q] == 2:
                _assert_same_bits(got[b, :, q * cpg:(q + 1) * cpg].float(), lrelu_beta[q * cpg:(q + 1) * cpg].expand(T, cpg),
                                  "constant group (%d, %d)" % (b, q))


def test_groupnorm_batch_rows_and_repeats_agree_to_one_ulp():
    """GroupNorm's per-utterance statistics are sums of fp64 atomics in no fixed order, so a batch row and the same row
    alone, or two identical calls, may differ where the rounding of the fp64 mean / rstd to fp32 flips: by at most one
    ulp of the group's largest output."""
    B, T, groups = 3, 700, 4
    g = torch.Generator(device=DEV).manual_seed(9)
    x = torch.randn(B, T, 256, generator=g, device=DEV)
    gamma, beta = torch.randn(256, generator=g, device=DEV), torch.randn(256, generator=g, device=DEV)
    full = _gn_run(x, groups, gamma, beta)
    tol = torch.from_numpy(np.spacing(full.abs().reshape(B, T, groups, 64).amax(dim=(1, 3)).cpu().numpy())).to(DEV)
    tol = tol.reshape(B, 1, groups, 1).expand(B, T, groups, 64).reshape(B, T, 256)
    assert ((_gn_run(x, groups, gamma, beta) - full).abs() <= tol).all()
    for b in range(B):
        alone = _gn_run(x[b:b + 1].contiguous(), groups, gamma, beta)[0]
        assert ((alone - full[b]).abs() <= tol[b]).all(), b


# ---------------------------------------------------------------------------------------------------------------------
# b2d_u2c_layernorm
# ---------------------------------------------------------------------------------------------------------------------
def _ln_run(x, gamma, beta):
    y = torch.empty_like(x)
    _call("b2d_u2c_layernorm", x.data_ptr(), y.data_ptr(), x.shape[0], x.shape[1], gamma.data_ptr(), beta.data_ptr(), 1e-5)
    return y


@pytest.mark.parametrize("n", [1, 7, 8, 9, 100003])
@pytest.mark.parametrize("C", [32, 256, 288, 1024])
def test_layernorm_against_float64(C, n):
    """One warp per token; each lane sums per = C/32 values, then a 5-step butterfly.  With m = C^-1 sum |x|:
    mean error <= (per + 6) u m; (x - mean)^2 summed the same way has relative error (per + 8) u plus
    (mean error)^2 / var; rsqrtf adds 4 u.  The output (x - mean) rstd gamma + beta adds three roundings:
      |err| <= 2 (|gamma| rstd ((per + 6) u m + |x - mean| ((per + 14) u + dmean^2 / (2 var))) + 2 u (|y| + |beta|)),
    where the factor 2 is headroom on the worst case.  Rows: random scales and offsets, offset rows (1e3 + N(0, 1)),
    constant rows of -1.25 (exact sums: output must be beta bit for bit) and of a random constant."""
    g = torch.Generator(device=DEV).manual_seed(C * 7 + n)
    x = torch.randn(n, C, generator=g, device=DEV) * torch.rand(n, 1, generator=g, device=DEV) * 3 + \
        torch.randn(n, 1, generator=g, device=DEV) * 2
    special = {1: "offset", 2: "const_exact", 3: "const_random", 4: "offset"}
    for r, what in special.items():
        if r < n:
            if what == "offset":
                x[r] = 1e3 + torch.randn(C, generator=g, device=DEV)
            else:
                x[r] = -1.25 if what == "const_exact" else float(torch.randn(1, generator=g, device=DEV))
    gamma, beta = torch.randn(C, generator=g, device=DEV), torch.randn(C, generator=g, device=DEV)
    got = _ln_run(x, gamma, beta).to(F64)
    xd = x.to(F64)
    mean = xd.mean(-1, keepdim=True)
    d = xd - mean
    var = (d * d).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    want = d * rstd * gamma.to(F64) + beta.to(F64)
    per = C // 32
    dmean = (per + 6) * U * xd.abs().mean(-1, keepdim=True)
    rel = (per + 14) * U + dmean ** 2 / (2 * (var + 1e-5))
    bound = 2 * (gamma.to(F64).abs() * rstd * (dmean + d.abs() * rel) + 2 * U * (want.abs() + beta.to(F64).abs()))
    _check("layernorm/C=%d,n=%d" % (C, n), (got - want).abs(), bound)
    if n > 2:
        _assert_same_bits(got[2].float(), beta, "constant row")


@pytest.mark.parametrize("C", [256, 1024])
def test_layernorm_batch_rows_are_bitwise_independent(C):
    g = torch.Generator(device=DEV).manual_seed(C)
    B, T = 3, 37
    x = torch.randn(B * T, C, generator=g, device=DEV) + 0.5
    gamma, beta = torch.randn(C, generator=g, device=DEV), torch.randn(C, generator=g, device=DEV)
    full = _ln_run(x, gamma, beta)
    _assert_same_bits(_ln_run(x, gamma, beta), full, "repeat")
    for b in range(B):
        _assert_same_bits(_ln_run(x[b * T:(b + 1) * T].contiguous(), gamma, beta), full[b * T:(b + 1) * T], "row %d" % b)


# ---------------------------------------------------------------------------------------------------------------------
# b2d_u2c_glu_dwconv_silu
# ---------------------------------------------------------------------------------------------------------------------
CANARY = 256


def _dw_inputs(B, T, Ci, seed):
    """value | gate channels; the gates include saturating +-60; utterance 1 is 1e3x utterance 0 (a halo that read
    across utterances would show in utterance 0 and 2); taps are random, so not symmetric."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(B, T, Ci, generator=g, device=DEV)
    gate = torch.randn(B, T, Ci, generator=g, device=DEV) * 3
    gate[:, ::5] = 60.0
    gate[:, 2::7] = -60.0
    if B > 1:
        a[1] *= 1e3
    w = torch.randn(Ci, 31, generator=g, device=DEV) * 0.3
    w[:, 0] += 1.0                                    # a strongly one-sided tap pattern on top
    bias = torch.randn(Ci, generator=g, device=DEV) * 0.1
    return torch.cat([a, gate], -1).contiguous(), w.contiguous(), bias


def _dw_run(inp, w, bias):
    B, T, C2 = inp.shape
    Ci = C2 // 2
    buf = torch.full((B * T * Ci + CANARY,), float("nan"), device=DEV)
    _call("b2d_u2c_glu_dwconv_silu", inp.data_ptr(), w.data_ptr(), bias.data_ptr(), buf.data_ptr(), B, T, Ci, 31)
    assert torch.isnan(buf[B * T * Ci:]).all(), "stores past the output"
    return buf[:B * T * Ci].reshape(B, T, Ci)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("Ci", [128, 512, 1024])
@pytest.mark.parametrize("T", [1, 2, 14, 15, 16, 30, 31, 32, 63, 64, 65, 129, 5168])
def test_glu_dwconv_silu_against_float64(T, Ci, B):
    """g = a sigmoid(gate) (relative error <= 5 u: expf, add, divide, multiply), acc = bias + sum_k w_k g[t - 15 + k]
    (31 fmaf: <= 31 u of l1 = |bias| + sum_k |w_k g|, plus the terms' own 7 u), y = acc sigmoid(acc) (SiLU's slope
    is below 1.1, plus 6 u |y|):
      |err| <= 1.1 * 40 u l1 + 6 u |y|.
    T < 31 puts both zero pads in one 64-frame tile; T = 64 ends exactly on a tile; a NaN canary after the output
    catches stores past T."""
    inp, w, bias = _dw_inputs(B, T, Ci, 100 * T + Ci + B)
    got = _dw_run(inp, w, bias).to(F64)
    a, gate = inp.to(F64).split(Ci, -1)
    gl = (a * torch.sigmoid(gate)).transpose(1, 2)
    wd = w.to(F64).unsqueeze(1)
    acc = F.conv1d(F.pad(gl, (15, 15)), wd, bias.to(F64), groups=Ci)
    l1 = F.conv1d(F.pad(gl.abs(), (15, 15)), wd.abs(), bias.to(F64).abs(), groups=Ci)
    want = (acc * torch.sigmoid(acc)).transpose(1, 2)
    bound = (1.1 * 40 * U * l1).transpose(1, 2) + 6 * U * want.abs()
    _check("glu_dwconv/T=%d,Ci=%d,B=%d" % (T, Ci, B), (got - want).abs(), bound)


def test_glu_dwconv_batch_rows_are_bitwise_independent():
    inp, w, bias = _dw_inputs(3, 100, 256, 5)
    full = _dw_run(inp, w, bias)
    _assert_same_bits(_dw_run(inp, w, bias), full, "repeat")
    for b in range(3):
        _assert_same_bits(_dw_run(inp[b:b + 1].contiguous(), w, bias)[0], full[b], "utterance %d" % b)


# ---------------------------------------------------------------------------------------------------------------------
# b2d_u2c_softmax_features
# ---------------------------------------------------------------------------------------------------------------------
def _sf_inputs(rows, J, d, is_query, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    data = torch.randn(rows, d, generator=g, device=DEV) * 0.6
    dd = torch.randn(rows, J, generator=g, device=DEV) * 1.5
    if rows > 1:
        dd[1] = dd[1] - dd[1].max() + 3.0
        dd[1, -1] = dd[1].max() + 5.0                 # the row's max is the last feature
    if is_query and rows > 2:
        dd[2] = torch.rand(J, generator=g, device=DEV) * 200.0   # up to +200: expf stays finite only after the max
        dd[2, -1] = 200.0
    return dd.contiguous(), data


def _sf_run(dd, data, is_query):
    rows, J = dd.shape
    out = dd.clone()
    _call("b2d_u2c_softmax_features", out.data_ptr(), data.data_ptr(), rows, J, data.shape[1], int(is_query), 1e-4)
    return out


@pytest.mark.parametrize("d", [16, 64])
@pytest.mark.parametrize("J", [1, 31, 33, 266])
@pytest.mark.parametrize("rows", [1, 7, 9, 8 * 5168])
@pytest.mark.parametrize("is_query", [1, 0], ids=["query", "key"])
def test_softmax_features_against_float64(is_query, rows, J, d):
    """diag = |data|^2 / 2 d^-1/2 (sum of d squares: (d/32 + 6) u relative, d^-1/2 via rsqrtf(sqrtf(d)) squared: 12 u);
    the exponent's argument p - diag - max (query) or p - diag + eps (key) is formed with two roundings, so its absolute
    error is <= 2 u (|p| + |diag| + |max|) + (d/32 + 18) u |diag|; expf (4 u), ratio = rsqrtf(J) (4 u), the product
    and the + eps add 12 u relative:  |err| <= 2 |y| (arg_err + 12 u), 2 = headroom."""
    dd, data = _sf_inputs(rows, J, d, is_query, 1000 * rows + 10 * J + d + is_query)
    got = _sf_run(dd, data, is_query).to(F64)
    p, x = dd.to(F64), data.to(F64)
    diag = (x * x).sum(-1, keepdim=True) / 2 * d ** -0.5
    ratio = J ** -0.5
    mx = p.amax(-1, keepdim=True)
    want = ratio * (torch.exp(p - diag - mx) + 1e-4) if is_query else ratio * torch.exp(p - diag + 1e-4)
    third = mx.abs() if is_query else torch.full_like(mx, 1e-4)
    arg_err = 2 * U * (p.abs() + diag.abs() + third) + (d / 32 + 18) * U * diag.abs()
    assert torch.isfinite(got).all()
    _check("softmax_features/%s,rows=%d,J=%d,d=%d" % ("q" if is_query else "k", rows, J, d), (got - want).abs(),
           2 * want.abs() * (arg_err + 12 * U))


@pytest.mark.parametrize("is_query", [1, 0], ids=["query", "key"])
def test_softmax_features_batch_rows_are_bitwise_independent(is_query):
    n, J, d = 41, 266, 64
    dd, data = _sf_inputs(3 * n, J, d, is_query, 77)
    full = _sf_run(dd, data, is_query)
    _assert_same_bits(_sf_run(dd, data, is_query), full, "repeat")
    for b in range(3):
        s = slice(b * n, (b + 1) * n)
        _assert_same_bits(_sf_run(dd[s].contiguous(), data[s].contiguous(), is_query), full[s], "utterance %d" % b)


# ---------------------------------------------------------------------------------------------------------------------
# b2d_u2c_linear_attention
# ---------------------------------------------------------------------------------------------------------------------
def _la_inputs(BH, T, J, seed):
    """feature maps like the performer's (positive, ratio exp(N(0, 1) - 1)) and values N(0, 1)"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    feat = lambda: (torch.exp(torch.randn(BH, T, J, generator=g, device=DEV) - 1.0) * J ** -0.5).contiguous()
    return feat(), feat(), torch.randn(BH, T, 64, generator=g, device=DEV).contiguous()


def _la_run(qf, kf, v, B, H):
    T, J = qf.shape[1], qf.shape[2]
    out = torch.empty(B, T, H, 64, device=DEV)
    _call("b2d_u2c_linear_attention", qf.data_ptr(), kf.data_ptr(), v.data_ptr(), out.data_ptr(), B, H, T, J, 64, 1e-8)
    return out


def _la_formula(qf, kf, v, B, H):
    """(q' . (k'^T v)) / (q' . sum_t k' + 1e-8) in the dtype of the inputs, with the library calls Unit2Control makes
    when fused_attention is off -> [B, T, H, 64]"""
    k_sum = kf.sum(dim=-2)
    d_inv = 1.0 / (torch.einsum("bnj,bj->bn", qf, k_sum) + 1e-8)
    out = torch.matmul(qf, torch.matmul(kf.transpose(-1, -2), v)) * d_inv.unsqueeze(-1)
    return out.reshape(B, H, -1, 64).permute(0, 2, 1, 3)


def _rel_rms(a, b):
    return (torch.sqrt(((a - b) ** 2).mean()) / torch.sqrt((b ** 2).mean())).item()


@pytest.mark.parametrize("BH", [1, 24])
@pytest.mark.parametrize("J", [8, 129, 266, 272])
@pytest.mark.parametrize("T", [1, 15, 16, 17, 150, 5168])
def test_linear_attention_against_float64(T, J, BH):
    """The kernel keeps k_sum and the context as per-thread fp32 running sums over all T frames, then finishes each row
    with J-long fmaf chains.  Its relative RMS error against float64 must stay within 3x that of the library path the
    module runs otherwise (kf.sum + fp32 torch.matmul, no TF32) on the same inputs, or within 8 u (short T, where both
    are a handful of roundings)."""
    B, H = (1, 1) if BH == 1 else (3, 8)
    qf, kf, v = _la_inputs(BH, T, J, 1000 * T + J + BH)
    got = _la_run(qf, kf, v, B, H)
    want = _la_formula(qf.to(F64), kf.to(F64), v.to(F64), B, H)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        lib_out = _la_formula(qf, kf, v, B, H)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    e_k, e_l = _rel_rms(got.to(F64), want), _rel_rms(lib_out.to(F64), want)
    bound = max(3 * e_l, 8 * U)
    report.record("u2c_kernels/linear_attention/T=%d,J=%d,BH=%d" % (T, J, BH), rel_rms=e_k, library_rel_rms=e_l, bound=bound)
    assert e_k <= bound, (e_k, e_l)


def test_linear_attention_batch_rows_are_bitwise_independent():
    B, H, T, J = 3, 8, 90, 266
    qf, kf, v = _la_inputs(B * H, T, J, 3)
    full = _la_run(qf, kf, v, B, H)
    _assert_same_bits(_la_run(qf, kf, v, B, H), full, "repeat")
    for b in range(B):
        s = slice(b * H, (b + 1) * H)
        _assert_same_bits(_la_run(qf[s].contiguous(), kf[s].contiguous(), v[s].contiguous(), 1, H)[0], full[b], "utterance %d" % b)


# ---------------------------------------------------------------------------------------------------------------------
# b2d_u2c_embed batch independence (the other kernels have theirs next to their float64 test)
# ---------------------------------------------------------------------------------------------------------------------
def test_embed_batch_rows_are_bitwise_independent():
    B, T = 3, 50
    I = _embed_inputs(B, T, 21)
    full = _embed_run(I, B, T, B, True)
    _assert_same_bits(_embed_run(I, B, T, B, True), full, "repeat")
    for b in range(B):
        s = slice(b * T, (b + 1) * T)
        Ib = {k: (v[s].contiguous() if k in ("x", "f0", "phase", "volume") else v) for k, v in I.items()}
        Ib["spk"], Ib["aug"] = I["spk"][b:b + 1].contiguous(), I["aug"][b:b + 1].contiguous()
        _assert_same_bits(_embed_run(Ib, 1, T, 1, True), full[s], "utterance %d" % b)

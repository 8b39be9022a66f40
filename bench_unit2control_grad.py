"""Training step of the control network (Unit2Control with the convolution-only decoder) on the kernels: its forward,
its backward, the backward's own kernels one by one, and the whole configs/combsub.yaml step (control network +
CombSubSuperFast + RSSLoss, forward and backward) -- alternated with the same step using a plain-torch control network
(oracle/unit2control.py, eager, same GPU: what a differentiable ``unit2ctrl=`` gives).  Prints one JSON line.

    python bench_unit2control_grad.py [--steps 20] [--warmup 3]

Shapes: the training batch of configs/combsub.yaml (24 x 2 s, 172 frames) and BASELINE config 3 (32 x 10 s), 768 units.
Every step is timed with CUDA events after the L2 was flushed (256 MiB memset, untimed); medians are reported.
``backward_library_gemms_and_glue_ms`` is the backward minus its kernels: the library GEMMs, the TF32 splits and the
gathers of the k = 3 convolutions.  Needs a CUDA device; there is no fallback."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SR, P, WIN, N_UNIT = 44100, 512, 2048, 768
SHAPES = [("combsub_yaml_train_b24_2s", 24, 172), ("baseline_cfg3_b32_10s", 32, 861)]
N_FFTS = [1800, 333, 1024, 1531]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=power.limit,power.max_limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        limit, max_limit, sm_clock = float(q[0]), float(q[1]), float(q[2])
    except Exception:
        limit = max_limit = sm_clock = None
    return {"name": name, "power_limit_w": limit, "power_max_limit_w": max_limit, "max_sm_clock_mhz": sm_clock}


def one(fn, prep, flush):
    import torch
    prep()
    flush.zero_()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def timed(fn, prep, flush, steps, warmup):
    for _ in range(warmup):
        prep()
        fn()
    return statistics.median(one(fn, prep, flush) for _ in range(steps))


def kernel_times(B, T, n_out, flush, steps, warmup):
    """the backward's kernels alone through the C ABI at this shape (per call; the step runs glu x 3, colsum x 9 or so)"""
    import torch
    from ddsp_svc_b200 import _lib
    L, N, dev = _lib.lib(), B * T, "cuda"
    r = lambda *s: torch.randn(*s, device=dev)
    n = L.b2d_u2c_backward_workspace_bytes(B, T, 512, n_out)
    ws = torch.empty(n, dtype=torch.uint8, device=dev)
    h, gout, gh, dwb, w, bias = r(N, 1024), r(N, 512), r(N, 1024), r(512, 32), r(512, 31), r(512)
    x, gy, gx, dgb, gamma = r(N, 256), r(N, 256), r(N, 256), r(2, 256), r(256)
    stats, f0, ge, out = torch.empty(B * 8, dtype=torch.float64, device=dev), r(N).abs() * 200, r(N, n_out), r(n_out)
    y = x.clone()
    L.b2d_u2c_groupnorm_lrelu(y.data_ptr(), B, T, 256, 4, gamma.data_ptr(), gamma.data_ptr(), 1e-5, 0.01, stats.data_ptr(), 0)
    gcat, dtable, rowsum = r(N, 768), r(7, 256), r(B, 256)
    p = lambda t: t.data_ptr()
    calls = {
        "glu_dwconv_silu_backward_ms": lambda: L.b2d_u2c_glu_dwconv_silu_backward(p(h), p(w), p(bias), p(gout), p(gh), p(dwb), B, T, 512,
                                                                                   31, p(ws), n, 0),
        "layernorm_backward_ms": lambda: L.b2d_u2c_layernorm_backward(p(x), p(gy), p(gamma), 1e-5, N, 256, p(gx), p(dgb), p(ws), n, 0),
        "groupnorm_lrelu_backward_ms": lambda: L.b2d_u2c_groupnorm_lrelu_backward(p(x), p(stats), p(gamma), p(gamma), 1e-5, 0.01, p(gy),
                                                                                   B, T, 256, 4, p(gx), p(dgb), p(ws), n, 0),
        "embed_backward_ms": lambda: L.b2d_u2c_embed_backward(p(gx), p(f0), p(f0), p(f0), 0, B, T, p(dtable), p(rowsum), p(ws), n, 0),
        "colsum_dense_out_ms": lambda: L.b2d_u2c_colsum(p(ge), N, n_out, p(out), p(ws), n, 0),
        "colsum_1024_ms": lambda: L.b2d_u2c_colsum(p(h), N, 1024, p(out), p(ws), n, 0),
        "colsum_256_ms": lambda: L.b2d_u2c_colsum(p(x), N, 256, p(out), p(ws), n, 0),
        "conv3_fold_ms": lambda: L.b2d_u2c_conv3_fold(p(gcat), B, T, 256, p(gx), 0),
    }
    res = {}
    for k, fn in calls.items():
        assert fn() == 0, k
        res[k] = timed(fn, lambda: None, flush, steps, warmup)
    # per backward: 3 decoder layers (glu, colsum 256 + 1024 each), dense_out, final LayerNorm, embed, second convolution
    # (colsum 256, fold, GroupNorm), first convolution (colsum 256)
    res["all_kernels_per_backward_ms"] = (3 * (res["glu_dwconv_silu_backward_ms"] + res["colsum_1024_ms"] + res["colsum_256_ms"]) +
                                          res["colsum_dense_out_ms"] + res["layernorm_backward_ms"] + res["embed_backward_ms"] +
                                          2 * res["colsum_256_ms"] + res["conv3_fold_ms"] + res["groupnorm_lrelu_backward_ms"])
    return res


def run_shape(label, B, nF, flush, steps, warmup):
    import torch
    import ddsp_svc_b200 as pkg
    from ddsp_svc_b200 import synthetic as syn
    from oracle.unit2control import NaiveUnit2Control
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(1)
    ours = pkg.CombSubSuperFast(SR, P, WIN, n_unit=N_UNIT, n_spk=2, use_pitch_aug=True).to(dev).train()
    u2c = ours.unit2ctrl
    eager_net = NaiveUnit2Control(N_UNIT, 2, u2c.output_splits, use_pitch_aug=True)
    eager_net.load_state_dict(u2c.state_dict())
    eager = pkg.CombSubSuperFast(SR, P, WIN, unit2ctrl=eager_net).to(dev).train()
    g = torch.Generator().manual_seed(2)
    units, volume = torch.randn(B, nF, N_UNIT, generator=g).to(dev), (0.2 * torch.rand(B, nF, 1, generator=g)).to(dev)
    f0, phase = syn.make_f0(B, nF, SR, P).to(dev), (torch.rand(B, nF, 1, generator=g) * 6 - 3).to(dev)
    spk, aug = torch.randint(1, 3, (B, 1), generator=g).to(dev), torch.randn(B, 1, 1, generator=g).to(dev)
    target = 0.1 * torch.randn(B, nF * P, generator=g).to(dev)
    cot_e, cot_h = torch.randn(B, nF, u2c.n_out, generator=g).to(dev), torch.randn(B, nF, 256, generator=g).to(dev)
    cots = list(torch.split(cot_e, list(u2c.output_splits.values()), dim=-1)) + [cot_h]
    crit = pkg.RSSLoss(256, 2048, 4)
    st = {}

    def net_fwd():
        c, h = u2c(units, f0, phase, volume, spk_id=spk, aug_shift=aug)
        st["out"] = list(c.values()) + [h]

    def net_bwd():
        torch.autograd.backward(st["out"], cots)        # as in a step: autograd gathers the views' cotangents into the dense one

    def step_of(model):
        def step():
            signal, hidden, _ = model(units, f0, volume, spk_id=spk, aug_shift=aug, infer=False)
            crit(signal, target, n_ffts=N_FFTS).backward()
        return step

    def clear():
        ours.zero_grad(set_to_none=True)
        eager.zero_grad(set_to_none=True)

    def prep_bwd():
        clear()
        net_fwd()

    with torch.no_grad():
        infer_ms = timed(net_fwd, lambda: None, flush, steps, warmup)
    fwd_ms = timed(net_fwd, clear, flush, steps, warmup)
    bwd_ms = timed(net_bwd, prep_bwd, flush, steps, warmup)
    st.clear()
    kern = kernel_times(B, nF, u2c.n_out, flush, steps, warmup)
    torch.cuda.empty_cache()
    a, b = step_of(ours), step_of(eager)
    for _ in range(warmup):
        clear(); a(); clear(); b()
    ta, tb = [], []
    for _ in range(steps):                                       # alternated: both see the same neighbours on the device
        ta.append(one(a, clear, flush))
        tb.append(one(b, clear, flush))
    clear()
    torch.cuda.empty_cache()
    step_ms, eager_ms = statistics.median(ta), statistics.median(tb)
    return {"B": B, "n_frames": nF, "seconds": nF * P / SR, "gemm_precision": u2c.gemm_precision,
            "network_forward_no_grad_ms": infer_ms, "network_forward_ms": fwd_ms,
            "network_backward_ms": bwd_ms, "backward_kernels": kern,
            "backward_library_gemms_and_glue_ms": bwd_ms - kern["all_kernels_per_backward_ms"],
            "combsub_yaml_step_ms": step_ms, "combsub_yaml_step_eager_torch_network_ms": eager_ms,
            "step_speedup_vs_eager_torch_network": eager_ms / step_ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_unit2control_grad.py needs a CUDA device (no fallback)")
    from ddsp_svc_b200 import _lib
    _lib.lib()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    line = {"metric": "unit2control_train_step", "card": card(),
            "timing": "median of %d steps after %d warm-up, CUDA events, L2 flushed before each step (untimed); network = "
                      "Unit2Control(use_naive_v2) alone with cotangents on the controls and on hidden; step = control network + "
                      "CombSubSuperFast + RSSLoss forward and backward, alternated with the same step on a plain-torch "
                      "control network run eagerly (torch defaults: fp32 matmul, cuDNN convolutions may use TF32)"
                      % (args.steps, args.warmup),
            "shapes": {label: run_shape(label, B, nF, flush, args.steps, args.warmup) for label, B, nF in SHAPES}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()

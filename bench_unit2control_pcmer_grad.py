"""Training step of the PCmer control network (Unit2Control with ``pcmer_backward``) on the kernels: its forward (no_grad
and under grad), its backward, the new attention-backward kernels one by one, and the whole configs/sins.yaml step
(control network + Sins + RSSLoss, forward and backward) -- alternated with the same step using the plain-torch PCmer
network (tests/u2c_pcmer_oracle.py: PCmerUnit2Control, eager, same GPU: what a differentiable ``unit2ctrl=`` gives).
Prints one JSON line.

    python bench_unit2control_pcmer_grad.py [--steps 20] [--warmup 3]

Shapes: the training batch of configs/sins.yaml (24 x 2 s, 172 frames) and BASELINE config 3 (32 x 10 s), 768 units.
Timing as bench_unit2control_grad.py (whose ``card`` also reports the max SM clock): CUDA events, L2 flushed before each
timed call, medians.  Kernel rates are the bytes each kernel must move (computed from shapes below) over its time.
``saved_activation_mb_per_layer`` is the memory the forward under grad keeps for the backward, over the no_grad forward,
divided by the three layers.  Needs a CUDA device; there is no fallback."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_unit2control_grad import card, one, timed  # noqa: E402

SR, P, N_UNIT, H, J = 44100, 512, 768, 8, 266
SHAPES = [("sins_yaml_train_b24_2s", 24, 172), ("baseline_cfg3_b32_10s", 32, 861)]
N_FFTS = [1800, 333, 1024, 1531]


def kernel_times(B, T, flush, steps, warmup):
    """the attention backward's kernels alone through the C ABI (one call each; a backward runs 3 x (readout, 2 x features,
    gather)) with the bytes each must read and write"""
    import torch
    from ddsp_svc_b200 import _lib
    L, R, dev = _lib.lib(), B * H * T, "cuda"
    r = lambda *s: torch.randn(*s, device=dev)
    g_out, out, d_inv, gn = r(B, T, H, 64), r(B, T, H, 64), r(B, H, T).abs() + 0.1, r(B, H, T, 65)
    g, phi, x, vec, scal, gx = r(R, J), r(R, J).abs(), r(R, 64), r(B * H, J).abs(), r(R), r(R, 64)
    gq, gk, gv, qkv, gqkv = r(R, 64), r(R, 64), r(R, 64), r(B, T, 3, H, 64), r(B, T, 3, H, 64)
    p = lambda t: t.data_ptr()
    f = 4
    calls = {
        "attn_readout_backward": (lambda: L.b2d_u2c_attn_readout_backward(p(g_out), p(out), p(d_inv), B, H, T, 64, p(gn), 0),
                                  f * R * (64 + 64 + 1 + 65)),
        "softmax_features_backward_query": (lambda: L.b2d_u2c_softmax_features_backward(p(g), p(phi), p(x), p(vec), p(scal), R, T, J,
                                                                                         64, 1, 1e-4, p(gx), 0),
                                            f * (R * (3 * J + 64 + 1 + 64) + B * H * J)),
        "qkv_gather_backward_normalized": (lambda: L.b2d_u2c_qkv_gather_backward(p(gq), p(gk), p(gv), p(qkv), B, H, T, 64, 1, p(gqkv), 0),
                                           f * R * 64 * (3 + 2 + 3)),
    }
    res = {}
    for k, (fn, nbytes) in calls.items():
        assert fn() == 0, k
        ms = timed(fn, lambda: None, flush, steps, warmup)
        res[k + "_ms"], res[k + "_tb_per_s"] = ms, nbytes / (ms * 1e-3) / 1e12
    res["all_kernels_per_backward_ms"] = 3 * (res["attn_readout_backward_ms"] + 2 * res["softmax_features_backward_query_ms"] +
                                              res["qkv_gather_backward_normalized_ms"])
    return res


def run_shape(label, B, nF, flush, steps, warmup):
    import torch
    import ddsp_svc_b200 as pkg
    from ddsp_svc_b200 import synthetic as syn
    from tests.u2c_pcmer_oracle import PCmerUnit2Control
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(1)
    ours = pkg.Sins(SR, P, 128, 256, 256, n_unit=N_UNIT, n_spk=2).to(dev).train()
    u2c = ours.unit2ctrl
    u2c.pcmer_backward = True
    eager_net = PCmerUnit2Control(N_UNIT, 2, u2c.output_splits)
    eager_net.load_state_dict(u2c.state_dict())
    eager = pkg.Sins(SR, P, 128, 256, 256, unit2ctrl=eager_net).to(dev).train()
    g = torch.Generator().manual_seed(2)
    units, volume = torch.randn(B, nF, N_UNIT, generator=g).to(dev), (0.2 * torch.rand(B, nF, 1, generator=g)).to(dev)
    f0, phase = syn.make_f0(B, nF, SR, P).to(dev), (torch.rand(B, nF, 1, generator=g) * 6 - 3).to(dev)
    spk = torch.randint(1, 3, (B, 1), generator=g).to(dev)
    target = 0.1 * torch.randn(B, nF * P, generator=g).to(dev)
    cot_e, cot_h = torch.randn(B, nF, u2c.n_out, generator=g).to(dev), torch.randn(B, nF, 256, generator=g).to(dev)
    cots = list(torch.split(cot_e, list(u2c.output_splits.values()), dim=-1)) + [cot_h]
    crit = pkg.RSSLoss(256, 2048, 4)
    st = {}

    def net_fwd():
        c, h = u2c(units, f0, phase, volume, spk_id=spk)
        st["out"] = list(c.values()) + [h]

    def net_bwd():
        torch.autograd.backward(st["out"], cots)

    def step_of(model):
        def step():
            signal, hidden, _ = model(units, f0, volume, spk_id=spk, infer=False)
            crit(signal, target, n_ffts=N_FFTS).backward()
        return step

    def clear():
        ours.zero_grad(set_to_none=True)
        eager.zero_grad(set_to_none=True)
        st.clear()

    def prep_bwd():
        clear()
        net_fwd()

    with torch.no_grad():
        infer_ms = timed(net_fwd, clear, flush, steps, warmup)
        clear()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        net_fwd()
        torch.cuda.synchronize()
        infer_bytes = torch.cuda.memory_allocated() - base
    clear()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    net_fwd()
    torch.cuda.synchronize()
    saved_mb = (torch.cuda.memory_allocated() - base - infer_bytes) / 3 / 2 ** 20
    clear()
    fwd_ms = timed(net_fwd, clear, flush, steps, warmup)
    bwd_ms = timed(net_bwd, prep_bwd, flush, steps, warmup)
    clear()
    kern = kernel_times(B, nF, flush, steps, warmup)
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
            "network_forward_no_grad_ms": infer_ms, "network_forward_ms": fwd_ms, "network_backward_ms": bwd_ms,
            "saved_activation_mb_per_layer": saved_mb, "backward_kernels": kern,
            "backward_library_gemms_and_glue_ms": bwd_ms - kern["all_kernels_per_backward_ms"],
            "sins_yaml_step_ms": step_ms, "sins_yaml_step_eager_torch_network_ms": eager_ms,
            "step_speedup_vs_eager_torch_network": eager_ms / step_ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_unit2control_pcmer_grad.py needs a CUDA device (no fallback)")
    from ddsp_svc_b200 import _lib
    _lib.lib()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    line = {"metric": "unit2control_pcmer_train_step", "card": card(),
            "timing": "median of %d steps after %d warm-up, CUDA events, L2 flushed before each step (untimed); network = "
                      "Unit2Control (PCmer, pcmer_backward) alone with cotangents on the controls and on hidden; step = control "
                      "network + Sins + RSSLoss forward and backward, alternated with the same step on the plain-torch PCmer "
                      "network run eagerly (torch defaults: fp32 matmul, cuDNN convolutions may use TF32)" % (args.steps, args.warmup),
            "shapes": {label: run_shape(label, B, nF, flush, args.steps, args.warmup) for label, B, nF in SHAPES}}
    print(json.dumps(line))


if __name__ == "__main__":
    main()

"""Training step of the reflow model on the kernels: the reflow loss (RectifiedFlow(infer=False) around NaiveV2Diff at
configs/reflow.yaml's width: 512 channels, 6 layers, 128 mel bins) forward and forward + backward, and the whole
configs/reflow.yaml step (control network -> CombSubSuperFast -> get_mel -> mse + reflow loss -> backward).  Each is
alternated with the same work using the velocity network written in plain torch (tests/reflow_oracle.py) run eagerly in
fp32 under torch's defaults -- cuDNN convolutions in TF32, what the reference runs today; in the step's eager arm the
control network is the plain-torch oracle/unit2control.py network as well (the synthesizer and mel are the package's in
both arms).  Prints one JSON line, with the card's name and power limit read in the same run.  Writes nothing.

    python bench_reflow_grad.py [--steps K] [--warmup W]

Shapes: the reflow.yaml batch (48 x 2 s, 172 frames) and 32 x 10 s (861 frames).  Every call is timed with CUDA events
after the L2 was flushed (256 MiB memset, untimed); the arms alternate call by call; medians of K calls after W warm-up
calls of each.  Also reported: the GEMM FLOP of one loss forward and backward from shapes, and the memory the training
forward holds for its backward (allocated after a forward under grad, minus the same after the no_grad forward).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

M, DIM, LAYERS, SR, P, WIN, N_UNIT = 128, 512, 6, 44100, 512, 2048, 768
SHAPES = [("reflow_yaml_b48_2s", 48, 172), ("b32_10s", 32, 861)]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        limit, sm_clock = float(q[0]), float(q[1])
    except Exception:
        limit = sm_clock = None
    return {"name": name, "power_limit_w": limit, "max_sm_clock_mhz": sm_clock}


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


def alternate(fa, fb, prep, flush, steps, warmup):
    for _ in range(warmup):
        prep(); fa(); prep(); fb()
    ta, tb = [], []
    for _ in range(steps):
        ta.append(one(fa, prep, flush))
        tb.append(one(fb, prep, flush))
    prep()
    return statistics.median(ta), statistics.median(tb), [min(ta), max(ta)], [min(tb), max(tb)]


def gemm_flop(B, T):
    """multiply-adds x 2 of the loss's GEMMs from shapes: forward (input, per-layer pw1 / pw2, output and the condition
    projections of all layers; the B-row step MLP is negligible) and backward (two products per forward product, none
    towards the input mel)"""
    N = B * T
    per_layer = DIM * 4 * DIM + 2 * DIM * DIM
    fwd = 2 * N * (M * DIM + LAYERS * per_layer + DIM * M + M * LAYERS * DIM)
    bwd = 2 * N * (M * DIM + 2 * LAYERS * per_layer + 2 * DIM * M + 2 * M * LAYERS * DIM)
    return fwd, bwd


def held(fn):
    """bytes allocated after fn() while its result is alive, over the allocation before"""
    import torch
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    n = torch.cuda.memory_allocated() - m0
    del out
    return n


def run_shape(B, T, flush, steps, warmup):
    import torch
    import ddsp_svc_b200 as pkg
    from ddsp_svc_b200 import mel as pm, synthetic as syn
    from oracle.unit2control import NaiveUnit2Control
    from tests.golden import make_golden_reflow as mk
    from tests.golden import make_golden_reflow_grad as GR
    dev = torch.device("cuda:0")
    net = pkg.NaiveV2Diff(use_mlp=False, **mk.model_kwargs("w512"))
    net.load_state_dict(mk.build_oracle("w512").state_dict(), strict=True)
    net.reflow_backward = True
    flow = pkg.RectifiedFlow(net.to(dev)).train()
    eager = mk.build_oracle("w512").to(dev).train()
    g = torch.Generator().manual_seed(B * T)
    ramp = torch.linspace(-8.0, 0.5, M)[None, None, :]
    cond = (ramp + 1.5 * torch.randn(B, T, M, generator=g)).to(dev)
    gt = (ramp + 1.5 * torch.randn(B, T, M, generator=g)).to(dev)
    torch.manual_seed(1)
    t = torch.clip(torch.rand(B, device=dev), 1e-7, 1 - 1e-7)
    x0 = torch.randn(B, T, M, device=dev)
    cg = cond.clone().requires_grad_(True)
    k_loss = lambda: flow._loss(cg, gt, t, x0)
    e_loss = lambda: GR.oracle_loss(eager, cg, gt, t, x0)

    def clear():
        flow.zero_grad(set_to_none=True)
        eager.zero_grad(set_to_none=True)
        cg.grad = None

    res = {"B": B, "frames": T}
    res["loss_forward_ms"], res["loss_forward_eager_ms"], sa, sb = alternate(k_loss, e_loss, clear, flush, steps, warmup)
    res["loss_fwd_bwd_ms"], res["loss_fwd_bwd_eager_ms"], sc, sd = alternate(lambda: k_loss().backward(),
                                                                            lambda: e_loss().backward(), clear, flush,
                                                                            steps, warmup)
    res["spreads_ms"] = {"loss_forward": sa, "loss_forward_eager": sb, "loss_fwd_bwd": sc, "loss_fwd_bwd_eager": sd}
    res["loss_fwd_bwd_speedup"] = res["loss_fwd_bwd_eager_ms"] / res["loss_fwd_bwd_ms"]
    fwd, bwd = gemm_flop(B, T)
    res["gemm_gflop_forward"], res["gemm_gflop_backward"] = fwd / 1e9, bwd / 1e9
    res["kernels_gemm_tflops_fwd_bwd"] = (fwd + bwd) / (res["loss_fwd_bwd_ms"] * 1e-3) / 1e12
    with torch.no_grad():
        base_k, base_e = held(k_loss), held(e_loss)
    res["saved_activations_mb"] = (held(k_loss) - base_k) / 2 ** 20
    res["saved_activations_eager_mb"] = (held(e_loss) - base_e) / 2 ** 20
    clear()
    with torch.no_grad():
        lk, le = k_loss(), e_loss()
    res["loss_rel_diff_kernels_vs_eager"] = abs(lk.item() - le.item()) / abs(le.item())
    del eager
    torch.cuda.empty_cache()

    # the whole reflow.yaml step: control network -> CombSubSuperFast -> get_mel -> mse + reflow loss -> backward
    torch.manual_seed(2)
    ours = pkg.CombSubSuperFast(SR, P, WIN, n_unit=N_UNIT, n_spk=2, use_pitch_aug=True).to(dev).train()
    u2c_eager = NaiveUnit2Control(N_UNIT, 2, ours.unit2ctrl.output_splits, use_pitch_aug=True)
    u2c_eager.load_state_dict(ours.unit2ctrl.state_dict())
    theirs = pkg.CombSubSuperFast(SR, P, WIN, unit2ctrl=u2c_eager).to(dev).train()
    vel_eager = mk.build_oracle("w512").to(dev).train()
    stft = pm.STFT(SR, M, 2048, 2048, P, 40, 16000)
    units, volume = torch.randn(B, T, N_UNIT, generator=g).to(dev), (0.2 * torch.rand(B, T, 1, generator=g)).to(dev)
    f0 = syn.make_f0(B, T, SR, P).to(dev)
    spk, aug = torch.randint(1, 3, (B, 1), generator=g).to(dev), torch.randn(B, 1, 1, generator=g).to(dev)
    with torch.no_grad():
        sig, _, _ = ours(units, f0, volume, spk_id=spk, aug_shift=aug)
        mel0 = stft.get_mel(sig).transpose(1, 2)
        gt_step = (mel0 + 0.5 * torch.randn_like(mel0)).contiguous()

    def step_of(model, reflow_loss):
        def step():
            signal, _, _ = model(units, f0, volume, spk_id=spk, aug_shift=aug, infer=False)
            mel = stft.get_mel(signal).transpose(1, 2)
            Tm = mel.shape[1]
            torch.manual_seed(3)
            tt = torch.clip(torch.rand(B, device=dev), 1e-7, 1 - 1e-7)
            xx = torch.empty_strided((B, 1, M, Tm), (Tm * M, Tm * M, 1, M), device=dev).normal_()[:, 0].transpose(1, 2)
            (torch.nn.functional.mse_loss(mel, gt_step) + reflow_loss(mel, gt_step, tt, xx)).backward()
        return step

    def clear_step():
        ours.zero_grad(set_to_none=True)
        theirs.zero_grad(set_to_none=True)
        flow.zero_grad(set_to_none=True)
        vel_eager.zero_grad(set_to_none=True)

    a = step_of(ours, lambda c, s, tt, xx: flow._loss(c, s, tt, xx))
    b = step_of(theirs, lambda c, s, tt, xx: GR.oracle_loss(vel_eager, c, s, tt, xx))
    res["reflow_yaml_step_ms"], res["reflow_yaml_step_eager_ms"], se, sf = alternate(a, b, clear_step, flush, steps, warmup)
    res["spreads_ms"].update(step=se, step_eager=sf)
    res["step_speedup"] = res["reflow_yaml_step_eager_ms"] / res["reflow_yaml_step_ms"]
    del ours, theirs, vel_eager
    torch.cuda.empty_cache()
    return {k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed calls per arm and shape")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_reflow_grad.py needs a CUDA device (no fallback)")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")   # > 50 MB L2
    res = {"bench": "reflow_train_step", "card": card(), "gemm_precision": "3xtf32 (default)",
           "timing": "median of %d calls per arm after %d warm-up calls, arms alternating, CUDA events, L2 flushed before "
                     "each call (untimed); eager arm: plain-torch networks in fp32 under torch's defaults"
                     % (args.steps, args.warmup),
           "shapes": {label: run_shape(B, T, flush, args.steps, args.warmup) for label, B, T in SHAPES}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Occupancy and per-launch time of the FFT-domain FIR at bench.py's headline size (Sins, B = 32 x 10 s, two jobs:
all-pass and noise filters + mix), kept apart from bench.py.

Runs the headline FIR launch under torch.profiler with CUDA activities and prints, for every ltv_fir_fft_kernel
launch, its grid, the hops per CTA (G = ceil(nF / grid.x)), registers per thread, shared memory per CTA and duration,
and the resident CTAs per SM that those resources allow on this device (the same limits
cudaOccupancyMaxActiveBlocksPerMultiprocessor applies: threads, registers in 256-register warp units, shared memory
with the 1 KB per-CTA reserve).  Output: one JSON line on stdout; the chrome trace goes to --out.

    python bench_fir_occupancy.py [--reps 5] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import tempfile

import torch

import bench


def resident_ctas(threads, regs, smem, props):
    warps = (threads + 31) // 32
    by_threads = props.max_threads_per_multi_processor // threads
    regs_per_warp = ((regs * 32 + 255) // 256) * 256
    by_regs = props.regs_per_multiprocessor // (regs_per_warp * warps) if regs else by_threads
    smem_sm = props.shared_memory_per_multiprocessor
    by_smem = smem_sm // (smem + 1024) if smem else by_threads
    return min(by_threads, by_regs, by_smem, 32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the chrome trace (default: a temporary directory)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    props = torch.cuda.get_device_properties(dev)
    w = bench.WORKLOADS["sins"]
    run = bench.Runner(w, dev, 0, torch)
    fir = run.kernels()["ltv_fir_x2_mix"]
    fir()
    torch.cuda.synchronize()
    out = args.out or tempfile.mkdtemp(prefix="fir_occupancy_")
    os.makedirs(out, exist_ok=True)
    trace = os.path.join(out, "fir_occupancy.pt.trace.json")
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            fir()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        events = json.load(f)["traceEvents"]
    launches = []
    for e in events:
        if e.get("cat") != "kernel" or "ltv_fir_fft_kernel" not in e.get("name", ""):
            continue
        a = e.get("args", {})
        grid, block = a.get("grid"), a.get("block")
        regs, smem = a.get("registers per thread"), a.get("shared memory")
        launches.append({"grid": grid, "block": block, "G": -(-run.nF // grid[0]) if grid else None,
                         "registers": regs, "smem_bytes": smem, "us": e.get("dur"),
                         "ctas_per_sm": resident_ctas(block[0], regs, smem, props) if block and regs is not None else None,
                         "est_achieved_occupancy_pct": a.get("est. achieved occupancy %")})
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        power = None
    print(json.dumps({"device": props.name, "sms": props.multi_processor_count, "nvidia_smi": power,
                      "B": run.B, "nF": run.nF, "launches": launches,
                      "median_us": statistics.median(l["us"] for l in launches) if launches else None}))


if __name__ == "__main__":
    main()

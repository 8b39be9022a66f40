"""Block time of gui.py's real-time callback for N independent sessions on one card, N in --sessions (default 1, 4,
16, 64), at the GUI defaults (44.1 kHz, block 0.3 s, crossfade 0.04 s, extra 2.0 s, enhancer on, key 0) with a synthetic
seeded Sins checkpoint (conversion_fixtures.write_synthetic, in a temporary directory).

Three arms, alternated block by block, each timed with CUDA events from before the first upload to after the last output
copy (the device's span of one block for all N sessions):
  batched   one BatchedRealtimeVC of N sessions: one upload, graphs A and B replayed once
  serial    N RealtimeVC objects, each replaying its graphs after the previous one finished
  streams   N RealtimeVC objects on their N streams at once
The RealtimeVC arms are run where the card's free memory holds N of them (each holds its own models and graphs).
Medians and p99 over --blocks blocks after --warmup blocks.  Prints one JSON line per N with the card's name and power
limit, then one with the largest N whose p99 stays under the block length, per arm."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def time_block(sessions, chain, enqueue):
    """device time (ms) of one block: every session stream starts after one event, the end waits for all of them;
    chain: each session starts after the previous one's work"""
    cur = torch.cuda.current_stream()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record(cur)
    prev = None
    for s in sessions:
        s.stream.wait_event(start)
        if chain and prev is not None:
            s.stream.wait_stream(prev.stream)
        enqueue(s)
        prev = s
    for s in sessions:
        cur.wait_stream(s.stream)
    end.record(cur)
    end.synchronize()
    return start.elapsed_time(end)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", type=int, nargs="+", default=[1, 4, 16, 64])
    ap.add_argument("--blocks", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--model", default="Sins")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_realtime_batch.py needs a CUDA device"
    from conversion_fixtures import write_synthetic
    from ddsp_svc_b200.realtime import BatchedRealtimeVC, RealtimeVC
    gpu = card()
    rng = np.random.default_rng(0)
    best = {}
    with tempfile.TemporaryDirectory() as d, contextlib.redirect_stdout(io.StringIO()) as quiet:
        model_path, rmvpe_path = write_synthetic(d, a.model)
        kw = dict(rmvpe_ckpt=rmvpe_path, device="cuda:0")
        singles, per_single = [], None
        for n in a.sessions:
            torch.cuda.synchronize()
            b = BatchedRealtimeVC(model_path, [dict(spk_id=1 + i % 2, pitch_adjust=i % 5) for i in range(n)], **kw)
            block_ms = 1e3 * b.block / b.sr
            # RealtimeVC objects up to n if the free memory holds the missing ones with a quarter to spare
            while len(singles) < n:
                free = torch.cuda.mem_get_info()[0]
                if per_single is not None and free < 1.25 * per_single * (n - len(singles)):
                    break
                before = torch.cuda.memory_allocated()
                s = RealtimeVC(model_path, **kw)
                s.process(np.zeros((s.block, 2), np.float32))              # captures its graphs
                per_single = per_single or (torch.cuda.memory_allocated() - before + (1 << 28))
                singles.append(s)
            arms = {"batched": ([b], False)}
            if len(singles) >= n:
                arms.update(serial=(singles[:n], True), streams=(singles[:n], False))
            x = {}

            def enqueue(s):
                if s is b:
                    b.upload(x["batch"])
                    b.run_a()
                    b.run_b()
                else:
                    s.upload(x["one"])
                    s.run_a()
                    s.run_b(s.pick_key())
            times = {k: [] for k in arms}
            order = list(arms)
            for i in range(a.warmup + a.blocks):
                x["one"] = (0.1 * rng.standard_normal((b.block, 2))).astype(np.float32)
                x["batch"] = np.repeat(x["one"][None], n, 0)
                for k in order[i % len(order):] + order[:i % len(order)]:     # alternate which arm goes first
                    t = time_block(*arms[k], enqueue)
                    if i >= a.warmup:
                        times[k].append(t)
            res = {"metric": "realtime block time for N sessions (ms, CUDA events)", "gpu": gpu, "model": a.model,
                   "sessions": n, "block_ms": block_ms,
                   "settings": "44.1 kHz, block 0.3 s, crossfade 0.04 s, extra 2.0 s, enhancer key 0",
                   "blocks": a.blocks}
            for k, v in times.items():
                med, p99 = float(np.median(v)), float(np.percentile(v, 99))
                res[k] = {"median_ms": med, "p99_ms": p99, "median_ms_per_session": med / n}
                if p99 < block_ms:
                    best[k] = max(best.get(k, 0), n)
            for k in ("serial", "streams"):
                res.setdefault(k, "not measured: %d RealtimeVC objects do not fit in the free memory" % n)
            print(json.dumps(res), file=sys.__stdout__, flush=True)
            del b, arms
            torch.cuda.empty_cache()
        quiet.truncate(0)
    print(json.dumps({"metric": "largest N with p99 block time under the block length", "gpu": gpu,
                      "sessions_tried": a.sessions, "largest_n": best}), flush=True)


if __name__ == "__main__":
    main()

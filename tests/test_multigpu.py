"""Multi-GPU tests of the waveform gather (need >= 2 CUDA devices; skipped otherwise).  Every mode bench.py can
choose -- the FIR kernel storing `signal` straight into rank 0's symmetric-memory buffer, chunked synthesis with
per-chunk peer stores or copy-engine pushes on one or two compute streams, and the NCCL fallbacks -- must deliver on
rank 0 exactly the single-GPU synthesis of the whole batch (bit for bit: the in-kernel noise is keyed by the global
utterance index and the FFT-domain FIR is chunking-invariant).

Run on a machine with two (and eight) GPUs:  python -m pytest tests/test_multigpu.py -q"""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

MODES = ["peer", "peer-chunks-1s", "peer-chunks-2s", "peer-copy-1s", "peer-copy-2s", "nccl", "nccl-chunks"]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, modes, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from ddsp_svc_b200 import FixedControls, Sins, sharding, synthetic as syn
        SR, P, nF, H, Bl, CH = 44100, 512, 20, 32, 6, 3
        sm = syn.sins_split_map(H, 256, 256)
        f0 = syn.make_f0(world * Bl, nF)
        dense = syn.make_ctrl(world * Bl, nF, sm)[0]
        lo, hi = sharding.shard_bounds(world * Bl, world, rank)
        f0_d, dense_d = f0[lo:hi].to(dev), dense[lo:hi].to(dev)
        fixed = FixedControls(syn.split_views(dense_d, sm), None)
        model = Sins(SR, P, H, 256, 256, unit2ctrl=fixed).to(dev)
        peer = sharding.PeerGather(Bl, nF * P, dev, dst=0)

        def rows(a, b, signal_out=None):          # local rows [a, b) with their GLOBAL utterance index
            fixed.ctrls = syn.split_views(dense_d[a:b], sm)
            kw = {"signal_out": signal_out} if signal_out is not None else {}
            return model(None, f0_d[a:b], None, utterance_offset=lo + a, **kw)[0]

        results = {}
        with torch.no_grad():
            for mode in modes:
                if rank == 0:
                    peer.result.zero_()
                torch.cuda.synchronize()
                dist.barrier()
                torch.manual_seed(11)   # same host seed stream on every rank -> same Philox keys; rows differ by utterance index
                if mode == "peer":
                    rows(0, Bl, signal_out=peer.my_rows)
                    out = peer.finish()
                elif mode.startswith("peer-"):
                    out = sharding.synthesize_and_push(rows, peer, Bl, dev, chunks=CH, streams=int(mode[-2]),
                                                       direct=mode.startswith("peer-chunks"))
                elif mode == "nccl":
                    out = sharding.gather_waveform(rows(0, Bl), world * Bl, dst=0)
                else:
                    out = sharding.synthesize_and_gather(rows, Bl, world * Bl, nF * P, dev, dst=0, chunks=CH)
                torch.cuda.synchronize()
                dist.barrier()
                if rank == 0:
                    chunked = mode not in ("peer", "nccl")
                    fixed_all = FixedControls(None, None)
                    ref_model = Sins(SR, P, H, 256, 256, unit2ctrl=fixed_all).to(dev)
                    want = []
                    for r in range(world):          # replay each rank's sequence of host-seed draws
                        a, b = sharding.shard_bounds(world * Bl, world, r)
                        torch.manual_seed(11)
                        spans = sharding._chunk_bounds(Bl, CH) if chunked else [(0, Bl)]
                        for ca, cb in spans:
                            fixed_all.ctrls = syn.split_views(dense[a + ca:a + cb].to(dev), sm)
                            want.append(ref_model(None, f0[a + ca:a + cb].to(dev), None, utterance_offset=a + ca)[0])
                    want = torch.cat(want)
                    results[mode] = (float((out - want).abs().max().item()), float(want.abs().max().item()))
        if rank == 0:
            ret.put(results)
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _run(world, modes):
    ctx = mp.get_context("spawn")
    ret = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, modes, ret)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(600)
        assert p.exitcode == 0
    return ret.get()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_gather_modes_two_gpus():
    res = _run(2, MODES)
    for mode in MODES:
        err, amp = res[mode]
        assert amp > 1e-3 and err == 0.0, (mode, err, amp)


@pytest.mark.skipif(torch.cuda.device_count() < 8, reason="needs eight GPUs")
def test_gather_modes_eight_gpus():
    res = _run(8, MODES)
    for mode in MODES:
        err, amp = res[mode]
        assert amp > 1e-3 and err == 0.0, (mode, err, amp)

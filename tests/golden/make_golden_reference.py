"""Generate the reference-side fixtures of the tests that compare this package with the upstream classes
(yxlllc/DDSP-SVC), so that those tests run without the reference:

    DDSP_REFERENCE_ROOT=<DDSP-SVC checkout> python tests/golden/make_golden_reference.py

* u2c_host_<variant>.npz -- tests/test_unit2control_host.py: the reference's Unit2Control (64 units) with this
  package's seeded initial weights loaded, its state-dict keys / shapes and its outputs for the test's calls;
* u2c_gpu_<variant>.npz -- tests/test_gpu_unit2control.py: the same at 768 units, outputs as a fixed seeded sample;
* u2c_sins_e2e.npz -- the reference's Sins.forward (this package's seeded weights) and the noise it drew;
* stft_live_reference.npz -- the reference's STFT.get_mel on the inputs of tests/test_oracle_mel.py;
* reference_state_dicts.json -- state-dict keys / shapes of the reference classes that tests/test_dropin.py loads;
* linear_attention_reference.npz -- the reference's pcmer.linear_attention (tests/test_emu_linear_attention.py);
* fresh_frontend_reference.npz -- Volume_Extractor, the silence-mask lines and main.py's cross_fade on the fresh inputs
  of tests/test_oracle_frontend.py;
* acceptance_<class>_<call>.npz, acceptance_source_module.npz -- tests/test_gpu_acceptance.py: the reference classes'
  forward (this package's seeded weights) on the test's inputs and calls, with the white noise it drew.
"""
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.dirname(os.path.abspath(__file__))

from oracle import ref_loader  # noqa: E402

U2C_HOST = {"pcmer": dict(), "naive_conformer": dict(use_naive_v2=True, use_conv_stack=True, use_pitch_aug=True),
            "pcmer_norm_plainconv": dict(pcmer_norm=True, use_conv_stack=False)}
U2C_SAMPLE = 16384          # sampled elements per output and call of the 768-unit fixtures


def keys_shapes(sd):
    return json.dumps([[k, list(v.shape)] for k, v in sd.items()])


def host_calls(kw):
    calls = [dict(spk_id=torch.LongTensor([[2], [3]])), dict(spk_id=torch.LongTensor([[1]]), spk_mix_dict={1: 0.3, 2: 0.7})]
    if kw.get("use_pitch_aug"):
        calls.append(dict(spk_id=torch.LongTensor([[1], [1]]), aug_shift=torch.tensor([[[2.0]], [[-3.0]]])))
    return calls


def host_inputs():
    g = torch.Generator().manual_seed(1)
    units, f0 = torch.randn(2, 50, 64, generator=g), 200 + 100 * torch.rand(2, 50, 1, generator=g)
    ph, vo = torch.rand(2, 50, 1, generator=g), torch.rand(2, 50, 1, generator=g)
    return units, f0, ph, vo


@contextlib.contextmanager
def record_random(store):
    """record what torch.rand / rand_like / randn_like return while the reference runs"""
    saved = torch.rand, torch.rand_like, torch.randn_like

    def wrap(name, fn):
        def f(*a, **k):
            t = fn(*a, **k); store.append((name, t)); return t
        return f
    torch.rand, torch.rand_like, torch.randn_like = (wrap(n, f) for n, f in zip(("rand", "rand_like", "randn_like"), saved))
    try:
        yield
    finally:
        torch.rand, torch.rand_like, torch.randn_like = saved


def sample_index(n, seed):
    return torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:U2C_SAMPLE].sort().values


def main():
    if not ref_loader.available():
        raise SystemExit("set DDSP_REFERENCE_ROOT to a DDSP-SVC checkout")
    from ddsp_svc_b200 import unit2control as U
    import ddsp_svc_b200 as pkg
    from oracle import mel as om
    from tests import test_gpu_unit2control as TG
    from tests import test_gpu_acceptance as TA
    with contextlib.redirect_stdout(io.StringIO()):
        V, _, _ = ref_loader.load()
    from ddsp.unit2control import Unit2Control as Ref
    import ddsp.pcmer as ref_pcmer
    import nsf_hifigan.models as nsf

    for name, kw in U2C_HOST.items():
        ref_pcmer.FLAG_PCMER_NORM = False
        torch.manual_seed(3)
        ours = U.Unit2Control(64, 3, {"a": 33, "b": 7}, **kw)
        ref = Ref(64, 3, {"a": 33, "b": 7}, **kw).eval()
        ref.load_state_dict(ours.state_dict())
        units, f0, ph, vo = host_inputs()
        out = {"keys_shapes": np.array(keys_shapes(ref.state_dict()))}
        for i, c in enumerate(host_calls(kw)):
            with torch.no_grad():
                wc, wh = ref(units, f0, ph, vo, **c)
            out["controls_%d" % i] = torch.cat(list(wc.values()), -1).numpy()
            out["hidden_%d" % i] = wh.numpy()
        np.savez_compressed(os.path.join(HERE, "u2c_host_%s.npz" % name), **out)

    for name, (kw, splits) in TG.VARIANTS.items():
        if name.endswith("fused_attention"):
            continue                                    # same reference outputs as its unfused twin
        ref_pcmer.FLAG_PCMER_NORM = False
        torch.manual_seed(3)
        ours = U.Unit2Control(768, 3, splits, **kw)
        ref = Ref(768, 3, splits, **kw).eval()
        ref.load_state_dict(ours.state_dict())
        units, f0, phase, volume = TG._inputs(2, 150, 768, 4)
        out = {"keys_shapes": np.array(keys_shapes(ref.state_dict()))}
        for i, c in enumerate(TG.calls_of(kw)):
            with torch.no_grad():
                wc, wh = ref(units, f0, phase, volume, **c)
            dense = torch.cat([wc[k] for k in wc], -1).reshape(-1)
            hid = wh.reshape(-1)
            out["controls_%d" % i] = dense[sample_index(dense.numel(), 100 + i)].numpy()
            out["hidden_%d" % i] = hid[sample_index(hid.numel(), 200 + i)].numpy()
            out["controls_rms_%d" % i] = np.float64(dense.pow(2).mean().sqrt())
            out["hidden_rms_%d" % i] = np.float64(hid.pow(2).mean().sqrt())
        np.savez_compressed(os.path.join(HERE, "u2c_gpu_%s.npz" % name.replace("_fused_attention", "")), **out)

    ref_pcmer.FLAG_PCMER_NORM = False
    torch.manual_seed(5)
    ours = pkg.Sins(44100, 512, 128, 256, 256, n_unit=768, n_spk=2)
    ref = V.Sins(44100, 512, 128, 256, 256, n_unit=768, n_spk=2).eval()
    ref.load_state_dict(ours.state_dict())
    units, f0, _, volume = TG._inputs(1, 90, 768, 6)
    drawn = []
    r0 = torch.rand_like

    def rec(*a, **k):
        t = r0(*a, **k); drawn.append(t); return t
    torch.rand_like = rec
    try:
        with torch.no_grad():
            want = ref(units, f0, volume, spk_id=torch.LongTensor([[2]]))[0]
    finally:
        torch.rand_like = r0
    np.savez_compressed(os.path.join(HERE, "u2c_sins_e2e.npz"), signal=want.numpy(),
                        noise=(drawn[0] * 2 - 1).reshape(1, -1).numpy())

    st_mod = om.load_reference_stft()
    g = torch.Generator().manual_seed(9)
    out = {}
    for i, (T, hop) in enumerate(((512 * 9 + 17, 512), (900, 512), (256 * 30, 256))):
        y = 0.2 * torch.randn(2, T, generator=g)
        with torch.no_grad():
            out["mel_%d" % i] = st_mod.STFT(44100, 128, 2048, 2048, hop, 40, 16000).get_mel(y).numpy()
    np.savez_compressed(os.path.join(HERE, "stft_live_reference.npz"), **out)

    with contextlib.redirect_stdout(io.StringIO()):
        sds = {"Sins": V.Sins(44100, 512, 128, 256, 256, n_unit=768, n_spk=1).state_dict(),
               "CombSub": V.CombSub(44100, 512, 256, 512, 256, n_unit=768, n_spk=2).state_dict(),
               "CombSubSuperFast": V.CombSubSuperFast(44100, 512, 2048, n_unit=768, n_spk=1).state_dict(),
               "CombSubFast": V.CombSubFast(44100, 512, n_unit=768, n_spk=1).state_dict(),
               "SourceModuleHnNSF": nsf.SourceModuleHnNSF(44100, harmonic_num=8).state_dict()}
    with open(os.path.join(HERE, "reference_state_dicts.json"), "w") as f:
        json.dump({k: [[n, list(v.shape)] for n, v in sd.items()] for k, sd in sds.items()}, f, indent=0)
        f.write("\n")

    g = torch.Generator().manual_seed(1)
    q = torch.rand(2, 3, 20, 266, generator=g, dtype=torch.float64)
    k = torch.rand(2, 3, 20, 266, generator=g, dtype=torch.float64)
    v = torch.randn(2, 3, 20, 64, generator=g, dtype=torch.float64)
    np.savez_compressed(os.path.join(HERE, "linear_attention_reference.npz"), out=ref_pcmer.linear_attention(q, k, v).numpy())

    from tests.golden.make_golden_frontend import inputs, reference_function, reference_mask_lines
    cf = reference_function("main.py", "cross_fade")
    out = {}
    for seed, T, hop in ((11, 9000, 512), (12, 777, 256), (13, 30011, 441)):
        vol = V.Volume_Extractor(hop).extract(inputs(seed, T))
        out["volume_%d" % seed], out["mask_%d" % seed] = vol, reference_mask_lines(vol, -45)
        rng = np.random.default_rng(seed)
        a, b = rng.standard_normal(400).astype(np.float32), rng.standard_normal(500).astype(np.float32)
        for idx in (0, 1, 250, 399):
            out["fade_%d_%d" % (seed, idx)] = cf(a, b, idx)
    np.savez_compressed(os.path.join(HERE, "fresh_frontend_reference.npz"), **out)


    units, f0, volume, _ = TA.inputs()
    for kind, case in TA.CASES.items():
        with contextlib.redirect_stdout(io.StringIO()):
            ref = case["make"](V).eval()
        ref.load_state_dict(TA.seeded_state_dict(kind))
        for i, kw in enumerate(TA.calls()):
            drawn = []
            with torch.no_grad(), record_random(drawn):
                sig, hidden, (harm, _) = ref(units, f0, volume, **kw)
            assert len(drawn) == 1 and drawn[0][0] == ("rand_like" if case["uniform"] else "randn_like")
            noise = drawn[0][1] * 2 - 1 if case["uniform"] else drawn[0][1]
            out = {"signal": sig.numpy(), "hidden": hidden.numpy(), "noise": noise.reshape(1, -1).numpy()}
            if case["parts"]:
                out["harmonic"] = harm.numpy()
            np.savez_compressed(os.path.join(HERE, "acceptance_%s_%d.npz" % (kind, i)), **out)

    torch.manual_seed(3)
    sd = pkg.SourceModuleHnNSF(44100, harmonic_num=8).state_dict()
    ref_sm = nsf.SourceModuleHnNSF(44100, harmonic_num=8).eval()
    ref_sm.load_state_dict(sd)
    f0, upp = TA.source_module_inputs()
    drawn = []
    with torch.no_grad(), record_random(drawn):
        out = ref_sm(f0, upp)
    rand_ini = [t for n, t in drawn if n == "rand"][0].clone()
    rand_ini[..., 0] = 0
    noise = [t for n, t in drawn if n == "randn_like"][0]
    np.savez_compressed(os.path.join(HERE, "acceptance_source_module.npz"), out=out.numpy(), rand_ini=rand_ini.numpy(),
                        noise=noise.numpy())


if __name__ == "__main__":
    main()

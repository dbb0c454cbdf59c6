"""Row a17 (second half): multi-band-diffusion vocoder.  PARITY UNPINNED (audiocraft / julius / mbd_comp_8.pt absent):
the CUDA implementation is checked against the CPU restatement oracle/mbd_port.py on a seeded synthetic checkpoint of a
parametrised configuration; the CPU test checks the restatement's own invariants."""
import numpy as np
import pytest
import torch

from mvb200 import synth
from oracle import mbd_port as M

SMALL = M.MBDConfig(n_models=2, unet=M.UnetCfg(hidden=16, depth=2, growth=2.0, kernel=8, stride=4, res_blocks=1, norm_groups=4),
                    proc_bands=4, eq_bands=8, step_list=[999, 749, 499, 249, 0])


def test_restatement_invariants():
    # SplitBands is a partition of the signal; the filters have unit DC gain; the default step list gives 20 model calls
    x = torch.from_numpy(synth.synthetic_waveform(0.5, 24000, seed=1))
    for n in (4, 8, 32):
        b = M.split_bands(x, n, 24000)
        assert b.shape == (n, x.numel()) and torch.allclose(b.sum(0), x, atol=1e-5)
        assert torch.allclose(M.lowpass_bank(n, 24000).sum(1), torch.ones(n - 1), atol=1e-5)
    assert len(M.schedule_coefficients(M.ScheduleCfg(), M.MBDConfig().steps())) == 20
    co = M.schedule_coefficients(M.ScheduleCfg(), M.MBDConfig().steps())
    assert co[-1][2] == 0.0 and all(c[2] > 0 for c in co[:-1])          # no noise after the last call
    # re_eq imposes the reference's band energies
    ref = torch.from_numpy(synth.synthetic_waveform(0.5, 24000, seed=2))
    y = M.re_eq(x, ref, 8, 24000)
    by, br = M.split_bands(y, 8, 24000), M.split_bands(ref, 8, 24000)
    assert y.shape == ref.shape and torch.isfinite(y).all()
    # UNet shape contract (odd length: right padding to the stride, cropped back)
    ck = synth.mbd_checkpoint(SMALL, 0)
    est = M.unet_forward(ck["models"][0], SMALL.unet, torch.randn(1, 1, 1001), 499, torch.randn(1, 128, 4))
    assert est.shape == (1, 1, 1001) and torch.isfinite(est).all()


@pytest.mark.gpu
@pytest.mark.parametrize("frames", [12, 40])
def test_mbd_device_vs_restatement(frames):
    from mvb200.mbd import MBDSettings, MultiBandDiffusionEngine, ScheduleSettings, UnetSettings
    ck = synth.mbd_checkpoint(SMALL, 0)
    settings = MBDSettings(n_models=2, unet=UnetSettings(hidden=16, depth=2, growth=2.0, kernel=8, stride=4, res_blocks=1, norm_groups=4),
                           schedule=ScheduleSettings(), proc_bands=4, eq_bands=8, step_list=[999, 749, 499, 249, 0])
    # the fp32 CUDA-core kernels (the tensor-core lowering has its own test below)
    eng = MultiBandDiffusionEngine(ck, settings, device="cuda:0", max_seconds=1.0, tensor_cores=False)
    T = frames * 320
    g = torch.Generator().manual_seed(frames)
    cond = torch.randn(128, frames, generator=g)
    wav_e = torch.from_numpy(synth.synthetic_waveform(T / 24000.0, 24000, seed=3))[:T]
    noise = torch.randn(2, 4, T, generator=g)
    want = M.MBDOracle(ck, SMALL).tokens_to_wav(wav_e, cond, noise)
    got = eng.tokens_to_wav(cond, wav_e, noise=noise).cpu()
    err = float((got - want).abs().max() / want.abs().max())
    print(f"MBD ({frames} frames, {T} samples): rel err vs restatement {err:.2e}")
    assert err < 2e-3
    a = eng.tokens_to_wav(cond, wav_e, seed=5).cpu()
    b = eng.tokens_to_wav(cond, wav_e, seed=5).cpu()
    assert torch.equal(a, b) and torch.isfinite(a).all()


def _round_conv_weights_to_bf16(ck):
    for sd in ck["models"]:
        for k in list(sd):
            if sd[k].ndim == 3:
                sd[k] = sd[k].to(torch.bfloat16).to(torch.float32)
    return ck


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,stride,frames,hidden", [(8, 4, 12, 64), (8, 4, 33, 64), (4, 2, 12, 64), (8, 4, 12, 48)])
def test_mbd_tensor_core_convs_vs_restatement(kernel, stride, frames, hidden):
    """Input widths >= 32 channels take the tensor-core path (csrc/mbd_tc.cuh): shifted-GEMM Conv1d (dilation 1
    and 2), the strided encoder convolution and the phase-decomposed ConvTranspose1d.  With conv weights representable in
    bf16 the path is exact to fp32 round-off against the fp32 restatement; with arbitrary fp32 weights the only deviation
    is the bf16 rounding of the taps (reported, bounded)."""
    from mvb200.mbd import MBDSettings, MultiBandDiffusionEngine, ScheduleSettings, UnetSettings
    ucfg = dict(hidden=hidden, depth=2, growth=2.0, kernel=kernel, stride=stride, res_blocks=2, norm_groups=4)
    cfg = M.MBDConfig(n_models=2, unet=M.UnetCfg(**ucfg), proc_bands=4, eq_bands=8, step_list=[999, 666, 333, 0])
    settings = MBDSettings(n_models=2, unet=UnetSettings(**ucfg), schedule=ScheduleSettings(), proc_bands=4, eq_bands=8,
                           step_list=[999, 666, 333, 0])
    T = frames * 320 - 7                      # not a multiple of the stride: right padding + crop
    g = torch.Generator().manual_seed(100 + frames)
    cond = torch.randn(128, frames, generator=g)
    wav_e = torch.from_numpy(synth.synthetic_waveform(frames * 320 / 24000.0, 24000, seed=4))[:T]
    noise = torch.randn(2, 3, T, generator=g)
    for exact in (True, False):
        ck = synth.mbd_checkpoint(cfg, 1)
        if exact:
            ck = _round_conv_weights_to_bf16(ck)
        eng = MultiBandDiffusionEngine(ck, settings, device="cuda:0", max_seconds=1.0)
        want = M.MBDOracle(ck, cfg).tokens_to_wav(wav_e, cond, noise)
        got = eng.tokens_to_wav(cond, wav_e, noise=noise).cpu()
        err = float((got - want).abs().max() / want.abs().max())
        print(f"MBD tensor-core (k={kernel}, s={stride}, {T} samples, bf16-representable taps={exact}): rel err {err:.2e}")
        assert err < (2e-3 if exact else 3e-2)


@pytest.mark.gpu
def test_mbd_default_config_vs_restatement():
    """The shipped UNet (default UnetSettings: hidden 48, growth 4, depth 4, widths 48 / 192 / 768 / 3072) end to end:
    workspace sizing (mbd_layout) and layer wiring at those widths, 2 band models, 2 sampler calls, 12 frames
    (3833 samples), bf16-representable taps."""
    from mvb200.mbd import MBDSettings, MultiBandDiffusionEngine
    steps = [999, 499, 0]
    cfg = M.MBDConfig(n_models=2, step_list=steps)
    settings = MBDSettings(n_models=2, step_list=steps)
    frames = 12
    T = frames * 320 - 7
    g = torch.Generator().manual_seed(7)
    cond = torch.randn(128, frames, generator=g)
    wav_e = torch.from_numpy(synth.synthetic_waveform(frames * 320 / 24000.0, 24000, seed=5))[:T]
    noise = torch.randn(2, len(steps) - 1, T, generator=g)
    ck = _round_conv_weights_to_bf16(synth.mbd_checkpoint(cfg, 2))
    eng = MultiBandDiffusionEngine(ck, settings, device="cuda:0", max_seconds=1.0)
    want = M.MBDOracle(ck, cfg).tokens_to_wav(wav_e, cond, noise)
    got = eng.tokens_to_wav(cond, wav_e, noise=noise).cpu()
    err = float((got - want).abs().max() / want.abs().max())
    print(f"MBD default configuration ({T} samples, 2 band models, 2 calls): rel err vs restatement {err:.2e}")
    assert err < 2e-3


def test_flop_accounting_matches_the_restatement_shapes():
    """bench.py's MBD roofline uses MultiBandDiffusionEngine.flops(): check it against a direct count over the restatement's
    own layer shapes for the default parametrised configuration (187 GFLOP per UNet pass, 80 passes per utterance)."""
    import types
    from mvb200.mbd import MBDSettings, MultiBandDiffusionEngine
    s = MBDSettings()
    got = MultiBandDiffusionEngine.flops(types.SimpleNamespace(s=s), 120000, 375)
    u, ch = s.unet, s.unet.channels()
    t, cin, per = 120000, u.chin, 0.0
    for c in ch:
        t = -(-t // u.stride)
        per += 2.0 * t * (u.kernel * cin * c)                    # Conv1d(cin, c, k, stride)
        per += 2 * u.res_blocks * 2 * 2.0 * t * (3 * c * c)      # encoder + decoder ResBlocks
        per += 2.0 * t * (u.kernel * c * cin)                    # ConvTranspose1d(c, cin, k, stride): every input sample x every tap
        cin = c
    per += 2.0 * 375 * u.codec_dim * ch[-1]
    want = per * s.n_models * (len(s.steps()) - 1)
    assert abs(got - want) / want < 1e-12 and 14.5e12 < got < 15.5e12

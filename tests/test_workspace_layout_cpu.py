"""CPU: the exact workspace size every engine asks its caller for.  Each slice keeps its order, size and 256-byte
alignment, so these byte counts only change when a layout is changed on purpose."""
import ctypes as C

import pytest

from mvb200 import _lib, synth
from mvb200.mbd import MBDSettings, _lowpass_bank, _schedule_table
from mvb200.vocoder import RATIOS


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _s1(d, max_utts, kv):
    return _lib.S1Config(d.n_layer, d.n_head, d.head_dim, d.dim, d.intermediate_size, d.vocab_size, d.block_size,
                         d.speaker_emb_dim, d.norm_eps, max_utts, kv, d.block_size)


S1_BYTES = {   # (dims, max_utts, kv_dtype) -> (mvb_s1_workspace_bytes, mvb_s1_int4_workspace_bytes)
    ("full", 1, _lib.MVB_KV_BF16): (66566656, 169327104),
    ("full", 1, _lib.MVB_KV_FP32): (66566656, 169327104),
    ("full", 8, _lib.MVB_KV_BF16): (71178240, 173938688),
    ("full", 8, _lib.MVB_KV_FP32): (71178240, 173938688),
    ("full", 64, _lib.MVB_KV_BF16): (108075264, 210835712),
    ("full", 64, _lib.MVB_KV_FP32): (108075264, 210835712),
    ("tiny", 1, _lib.MVB_KV_FP32): (8898560, 10602496),
}


@pytest.mark.parametrize("key", list(S1_BYTES), ids=lambda k: f"{k[0]}-u{k[1]}-kv{k[2]}")
def test_stage1_workspace_bytes(lib, key):
    dims = {"full": synth.FULL, "tiny": synth.TINY}[key[0]]
    cfg = _s1(dims, key[1], key[2])
    assert (lib.mvb_s1_workspace_bytes(C.byref(cfg)), lib.mvb_s1_int4_workspace_bytes(C.byref(cfg))) == S1_BYTES[key]


@pytest.mark.parametrize("max_batch,want", [(1, 40955904), (2, 78240256)])
def test_stage2_workspace_bytes(lib, max_batch, want):
    d = synth.S2_FULL      # the configuration SecondStage builds from a checkpoint of these dimensions
    cfg = _lib.S2Config()
    cfg.n_layer, cfg.n_head, cfg.n_embd, cfg.hidden = d.n_layer, d.n_head, d.n_embd, d.hidden
    cfg.block_size, cfg.n_in, cfg.n_out = d.block_size, len(d.vocab_sizes), len(d.target_vocab_sizes)
    for i, v in enumerate(d.vocab_sizes):
        cfg.vocab_in[i] = v
    for i, v in enumerate(d.target_vocab_sizes):
        cfg.vocab_out[i] = v
    cfg.spk_dim, cfg.norm_eps, cfg.max_batch = d.speaker_emb_dim, d.rmsnorm_eps, max_batch
    assert lib.mvb_s2_workspace_bytes(C.byref(cfg)) == want


@pytest.mark.parametrize("max_frames,want", [(2048, 268440320), (256, 33559296)])
def test_vocoder_workspace_bytes(lib, max_frames, want):
    cfg = _lib.VocConfig()     # EncodecDecodeEngine's configuration for the 24 kHz codec
    cfg.n_q, cfg.hidden, cfg.n_filters, cfg.n_ratios = 8, 128, 32, len(RATIOS)
    for k, r in enumerate(RATIOS):
        cfg.ratios[k] = r
    cfg.kernel, cfg.res_kernel, cfg.last_kernel, cfg.compress, cfg.max_frames = 7, 3, 7, 2, max_frames
    assert lib.mvb_voc_workspace_bytes(C.byref(cfg)) == want


def _mbd_cfg(max_seconds):
    s, u = MBDSettings(), MBDSettings().unet     # MultiBandDiffusionEngine's configuration for the default settings
    taps_p = _lowpass_bank(s.proc_bands, s.sample_rate).shape[1]
    taps_e = _lowpass_bank(s.eq_bands, s.sample_rate).shape[1]
    n_calls = _schedule_table(s.schedule, s.steps()).shape[0]
    return _lib.MbdConfig(s.n_models, u.chin, u.hidden, u.depth, u.res_blocks, u.norm_groups, u.kernel, u.stride, float(u.growth),
                          int(u.emb_all_layers), u.codec_dim, u.num_steps, n_calls, float(s.schedule.noise_scale),
                          float(s.schedule.clip), s.proc_bands, taps_p, s.eq_bands, taps_e, int(max_seconds * s.sample_rate))


@pytest.mark.parametrize("options,max_seconds,want", [
    (0, 30.0, 3849490688), (0, 12.0, 2317570304),
    (_lib.MVB_MBD_CUDA_CORES, 30.0, 2560819456),
    (_lib.MVB_MBD_ONE_STREAM, 30.0, 1928876288),
    (_lib.MVB_MBD_CUDA_CORES | _lib.MVB_MBD_ONE_STREAM, 30.0, 640205056),
], ids=["default-30s", "default-12s", "no_tc", "one_stream", "no_tc-one_stream"])
def test_mbd_workspace_bytes(lib, options, max_seconds, want):
    cfg = _mbd_cfg(max_seconds)
    cfg.options = options
    assert lib.mvb_mbd_workspace_bytes(C.byref(cfg)) == want


@pytest.mark.parametrize("max_seconds,want", [(180.0, 3932928), (30.0, 1532928)])
def test_speaker_workspace_bytes(lib, max_seconds, want):
    # SpeakerEncoder's front end and network at an explicit capacity (SpeakerEncoder(max_seconds=s) itself asks for
    # s * 16000 samples plus one 160-frame window, the most embed_utterance pads an s-second reference to)
    cfg = _lib.SpkConfig(40, 256, 3, 256, 400, 160, 160, int(max_seconds * 16000))
    assert lib.mvb_spk_workspace_bytes(C.byref(cfg)) == want


@pytest.mark.parametrize("n,want", [(1, 65792), (24000, 161536), (24000 * 60 + 7, 5825792)])
def test_audio_post_workspace_bytes(lib, n, want):
    assert lib.mvb_audio_post_workspace_bytes(n) == want

"""CPU: the C-ABI library loads and exports every symbol include/mvb200.h declares (no compute calls)."""
import ctypes
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "mvb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mvb_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_boundary():
    names = _declared()
    for must in ("mvb_s1_create", "mvb_s1_forward", "mvb_s1_sample", "mvb_s1_generate", "mvb_s1_decode",
                 "mvb_last_error"):
        assert must in names


def test_library_exports_every_declared_symbol():
    from mvb200 import _lib
    if not os.path.isfile(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in _declared():
        assert hasattr(lib, name), f"{name} declared in include/mvb200.h but not exported"
    assert set(_declared()) == set(_lib.SIGNATURES), "python binding table out of sync with the header"
    for hook in ("mvb_gemm_test", "mvb_mbd_conv_test", "mvb_mbd_op_test", "mvb_mbd_unet_test", "mvb_s2_attn_test", "mvb_s2_sample_test", "mvb_s2_embed_test",
                 "mvb_voc_op_test",
                 "mvb_audio_post_test", "mvb_spk_op_test"):
        assert hook in _lib.SIGNATURES and hasattr(lib, hook), f"test hook {hook} missing"
    assert lib.mvb_abi_version() == _lib.ABI_VERSION == 3


def test_config_validation_without_gpu():
    from mvb200 import _lib
    lib = _lib.load()
    ok = _lib.S1Config(24, 16, 128, 2048, 5632, 2562, 2048, 256, 1e-5, 1, 0, 2048)
    # 24 layers x {K,V} x 2 rows x 16 heads x 2048 slots x 128 x 2 B = 805,306,368 (SURVEY.md D5)
    assert lib.mvb_s1_kv_bytes(ctypes.byref(ok)) == 805306368
    assert lib.mvb_s1_workspace_bytes(ctypes.byref(ok)) > 0
    bad = _lib.S1Config(24, 16, 64, 1024, 5632, 2562, 2048, 256, 1e-5, 1, 0, 2048)
    assert lib.mvb_s1_kv_bytes(ctypes.byref(bad)) == 0
    assert b"head_dim" in lib.mvb_last_error()
    # speaker encoder: 1..64 mel bands (k_spk_lstm's input buffer), 2..2048-point frames, hop >= 1, and only the
    # reference's 256-wide 3-layer network
    def spk(**kw):
        return _lib.SpkConfig(**{**dict(n_mels=40, hidden=256, n_layers=3, emb=256, n_fft=400, hop=160, partial_frames=160,
                                        max_samples=16000), **kw})

    assert lib.mvb_spk_workspace_bytes(ctypes.byref(spk())) > 0
    for kw in (dict(n_mels=64), dict(n_mels=1), dict(n_fft=2), dict(n_fft=2048), dict(hop=1)):
        assert lib.mvb_spk_workspace_bytes(ctypes.byref(spk(**kw))) > 0, kw
    for kw, msg in ((dict(n_mels=0), b"front-end"), (dict(n_mels=65), b"front-end"), (dict(n_fft=1), b"front-end"),
                    (dict(n_fft=2049), b"front-end"), (dict(hop=0), b"front-end"), (dict(hidden=128), b"3 layers"),
                    (dict(n_layers=2), b"3 layers")):
        assert lib.mvb_spk_workspace_bytes(ctypes.byref(spk(**kw))) == 0, kw
        assert msg in lib.mvb_last_error(), (kw, lib.mvb_last_error())


_MBD_VALIDATE = r"""
import ctypes as C, sys
sys.path[:0] = [{root!r}, {pkg!r}]
from mvb200 import _lib
from mvb200.mbd import MBDSettings, _lowpass_bank, _schedule_table
lib = _lib.load()
s, u = MBDSettings(), MBDSettings().unet
cfg = _lib.MbdConfig(s.n_models, u.chin, u.hidden, u.depth, u.res_blocks, u.norm_groups, u.kernel, u.stride, float(u.growth),
                     int(u.emb_all_layers), u.codec_dim, u.num_steps, _schedule_table(s.schedule, s.steps()).shape[0],
                     float(s.schedule.noise_scale), float(s.schedule.clip), s.proc_bands,
                     _lowpass_bank(s.proc_bands, s.sample_rate).shape[1], s.eq_bands,
                     _lowpass_bank(s.eq_bands, s.sample_rate).shape[1], 12 * s.sample_rate)
for field, value in {overrides!r}:
    setattr(cfg, field, value)
print(lib.mvb_mbd_workspace_bytes(C.byref(cfg)), lib.mvb_last_error().decode())
"""


@pytest.mark.parametrize("overrides,want_error", [
    ([("norm_groups", 0)], "norm_groups"),
    ([("norm_groups", -1)], "norm_groups"),
    ([("norm_groups", 33), ("hidden", 33 * 4)], "norm_groups"),
    ([("proc_taps", 0)], "filter length"),
    ([("eq_taps", 19030)], "filter length"),
    ([("norm_groups", 32), ("hidden", 32 * 3), ("eq_taps", 19029)], None),
    ([("proc_bands", 64), ("proc_taps", 5921), ("eq_bands", 64), ("eq_taps", 5921)], None),
], ids=["groups0", "groups-1", "groups33", "taps0", "taps19030", "groups32-taps19029", "bands64"])
def test_mbd_config_validation(overrides, want_error):
    """mvb_mbd_workspace_bytes rejects GroupNorm group counts outside 1 .. 32 (the workspace's statistics slots and
    partials hold 32 groups; 0 used to divide by zero) and filters longer than k_fir_bank's shared memory can hold
    (227 KB: 19029 taps), and accepts the limits and a 64-band bank.  Each configuration runs in a child process, so that
    a crash of the validation cannot take the test session down with it."""
    from mvb200 import _lib
    if not os.path.isfile(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    code = _MBD_VALIDATE.format(root=ROOT, pkg=os.path.join(ROOT, "metavoice-src_b200"), overrides=overrides)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, f"child exited with {r.returncode}: {r.stderr[-2000:]}"
    nbytes, _, err = r.stdout.strip().partition(" ")
    if want_error is None:
        assert int(nbytes) > 0, err
    else:
        assert int(nbytes) == 0 and want_error in err, r.stdout


def _engine_configs():
    """Production configurations (options = 0) of the three engines whose config carries `options`: stage 1 at 8
    utterances, stage 2 at batch 1, MBD at its default settings and 12 s."""
    from mvb200 import _lib, synth
    from mvb200.mbd import MBDSettings, _lowpass_bank, _schedule_table
    d = synth.FULL
    s1 = _lib.S1Config(d.n_layer, d.n_head, d.head_dim, d.dim, d.intermediate_size, d.vocab_size, d.block_size,
                       d.speaker_emb_dim, d.norm_eps, 8, _lib.MVB_KV_BF16, d.block_size)
    e = synth.S2_FULL
    s2 = _lib.S2Config()
    s2.n_layer, s2.n_head, s2.n_embd, s2.hidden = e.n_layer, e.n_head, e.n_embd, e.hidden
    s2.block_size, s2.n_in, s2.n_out = e.block_size, len(e.vocab_sizes), len(e.target_vocab_sizes)
    for i, v in enumerate(e.vocab_sizes):
        s2.vocab_in[i] = v
    for i, v in enumerate(e.target_vocab_sizes):
        s2.vocab_out[i] = v
    s2.spk_dim, s2.norm_eps, s2.max_batch = e.speaker_emb_dim, e.rmsnorm_eps, 1
    s, u = MBDSettings(), MBDSettings().unet
    mbd = _lib.MbdConfig(s.n_models, u.chin, u.hidden, u.depth, u.res_blocks, u.norm_groups, u.kernel, u.stride, float(u.growth),
                         int(u.emb_all_layers), u.codec_dim, u.num_steps, _schedule_table(s.schedule, s.steps()).shape[0],
                         float(s.schedule.noise_scale), float(s.schedule.clip), s.proc_bands,
                         _lowpass_bank(s.proc_bands, s.sample_rate).shape[1], s.eq_bands,
                         _lowpass_bank(s.eq_bands, s.sample_rate).shape[1], 12 * s.sample_rate)
    return s1, s2, mbd


def _workspace_sizes():
    from mvb200 import _lib
    lib = _lib.load()
    s1, s2, mbd = (ctypes.byref(c) for c in _engine_configs())
    return {"s1_kv": lib.mvb_s1_kv_bytes(s1), "s1": lib.mvb_s1_workspace_bytes(s1), "s1_int4": lib.mvb_s1_int4_workspace_bytes(s1),
            "s2": lib.mvb_s2_workspace_bytes(s2), "mbd": lib.mvb_mbd_workspace_bytes(mbd)}


# environment variables that earlier versions of the library read when an engine was created
_OLD_SWITCHES = {"MVB_PATHB": "0", "MVB_PATHC": "0", "MVB_PC_FUSED": "0", "MVB_PC_TRACE": "1", "MVB_PDL": "0",
                 "MVB_S2_NO_GRAPH": "1", "MVB_MBD_NO_TC": "1", "MVB_MBD_STREAMS": "0"}


def test_workspace_sizes_ignore_the_process_environment():
    """Engine paths are chosen by the config's `options` alone: in a process whose environment sets every variable an
    earlier library read, each workspace size equals the one for options = 0.  The MBD workspace used to follow two of
    them, so a buffer sized under one environment could be too small for the engine created under another."""
    want = _workspace_sizes()
    assert all(v > 0 for v in want.values()), want
    code = (f"import sys; sys.path[:0] = {[ROOT, os.path.join(ROOT, 'metavoice-src_b200'), os.path.join(ROOT, 'tests')]!r}\n"
            "import json, test_capi_abi as t; print(json.dumps(t._workspace_sizes()))")
    r = subprocess.run([sys.executable, "-c", code], env={**os.environ, **_OLD_SWITCHES}, capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert json.loads(r.stdout) == want


def test_undefined_option_bits_are_rejected():
    """`options` comes from outside the library: a bit no engine defines makes the workspace query fail and names the
    field, before any engine could be created with it."""
    from mvb200 import _lib
    lib = _lib.load()
    s1, s2, mbd = _engine_configs()
    for cfg, fn, bits in ((s1, lib.mvb_s1_workspace_bytes, (0x10, -2 ** 31)), (s2, lib.mvb_s2_workspace_bytes, (0x2, -2 ** 31)),
                          (mbd, lib.mvb_mbd_workspace_bytes, (0x4, -2 ** 31))):
        assert fn(ctypes.byref(cfg)) > 0
        for bit in bits:
            cfg.options = bit
            assert fn(ctypes.byref(cfg)) == 0, (fn.__name__, bit)
            assert b"options" in lib.mvb_last_error(), (fn.__name__, bit, lib.mvb_last_error())
        cfg.options = 0


def test_missing_library_fails_loudly(monkeypatch):
    from mvb200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libmvb200.so")
    with pytest.raises(_lib.MvbError, match="no CPU or PyTorch fallback"):
        _lib.load()

"""tests/golden/speaker_device_bits.npz: the partial and utterance embeddings that the device speaker encoder
(csrc/speaker.cu through mvb200.speaker_encoder.SpeakerEncoder) produced on an H100 before k_spk_lstm gained its optional
state trace, on the golden 6.4 s waveform and on a 30 s one.  tests/test_speaker_ops_gpu.py holds the current library to
these bits, so that production (no trace) computes exactly what it computed before.

GPU only, with MVB200_LIB naming the library to record (built from the commit before the trace with
`make BUILD=build_alt OUT=../mvb200/libmvb200_alt.so`):
    MVB200_LIB=<path> python oracle/make_golden_speaker_bits.py [out.npz]
Regenerate only on a deliberate change of the speaker encoder's arithmetic."""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "metavoice-src_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def waveforms():
    from mvb200 import synth
    g = np.load(os.path.join(ROOT, "tests", "golden", "speaker.npz"))
    return {"golden": g["wav"], "s30": synth.synthetic_waveform(30.0, 16000, seed=7)}


def main(out):
    from mvb200 import _lib, synth
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in [n for n in _lib.SIGNATURES if not hasattr(lib, n)]:   # an older build lacks the newer test hooks
        del _lib.SIGNATURES[name]
    from mvb200.speaker_encoder import SpeakerEncoder
    enc = SpeakerEncoder(model_state=synth.speaker_encoder_state_dict(3), device="cuda:0", verbose=False)
    arrays = {}
    for name, wav in waveforms().items():
        e, p, _ = enc.embed_utterance(wav, return_partials=True)
        arrays[f"{name}_embed"], arrays[f"{name}_partials"] = e, p
    enc.close()
    np.savez_compressed(out, **arrays)
    print(f"{_lib.LIB_PATH}: " + ", ".join(f"{k} {v.shape}" for k, v in arrays.items()))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "speaker_device_bits.npz"))

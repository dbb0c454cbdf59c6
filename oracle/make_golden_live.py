"""Record what the reference's own code returns for the checks that used to call it live, so that the tests run
self-contained: tests/golden/reference_calls.npz.  Needs the reference tree (see ref_harness); CPU only:

    python oracle/make_golden_live.py

  * stage-1 port vs the reference Transformer (tiny seeded checkpoint): logits of a 9-token prefill, and the tokens of
    the reference generate() under torch.manual_seed(5);
  * SpeakerEncoder.compute_partial_slices for a grid of lengths / rates / coverages;
  * the two adapters' decode() on seeded random token lists;
  * the stage-2 input tensor of the reference's Model for three texts / code lengths.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "metavoice-src_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from mvb200 import synth  # noqa: E402

SLICE_LENS = (16000, 25601, 102400, 480000, 777777)
SLICE_PARAMS = ((1.3, 0.75), (2.0, 0.5))
S2_TEXTS = ["a b c", "the quick brown fox", "x"]
S2_CODE_LENS = (10, 300, 255)


def stage1_inputs():
    d = synth.TINY
    return d, synth.stage1_state_dict(d, 3), synth.synthetic_prompt(9, seed=5), synth.synthetic_speaker(seed=2)


def adapter_inputs():
    g = torch.Generator().manual_seed(0)
    flat = torch.randint(0, 2562, (300,), generator=g).tolist()
    hier = torch.randint(0, 1100, (8, 200), generator=g).tolist()
    return flat, hier


def stage2_inputs():
    from mvb200.tokenise import TrainedBPETokeniser
    tok = TrainedBPETokeniser(**synth.synthetic_tokenizer_meta(n_text_tokens=512, offset=1025))
    g = torch.Generator().manual_seed(77)
    codes = [torch.randint(0, 1024, (1, 2, n), generator=g) for n in S2_CODE_LENS]
    return tok, codes


def main():
    from oracle import ref_harness
    out = {}
    d, sd, prompt, spk = stage1_inputs()
    ref = ref_harness.build_reference_model(sd, d, torch.float32)
    idx = prompt.view(1, -1).repeat(2, 1)
    with torch.no_grad():
        out["s1_logits"] = ref(idx, spk, torch.arange(9)).float().numpy()
    fiu = ref_harness.reference_functions()
    ref2 = ref_harness.build_reference_model(sd, d, torch.float32)
    kw = dict(temperature=torch.tensor(0.8), top_p=torch.tensor(0.9), guidance_scale=torch.tensor(2.0), top_k=None)
    torch.manual_seed(5)
    out["s1_tokens"] = np.asarray(fiu.generate(ref2, prompt, spk, max_new_tokens=12, end_of_audio_token=9999, **kw).tolist(),
                                  dtype=np.int64)

    from fam.quantiser.audio.speaker_encoder.model import SpeakerEncoder as Ref
    slices = []
    for n in SLICE_LENS:
        for rate, cov in SLICE_PARAMS:
            w, m = Ref.compute_partial_slices(n, rate, cov)
            slices.append([[(s.start, s.stop) for s in w], [(s.start, s.stop) for s in m]])
    for i, (w, m) in enumerate(slices):
        out[f"slices_{i}_wav"] = np.asarray(w, dtype=np.int64).reshape(-1, 2)
        out[f"slices_{i}_mel"] = np.asarray(m, dtype=np.int64).reshape(-1, 2)

    from fam.llm.adapters import FlattenedInterleavedEncodec2Codebook, TiltedEncodec
    flat, hier = adapter_inputs()
    text, cb = FlattenedInterleavedEncodec2Codebook(end_of_audio_token=1024).decode([flat])
    out["flat_text"] = np.asarray(text, dtype=np.int64)
    for i, c in enumerate(cb):
        out[f"flat_cb_{i}"] = np.asarray(c, dtype=np.int64)
    out["flat_n_cb"] = np.int64(len(cb))
    text, codes = TiltedEncodec(end_of_audio_token=1024).decode(hier)
    out["tilted_text"] = np.asarray(text, dtype=np.int64)
    for i, c in enumerate(codes):
        out[f"tilted_codes_{i}"] = np.asarray(c, dtype=np.int64)
    out["tilted_n_codes"] = np.int64(len(codes))

    import importlib.util
    spec = importlib.util.spec_from_file_location("mk_s2in", os.path.join(ROOT, "oracle", "make_golden_stage2_input.py"))
    mk = importlib.util.module_from_spec(spec); spec.loader.exec_module(mk)
    tok, codes = stage2_inputs()
    in_x = mk.reference_in_x(mk.reference_model_class(), tok, S2_TEXTS, codes, 256)
    for i in range(len(S2_TEXTS)):
        out[f"s2_in_x_{i}"] = in_x[i].numpy().astype(np.int64)

    path = os.path.join(ROOT, "tests", "golden", "reference_calls.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

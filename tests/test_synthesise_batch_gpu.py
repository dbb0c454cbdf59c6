"""GPU: `TTS.synthesise_batch` on a tiny synthetic snapshot (3 texts, 2 speakers, fixed seed).

Each returned file must equal, byte for byte, the same utterance run alone through the public pieces: stage 1 through a
`ContinuousBatcher` over a one-slot engine with the same per-request draws (`serving.seeded_noise(seed + i)`), stage 2
through `SecondStage.non_causal_sample`, then `EncodecDecodeEngine.decode` and `audio_out.wav_bytes_on_device`.  Stage 2
is called over the same three utterances with the same seed as the batch: its sampler keys its stream on the row within
the batch, so that call is what fixes an utterance's stage-2 codes.  Results come back in input order, and an
utterance forced below 400 ms yields None while the others are still written."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

TEXTS = ["Hello, what's up?", "The quick brown fox.", "A third, somewhat longer sentence to say."]
SEED = 1234


@pytest.fixture(scope="module")
def snap(tmp_path_factory):
    from mvb200 import synth
    d = tmp_path_factory.mktemp("snapshot")
    torch.save(synth.stage1_checkpoint(synth.TINY, 0), str(d / "first_stage.pt"))
    torch.save(synth.stage2_checkpoint(synth.S2_TINY, 1), str(d / "second_stage.pt"))
    _, enc_sd = synth.encodec_model_and_state_dict(0)
    spks = [str(d / "spk_a.pt"), str(d / "spk_b.pt")]
    torch.save(synth.synthetic_speaker(seed=11), spks[0])
    torch.save(synth.synthetic_speaker(seed=12), spks[1])
    return d, enc_sd, [spks[0], spks[1], spks[0]]


def _solo_reference(tts, snap_dir, spk_paths):
    """Per utterance: stage-1 tokens from a one-slot engine, stage-2 codes, and the wav file bytes."""
    from mvb200.audio_out import wav_bytes_on_device
    from mvb200.fast_inference import load_speaker_embedding, normalize_text
    from mvb200.fast_inference_utils import build_model, encode_tokens
    from mvb200.second_stage import flattened_interleaved_decode
    from mvb200.serving import ContinuousBatcher, seeded_noise
    model, tok, _, _ = build_model(checkpoint_path=snap_dir / "first_stage.pt", device="cuda:0", max_utts=1)
    model._cfg.max_new = 256
    texts = [normalize_text(t) for t in TEXTS]
    spk = [load_speaker_embedding(p) for p in spk_paths]
    extracted = []
    for i, (t, e) in enumerate(zip(texts, spk)):
        prompt = encode_tokens(tok, t, device="cpu")
        noise = seeded_noise(model, prompt.numel(), SEED + i)
        cb = ContinuousBatcher(model)
        rid = cb.submit(prompt, e, max_new_tokens=noise.shape[0], noise=noise, top_p=0.95, guidance_scale=3.0, temperature=1.0)
        extracted.append(flattened_interleaved_decode(cb.run_until_done()[rid].tolist(), 1024)[1])
    model.close()
    codes = tts.llm_second_stage.non_causal_sample(
        texts=texts, encodec_tokens=[torch.tensor(x, dtype=torch.int32).unsqueeze(0) for x in extracted],
        speaker_embs=torch.stack(spk), batch_size=3, top_k=200, temperature=1.0, seed=SEED)
    return codes, [wav_bytes_on_device(tts.codec.decode(c), 24000) for c in codes]


def test_synthesise_batch_equals_solo_runs_in_order(snap, tmp_path):
    from mvb200.fast_inference import TTS
    snap_dir, enc_sd, spk_paths = snap
    tts = TTS(str(snap_dir), output_dir=str(tmp_path / "out"), encodec_state_dict=enc_sd, device="cuda:0", max_utts=3)
    tts.model._cfg.max_new = 256
    assert tts.codec.max_batch == 3 and tts.llm_second_stage.cfg.max_batch == 3
    codes, want = _solo_reference(tts, snap_dir, spk_paths)
    frames = [c.shape[-1] for c in codes]
    print(f"stage-2 frames per utterance: {frames}")
    assert min(frames) >= 30, "the seeded utterances must be long enough to be written"
    paths = tts.synthesise_batch(TEXTS, spk_paths, top_p=0.95, guidance_scale=3.0, temperature=1.0, seed=SEED)
    assert len(paths) == 3
    for i, p in enumerate(paths):
        assert p is not None and os.path.isfile(p) and p.endswith(".wav")
        assert open(p, "rb").read() == want[i], f"utterance {i}: the file differs from its solo run"
    # same seed, same files; a different seed changes them
    again = tts.synthesise_batch(TEXTS, spk_paths, seed=SEED)
    assert [open(p, "rb").read() for p in again] == want
    other = tts.synthesise_batch(TEXTS, spk_paths, seed=SEED + 100)
    assert [open(p, "rb").read() for p in other] != want

    # an utterance forced below 400 ms (29 frames = 9280 samples) yields None; the others are still written
    real = tts.llm_second_stage.non_causal_sample

    def short_middle(**kw):
        out = real(**kw)
        out[1] = out[1][:, :29]
        return out

    tts.llm_second_stage.non_causal_sample = short_middle
    try:
        paths = tts.synthesise_batch(TEXTS, spk_paths, seed=SEED)
    finally:
        tts.llm_second_stage.non_causal_sample = real
    assert paths[1] is None
    assert open(paths[0], "rb").read() == want[0] and open(paths[2], "rb").read() == want[2]

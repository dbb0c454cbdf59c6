"""GPU: SpeakerEncoder.embed_files, get_cached_embeddings and TTS.embed_speakers on files.

embed_files runs the reference front-end on the device (fp32 polyphase resampling, fp32 trim, batched embedding) where
embed_utterance_from_file resamples in float64 and trims on the host.  On these signals no trim frame lies near the
threshold, so both paths embed the same span and differ only by the resampler's fp32 rounding, which the free-running
network carries into the embedding.  FILE_BOUND bounds the normwise difference of the embeddings; the observed value
is printed."""
import os
import struct

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
FILE_BOUND = 1e-4


def _write_wav(path, x, sr):
    """PCM16 RIFF/WAVE; x is [n] (mono) or [channels, n]."""
    x = np.atleast_2d(x)
    pcm = np.clip(np.round(x.T * 32767), -32768, 32767).astype("<i2").tobytes()
    ch = x.shape[0]
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 36 + len(pcm)) + b"WAVE")
        f.write(b"fmt " + struct.pack("<IHHIIHH", 16, 1, ch, sr, sr * ch * 2, ch * 2, 16))
        f.write(b"data" + struct.pack("<I", len(pcm)) + pcm)


def _reference(sr, seconds, seed, stereo):
    from mvb200 import synth
    x = synth.synthetic_waveform(seconds, sr, seed=seed)
    lead, tail = int(0.7 * sr), int(1.1 * sr)
    x[:lead] = 0
    x[-tail:] = 0
    if stereo:
        return np.stack([x, 0.5 * np.roll(x, 37)])
    return x


@pytest.fixture(scope="module")
def enc():
    from mvb200 import synth
    from mvb200.speaker_encoder import SpeakerEncoder
    e = SpeakerEncoder(model_state=synth.speaker_encoder_state_dict(3), device=DEV, verbose=False)
    yield e
    e.close()


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("refs")
    out = []
    for k, (sr, stereo) in enumerate([(16000, False), (22050, True), (44100, False), (48000, True), (44100, True),
                                      (16000, True), (22050, False), (48000, False)]):
        p = str(d / f"ref{k}_{sr}_{'st' if stereo else 'mo'}.wav")
        _write_wav(p, _reference(sr, 30.5 + k % 3, seed=20 + k, stereo=stereo), sr)
        out.append(p)
    return out


def test_embed_files_vs_host_front_end(enc, files):
    got = enc.embed_files(files).cpu().numpy()
    assert got.shape == (len(files), 256)
    worst = 0.0
    for i, p in enumerate(files):
        want = enc.embed_utterance_from_file(p, numpy=True)
        nw = float(np.linalg.norm(got[i] - want) / np.linalg.norm(want))
        print(f"embed_files {os.path.basename(p)}: normwise {nw:.2e} against embed_utterance_from_file")
        worst = max(worst, nw)
        assert nw < FILE_BOUND, (p, nw)
    print(f"embed_files: worst normwise {worst:.2e}, bound {FILE_BOUND:.0e}")
    # the input order is kept whatever the rates
    rev = enc.embed_files(files[::-1]).cpu().numpy()
    assert np.array_equal(rev, got[::-1])


def test_embed_files_errors_name_the_file(enc, tmp_path):
    short = str(tmp_path / "short.wav")
    _write_wav(short, _reference(16000, 5, 1, False), 16000)
    with pytest.raises(Exception, match="short.wav.*too short"):
        enc.embed_files([short])
    odd = str(tmp_path / "odd_rate.wav")
    _write_wav(odd, _reference(44099, 31, 2, False), 44099)
    with pytest.raises(ValueError, match="odd_rate.wav.*taps"):
        enc.embed_files([odd])
    long = str(tmp_path / "long.wav")
    _write_wav(long, _reference(8000, 181, 3, False), 8000)
    with pytest.raises(ValueError, match="long.wav.*longer than 180 s"):
        enc.embed_files([long])


def test_get_cached_embeddings(enc, files, tmp_path, monkeypatch):
    from mvb200.speaker_encoder import _embedding_cache_path, get_cached_embedding, get_cached_embeddings
    monkeypatch.setenv("HOME", str(tmp_path))
    a, b, c = files[0], files[2], files[3]
    hit = get_cached_embedding(a, enc)                    # written by the single-file path
    assert os.path.isfile(_embedding_cache_path(a)) and not os.path.isfile(_embedding_cache_path(b))
    got = get_cached_embeddings([b, a, c, b], enc)
    assert got.shape == (4, 256) and got.device.type == "cpu"
    assert torch.equal(got[1], hit[0])
    assert torch.equal(got[0], got[3])
    want = enc.embed_files([b, c]).cpu()
    assert torch.equal(got[0], want[0]) and torch.equal(got[2], want[1])
    for p, row in ((b, got[0]), (c, got[2])):             # written back, readable by the single-file path
        assert torch.equal(get_cached_embedding(p, enc)[0], row)
    again = get_cached_embeddings([c, a, b], enc)
    assert torch.equal(again, got[[2, 1, 0]])


def test_embed_speakers_feeds_synthesise_batch(files, tmp_path, monkeypatch):
    from mvb200 import synth
    from mvb200.fast_inference import TTS, load_speaker_embedding
    monkeypatch.setenv("HOME", str(tmp_path))
    d = tmp_path / "snapshot"
    d.mkdir()
    torch.save(synth.stage1_checkpoint(synth.TINY, 0), str(d / "first_stage.pt"))
    torch.save(synth.stage2_checkpoint(synth.S2_TINY, 1), str(d / "second_stage.pt"))
    torch.save({"model_state": synth.speaker_encoder_state_dict(3)}, str(d / "speaker_encoder.pt"))
    _, enc_sd = synth.encodec_model_and_state_dict(0)
    pt, npy = str(tmp_path / "spk.pt"), str(tmp_path / "spk.npy")
    torch.save(synth.synthetic_speaker(seed=11), pt)
    np.save(npy, synth.synthetic_speaker(seed=12).numpy())
    tts = TTS(str(d), output_dir=str(tmp_path / "out"), encodec_state_dict=enc_sd, device="cuda:0", max_utts=3)
    tts.model._cfg.max_new = 256
    refs = [pt, npy, files[2]]
    embs = tts.embed_speakers(refs)
    assert embs.shape == (3, 256)
    assert torch.equal(embs[0], load_speaker_embedding(pt)[0]) and torch.equal(embs[1], load_speaker_embedding(npy)[0])
    saved = []
    for i, e in enumerate(embs):
        p = str(tmp_path / f"emb{i}.pt")
        torch.save(e.clone(), p)
        saved.append(p)
    texts = ["Hello, what's up?", "The quick brown fox.", "A third sentence."]
    # the wav reference is read back from the cache embed_speakers filled, so both runs see the same embeddings
    want = tts.synthesise_batch(texts, refs, seed=77)
    got = tts.synthesise_batch(texts, saved, seed=77)
    assert all(p is not None for p in want + got)
    assert [open(p, "rb").read() for p in got] == [open(p, "rb").read() for p in want]

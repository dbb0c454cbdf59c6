"""Host-side mirror of the façade ``fam/llm/fast_inference.py::TTS`` over libmvb200.

Same constructor keywords and the same ``synthesise(text, spk_ref_path, top_p, guidance_scale, temperature) -> path``
contract (fast_inference.py:41-50, 111-119, 195).  Differences, all stated where they occur:
  * checkpoints are read from a local directory (the reference calls ``snapshot_download``, :71; no network here);
  * the speaker reference may be a RIFF/WAVE file (>= 30 s, utils.py:55-70), embedded by the on-device speaker encoder
    (mvb200/speaker_encoder.py, SURVEY.md N3) and disk-cached like the reference (inference.py:419-435), or an already
    computed embedding (``.pt`` tensor / ``.npy``); mp3 / flac / URLs need a decoder / network that this image lacks;
  * the vocoder stage is the EnCodec decoder followed by the multi-band-diffusion refinement (mvb200/mbd.py; parity
    UNPINNED, its configuration is read from ``multiband_diffusion.pt`` in the model directory or passed in) when such a
    checkpoint is available; the DeepFilterNet enhancer (fast_inference.py:158-163) is not implemented (N1);
  * the wav goes through the reference's ``audio_write`` post-processing (loudness normalisation to -14 LUFS, tanh
    compressor, PCM16; decoders.py:40-47) in mvb200/audio_out.py.
Extension keywords: ``max_utts`` (KV slots of the stage-1 engine, the batch of ``synthesise_batch``), ``kv_dtype``
("bf16", the reference's cache; "fp8", e4m3 with one bf16 scale per head vector at half the cache bytes; "fp32") and
``voices`` ({name: first_stage.pt} of last-N-block finetunes that fam/llm/finetune.py writes, served by the one stage-1
engine; ``voice=`` / ``voices=`` of the synthesis calls select them by name, None being the base checkpoint).
"""
from __future__ import annotations

import os
import re
import time
import uuid
from datetime import datetime
from pathlib import Path
from typing import Dict, List, Literal, Optional

import numpy as np
import torch

from .fast_inference_utils import build_model, main, split_guidance
from .second_stage import SecondStage, flattened_interleaved_decode
from .tokenise import TrainedBPETokeniser
from .vocoder import EncodecDecodeEngine

_UNICODE = {8175: "'", 8189: "'", 8190: "'", 8208: "-", 8209: "-", 8210: "-", 8211: "-", 8212: "-", 8213: "-", 8214: "||",
            8216: "'", 8217: "'", 8218: ",", 8219: "`", 8220: '"', 8221: '"', 8222: ",,", 8223: '"', 8228: ".", 8229: "..",
            8230: "...", 8242: "'", 8243: '"', 8245: "'", 8246: '"', 180: "'", 2122: "TM"}


from .audio_out import audio_write_wav  # noqa: E402


def normalize_text(text: str) -> str:
    """fam/llm/utils.py:12-52: map typographic punctuation, reject code points >= 256, collapse whitespace."""
    text = text.translate(_UNICODE)
    bad = {c for c in text if ord(c) >= 256}
    if bad:
        raise ValueError(f"Non-supported character found: {[(c, ord(c)) for c in bad]}")
    text = text.replace("\t", " ").replace("\n", " ").replace("\r", " ").replace("*", " ").strip()
    return re.sub(r"\s\s+", " ", text)


def load_speaker_embedding(path: str, smodel=None) -> torch.Tensor:
    if not os.path.exists(path):
        raise FileNotFoundError(f"File {path} not found!")      # inference.py:412-415, 420-421
    if path.endswith(".npy"):
        e = torch.from_numpy(np.load(path))
    elif path.endswith(".pt"):
        e = torch.load(path, map_location="cpu")
    else:
        if smodel is None:
            raise FileNotFoundError("speaker_encoder.pt not found in the model directory: pass a precomputed embedding (.pt / .npy)")
        from .speaker_encoder import check_audio_file, get_cached_embedding
        check_audio_file(path)                                  # fast_inference.py:123: >= 30 s of reference audio
        e = get_cached_embedding(path, smodel)                  # fast_inference.py:124-127
    return e.reshape(1, -1).float()


class TTS:
    END_OF_AUDIO_TOKEN = 1024

    def __init__(self, model_name: str = "metavoiceio/metavoice-1B-v0.1", *, seed: int = 1337, output_dir: str = "outputs",
                 quantisation_mode: Optional[Literal["int4", "int8", "fp8"]] = None, first_stage_path: Optional[str] = None,
                 telemetry_origin: Optional[str] = None, encodec_state_dict=None, device: str = "cuda", max_utts: int = 1,
                 mbd_checkpoint: Optional[dict] = None, mbd_settings=None,
                 kv_dtype: Literal["bf16", "fp32", "fp8"] = "bf16", voices: Optional[Dict[str, str]] = None):
        if voices and quantisation_mode is not None:    # before any checkpoint is read
            raise NotImplementedError(f"voices are served by bf16-weight engines only (quantisation_mode={quantisation_mode!r})")
        self._device = device
        self._model_dir = model_name
        if not os.path.isdir(model_name):
            raise FileNotFoundError(f"{model_name}: pass a local snapshot directory holding first_stage.pt / second_stage.pt "
                                    "(there is no network access for snapshot_download)")
        self.output_dir = output_dir
        os.makedirs(self.output_dir, exist_ok=True)
        self._first_stage_ckpt = first_stage_path or f"{self._model_dir}/first_stage.pt"
        torch.manual_seed(seed)                                                        # inference.py:69-70
        ck2 = torch.load(f"{self._model_dir}/second_stage.pt", map_location="cpu", weights_only=False)
        tok2 = TrainedBPETokeniser(**ck2["meta"]["tokenizer"])
        self.llm_second_stage = SecondStage(ck2, device=device, tokenizer=tok2, max_batch=max_utts)
        if encodec_state_dict is None:
            encodec_state_dict = torch.load(f"{self._model_dir}/encodec_24khz.pt", map_location="cpu", weights_only=False)
        # synthesise_batch decodes up to max_utts utterances (at most 32) per launch set, 10 s of audio each on average;
        # longer batches are split
        codec_batch = min(max_utts, 32)
        self.codec = EncodecDecodeEngine(encodec_state_dict, device=device, max_batch=codec_batch,
                                         max_total_frames=codec_batch * 750 if codec_batch > 1 else None)
        # decoders.py:13: MultiBandDiffusion.get_mbd_24khz(bw=6) -- here: {"models", "proc", "settings"} (see mvb200/mbd.py)
        self.mbd = None
        mbd_path = f"{self._model_dir}/multiband_diffusion.pt"
        if mbd_checkpoint is None and os.path.isfile(mbd_path):
            mbd_checkpoint = torch.load(mbd_path, map_location="cpu", weights_only=False)
            mbd_settings = mbd_settings or mbd_checkpoint.get("settings")
        if mbd_checkpoint is not None:
            from .mbd import MBDSettings, MultiBandDiffusionEngine
            self.mbd = MultiBandDiffusionEngine(mbd_checkpoint, mbd_settings or MBDSettings(), device=device, max_seconds=30.0)
        self.precision = torch.bfloat16
        self.model, self.tokenizer, self.smodel, self.model_size = build_model(
            precision=self.precision, checkpoint_path=Path(self._first_stage_ckpt),
            spk_emb_ckpt_path=Path(f"{self._model_dir}/speaker_encoder.pt"), device=device, compile=True,
            compile_prefill=True, quantisation_mode=quantisation_mode, max_utts=max_utts, kv_dtype=kv_dtype)
        self._seed = seed
        # last-N-block finetunes of the first stage, each an overlay of its finetuned blocks and ln_f on the one engine
        self.voices: Dict[str, int] = {}
        for name, path in (voices or {}).items():
            self.voices[name] = self.model.add_voice(torch.load(str(path), map_location="cpu", mmap=True, weights_only=False))
        spk_ckpt = f"{self._model_dir}/speaker_encoder.pt"
        if os.path.isfile(spk_ckpt):                                                   # fast_inference_utils.py:314-318
            from .speaker_encoder import SpeakerEncoder
            self.smodel = SpeakerEncoder(weights_fpath=spk_ckpt, device=device, eval=True, verbose=False)

    def _check_guidance(self, guidance_scale) -> None:
        """``guidance_scale`` is a float or the reference's ``(s, p)`` (inference.py:646-647).  With p > 1 every text is
        decoded on two KV slots (its own and the prompt-guidance companion), which a one-slot engine does not have."""
        _, p = split_guidance(guidance_scale, self.tokenizer.eot_token)
        if p is not None and self.model.max_utts < 2:
            raise ValueError(f"guidance_scale={tuple(guidance_scale)!r} (prompt guidance) decodes each text on two KV slots; "
                             "create the TTS with max_utts=2 or more")

    def _voice(self, name: Optional[str]) -> int:
        """Voice id of a name given to ``TTS(voices=...)``; None is the base checkpoint.  KeyError for any other name."""
        if name is None:
            return 0
        if name not in self.voices:
            raise KeyError(f"voice {name!r} is not one of the TTS's voices {sorted(self.voices)}")
        return self.voices[name]

    def synthesise(self, text: str, spk_ref_path: str, top_p=0.95, guidance_scale=3.0, temperature=1.0,
                   voice: Optional[str] = None) -> str:
        vid = self._voice(voice)
        self._check_guidance(guidance_scale)
        text = normalize_text(text)
        spk_emb = load_speaker_embedding(spk_ref_path, self.smodel)
        start = time.time()
        tokens = main(model=self.model, tokenizer=self.tokenizer, model_size=self.model_size, prompt=text, spk_emb=spk_emb,
                      top_p=top_p, guidance_scale=guidance_scale, temperature=temperature, device=self._device, voice=vid)
        _, extracted = flattened_interleaved_decode(tokens, self.END_OF_AUDIO_TOKEN)
        codes = self.llm_second_stage.non_causal_sample(
            texts=[text], encodec_tokens=[torch.tensor(extracted, dtype=torch.int32).unsqueeze(0)],
            speaker_embs=spk_emb.unsqueeze(0), batch_size=1, top_k=200, temperature=1.0)[0]
        wav = self._tokens_to_wav(codes)
        if wav.shape[-1] < 9600:
            raise Exception("wav predicted is shorter than 400ms!")                    # decoders.py:88-91
        name = f"synth_{datetime.now().strftime('%y-%m-%d--%H-%M-%S')}_{text.replace(' ', '_')[:25]}_{uuid.uuid4()}"
        # decoders.py:40-47: audio_write(strategy="loudness", loudness_compressor=True) -> <name>.wav
        path = audio_write_wav(str(Path(self.output_dir).resolve() / name), wav.reshape(1, -1), 24000,
                               strategy="loudness", loudness_compressor=True)
        print(f"\nSaved audio to {path}")
        dt = time.time() - start
        dur = wav.shape[-1] / 24000.0
        print(f"\nTotal time to synth (s): {dt}")
        print(f"Real-time factor: {dt / dur:.2f}")
        return path

    def _tokens_to_wav(self, codes: torch.Tensor) -> torch.Tensor:
        """decoders.py:84-85 ``mbd.tokens_to_wav(tokens)``: codec decode, then (when a diffusion checkpoint is loaded) the
        multi-band-diffusion refinement conditioned on the codec latent and re-equalised against the codec waveform."""
        wav = self.codec.decode(codes)
        if self.mbd is not None:
            wav = self.mbd.tokens_to_wav(self.codec.decode_latent(codes), wav)
        return wav

    def synthesise_long(self, text: str, spk_ref_path: str, top_p=0.95, guidance_scale=3.0, temperature=1.0,
                        max_chars: int = 220, voice: Optional[str] = None) -> str:
        """Long-form synthesis (the reference truncates at 220 characters, inference.py:535-541: "Long form synthesis
        coming soon"): the text is cut into <= ``max_chars`` chunks at sentence boundaries, the chunks are decoded as one
        continuous batch over the engine's KV slots (``TTS(max_utts=...)``), every chunk goes through stage 2 and the
        vocoder, and the waveforms are concatenated into one file."""
        from .fast_inference_utils import encode_tokens
        from .serving import ContinuousBatcher, chunk_text
        vid = self._voice(voice)
        self._check_guidance(guidance_scale)
        chunks = chunk_text(normalize_text(text), max_chars)
        if not chunks:
            raise ValueError("empty text")
        spk_emb = load_speaker_embedding(spk_ref_path, self.smodel)
        start = time.time()
        cb = ContinuousBatcher(self.model)
        ids = [cb.submit(encode_tokens(self.tokenizer, c, device="cpu"), spk_emb, top_p=top_p, guidance_scale=guidance_scale,
                         temperature=temperature, end_of_text_token=self.tokenizer.eot_token, voice=vid) for c in chunks]
        toks = cb.run_until_done()
        wavs = []
        for c, rid in zip(chunks, ids):
            _, extracted = flattened_interleaved_decode(toks[rid].tolist(), self.END_OF_AUDIO_TOKEN)
            codes = self.llm_second_stage.non_causal_sample(
                texts=[c], encodec_tokens=[torch.tensor(extracted, dtype=torch.int32).unsqueeze(0)],
                speaker_embs=spk_emb.unsqueeze(0), batch_size=1, top_k=200, temperature=1.0)[0]
            wavs.append(self._tokens_to_wav(codes).reshape(-1))
        wav = torch.cat(wavs)
        if wav.shape[-1] < 9600:
            raise Exception("wav predicted is shorter than 400ms!")                    # decoders.py:88-91
        name = f"synth_{datetime.now().strftime('%y-%m-%d--%H-%M-%S')}_{chunks[0].replace(' ', '_')[:25]}_{uuid.uuid4()}"
        path = audio_write_wav(str(Path(self.output_dir).resolve() / name), wav.reshape(1, -1), 24000,
                               strategy="loudness", loudness_compressor=True)
        dt = time.time() - start
        print(f"\nSaved audio to {path} ({len(chunks)} chunks, {wav.shape[-1] / 24000.0:.1f} s of audio in {dt:.2f} s)")
        return path

    def embed_speakers(self, spk_ref_paths: List[str]) -> torch.Tensor:
        """One speaker embedding per reference -> fp32 [n, 256] on the CPU in input order: ``.pt`` / ``.npy`` files load
        as ``synthesise`` loads them, and every audio file goes through ``get_cached_embeddings`` (the same disk cache,
        with all misses embedded in one batched front-end pass on the device).  A serving loop can embed the
        references of a batch this way and pass the embeddings on as ``.pt`` files."""
        from .speaker_encoder import get_cached_embeddings
        audio = [p for p in spk_ref_paths if not p.endswith((".pt", ".npy"))]
        if audio and self.smodel is None:
            raise FileNotFoundError("speaker_encoder.pt not found in the model directory: pass a precomputed embedding (.pt / .npy)")
        rows = dict(zip(audio, get_cached_embeddings(audio, self.smodel))) if audio else {}
        out = [rows[p].reshape(1, -1).float() if p in rows else load_speaker_embedding(p) for p in spk_ref_paths]
        return torch.cat(out) if out else torch.empty((0, 256))

    def synthesise_batch(self, texts: List[str], spk_ref_paths: List[str], top_p=0.95, guidance_scale=3.0, temperature=1.0,
                         seed: Optional[int] = None, voices: Optional[List[Optional[str]]] = None) -> List[Optional[str]]:
        """N texts with N speaker references in one batch, one wav file per text, returned in input order (the reference's
        ``_sample_utterance_batch``, inference.py:438-517): stage 1 as one continuous batch over the ``max_utts`` KV
        slots, stage 2 in batches of ``max_utts``, the EnCodec decode and the loudness post-processing batched on the
        device (the diffusion refinement, when loaded, per utterance).  An utterance shorter than 400 ms, or one whose
        loudness is undefined, gets None and the others are still written (the reference returns None where decoding
        fails, inference.py:330-336).  ``seed`` fixes the result: request i's stage-1 draws come from a Philox stream
        seeded with ``seed + i`` (``serving.seeded_noise``) and stage 2 samples with ``seed``.  ``voices``: one voice
        name per text (None: the base checkpoint); texts of different voices share the stage-1 batch."""
        from .audio_out import LOUDNESS_HEADROOM_DB, _post_batch
        from .fast_inference_utils import encode_tokens
        from .serving import ContinuousBatcher, seeded_noise
        if len(texts) != len(spk_ref_paths):
            raise ValueError(f"{len(texts)} texts but {len(spk_ref_paths)} speaker references")
        if voices is not None and len(voices) != len(texts):
            raise ValueError(f"{len(texts)} texts but {len(voices)} voices")
        vids = [self._voice(v) for v in (voices if voices is not None else [None] * len(texts))]
        self._check_guidance(guidance_scale)
        if not texts:
            return []
        texts = [normalize_text(t) for t in texts]
        embs = {}
        for p in spk_ref_paths:                                # one embedding per distinct reference (disk-cached for audio)
            if p not in embs:
                embs[p] = load_speaker_embedding(p, self.smodel)
        spk = [embs[p] for p in spk_ref_paths]
        start = time.time()
        cb = ContinuousBatcher(self.model)
        ids = []
        for i, (t, e) in enumerate(zip(texts, spk)):
            prompt = encode_tokens(self.tokenizer, t, device="cpu")
            kw = dict(top_p=top_p, guidance_scale=guidance_scale, temperature=temperature,
                      end_of_text_token=self.tokenizer.eot_token, voice=vids[i])
            if seed is not None:
                noise = seeded_noise(self.model, prompt.numel(), seed + i)
                kw.update(max_new_tokens=noise.shape[0], noise=noise)
            ids.append(cb.submit(prompt, e, **kw))
        toks = cb.run_until_done()
        extracted = [flattened_interleaved_decode(toks[rid].tolist(), self.END_OF_AUDIO_TOKEN)[1] for rid in ids]
        codes = self.llm_second_stage.non_causal_sample(
            texts=texts, encodec_tokens=[torch.tensor(x, dtype=torch.int32).unsqueeze(0) for x in extracted],
            speaker_embs=torch.stack(spk), batch_size=len(texts), top_k=200, temperature=1.0, seed=seed)
        # 400 ms = 9600 samples = 30 frames at 320 samples per frame (decoders.py:88-91)
        ok = [i for i, c in enumerate(codes) if c.shape[-1] * self.codec.upsample >= 9600]
        wavs = self.codec.decode_batch([codes[i] for i in ok])
        if self.mbd is not None:
            wavs = [self.mbd.tokens_to_wav(self.codec.decode_latent(codes[i]), w) for i, w in zip(ok, wavs)]
        files, _, _ = _post_batch(wavs, 24000, LOUDNESS_HEADROOM_DB, True) if wavs else ([], [], [])
        paths: List[Optional[str]] = [None] * len(texts)
        for i in range(len(texts)):
            if i not in ok:
                print(f"utterance {i}: wav predicted is shorter than 400ms! ({codes[i].shape[-1]} frames)")
        for i, f in zip(ok, files):
            if isinstance(f, Exception):
                print(f"utterance {i}: post-processing failed: {f}")
                continue
            name = f"synth_{datetime.now().strftime('%y-%m-%d--%H-%M-%S')}_{texts[i].replace(' ', '_')[:25]}_{uuid.uuid4()}"
            path = str(Path(self.output_dir).resolve() / name) + ".wav"
            with open(path, "wb") as fh:
                fh.write(f)
            paths[i] = path
        dt = time.time() - start
        print(f"\nSaved {sum(p is not None for p in paths)} of {len(texts)} utterances in {dt:.2f} s")
        return paths

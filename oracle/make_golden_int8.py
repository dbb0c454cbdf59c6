"""ORACLE (test infrastructure): generate tests/golden/int8_quant.npz and tests/golden/int8_stage1_tiny.npz by executing the
REFERENCE'S OWN int8 code (fam.llm.fast_quantize, CPU) through oracle/ref_harness.py.  Run in the build container only:

    python oracle/make_golden_int8.py

int8_quant.npz: ``dynamically_quantize_per_channel(w.float(), -128, 127, torch.int8)`` with the scales cast to bf16 as
``WeightOnlyInt8QuantHandler.create_quantized_state_dict`` does, on seeded bf16 slices of the production shapes and on edge
rows; plus the names of the modules the handler quantises on the tiny reference ``Transformer`` and that model's
``model_size`` (fast_inference_utils.py:348).

int8_stage1_tiny.npz: the tiny synthetic checkpoint built in bf16, quantised by the handler (create_quantized_state_dict,
convert_for_runtime, load_state_dict(assign=True)), then cast to fp32 for the forward (the int8 weights and the bf16 scales
stay exact, so this is the exact function).  Stored: prefill logits, logits at teacher-forced steps 1 / 8 / 64 / 255, the
256 tokens sampled under seeded Exp(1) noise, and the reference's own bf16-vs-fp32 gap on the same int8 model.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "metavoice-src_b200"))

from mvb200 import synth  # noqa: E402
from oracle import ref_harness as R  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
NOISE_SEED = 4
N_NEW, T, KEEP = 256, 12, [1, 8, 64, 255]


def _bits(t: torch.Tensor) -> np.ndarray:
    return t.contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def edge_rows(K: int = 256) -> torch.Tensor:
    g = torch.Generator().manual_seed(5)
    rnd = lambda scale: torch.randn(K, generator=g) * scale                                      # noqa: E731
    eps = torch.finfo(torch.float32).eps
    amp = rnd(0.02)
    rows = [
        torch.zeros(K),                                                  # all zero: scale clamped to FLT_EPSILON
        torch.full((K,), 0.0371),                                        # constant positive
        torch.full((K,), -3.25),                                         # constant negative
        torch.cat([rnd(0.01)[:K - 1], torch.tensor([3.5])]),             # one outlier
        torch.cat([amp[:K - 2], torch.tensor([-0.75, 0.75])]),           # minimum exactly -maximum
        -(rnd(0.05).abs() + 0.01),                                       # negative only
        rnd(1.0).clamp(-3, 3) * 1e38,                                    # near the top of the bf16 range
        rnd(1.0) * (0.25 * eps * 127.5),                                 # below FLT_EPSILON * 127.5: clamped scale
        torch.linspace(-1, 1, K),                                        # exact grid ties
        torch.arange(K, dtype=torch.float32) / 2 - 64,                   # halves: round-half-even ties
    ]
    return torch.stack(rows).to(torch.bfloat16)


def golden_quant():
    fm, _ = R._import_reference()
    from fam.llm.fast_quantize import WeightOnlyInt8QuantHandler, dynamically_quantize_per_channel
    g = torch.Generator().manual_seed(2024)
    cases = {
        "k256": (torch.randn(64, 256, generator=g) * 0.05).to(torch.bfloat16),      # speaker_cond_pos slice
        "k2048": (torch.randn(48, 2048, generator=g) * 0.02).to(torch.bfloat16),    # wqkv / wo / w1 / w3 slice
        "k5632": (torch.randn(16, 5632, generator=g) * 0.02).to(torch.bfloat16),    # w2 slice
        "head": (torch.randn(2562, 64, generator=g) * 0.02).to(torch.bfloat16),     # all 2562 lm_head rows, 64 inputs
        "edge": edge_rows(),
    }
    out = {}
    for name, w in cases.items():
        q, s, _ = dynamically_quantize_per_channel(w.float(), -128, 127, torch.int8)
        out[f"{name}_w"] = _bits(w)
        out[f"{name}_q"] = q.numpy()
        out[f"{name}_scales"] = _bits(s.to(torch.bfloat16))
    d = synth.TINY
    model = _bf16_model(fm, synth.stage1_state_dict(d, 0), d)
    h = WeightOnlyInt8QuantHandler(model)
    qsd = h.create_quantized_state_dict()
    names = sorted(k[:-len(".scales")] for k in qsd if k.endswith(".scales"))
    model = h.convert_for_runtime()
    model.load_state_dict(qsd, assign=True)
    out["tiny_quantised_modules"] = np.array(names)
    out["tiny_model_size"] = np.int64(sum(p.numel() * p.dtype.itemsize for p in list(model.parameters()) + list(model.buffers())))
    np.savez_compressed(os.path.join(GOLD, "int8_quant.npz"), **out)
    print("wrote int8_quant.npz:", names, int(out["tiny_model_size"]))


def _bf16_model(fm, sd, d):
    args = fm.ModelArgs(block_size=d.block_size, vocab_size=d.vocab_size, n_layer=d.n_layer, n_head=d.n_head, dim=d.dim,
                        speaker_emb_dim=d.speaker_emb_dim, norm_eps=d.norm_eps)
    with torch.device("meta"):
        model = fm.Transformer(args)
    model.load_state_dict(R.rename_to_fast(sd), assign=True)
    return model.to(dtype=torch.bfloat16).eval()


def _int8_model(fm, sd, d, dtype):
    """fast_inference_utils.py:283-296 on the bf16 model, then cast to `dtype` (int8 buffers are not floating point)."""
    from fam.llm.fast_quantize import WeightOnlyInt8QuantHandler
    model = _bf16_model(fm, sd, d)
    h = WeightOnlyInt8QuantHandler(model)
    qsd = h.create_quantized_state_dict()
    model = h.convert_for_runtime()
    model.load_state_dict(qsd, assign=True)
    model = model.to(dtype=dtype).eval()
    model.config.dtype = dtype
    model.setup_spk_cond_mask()
    model.setup_caches(max_batch_size=2, max_seq_length=d.block_size)
    return model


def golden_stage1_tiny():
    torch.set_grad_enabled(False)
    fm, fiu = R._import_reference()
    d = synth.TINY
    sd = synth.stage1_state_dict(d, 0)
    prompt, spk = synth.synthetic_prompt(T), synth.synthetic_speaker()
    noise = torch.empty(N_NEW, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(NOISE_SEED))
    model = _int8_model(fm, sd, d, torch.float32)
    assert model.output.weight.dtype == torch.int8 and model.output.scales.dtype == torch.float32
    logs = []
    hook = model.register_forward_hook(lambda m, i, o: logs.append(o.float().clone()))
    step = [0]
    orig = fiu.multinomial_sample_one_no_sync

    def injected(probs_sort):   # == fast_inference_utils.py:61-65 with q taken from the seeded draws
        q = noise[step[0]].view_as(probs_sort).to(probs_sort.dtype)
        step[0] += 1
        return torch.argmax(probs_sort / q, dim=-1, keepdim=True).to(dtype=torch.int)

    fiu.multinomial_sample_one_no_sync = injected
    try:
        y = fiu.generate(model, prompt, spk, max_new_tokens=N_NEW, end_of_audio_token=9999, temperature=torch.tensor(1.0),
                         top_p=torch.tensor(0.95), guidance_scale=torch.tensor(3.0), top_k=None)
    finally:
        fiu.multinomial_sample_one_no_sync = orig
    hook.remove()
    gen = y[T:].to(torch.int32)
    assert gen.numel() == N_NEW and len(logs) == N_NEW and step[0] == N_NEW
    out = dict(prompt=prompt.numpy(), spk=spk.numpy(), tokens=gen.numpy(), noise_seed=np.int64(NOISE_SEED),
               prefill_logits=logs[0].numpy(), steps=np.asarray(KEEP, np.int32),
               logits=torch.stack([logs[s][:, -1] for s in KEEP]).numpy(),
               weight_checksum=np.float64(synth.state_dict_checksum(sd)))
    # the reference's production precision on the same int8 model, teacher-forced with the fp32 run's tokens
    mb = _int8_model(fm, sd, d, torch.bfloat16)
    spk_b = spk.to(torch.bfloat16)
    lb = {}
    mb(prompt.view(1, -1).repeat(2, 1), spk_b, torch.arange(T))
    for s in range(1, max(KEEP) + 1):
        lg = mb(gen[s - 1].view(1, 1).repeat(2, 1), spk_b, torch.tensor([T + s - 1]))
        if s in KEEP:
            lb[s] = lg[:, -1].float()
    out["logits_ref_bf16"] = torch.stack([lb[s] for s in KEEP]).numpy()
    gap = [float(np.abs(a - b).max() / np.abs(a).max()) for a, b in zip(out["logits"], out["logits_ref_bf16"])]
    out["ref_bf16_gap"] = np.asarray(gap, np.float64)
    np.savez_compressed(os.path.join(GOLD, "int8_stage1_tiny.npz"), **out)
    print(f"wrote int8_stage1_tiny.npz: reference int8 bf16-vs-fp32 gap per kept step {gap}")


if __name__ == "__main__":
    os.makedirs(GOLD, exist_ok=True)
    golden_quant()
    golden_stage1_tiny()

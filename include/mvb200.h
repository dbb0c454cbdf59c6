/*
 * mvb200.h -- C ABI of libmvb200.so: the H100 (sm_90a) engine behind MetaVoice-1B's
 * TTS.synthesise() hot path.  Plain pointers and sizes only; no torch types.
 *
 * Every entry point names the reference interface it replaces (paths relative to the
 * reference tree metavoiceio/metavoice-src @ de3fa211).  Device buffers are owned by the
 * caller (the Python shim allocates them as torch tensors and passes data_ptr()); the
 * library never frees caller memory.  All functions return 0 on success, non-zero on
 * failure with the message available from mvb_last_error().  A handle is re-entrant per
 * handle, not thread-safe per handle (the reference is single-threaded per model,
 * SURVEY.md 8b "Threading / state").
 */
#ifndef MVB200_H
#define MVB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MVB_ABI_VERSION 3

/* KV-cache element type.  bf16 is what the reference stores (fast_model.py:97-102);
 * fp32 is the validation mode used for the <=1e-3 parity gate against the fp32 oracle;
 * fp8 (an extension: the reference has no fp8 cache) stores e4m3 codes with one bf16 scale per head vector, layout and
 * quantiser at mvb_s1_kv_bytes. */
enum { MVB_KV_BF16 = 0, MVB_KV_FP32 = 1, MVB_KV_FP8 = 2 };

/* Shape of the stage-1 causal LM: fam/llm/fast_model.py:52-94 (ModelArgs / "metavoice-1B"). */
typedef struct mvb_s1_config {
  int32_t n_layer;       /* 24 */
  int32_t n_head;        /* 16 (MHA: n_local_heads == n_head) */
  int32_t head_dim;      /* 128 (only 128 is supported) */
  int32_t dim;           /* 2048 */
  int32_t intermediate;  /* 5632 */
  int32_t vocab;         /* 2562 */
  int32_t block_size;    /* 2048: learned-position table length and KV slots per row */
  int32_t spk_dim;       /* 256 */
  float   norm_eps;      /* 1e-5 */
  int32_t max_utts;      /* utterance slots; each owns 2 CFG rows {cond, uncond} (fast_model.py:132-134) */
  int32_t kv_dtype;      /* MVB_KV_BF16 | MVB_KV_FP32 | MVB_KV_FP8 */
  int32_t max_new;       /* capacity of the per-utterance generated-token ring (<= block_size) */
  int32_t options;       /* MVB_S1_* bits below; 0 = the production engine */
} mvb_s1_config;

/* Stage-1 options: reference and identity paths for tests and tools, fixed at create time.  The workspace and KV sizes
 * do not depend on them; any other bit is MVB_ERR_ARG. */
#define MVB_S1_NO_ROWS_PATH    0x1 /* no tensor-core rows path: prefill and batched decode run on the CUDA-core kernels */
#define MVB_S1_NO_RESIDENT     0x2 /* no resident (persistent) decode kernel: decode runs on the per-layer path */
#define MVB_S1_UNFUSED_SAMPLER 0x4 /* the resident kernel leaves the logits to k_sample instead of sampling in the kernel */
#define MVB_S1_TRACE           0x8 /* the resident kernel records per-phase clocks for mvb_s1_trace_fetch */

/* Byte offsets (into one bf16 weight arena) of every stage-1 tensor, row-major [out, in]
 * exactly as stored in first_stage.pt (SURVEY.md App. B).  Built by the checkpoint loader that
 * replaces fast_inference_utils.py:236-281 (_load_model).  Per layer, in this order:
 * attn_norm[dim], wqkv[3*dim, dim], wo[dim, dim], ffn_norm[dim], w1[inter, dim], w3[inter, dim],
 * w2[dim, inter]. */
#define MVB_S1_GLOBAL_TENSORS 5 /* tok_emb[vocab,dim], pos_emb[block,dim], spk_proj[dim,spk_dim], out_norm[dim], lm_head[vocab,dim] */
#define MVB_S1_LAYER_TENSORS 7

/* Sampling parameters of fast_inference_utils.py:107-120 (sample) for one utterance. */
typedef struct mvb_sampling {
  float    guidance_scale; /* g in g*cond + (1-g)*uncond */
  float    temperature;    /* clamped below at 1e-5 (utils:92) */
  float    top_p;          /* <= 0 disables (top_p=None) */
  int32_t  top_k;          /* <= 0 disables (top_k=None) */
  int32_t  end_of_audio;   /* token id that latches termination (2048; 9999 disables), utils:161 */
  uint64_t seed;           /* Philox key for on-device Exp(1) noise when no noise buffer is supplied */
} mvb_sampling;

typedef struct mvb_s1 mvb_s1; /* opaque engine handle */

int         mvb_abi_version(void);
const char* mvb_last_error(void);

/* Sizes the caller must allocate (device memory) before mvb_s1_create.
 * Replaces Transformer.setup_caches (fast_model.py:136-148): KV = n_layer x {K,V} x rows x heads x
 * block_size x head_dim elements, rows = 2 max_utts, element [layer][K|V][row][head][pos][head_dim].
 * MVB_KV_FP8: with N = n_layer * 2 * rows * heads * block_size head vectors, bytes [0, 128 N) hold one e4m3 code per
 * element in that layout, and bytes [128 N, 130 N) one bf16 scale per head vector, [layer][K|V][row][head][pos] (scale
 * of vector i at byte 128 N + 2 i); mvb_s1_kv_bytes = 130 N (408,944,640 per utterance slot at the production shape,
 * 0.508x the bf16 cache).  Each vector x (fp32, as the qkv projection produced it) is stored as
 * s = bf16_rn(max(amax|x| / 448, FLT_EPSILON)), q = e4m3_rn(clamp(x / s, -448, 448)) (mvb200/quantize.py
 * quantize_kv_fp8); a NaN anywhere in x stores s = NaN (0x7fc0) and every code 0x7f, an infinite element makes s = +inf.
 * The workspace sizes do not depend on kv_dtype.  An fp8-cache engine never uses the resident decode kernel: one
 * utterance decodes on the per-layer CUDA-core path. */
size_t mvb_s1_kv_bytes(const mvb_s1_config* cfg);
size_t mvb_s1_workspace_bytes(const mvb_s1_config* cfg);

/* Build an engine over caller-owned device memory.  `offsets` is a HOST array of
 * MVB_S1_GLOBAL_TENSORS + n_layer*MVB_S1_LAYER_TENSORS byte offsets into d_arena.  d_workspace must
 * be zero-filled; with a bf16 cache the call zero-fills d_kv itself (the attention kernel reads whole 64-position tiles,
 * so positions that were never written must hold finite values).  Replaces build_model()/Transformer.__init__/setup_caches/setup_spk_cond_mask
 * (fast_inference_utils.py:324-352, fast_model.py:116-148); there is no JIT/compile step. */
int mvb_s1_create(const mvb_s1_config* cfg, const void* d_arena, size_t arena_bytes,
                  const uint64_t* offsets, void* d_kv, void* d_workspace, mvb_s1** out);
int mvb_s1_destroy(mvb_s1* h);

/* Stage-1 architecture: the GPTConfig fields (fam/llm/model.py:26-46) norm_type, nonlinearity_type and bias of the
 * reference's causal GPT (model.py:195-314, layers/attn.py, layers/combined.py, layers/layers.py), served by its slow
 * path fam.llm.inference (inference.py:102-156).  All zero = rmsnorm, swiglu, no bias: the production engine.  A field
 * outside its values is MVB_ERR_ARG naming it. */
typedef struct mvb_s1_arch {
  int32_t norm;            /* MVB_S1_NORM_*: ln_1, ln_2 and ln_f */
  int32_t mlp;             /* MVB_S1_MLP_* */
  int32_t bias;            /* 1: biases on attn.c_attn (k and v are cached with theirs), attn.c_proj, every MLP Linear and
                            * (LayerNorm) ln_1, ln_2, ln_f; speaker_cond_pos and the head (tied to wtes.0) never have one */
} mvb_s1_arch;
#define MVB_S1_NORM_RMS    0   /* RMSNorm(eps = norm_eps), layers.py:20-30 */
#define MVB_S1_NORM_LAYER  1   /* LayerNorm(eps = 1e-5), with a beta when bias, layers.py:8-17 */
#define MVB_S1_MLP_SWIGLU  0   /* c_proj(silu(w1 x) * (w3 x)) */
#define MVB_S1_MLP_GELU    1   /* c_proj(GELU(c_fc x)), exact erf GELU (nn.GELU()); cfg->intermediate = 4 dim */
/* mvb_s1_create with an architecture; mvb_s1_create == mvb_s1_create_ex with arch NULL (all zero).  The offset list is
 * mvb_s1_create's (MVB_S1_GLOBAL_TENSORS, then per layer {ln_1, attn.c_attn, attn.c_proj, ln_2, mlp.swiglu.w1,
 * mlp.swiglu.w3, mlp.c_proj}; GELU: {ln_1, attn.c_attn, attn.c_proj, ln_2, mlp.c_fc, mlp.c_proj}); then, when
 * arch->bias: ln_f.bias (LayerNorm only), and per layer {ln_1.bias (LayerNorm only), attn.c_attn.bias, attn.c_proj.bias,
 * ln_2.bias (LayerNorm only), mlp.c_fc.bias | mlp.swiglu.w1.bias, mlp.swiglu.w3.bias, mlp.c_proj.bias}, all bf16.  The
 * KV and workspace sizes do not depend on arch.  Any architecture but the production one decodes one utterance on the
 * CUDA-core GEMVs and a batch on the tensor-core rows path (MVB_S1_NO_ROWS_PATH: everything on the GEMVs), never in the
 * resident decode kernel, and prefills on the tensor cores. */
int mvb_s1_create_ex(const mvb_s1_config* cfg, const mvb_s1_arch* arch, const void* d_arena, size_t arena_bytes,
                     const uint64_t* offsets, void* d_kv, void* d_workspace, mvb_s1** out);

/* Voices: last-N-block finetunes of the engine's checkpoint (fam/llm/finetune.py trains ln_f and the last
 * last_n_blocks_to_finetune blocks and freezes the rest) served from one bf16 engine.  Voice 0 is the checkpoint the
 * engine was created from; every other voice overlays blocks [first_layer, n_layer) and ln_f.
 *   mvb_s1_add_voice  registers an overlay held in caller-owned device memory d_overlay (like the arena: it must outlive
 *                     the handle).  `offsets` is a HOST array of byte offsets into it: for each overlaid layer, that
 *                     layer's tensors in mvb_s1_create_ex's order (its weights; then, when arch->bias, its biases), then
 *                     ln_f.weight and (LayerNorm with bias) ln_f.bias; n_offsets must be exactly that count.  Offsets
 *                     are checked as the arena's are (16-byte aligned, inside the overlay).  *voice receives the id
 *                     (1, 2, ...).  At most MVB_S1_MAX_VOICES voices, voice 0 included: past that, MVB_ERR_ARG.  An
 *                     int4, int8 or fp8 engine returns MVB_ERR_UNSUPPORTED.
 *   mvb_s1_set_voice  selects the voice of slot `utt`.  It takes effect at the slot's next admission (mvb_s1_admit,
 *                     mvb_s1_admit_guided, mvb_s1_generate) or mvb_s1_begin; a prompt-guided companion always takes its
 *                     primary's voice.  A new handle starts every slot on voice 0.
 * A decode batch may mix voices; each slot computes exactly what an engine created from its voice's full checkpoint
 * computes on the same path.  A burst whose slots are all on voice 0 is unchanged (resident decode kernel included);
 * any other burst runs on the per-layer paths. */
#define MVB_S1_MAX_VOICES 16
int mvb_s1_add_voice(mvb_s1* h, const void* d_overlay, size_t overlay_bytes, int32_t first_layer, const uint64_t* offsets,
                     int32_t n_offsets, int32_t* voice);
int mvb_s1_set_voice(mvb_s1* h, int32_t utt, int32_t voice);

/* Hoisted speaker conditioning: spk_proj[utt] = W_spk * spk_emb (fast_model.py:152-157 recomputes it
 * every step; it only changes per utterance).  d_spk_emb: fp32 [spk_dim] on device. */
int mvb_s1_set_speaker(mvb_s1* h, int32_t utt, const float* d_spk_emb, void* stream);

/* Parity hook == Transformer.forward(idx[2,S], spk_emb, input_pos=arange(pos0, pos0+S)) for slot
 * `utt` (fast_model.py:150-163).  d_idx: int32 [2, S] on device (row 0 = cond, row 1 = uncond).
 * Writes the KV cache at positions pos0..pos0+S-1.  d_logits: fp32 [2, S, vocab] when
 * all_positions != 0, else fp32 [2, vocab] for the last position only. */
int mvb_s1_forward(mvb_s1* h, int32_t utt, const int32_t* d_idx, int32_t S, int32_t pos0,
                   float* d_logits, int32_t all_positions, void* stream);

/* == sample() (fast_inference_utils.py:107-120) on device.  d_logits fp32 [2, vocab];
 * d_noise: fp32 [vocab] Exp(1) draws (the reference's `q`, utils:64) or NULL for on-device Philox;
 * d_token_out int32 [1]; d_probs_out fp32 [vocab] or NULL. */
int mvb_s1_sample(mvb_s1* h, const float* d_logits, const mvb_sampling* p, const float* d_noise,
                  uint64_t step, int32_t* d_token_out, float* d_probs_out, void* stream);

/* Plugin call with HOST buffers == generate() (fast_inference_utils.py:181-228) for n_utts independent
 * utterances decoded together (per-row positions; semantics of mixins/causal.py:179-287, which equal
 * running each utterance alone).  Host->device copies of prompts/speaker vectors and the device->host
 * copy of the tokens happen inside this call.
 *   prompts      host int32, concatenated; prompt_lens[n_utts]
 *   spk_embs     host fp32 [n_utts, spk_dim]
 *   params       [n_utts]
 *   noise        NULL, or fp32 [n_utts, max_new_tokens, vocab] Exp(1) draws in the reference's call order
 *                (utils:61-65: one `q` per generated token).  noise_on_device == 0: HOST buffer, staged to the device
 *                one burst of decode steps at a time; != 0: DEVICE buffer used in place (how the Python shim hands
 *                over the draws it makes with torch's generator, so that torch.manual_seed reproduces the reference)
 *   forced       host or NULL: int32 [n_utts, max_new_tokens] teacher-forced feedback tokens (test hook)
 *   out_tokens   host int32 [n_utts, max_new_tokens]; out_lens[n_utts] = tokens produced (EOA included, utils:226)
 * Raises (returns MVB_ERR_PROMPT_TOO_LONG) when a prompt leaves no room: utils:203-204. */
int mvb_s1_generate(mvb_s1* h, int32_t n_utts, const int32_t* prompts, const int32_t* prompt_lens,
                    const float* spk_embs, const mvb_sampling* params, int32_t max_new_tokens,
                    const float* noise, int32_t noise_on_device, const int32_t* forced, int32_t* out_tokens,
                    int32_t* out_lens, void* stream);

/* Same loop with inputs already resident: prompts/speakers must have been installed with
 * mvb_s1_set_speaker + mvb_s1_forward (prefill).  Runs `n_steps` decode steps for utterances
 * [0, n_utts) entirely on device (sampler, EOA latch and position bump included) and returns without
 * a host sync.  Used by bench.py for the HBM-resident `value` and by the shim's generate(). */
int mvb_s1_decode(mvb_s1* h, int32_t n_utts, int32_t n_steps, void* stream);

/* Continuous batching (SURVEY.md row N4; the reference serialises requests, serving.py:59-109): utterances enter and
 * leave KV slots between decode bursts of the persistent kernel.
 *   mvb_s1_admit   == the per-utterance prologue of generate() (utils:196-212) for slot `utt`: HOST prompt int32 [T] and
 *                  speaker vector fp32 [spk_dim] are uploaded, the prompt is prefilled and the first token is sampled;
 *                  d_noise: optional DEVICE Exp(1) draws [max_new_tokens, vocab] (NULL = on-device Philox, params->seed).
 *                  Returns MVB_ERR_PROMPT_TOO_LONG like generate().
 *   mvb_s1_decode  then advances every slot [0, n_slots) by a burst; finished / parked slots are skipped by the sampler.
 *   mvb_s1_poll    done flags + generated-token counts of slots [0, n_slots) (one device->host round trip).
 *   mvb_s1_release parks a slot (done latch set) until the next admit. */
int mvb_s1_admit(mvb_s1* h, int32_t utt, const int32_t* prompt, int32_t T, const float* spk_emb,
                 const mvb_sampling* params, int32_t max_new_tokens, const float* d_noise, void* stream);
int mvb_s1_release(mvb_s1* h, int32_t utt, void* stream);
int mvb_s1_poll(mvb_s1* h, int32_t n_slots, int32_t* done_out, int32_t* n_gen_out, void* stream);

/* Prompt guidance: the reference's guidance_scale = (s, p) of _sample_batch (fam/llm/mixins/causal.py:89-105, 224-262;
 * inference.py:438-560), logits = (s + p - 1) cond + (1 - s) uncond_speaker + (1 - p) uncond_prompt, with the fast path's
 * temperature / top-k / top-p / Exp(1) tail after the mix.  A guided utterance owns two slots: its own (`utt`, rows
 * cond and uncond speaker) and a companion whose speaker-on row is the uncond-prompt row (its other row is computed and
 * ignored).  The forward passes see two ordinary slots; the sampler of the primary reads the three rows, does the
 * bookkeeping of both slots and feeds the companion `fed > end_of_audio ? end_of_text_token : fed` (causal.py:262).
 * Guided slots are sampled by k_sample, never by the resident kernel's fused sampler.
 *   mvb_s1_admit_guided  == mvb_s1_admit for slot `utt` (params->guidance_scale = s) plus companion slot `companion`,
 *                        prefilled with the prompt's tokens > params->end_of_audio replaced by end_of_text_token, under
 *                        the same speaker.  The first token is sampled from the three rows of the last prompt position.
 *                        p == 1 is exactly mvb_s1_admit (no companion is touched).
 *   mvb_s1_sample_guided == mvb_s1_sample over three rows: d_logits fp32 [3, vocab] = {cond, uncond speaker, uncond
 *                        prompt}; p == 1 reads rows 0 and 1 only and equals mvb_s1_sample.
 * MVB_ERR_ARG, before anything is launched, unless both scales are finite and >= 1 (the reference asserts s >= 1 and
 * p >= 1), `companion` != `utt` and both are slots of the handle, and end_of_text_token is in the vocabulary; T and
 * max_new_tokens are checked as mvb_s1_admit checks them.  mvb_s1_poll reports the companion done whenever the primary
 * is.  The link is dissolved on both sides (a former companion is parked) when mvb_s1_poll or mvb_s1_fetch reads the
 * primary's done flag set, when the primary is released, or when either slot is admitted or begun again; after that the
 * old companion is an ordinary free slot and unguided bursts sample in the resident kernel again.  While a link lives,
 * mvb_s1_decode returns MVB_ERR_ARG when one of its slots is inside [0, n_utts) and the other is not.  s and p are
 * passed as fp32: for a scale fp32 cannot represent exactly, a mix coefficient can differ from the reference's (formed
 * from Python doubles) by one fp32 ulp. */
int mvb_s1_admit_guided(mvb_s1* h, int32_t utt, int32_t companion, const int32_t* prompt, int32_t T,
                        const float* spk_emb, const mvb_sampling* params, float prompt_guidance_scale,
                        int32_t end_of_text_token, int32_t max_new_tokens, const float* d_noise, void* stream);
int mvb_s1_sample_guided(mvb_s1* h, const float* d_logits, const mvb_sampling* p, float prompt_guidance_scale,
                         const float* d_noise, uint64_t step, int32_t* d_token_out, float* d_probs_out, void* stream);

/* Install per-utterance decode state after prefill: first token, sampling params, optional device
 * noise [max_new, vocab] / forced-token [max_new] buffers (NULL = none). */
int mvb_s1_begin(mvb_s1* h, int32_t utt, int32_t first_token, int32_t pos, const mvb_sampling* p,
                 const float* d_noise, const int32_t* d_forced, void* stream);

/* Read back decode state: tokens generated so far for `utt` (host buffer, capacity cap). */
int mvb_s1_fetch(mvb_s1* h, int32_t utt, int32_t* out_tokens, int32_t cap, int32_t* n_out,
                 int32_t* done, void* stream);

/* Parity hook for the decode body: one decode position (== Transformer.forward with S = 1, fast_model.py:150-163)
 * for utterances [0, n_utts) from the state installed by mvb_s1_begin, through the body mvb_s1_decode runs for that
 * batch: the persistent fused kernel up to 8 utterances (when enabled and its per-CTA attention tile table can hold every
 * position of the context), the per-layer path otherwise (tensor-core
 * rows path up to max_utts = 64 utterances); logits fp32 [2*n_utts, vocab] are copied to d_logits, nothing is sampled,
 * positions do not advance (the KV cache is appended at the current positions). */
int mvb_s1_step_logits(mvb_s1* h, int32_t n_utts, float* d_logits, void* stream);

/* Weight-only int4 engine (quantisation_mode="int4", fast_inference_utils.py:297-306).  Same offset table as mvb_s1_create,
 * but the entries of every layer's wqkv, wo, w1, w3 and w2 point at an int4 PACKED MATRIX [M, K] (K % 256 == 0):
 *   nibbles  uint32 [M][K/8], q in [0, 15]: word w of row m holds q(m, 8w + 2i) in bits 4i..4i+3 and q(m, 8w + 2i + 1)
 *            in bits 16+4i..19+4i, i = 0..3 (a pair of consecutive k lands in the two bf16 halves of a register);
 *   then, at the next 256-byte boundary, bf16 [M][K/128][2] = {scale s, zero z} of every 128-wide group of a row.
 * (produced only by mvb200/quantize.py:pack_matrix; the quantiser is the reference's group_quantize_tensor(w, 4, 128)).
 * Dequantised weight: W_deq = bf16_rn((q - 8) s + z) -- the exact value rounded once to bf16 -- in every kernel.  All other
 * tensors are bf16 as for mvb_s1_create (speaker_cond_pos holds its W_deq; lm_head stays unquantised).
 * Decode always runs the per-layer CUDA-core path through the int4 GEMV (never the persistent kernel, never the tensor-core
 * rows path); prefill runs the tensor-core GEMM over one layer at a time dequantised into a scratch that is part of the
 * workspace: mvb_s1_int4_workspace_bytes = the bf16 workspace + one layer of bf16 weights.  Every other mvb_s1_* call
 * accepts the handle. */
size_t mvb_s1_int4_workspace_bytes(const mvb_s1_config* cfg);
int mvb_s1_create_int4(const mvb_s1_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets,
                       void* d_kv, void* d_workspace, mvb_s1** out);

/* Weight-only int8 engine (quantisation_mode="int8", fast_inference_utils.py:283-296).  Same offset table as mvb_s1_create,
 * but the entry of EVERY Linear weight -- wqkv, wo, w1, w3, w2 of every layer, speaker_cond_pos and lm_head -- points at an
 * INT8 MATRIX [M, K]: int8 q [M][K] row-major, then at the next 256-byte boundary bf16 [M] row scales s (produced only by
 * mvb200/quantize.py:pack_int8_matrix; the quantiser is the reference's dynamically_quantize_per_channel(w.float(), -128,
 * 127) with the scales cast to bf16).  Every kernel computes y_j = s_j * sum_k x_k q_jk: fp32 sums over the exact integer
 * weights, the scale applied once per output after the whole sum (and after any split-K reduction).  Embeddings and norms
 * are bf16.  Decode always runs the per-layer CUDA-core path through the int8 GEMV (never the persistent kernel, never the
 * tensor-core rows path); prefill runs the tensor-core GEMM over one layer's q at a time, widened to bf16 into the scratch
 * the int4 engine uses, and lm_head's q widened once at create: mvb_s1_int8_workspace_bytes = the int4 workspace + vocab x
 * dim bf16.  Every other mvb_s1_* call accepts the handle. */
size_t mvb_s1_int8_workspace_bytes(const mvb_s1_config* cfg);
int mvb_s1_create_int8(const mvb_s1_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets,
                       void* d_kv, void* d_workspace, mvb_s1** out);

/* Weight-only fp8 engine (quantisation_mode="fp8"; an extension, the reference has no fp8 mode).  Same offset table and
 * Linear weights as mvb_s1_create_int8, but each entry points at an FP8 MATRIX [M, K] (M even, K % 256 == 0): the int8
 * matrix layout -- M * K one-byte codes, then at the next 256-byte boundary bf16 [M] row scales s -- whose codes are
 * float8 e4m3fn values q in a fragment-native order (produced only by mvb200/quantize.py:pack_fp8_matrix):
 *   rows [0, M16), M16 = M & ~15, in 16-row blocks b, each block's K in 32-wide chunks c; chunk c of block b is 512 bytes
 *   at (b * K / 32 + c) * 512, in which lane l = 4 g + t (g = l / 4, t = l % 4) owns bytes [16 l, 16 l + 16): word 2 s + h
 *   (s, h in {0, 1}) holds the codes of (row g, k0), (row g + 8, k0), (row g, k0 + 1), (row g + 8, k0 + 1), k0 = 16 s +
 *   8 h + 2 t within the chunk -- the bf16 A fragment of mma.m16n8k16 for k-step s once each pair is widened;
 *   rows [M16, M) after them, row-major.
 * Quantiser, per output row j: s_j = bf16(max(amax_j / 448, FLT_EPSILON)), q_jk = e4m3(clamp(w_jk / s_j, -448, 448)) with
 * round-to-nearest-even; NaN or Inf weights are rejected.  Every kernel computes y_j = s_j * sum_k x_k q_jk: fp32 sums over
 * the exact e4m3 values, the scale applied once per output after the whole sum.  Decode of 1 to 8 slots runs the
 * per-layer path through the tensor-core fp8 GEMV, which reads every weight once per step for all of them; prefill and a
 * decode of more than 8 slots run the tensor-core GEMM over one layer's q at a time, widened to bf16 as the int8 engine
 * does.  Never the persistent kernel.  mvb_s1_fp8_workspace_bytes = the int8 workspace + dim x spk_dim bf16
 * (speaker_cond_pos's q, widened once at create).  Every other mvb_s1_* call accepts the handle. */
size_t mvb_s1_fp8_workspace_bytes(const mvb_s1_config* cfg);
int mvb_s1_create_fp8(const mvb_s1_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets,
                      void* d_kv, void* d_workspace, mvb_s1** out);

/* Kernel launches issued by this handle since creation (bench.py "gpu_launches"). */
uint64_t mvb_s1_launch_count(const mvb_s1* h);

/* Test / debug hooks (not part of the drop-in surface; used by tests/ and tools/ only):
 *   mvb_s1_fetch_sampled : the sampler's own draws for `utt` (they differ from the fed-back tokens of mvb_s1_fetch only
 *                          under teacher forcing), host int32 [cap];
 *   mvb_s1_trace_fetch   : per-CTA clock64 phase stamps of the last persistent-kernel step (MVB_S1_TRACE), host
 *                          int64 [max_ctas, 512]; the last 6 entries of a CTA's row are its producer warp's stall cycles
 *                          of the whole launch per phase (qkv, KV tiles, wo, w1|w3, w2, head); returns the number of CTAs
 *                          copied. */
int mvb_s1_fetch_sampled(mvb_s1* h, int32_t utt, int32_t* out_tokens, int32_t cap, void* stream);
int mvb_s1_trace_fetch(mvb_s1* h, long long* out, int32_t max_ctas, void* stream);

/* Tensor-core linear operator (TMA weight streaming + mma.sync), the building block of the batched /
 * prefill path and of the stage-2 model: y[R, M] (+)= f(x)[R, K] . W[M, K]^T, W bf16 row-major [out, in]
 * as every nn.Linear weight in the reference checkpoints (e.g. fast_model.py:194-195, layers/attn.py:61-64).
 * f = optional RMSNorm with bf16 gain (fast_model.py:250-261) when d_gain != NULL.  split_lo != 0 carries the
 * activations as two bf16 terms (hi + lo) so the result matches an fp32-activation product to ~1e-5.
 * K % 64 == 0, 1 <= R <= 128.  ksplit_override <= 0 selects the split automatically.  Synchronises `stream`. */
int mvb_linear(const void* d_W, int32_t M, int32_t K, const float* d_x, int32_t ldx, int32_t R,
               const void* d_gain, float eps, int32_t split_lo, int32_t ksplit_override, float* d_out,
               int32_t ldo, int32_t accumulate, void* stream);

/* Test hook (not part of the drop-in surface): cap the SM count the library plans for.  While n > 0, every engine
 * create and test hook reads the device's SM count as min(real, n), so the persistent decode kernel's grid, its K
 * splits, attention units and fused-sampler choice, and every split-K GEMM plan are those of a part with n SMs.  The
 * cap never raises the count (those kernels need every CTA co-resident).  n = 0 removes it; n < 0 is MVB_ERR_ARG.
 * A handle keeps the count it was created with.  Process-wide; no device setting is touched. */
int mvb_test_set_sm_limit(int32_t n);

/* Test hooks for the op-level tests of two tensor-core kernels (not part of the drop-in surface):
 *   mvb_gemm_test     : mvb_linear's operator with any epilogue of the weight-streaming GEMM (csrc/tc_gemm.cuh):
 *                       epi 0 store, 1 residual add, 2 SwiGLU  out = silu(x W^T) * (x W3^T)  (d_W3 bf16 [M, K]),
 *                       3 QKV  out = x W^T plus the K / V thirds scattered to d_kcache / d_vcache
 *                       [rows][H][S_max][128] (fp32 when kv_fp32, else bf16) at cache row d_row_cache[n], position
 *                       d_row_pos[n] (device int32 [R]; D = 128 H, M = 3 D).  Unused pointers may be NULL.
 *   mvb_mbd_conv_test : one multi-band-diffusion convolution (csrc/mbd.cu) without an mvb_mbd handle.  kind 0: Conv1d,
 *                       stride 1, pad = dil (K - 1) / 2; 1: Conv1d(K = 2 stride) over the input right-padded to a
 *                       multiple of stride; 2: ConvTranspose1d(K = 2 stride), no bias / emb / resid.  d_x fp32
 *                       [Cin, Tin]; d_w fp32 in PyTorch layout ([Cout, Cin, K], transposed [Cin, Cout, K]); optional
 *                       input transform relu(GroupNorm) from caller-supplied d_gn_stats [groups][mean, rstd], d_gn_w,
 *                       d_gn_b [Cin]; optional d_bias, d_emb [Cout], d_resid [Cout, Tout]; d_y fp32 [Cout, Tout], Tout =
 *                       Tin, ceil(Tin / stride), Tin * stride.  use_tc != 0: the tensor-core kernel with the engine's
 *                       weight packing; 0: the CUDA-core kernels.
 *   mvb_mbd_op_test   : one launch of a non-convolution multi-band-diffusion kernel (csrc/mbd.cu) with the engine's launch
 *                       configuration, without an mvb_mbd handle.  Inputs d_a .. d_e, output d_out (updated in place
 *                       where noted), sizes i0 .. i2, scalars f0 .. f4; all tensors fp32.  op 0: GroupNorm statistics
 *                       of d_a [i0, i1] in i2 groups (1 .. 64), eps f0 -> d_out [i2][mean, rstd]; 1: relu(GroupNorm) in
 *                       place on d_out [i0, i1], i2 groups, statistics d_a, gain d_b, bias d_c; 2: FIR bank, d_out [i0, i1]
 *                       = d_a [i1] through each row of d_b [i0, i2] with replicate padding (i0 <= 63); 3: unbiased std
 *                       of the i0 SplitBands bands of x = d_b [i1] from its low-passed copies d_a [i0 - 1, i1] -> d_out
 *                       [i0]; 4: band mix, d_out [i1] (+= when i2 != 0) sum_b band_b * (d_c / d_d)[b] + d_e[b] over i0
 *                       bands of (d_a, d_b) as in op 3 (d_d, d_e may be NULL: scale d_c, shift 0); 5: d_out [i0, i1] +=
 *                       nearest-interpolated d_a [i0, i2]; 6: d_out [i0, i1] = d_a [i0, i2] cropped to i1 + d_b [i0,
 *                       i1]; 7: schedule step on d_out [i1] with estimate d_a, noise d_b (never read when f2 <= 0),
 *                       (a, b, sigma, noise scale, clip) = f0 .. f4; 8: d_out [i1] = Box-Muller normals of Philox stream
 *                       i2 under `seed`; 9: d_out [i1] = sum of the i0 blocks at d_out + m i2 floats; 10: d_out [i1] =
 *                       d_a * f0.  The fp64 GroupNorm partials are allocated per call.
 *   mvb_mbd_unet_test : one UNet evaluation of mvb_mbd_tokens_to_wav on handle h: band model `model`, at the step of
 *                       schedule row `call`, in that model's workspace block, d_est [n_samples] <- UNet(d_cur [n_samples],
 *                       step, d_cond [codec_dim, n_frames]); the argument checks of mvb_mbd_tokens_to_wav.
 * All four synchronise `stream`. */
int mvb_gemm_test(int32_t epi, const void* d_W, const void* d_W3, int32_t M, int32_t K, const float* d_x, int32_t ldx,
                  int32_t R, const void* d_gain, float eps, int32_t split_lo, int32_t ksplit_override, float* d_out,
                  int32_t ldo, void* d_kcache, void* d_vcache, const int32_t* d_row_cache, const int32_t* d_row_pos,
                  int32_t H, int32_t S_max, int32_t D, int32_t kv_fp32, void* stream);
/* Test hooks for the int4 kernels (not part of the drop-in surface):
 *   mvb_w4_gemv_test    : the int4 GEMV (csrc/gemv_w4.cuh k_gemv_w4) as the int4 engine's decode launches it, for
 *                         utterances u in [0, n_utts): rows 2 s, 2 s + 1 (s = d_slot_map[u]) of d_x fp32 [*, ldx] and d_out
 *                         [*, ldo]; epi 0 store, 1 residual add, 2 SwiGLU with d_W3, 3 QKV plus the K / V thirds scattered to
 *                         d_kcache / d_vcache [rows][H][S_max][128] at position d_pos[s] (D = 128 H, M = 3 D).  d_W / d_W3 are
 *                         packed matrices [M, K]; d_gain optional bf16 [K] (RMSNorm prologue).  K % 256 == 0, 2 K floats <= 48 KB.
 *   mvb_w4_dequant_test : k_w4_dequant of one packed matrix into d_out bf16 row-major [M, K].
 * Both synchronise `stream`. */
int mvb_w4_gemv_test(int32_t epi, const void* d_W, const void* d_W3, int32_t M, int32_t K, const float* d_x, int32_t ldx,
                     int32_t n_utts, const void* d_gain, float eps, float* d_out, int32_t ldo, void* d_kcache, void* d_vcache,
                     const int32_t* d_slot_map, const int32_t* d_pos, int32_t H, int32_t S_max, int32_t D, int32_t kv_fp32,
                     void* stream);
int mvb_w4_dequant_test(const void* d_W, int32_t M, int32_t K, void* d_out, void* stream);
/* Test hooks for the int8 kernels (not part of the drop-in surface):
 *   mvb_w8_gemv_test  : the int8 GEMV (csrc/gemv_w8.cuh k_gemv_w8) as the int8 engine's decode launches it; the arguments
 *                       of mvb_w4_gemv_test with d_W / d_W3 int8 matrices [M, K].
 *   mvb_w8_gemm_test  : mvb_gemm_test's operator with the row-scale epilogue of the int8 engine: d_W (d_W3) bf16 [M, K]
 *                       holding q, d_scale (d_scale3 for SwiGLU) bf16 [M]; out = epilogue(s_j * (f(x) . W_j)).
 *   mvb_w8_widen_test : k_w8_widen of one int8 matrix into d_out bf16 row-major [M, K] (q exactly).
 * All three synchronise `stream`. */
int mvb_w8_gemv_test(int32_t epi, const void* d_W, const void* d_W3, int32_t M, int32_t K, const float* d_x, int32_t ldx,
                     int32_t n_utts, const void* d_gain, float eps, float* d_out, int32_t ldo, void* d_kcache, void* d_vcache,
                     const int32_t* d_slot_map, const int32_t* d_pos, int32_t H, int32_t S_max, int32_t D, int32_t kv_fp32,
                     void* stream);
int mvb_w8_gemm_test(int32_t epi, const void* d_W, const void* d_W3, const void* d_scale, const void* d_scale3, int32_t M,
                     int32_t K, const float* d_x, int32_t ldx, int32_t R, const void* d_gain, float eps, int32_t split_lo,
                     int32_t ksplit_override, float* d_out, int32_t ldo, void* d_kcache, void* d_vcache,
                     const int32_t* d_row_cache, const int32_t* d_row_pos, int32_t H, int32_t S_max, int32_t D,
                     int32_t kv_fp32, void* stream);
int mvb_w8_widen_test(const void* d_W, int32_t M, int32_t K, void* d_out, void* stream);
/* Test hooks for the fp8 kernels (not part of the drop-in surface):
 *   mvb_f8_gemv_test  : the fp8 GEMV (csrc/gemv_f8.cuh k_gemv_f8) as the fp8 engine's decode launches it, for any n_utts
 *                       in [1, 64] (one launch row per 8); the arguments of mvb_w4_gemv_test with d_W / d_W3 fp8 matrices
 *                       [M, K], any K % 256 == 0 and an even ldx.
 *   mvb_f8_widen_test : k_f8_widen of one fp8 matrix into d_out bf16 row-major [M, K] (q exactly).
 * Both synchronise `stream`. */
int mvb_f8_gemv_test(int32_t epi, const void* d_W, const void* d_W3, int32_t M, int32_t K, const float* d_x, int32_t ldx,
                     int32_t n_utts, const void* d_gain, float eps, float* d_out, int32_t ldo, void* d_kcache, void* d_vcache,
                     const int32_t* d_slot_map, const int32_t* d_pos, int32_t H, int32_t S_max, int32_t D, int32_t kv_fp32,
                     void* stream);
int mvb_f8_widen_test(const void* d_W, int32_t M, int32_t K, void* d_out, void* stream);
/* Test hook for the fp8 KV cache (not part of the drop-in surface):
 *   mvb_s1_kv_f8_store_test : k_kv_store_f8 as path B launches it.  Row n in [0, R) of d_qkv fp32 [R, 3 D] (D = 128 H)
 *                             stores its k and v third, head by head, at cache row d_cache_row[n] (< n_cache_rows),
 *                             position d_pos[n] (< S_max) of d_codes [K|V][n_cache_rows][H][S_max][128] e4m3 and
 *                             d_scales [K|V][n_cache_rows][H][S_max] bf16, with the quantiser of mvb_s1_kv_bytes.
 *                             1 <= R <= 128.  Synchronises `stream`. */
int mvb_s1_kv_f8_store_test(const float* d_qkv, int32_t R, int32_t H, int32_t n_cache_rows, int32_t S_max,
                            const int32_t* d_cache_row, const int32_t* d_pos, void* d_codes, void* d_scales, void* stream);
/* Test hook for the projections of a non-production stage-1 architecture (not part of the drop-in surface):
 *   path 0: k_gemv as path A launches it, for utterances u in [0, n_utts): rows 2 s, 2 s + 1 (s = d_slot_map[u]) of d_x
 *           fp32 [*, ldx] and d_out [*, ldo]; out = epilogue(f(x) . W^T + bias); norm 0 none, 1 RMSNorm (d_gain, eps),
 *           2 LayerNorm (d_gain, optional d_beta, eps); epi 0 store, 1 residual add, 2 SwiGLU silu(x W^T + bias) *
 *           (x W3^T + bias3), 3 QKV plus the K / V thirds (with their bias) scattered to d_kcache / d_vcache
 *           [rows][H][S_max][128] at position d_pos[s] (D = 128 H, M = 3 D), 4 GELU (exact erf).  d_bias, d_bias3 bf16
 *           [M] or NULL.  K % 256 == 0, 2 K floats <= 96 KB.
 *   path 1: the QKV epilogue of k_tc_gemm (epi must be 3) over R = 2 n_utts activation rows n of d_x / d_out, row n
 *           scattering to cache row 2 s + (n & 1) at position d_pos[s], s = d_slot_map[n >> 1]; the norm as above (the
 *           k_prep_b prologue), the bias added once per output after the split-K sum; ksplit_override > 0 forces the K
 *           split.  K % 64 == 0.  Row scratch is allocated per call.
 * Synchronises `stream`. */
int mvb_s1_arch_gemv_test(int32_t path, int32_t epi, int32_t norm, const void* d_W, const void* d_W3, const void* d_bias,
                          const void* d_bias3, int32_t M, int32_t K, const float* d_x, int32_t ldx, int32_t n_utts,
                          const void* d_gain, const void* d_beta, float eps, float* d_out, int32_t ldo, void* d_kcache,
                          void* d_vcache, const int32_t* d_slot_map, const int32_t* d_pos, int32_t H, int32_t S_max,
                          int32_t D, int32_t kv_fp32, int32_t ksplit_override, void* stream);
int mvb_mbd_conv_test(int32_t kind, const float* d_x, int32_t Cin, int32_t Tin, const float* d_w, int32_t Cout, int32_t K,
                      int32_t stride, int32_t dil, int32_t pad, const float* d_gn_stats, const float* d_gn_w,
                      const float* d_gn_b, int32_t groups, const float* d_bias, const float* d_emb, const float* d_resid,
                      float* d_y, int32_t use_tc, void* stream);
int mvb_mbd_op_test(int32_t op, const float* d_a, const float* d_b, const float* d_c, const float* d_d, const float* d_e,
                    float* d_out, int32_t i0, int32_t i1, int32_t i2, float f0, float f1, float f2, float f3, float f4,
                    uint64_t seed, void* stream);
struct mvb_mbd;
int mvb_mbd_unet_test(struct mvb_mbd* h, int32_t model, int32_t call, const float* d_cur, int32_t n_samples, const float* d_cond,
                      int32_t n_frames, float* d_est, void* stream);
/* Test hooks for the EnCodec decoder and audio post-processing kernels (not part of the drop-in surface):
 *   mvb_voc_op_test     : one launch of a csrc/vocoder.cu kernel with a single segment, through the launch helpers of
 *                         mvb_voc_decode and mvb_voc_decode_batch (every kernel serves both).  op 0: k_conv1d<k>, k = 1 / 3 / 7,
 *                         d_x [Cin, T] -> d_y [Cout, T], d_w [Cout, Cin, k], d_b [Cout] or NULL, ELU on the input when
 *                         elu_in, added to d_y when accumulate; op 1: k_convtr1d (ELU fused) at ratio r = k in 1..8,
 *                         d_x [Cin, T] -> d_y [Cout, T r], d_w [Cin, Cout, 2 r], d_b [Cout]; op 2: k_lstm_layer, H = Cin
 *                         (H % 32 == 0, its H / 4 CTAs co-resident), d_x = pre [4 H, T], d_w = W_hh [4 H, H], d_skip
 *                         [H, T] or NULL, d_y [H, T].  Scratch (h exchange, barrier word) is allocated per call.
 *   mvb_audio_post_test : mvb_audio_post with a workspace of its own, plus the K-weighted signal d_y fp32 [n_samples],
 *                         the block energies d_energy fp32 [n_blocks + 1] (the last entry: sum of x^2 over the whole
 *                         signal) and d_res fp32 [3] = {LKFS, gain, compressor flag}; *n_blocks_out (host) = number of
 *                         complete 400 ms gating blocks.
 * Both synchronise `stream`. */
int mvb_voc_op_test(int32_t op, const float* d_x, int32_t Cin, int32_t T, const float* d_w, const float* d_b, int32_t Cout,
                    int32_t k, int32_t elu_in, int32_t accumulate, const float* d_skip, float* d_y, void* stream);
int mvb_audio_post_test(const float* d_wav, int32_t n_samples, int32_t sample_rate, float loudness_headroom_db,
                        int32_t loudness_compressor, int16_t* d_pcm16, float* d_wav_out, float* d_y, float* d_energy,
                        float* d_res, int32_t* n_blocks_out, void* stream);
/* Test hook for the EnCodec encoder kernels (not part of the drop-in surface): one launch of a csrc/encoder.cu kernel on
 * a single segment of T samples of which the first V are valid (1 <= V <= T; samples past V are never read into a
 * written output), through the launch helpers of mvb_enc_encode.
 *   op 0: k_conv1d_down<k>, stride k in {2, 4, 5, 8} (ELU on the input fused): d_x [Cin, T] (T % k == 0) -> d_y
 *         [Cout, T / k], of which the first ceil(V / k) columns are written; d_w [Cout, Cin, 2k], d_b [Cout].
 *   op 1: k_conv1d<k>, k = 1 / 3 / 7, ELU on the input when elu_in: d_x [Cin, T] -> the first V columns of d_y [Cout, T];
 *         d_w [Cout, Cin, k], d_b [Cout] or NULL.
 *   op 2: k_rvq_encode over k codebooks: d_x = embeddings [Cin, T] (Cin <= 128), d_w = codebooks [k, 1024, Cin],
 *         d_codes int32 [k, T], d_y = the residual after the last codebook [Cin, T] or NULL.  |e|^2 is computed as
 *         mvb_enc_create computes it, into scratch allocated per call.
 * Synchronises `stream`. */
int mvb_enc_op_test(int32_t op, const float* d_x, int32_t Cin, int32_t T, int32_t V, const float* d_w, const float* d_b,
                    int32_t Cout, int32_t k, int32_t elu_in, float* d_y, int32_t* d_codes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Stage 2: the non-causal codebook-expansion model (fam/llm/model.py:195-314 with causal=False) and its sampler
 * (fam/llm/mixins/non_causal.py:15-67).  Shapes come from second_stage.pt["model_args"] (inference.py:124-128).
 * Supported: every GPTConfig (model.py:26-46) the reference's non-causal GPT builds with a speaker projection --
 * norm_type "rmsnorm" or "layernorm", nonlinearity_type "swiglu" or "gelu", bias True or False (mvb_s2_arch) -- with
 * head size 64 or 128 and equal target vocabularies (anything else fails loudly). */
typedef struct mvb_s2_config {
  int32_t n_layer, n_head, n_embd;
  int32_t hidden;          /* MLP width: SwiGLU's (layers.py:51-53), or 4 n_embd for GELU (layers.py:46) */
  int32_t block_size;      /* sequence length t of the single non-causal pass (non_causal.py:31) */
  int32_t n_in;            /* input hierarchies (2) */
  int32_t vocab_in[8];
  int32_t n_out;           /* predicted hierarchies (6) */
  int32_t vocab_out[8];
  int32_t spk_dim;
  float   norm_eps;        /* RMSNorm eps; LayerNorm always uses 1e-5 (layers.py:17) */
  int32_t max_batch;
  int32_t options;         /* MVB_S2_* bits below; 0 = the production engine */
} mvb_s2_config;
/* Stage-2 option (fixed at create time; the workspace size does not depend on it; any other bit is MVB_ERR_ARG): */
#define MVB_S2_EAGER 0x1   /* launch the forward pass kernel by kernel instead of replaying a captured CUDA graph */
typedef struct mvb_s2 mvb_s2;
/* Stage-2 architecture (GPTConfig.norm_type, nonlinearity_type, bias); all zero = rmsnorm, swiglu, no bias.  A field
 * outside its values is MVB_ERR_ARG naming it. */
typedef struct mvb_s2_arch {
  int32_t norm;            /* MVB_S2_NORM_*: ln_1, ln_2 and ln_f */
  int32_t mlp;             /* MVB_S2_MLP_* */
  int32_t bias;            /* 1: biases on c_attn, attn.c_proj, the MLP Linears and (LayerNorm) ln_1, ln_2, ln_f */
} mvb_s2_arch;
#define MVB_S2_NORM_RMS    0   /* RMSNorm(eps = norm_eps), layers.py:20-30 */
#define MVB_S2_NORM_LAYER  1   /* LayerNorm(eps = 1e-5), with a beta when bias, layers.py:8-17 */
#define MVB_S2_MLP_SWIGLU  0   /* c_proj(silu(w1 x) * (w3 x)) */
#define MVB_S2_MLP_GELU    1   /* c_proj(GELU(c_fc x)), exact erf GELU (nn.GELU()) */

size_t mvb_s2_workspace_bytes(const mvb_s2_config* cfg);
/* offsets (host), bf16 arena as for stage 1: wte[n_in], wpe, speaker_cond_pos, ln_f, lm_heads[n_out], then per layer
 * {ln_1, attn.c_attn, attn.c_proj, ln_2, mlp.swiglu.w1, mlp.swiglu.w3, mlp.c_proj} (GELU: {ln_1, attn.c_attn,
 * attn.c_proj, ln_2, mlp.c_fc, mlp.c_proj}); then, when arch->bias: ln_f.bias (LayerNorm only), and per layer
 * {ln_1.bias (LayerNorm only), attn.c_attn.bias, attn.c_proj.bias, ln_2.bias (LayerNorm only), mlp.c_fc.bias |
 * mlp.swiglu.w1.bias, mlp.swiglu.w3.bias, mlp.c_proj.bias}.  speaker_cond_pos and lm_heads never have a bias.
 * arch NULL = all zero.  d_workspace must be zero-filled; its size does not depend on arch.  Replaces Model._init_model
 * (inference.py:102-141).  mvb_s2_create == mvb_s2_create_ex with arch NULL. */
int mvb_s2_create_ex(const mvb_s2_config* cfg, const mvb_s2_arch* arch, const void* d_arena, size_t arena_bytes,
                     const uint64_t* offsets, void* d_workspace, mvb_s2** out);
int mvb_s2_create(const mvb_s2_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets,
                  void* d_workspace, mvb_s2** out);
int mvb_s2_destroy(mvb_s2* h);
/* == GPT.generate -> _non_causal_sample for `batch` rows: d_idx int32 [batch, n_in, block_size] (built as
 * inference.py:283-306), d_spk fp32 [batch, spk_dim] or NULL, top_k <= 0 disables, d_noise fp32
 * [n_out, batch*block_size, vocab_out] = the Exp(1) draws torch.multinomial consumes (NULL = on-device Philox),
 * d_tokens int32 [batch, n_out, block_size]; d_logits_out optional fp32 [n_out, batch*block_size, vocab_out]. */
int mvb_s2_forward(mvb_s2* h, int32_t batch, const int32_t* d_idx, const float* d_spk, float temperature,
                   int32_t top_k, const float* d_noise, uint64_t seed, int32_t* d_tokens, float* d_logits_out,
                   void* stream);
/* Test hook (not part of the drop-in surface): one stage-2 bidirectional attention (k_s2_attn, launched as
 * mvb_s2_forward launches it) without an mvb_s2 handle.  d_qkv fp32 [B * t, 3 E] rows {q | k | v}, head h at columns
 * h * hs of each third (hs = E / n_head, 64 or 128); d_out fp32 [B * t, E] = softmax(q k^T / sqrt(hs)) v per (row block,
 * head).  Synchronises `stream`. */
int mvb_s2_attn_test(const float* d_qkv, int32_t B, int32_t t, int32_t E, int32_t n_head, float* d_out, void* stream);
/* Test hook (not part of the drop-in surface): the stage-2 sampler (k_s2_sample, launched as mvb_s2_forward launches
 * it) on caller logits without an mvb_s2 handle.  d_logits fp32 [n_hier, n_rows, V], 1 <= V <= 2048; d_params DEVICE
 * buffer of 16 bytes {float temperature; int32 top_k (<= 0 disables); uint64 seed}; d_noise fp32 [n_hier, n_rows, V]
 * Exp(1) draws or NULL (on-device Philox keyed on (entry, row, hierarchy, seed)); d_tokens int32 [n_hier, n_rows].
 * Allocates nothing; synchronises `stream`. */
int mvb_s2_sample_test(const float* d_logits, int32_t n_hier, int32_t n_rows, int32_t V, const void* d_params,
                       const float* d_noise, int32_t* d_tokens, void* stream);
/* Test hook (not part of the drop-in surface): the stage-2 front end (k_s2_spk, then k_s2_embed, launched as
 * mvb_s2_forward launches them) without an mvb_s2 handle.  d_idx int32 [B, n_in, t]; d_wte DEVICE array of n_in bf16
 * table pointers ([vocab_h, E] each); d_wpe bf16 [>= t, E]; d_W_spk bf16 [E, spk_dim]; d_spk fp32 [B, spk_dim] or NULL
 * (no speaker term; d_W_spk and d_spk_proj are then not read); d_spk_proj fp32 [B, E] = W_spk . spk[b];
 * d_x fp32 [B * t, E] = sum_h wte_h[idx[b, h, i]] + wpe[i] (+ spk_proj[b]).  MVB_ERR_ARG for a null pointer, B, t, E or
 * spk_dim < 1, or n_in outside 1..8.  Allocates nothing; synchronises `stream`. */
int mvb_s2_embed_test(const int32_t* d_idx, int32_t B, int32_t n_in, int32_t t, const void* d_wte, const void* d_wpe,
                      const void* d_W_spk, const float* d_spk, int32_t spk_dim, int32_t E, float* d_spk_proj, float* d_x,
                      void* stream);
/* Test hook (not part of the drop-in surface): mvb_gemm_test's operator with the stage-2 prologues and epilogues.
 * out[R, M] (+)= epilogue(f(x) . W^T + bias): norm 0 none, 1 RMSNorm (gain, eps), 2 LayerNorm (gain, optional beta,
 * eps); epi 0 store, 1 residual add, 2 SwiGLU silu(x W^T + bias) * (x W3^T + bias3), 4 GELU (exact erf).  d_bias,
 * d_bias3 bf16 [M] or NULL (d_bias3 is required by SwiGLU with a bias).  ksplit_override > 0 forces the K split.
 * Synchronises `stream`. */
int mvb_s2_linear_test(int32_t epi, int32_t norm, const void* d_W, const void* d_W3, const void* d_bias, const void* d_bias3,
                       int32_t M, int32_t K, const float* d_x, int32_t ldx, int32_t R, const void* d_gain, const void* d_beta,
                       float eps, int32_t split_lo, int32_t ksplit_override, float* d_out, int32_t ldo, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Vocoder, EnCodec-24 kHz decode path: RVQ decode (the diffusion condition `decode_latent`) and the SEANet decoder
 * (causal conv stack + 2-layer LSTM), i.e. what mbd.tokens_to_wav (fam/llm/decoders.py:85, audiocraft 1.2.0 ->
 * transformers EncodecModel.decode) evaluates first.  The multi-band diffusion UNets themselves are NOT implemented
 * (their source/weights are unavailable: parity unpinned, see DESIGN.md).  fp32 arena, weight norm folded. */
typedef struct mvb_voc_config {
  int32_t n_q;          /* 8 codebooks at 6 kbps */
  int32_t hidden;       /* codebook / latent dim 128 */
  int32_t n_filters;    /* 32 */
  int32_t n_ratios;     /* 4 */
  int32_t ratios[8];    /* 8, 5, 4, 2 */
  int32_t kernel, res_kernel, last_kernel; /* 7, 3, 7 */
  int32_t compress;     /* 2 */
  int32_t max_frames;   /* workspace capacity in 75 Hz frames */
} mvb_voc_config;
typedef struct mvb_voc mvb_voc;

size_t mvb_voc_workspace_bytes(const mvb_voc_config* cfg);
/* offsets (host), fp32 tensors: codebooks[n_q] [1024,hidden] | conv_in {w[512,hidden,7], b} | lstm layer 0
 * {w_ih, w_hh, b_ih+b_hh} | lstm layer 1 {..} | per ratio: up {w[Cin,Cout,2r], b}, res.block1 {w,b}, res.block3 {w,b},
 * res.shortcut {w,b} | conv_out {w[1,32,7], b}. */
int mvb_voc_create(const mvb_voc_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets,
                   void* d_workspace, mvb_voc** out);
int mvb_voc_destroy(mvb_voc* h);
/* d_codes int32 [n_q, T] -> d_latent fp32 [hidden, T]  (EncodecResidualVectorQuantizer.decode) */
int mvb_voc_decode_latent(mvb_voc* h, const int32_t* d_codes, int32_t T, float* d_latent, void* stream);
/* d_codes int32 [n_q, T] -> d_wav fp32 [T * prod(ratios)]  (EncodecModel.decode, one chunk, 24 kHz) */
int mvb_voc_decode(mvb_voc* h, const int32_t* d_codes, int32_t T, float* d_wav, void* stream);
/* Batched decode (fam/llm/inference.py:438-517 `_sample_utterance_batch` decodes a batch of utterances): n utterances in
 * one launch set, the two LSTM layers as one grid-barrier loop over max T_i for all of them.  mvb_voc_decode /
 * mvb_voc_decode_latent run the same launch sequence over one utterance, and utterance i is bit-identical to them on it
 * alone.  Layout, with off_i = T_0 + ... + T_{i-1}:
 *   d_codes  int32, utterance i as [n_q, T_i] at n_q off_i;  T: HOST int32 [n];
 *   d_wav    fp32, utterance i as [T_i prod(ratios)] at off_i prod(ratios);  d_latent fp32 [hidden, T_i] at hidden off_i.
 * d_batch_ws: a caller workspace of mvb_voc_batch_workspace_bytes(cfg, max_batch, max_total_frames) bytes (the handle's
 * own workspace is not used), passed with the two capacities it was sized for.  MVB_ERR_ARG, before anything is
 * launched, unless 1 <= n <= max_batch <= 32, every 8 <= T_i <= max_frames and sum T_i <= max_total_frames.  Calls on one
 * batch workspace must be ordered (same stream).  mvb_voc_batch_workspace_bytes returns 0 for max_batch > 32. */
size_t mvb_voc_batch_workspace_bytes(const mvb_voc_config* cfg, int32_t max_batch, int32_t max_total_frames);
int mvb_voc_decode_batch(mvb_voc* h, int32_t n, const int32_t* d_codes, const int32_t* T, void* d_batch_ws, int32_t max_batch,
                         int32_t max_total_frames, float* d_wav, void* stream);
int mvb_voc_decode_latent_batch(mvb_voc* h, int32_t n, const int32_t* d_codes, const int32_t* T, void* d_batch_ws,
                                int32_t max_batch, int32_t max_total_frames, float* d_latent, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Codec, EnCodec-24 kHz encode path: SEANet encoder (causal conv stack with strided downsampling + 2-layer LSTM) and
 * the residual vector quantiser's encode, i.e. what `EncodecDecoder.get_tokens` (fam/llm/decoders.py:49-64) and the
 * fine-tuning loader's `_extract_encodec_tokens` (fam/llm/loaders/training_data.py:98-112) evaluate through
 * transformers EncodecModel.encode (normalize=False, one chunk).  Same checkpoint as mvb_voc; fp32 arena, weight norm
 * folded.  An input of L samples gives F = ceil(L / prod(ratios)) frames. */
typedef struct mvb_enc_config {
  int32_t n_q;          /* codebooks emitted: floor(bandwidth * 1000 / 750), 8 at 6 kbps */
  int32_t hidden;       /* codebook / embedding dim 128 (<= 128) */
  int32_t n_filters;    /* 32 */
  int32_t n_ratios;     /* 4 */
  int32_t ratios[8];    /* 8, 5, 4, 2 (EncodecConfig.upsampling_ratios; the encoder downsamples by them in reverse), each 2, 4, 5 or 8 */
  int32_t kernel, res_kernel, last_kernel; /* 7, 3, 7 */
  int32_t compress;     /* 2 */
  int32_t max_frames;   /* workspace capacity of mvb_enc_encode in frames */
} mvb_enc_config;
typedef struct mvb_enc mvb_enc;

/* The handle's workspace also holds the codebook pointer table and |e_j|^2 of every codebook row, computed in double and
 * rounded once to fp32 by mvb_enc_create (which synchronises the device). */
size_t mvb_enc_workspace_bytes(const mvb_enc_config* cfg);
/* offsets (host), fp32 tensors: codebooks[n_q] [1024, hidden] | conv_in {w[32,1,7], b} | per level, ratios in reverse
 * (2, 4, 5, 8 at C = 32, 64, 128, 256): res.block1 {w[C/2,C,3], b}, res.block3 {w[C,C/2,1], b}, res.shortcut {w[C,C,1], b},
 * down {w[2C,C,2r], b} | lstm layer 0 {w_ih, w_hh, b_ih+b_hh} | lstm layer 1 {..} | conv_out {w[hidden,512,7], b}. */
int mvb_enc_create(const mvb_enc_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets,
                   void* d_workspace, mvb_enc** out);
int mvb_enc_destroy(mvb_enc* h);
/* d_wav fp32 [L] (mono, 24 kHz) -> d_codes int32 [n_q, F]; d_emb fp32 [hidden, F] (the encoder output before
 * quantisation, the layout of mvb_voc_decode_latent) or NULL.  1 <= L <= prod(ratios) * max_frames.  The batch of one of
 * mvb_enc_encode_batch, on the handle's workspace. */
int mvb_enc_encode(mvb_enc* h, const float* d_wav, int32_t L, int32_t* d_codes, float* d_emb, void* stream);
/* Batched encode: n utterances in one launch set, the LSTM as one grid-barrier loop over max F_i.  Utterance i is
 * bit-identical to mvb_enc_encode on it alone.  Layout, with off_i = F_0 + ... + F_{i-1}:
 *   d_wav    fp32, utterance i's L_i samples at L_0 + ... + L_{i-1};  L: HOST int32 [n];
 *   d_codes  int32, utterance i as [n_q, F_i] at n_q off_i (the d_codes layout of mvb_voc_decode_batch);
 *   d_emb    fp32 [hidden, F_i] at hidden off_i, or NULL.
 * d_batch_ws: mvb_enc_batch_workspace_bytes(cfg, max_batch, max_total_frames) bytes, passed with the capacities it was
 * sized for.  MVB_ERR_ARG, before anything is launched, unless 1 <= n <= max_batch <= 32, every
 * 1 <= L_i <= prod(ratios) * max_frames and sum F_i <= max_total_frames.  Calls on one batch workspace must be ordered. */
size_t mvb_enc_batch_workspace_bytes(const mvb_enc_config* cfg, int32_t max_batch, int32_t max_total_frames);
int mvb_enc_encode_batch(mvb_enc* h, int32_t n, const float* d_wav, const int32_t* L, void* d_batch_ws, int32_t max_batch,
                         int32_t max_total_frames, int32_t* d_codes, float* d_emb, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Multi-band-diffusion vocoder (SURVEY.md row a17, second half) == `mbd.tokens_to_wav` (fam/llm/decoders.py:84-85 ->
 * audiocraft 1.2.0 MultiBandDiffusion.tokens_to_wav) after the codec decode: n_models band UNets x n_calls sampler steps
 * conditioned on the codec latent, per-band output processors, sum, 32-band re-EQ against the EnCodec waveform.
 * PARITY UNPINNED (audiocraft / julius / mbd_comp_8.pt are not available): the configuration is a parameter. */
typedef struct mvb_mbd_config {
  int32_t n_models;        /* band models summed by MultiBandDiffusion.generate (4) */
  int32_t chin, hidden, depth, res_blocks, norm_groups, kernel, stride;   /* DiffusionUnet kwargs; (kernel, stride) in {(8,4), (4,2)} */
  float   growth;
  int32_t emb_all_layers;  /* step embedding added after every encoder level (else only the first) */
  int32_t codec_dim;       /* 128: channels of the condition (codec latent) */
  int32_t num_steps;       /* rows of the step-embedding tables (1000) */
  int32_t n_calls;         /* UNet evaluations per band model (20 for step_list = range(1000)[::-50] + [0]) */
  float   noise_scale, clip;
  int32_t proc_bands, proc_taps;   /* MultiBandProcessor: SplitBands(n_bands) and its filter length */
  int32_t eq_bands, eq_taps;       /* re_eq: 32 bands and the filter length */
  int32_t max_samples;     /* workspace capacity (samples at 24 kHz) */
  int32_t options;         /* MVB_MBD_* bits below; 0 = the production engine */
} mvb_mbd_config;
/* MBD options, fixed at create time.  Both change the workspace layout, which mvb_mbd_workspace_bytes computes from the
 * same config; any other bit is MVB_ERR_ARG. */
#define MVB_MBD_CUDA_CORES 0x1 /* every convolution on the fp32 CUDA-core kernels (no packed bf16 taps, no tensor cores) */
#define MVB_MBD_ONE_STREAM 0x2 /* band models back to back on the caller's stream with one activation block */
typedef struct mvb_mbd mvb_mbd;
/* fp32 arena tensors (offsets, host): for every band model, in this order
 *   per encoder level: conv.weight [C, Cin, k], norm.weight, norm.bias, res_blocks x {norm1.w, norm1.b, conv1.w [C,C,3], conv1.b,
 *                      norm2.w, norm2.b, conv2.w, conv2.b}, step-embedding table [num_steps, C]
 *   conv_codec.weight [C_bottleneck, codec_dim, 1], conv_codec.bias
 *   per decoder level (deepest first): res_blocks x {8 tensors}, norm.weight, norm.bias, convtr.weight [C, C_out, k]
 *   processor scale [proc_bands] = (std / target_std) ** power_std, processor mean [proc_bands]
 * then three globals: processor low-pass bank [proc_bands - 1, proc_taps], re-EQ bank [eq_bands - 1, eq_taps],
 * schedule table [n_calls, 4] = {a, b, sigma, step}:  previous = clamp((current - a * estimate) * b + sigma * noise). */
size_t mvb_mbd_workspace_bytes(const mvb_mbd_config* cfg);
int mvb_mbd_create(const mvb_mbd_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets, void* d_workspace,
                   mvb_mbd** out);
int mvb_mbd_destroy(mvb_mbd* h);
/* d_cond fp32 [codec_dim, n_frames] (mvb_voc_decode_latent), d_wav_encodec fp32 [n_samples] (mvb_voc_decode),
 * d_noise fp32 [n_models, n_calls, n_samples] standard-normal draws (row 0 = initial sample, row i = the draw added after
 * call i - 1 ... see oracle/mbd_port.py) or NULL for on-device Philox (seed); d_wav_out fp32 [n_samples].
 * MVB_ERR_ARG, before anything is enqueued, unless 16 stride <= n_samples <= max_samples and 1 <= n_frames <=
 * min(max_samples / 320 + 8, 2 Tl): the workspace holds the projected condition for max_samples / 320 + 8 frames, and the
 * condition may be at most 2x longer than the bottleneck, Tl = n_samples divided depth times by stride, rounded up. */
int mvb_mbd_tokens_to_wav(mvb_mbd* h, const float* d_cond, int32_t n_frames, const float* d_wav_encodec, int32_t n_samples,
                          const float* d_noise, uint64_t seed, float* d_wav_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Speaker encoder (SURVEY.md row N3): fam/quantiser/audio/speaker_encoder/{audio.py:10-22, model.py:50-103}.
 * 16 kHz mono fp32 waveform -> power mel spectrogram (n_fft 400, hop 160, 40 Slaney bands, centered, zero padded) ->
 * 3-layer LSTM(40 -> 256) over partial windows of 160 frames -> linear -> ReLU -> L2 norm -> mean -> L2 norm. */
typedef struct mvb_spk_config {
  int32_t n_mels;          /* 40 */
  int32_t hidden;          /* 256 */
  int32_t n_layers;        /* 3 */
  int32_t emb;             /* 256 */
  int32_t n_fft;           /* 400 = 25 ms at 16 kHz */
  int32_t hop;             /* 160 = 10 ms */
  int32_t partial_frames;  /* 160 */
  int32_t max_samples;     /* workspace capacity (samples at 16 kHz) */
} mvb_spk_config;
typedef struct mvb_spk mvb_spk;
/* fp32 arena tensors, in this order: per LSTM layer {weight_ih [4H, in], weight_hh [4H, H], bias_ih + bias_hh [4H]},
 * linear.weight [256, 256], linear.bias [256], mel filterbank [n_mels, n_fft/2 + 1], analysis window [n_fft],
 * cos(2 pi i / n_fft) [n_fft], -sin(2 pi i / n_fft) [n_fft]. */
#define MVB_SPK_TENSORS 15
size_t mvb_spk_workspace_bytes(const mvb_spk_config* cfg);
int mvb_spk_create(const mvb_spk_config* cfg, const void* d_arena, size_t arena_bytes, const uint64_t* offsets,
                   void* d_workspace, mvb_spk** out);
int mvb_spk_destroy(mvb_spk* h);
/* == audio.wav_to_mel_spectrogram: d_wav fp32 [n_samples] -> d_mel fp32 [1 + n_samples / hop, n_mels] (parity hook). */
int mvb_spk_mel(mvb_spk* h, const float* d_wav, int32_t n_samples, float* d_mel, void* stream);
/* == SpeakerEncoder.embed_utterance on an already padded waveform: slice_starts (HOST int32 [n_partials]) are the first mel
 * frames of the partial windows (compute_partial_slices, model.py:55-79); d_embed fp32 [256]; d_partials_out optional
 * fp32 [n_partials, 256].  MVB_ERR_ARG before anything is launched unless 1 <= n_partials <= 1024 and every window lies
 * in the spectrogram: 0 <= start and start + partial_frames <= 1 + n_samples / hop. */
int mvb_spk_embed(mvb_spk* h, const float* d_wav, int32_t n_samples, const int32_t* slice_starts, int32_t n_partials,
                  float* d_embed, float* d_partials_out, void* stream);
/* Test hook for the speaker-encoder kernels (not part of the drop-in surface), through the launch helper of mvb_spk_embed
 * with the handle's weights and configuration:
 *   op 0: k_spk_lstm over a caller mel d_in fp32 [n_frames, n_mels] at the windows `starts` (HOST int32 [n_partials],
 *         checked as mvb_spk_embed checks them) -> d_out fp32 [n_partials, 256]; d_trace optional fp32
 *         [n_partials][partial_frames][3 layers][h, c][256], the LSTM state after every layer step.
 *   op 1: k_spk_mean over d_in fp32 [n_partials, 256] -> d_out fp32 [256]; n_frames, starts and d_trace are not used.
 * Synchronises `stream`. */
int mvb_spk_op_test(mvb_spk* h, int32_t op, const float* d_in, int32_t n_frames, const int32_t* starts, int32_t n_partials,
                    float* d_out, float* d_trace, void* stream);

/* Batched speaker front-end: a file's waveform -> 16 kHz (mvb_resample_batch) -> silence trimmed (mvb_spk_trim_batch) ->
 * embedded (mvb_spk_embed_batch).  Each call takes up to MVB_SPK_MAX_BATCH signals with their lengths in HOST arrays,
 * validates everything before anything is launched (MVB_ERR_ARG / MVB_ERR_UNSUPPORTED, outputs untouched) and launches
 * one kernel per stage for the whole batch; signal i is computed exactly as it is alone.  "Packed" means signal i's
 * samples start at n_0 + ... + n_{i-1}. */
#define MVB_SPK_MAX_BATCH 32
/* Longest filter the resampler takes: 20 max(up, down) + 1 <= 16384 taps, i.e. max(up, down) <= 819 after reduction.
 * Every standard rate from 8 to 96 kHz to 16 kHz fits (11.025 kHz: 640/441, 12,801 taps). */
#define MVB_RESAMPLE_MAX_TAPS 16384
/* == scipy.signal.resample_poly(x, up, down) with its defaults, per signal, in fp32 (fp32 products and sums).  up / down
 * are reduced by their gcd.  The caller designs the filter in float64,
 *   h = firwin(n_taps, 1 / max(up, down), window=("kaiser", 5.0)) * up,   n_taps = 20 max(up, down) + 1,
 * and passes it in polyphase order: d_taps fp32 [up][P], P = ceil(n_taps / up), d_taps[r][q] = h[r + q up] (0 past the
 * end).  Output j of a signal of n_in samples is sum_q h[r + q up] x[m - q] over 0 <= m - q < n_in, with
 * t = j down + (n_taps - 1) / 2 (scipy's delay compensation), r = t mod up, m = t div up: q ascending, one fmaf chain
 * from 0.  d_in packed fp32 with n_in (HOST int32 [n], each >= 1) -> d_out packed fp32, n_out_i = ceil(n_in_i up / down).
 * When up == down the signals are copied (no kernel); d_taps and n_taps are then not read.  MVB_ERR_UNSUPPORTED when the
 * filter would exceed MVB_RESAMPLE_MAX_TAPS; MVB_ERR_ARG for n_taps != 20 max(up, down) + 1. */
int mvb_resample_batch(int32_t n, const float* d_in, const int32_t* n_in, int32_t up, int32_t down, const float* d_taps,
                       int32_t n_taps, float* d_out, void* stream);
/* Bytes of the batch workspace of mvb_spk_trim_batch / mvb_spk_embed_batch for at most max_batch (<= 32) signals of
 * max_total_samples (<= INT32_MAX) 16 kHz samples in all; 0 on an invalid argument.  It holds max_batch +
 * max_total_samples / hop mel frames, as many windows, and the trim's RMS frames.  Calls on one workspace must be ordered. */
size_t mvb_spk_batch_workspace_bytes(const mvb_spk_config* cfg, int32_t max_batch, int64_t max_total_samples);
/* == trim_silence / librosa.effects.trim(y, top_db) per signal: frames of 2048 samples centered every 512 (zero padded),
 * RMS in fp32, ref = the signal's loudest frame; kept are the frames with 20 log10(max(rms, 1e-10) / ref) > -top_db,
 * evaluated as max(rms, 1e-10) / ref > 10^(-top_db / 20) with the threshold rounded to fp32 once.
 * d_wav packed fp32 with n_samples (HOST int32 [n], each >= 1, sum <= max_total_samples) -> d_spans int32 [n][2]:
 * {first kept frame * 512, min(n_i, (last kept frame + 1) * 512)}, {0, 0} when nothing is kept (an all-zero signal).
 * top_db must be finite and > 0. */
int mvb_spk_trim_batch(mvb_spk* h, int32_t n, const float* d_wav, const int32_t* n_samples, float top_db, void* d_batch_ws,
                       int32_t max_batch, int64_t max_total_samples, int32_t* d_spans, void* stream);
/* Batched SpeakerEncoder.embed_utterance: utterance i is the n_wav_i (>= 0) samples at d_wav + wav_off_i (HOST int64 [n],
 * so trimmed spans are read in place), zero-extended to max(n_wav_i, (last start + partial_frames) * hop) samples as
 * embed_utterance pads it; that length must be <= max_samples, and the padded lengths sum to <= max_total_samples.
 * Its n_partials_i (HOST int32 [n], >= 1) window starts follow those of utterance i - 1 in `starts` (HOST int32, flat),
 * each >= 0; at most max_batch + max_total_samples / hop windows in all.  d_embed fp32 [n, 256]; d_partials_out
 * optional fp32 [sum n_partials, 256] in the same order.  Utterance i is bit-identical to mvb_spk_embed on its padded
 * waveform alone: one k_spk_mel launch over all utterances, one k_spk_lstm over all windows, one k_spk_mean. */
int mvb_spk_embed_batch(mvb_spk* h, int32_t n, const float* d_wav, const int64_t* wav_off, const int32_t* n_wav,
                        const int32_t* starts, const int32_t* n_partials, void* d_batch_ws, int32_t max_batch,
                        int64_t max_total_samples, float* d_embed, float* d_partials_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Audio post-processing on the device (SURVEY.md row N2) == `_save_audio` (fam/llm/decoders.py:40-47 -> audiocraft
 * audio_write(strategy="loudness", loudness_compressor=True)): BS.1770-4 integrated loudness exactly as
 * torchaudio.functional.loudness computes it (the function audiocraft calls), gain to -loudness_headroom_db LUFS, tanh
 * compressor, clip, PCM16.  d_wav fp32 mono [n_samples]; d_pcm16 int16 [n_samples]; d_wav_out optional fp32 [n_samples];
 * d_lkfs_gain optional fp32 [2] = {measured LKFS, applied linear gain}.  Edge cases:
 *   LKFS = -inf: the RMS is below the 2e-3 energy floor; gain 1, no compressor (the signal passes through, clipped).
 *   LKFS = NaN : the meter is undefined -- a non-finite sample, no complete 400 ms block, or every block below the
 *                -70 LKFS gate (where torchaudio raises or returns NaN and audiocraft's normalize_loudness fails); gain 1,
 *                no compressor, NaN samples written as 0.  Callers that mirror the host writer must raise here.
 * n_samples beyond 15,996 gating blocks returns MVB_ERR_UNSUPPORTED before anything is launched. */
size_t mvb_audio_post_workspace_bytes(int32_t max_samples);
int mvb_audio_post(const float* d_wav, int32_t n_samples, int32_t sample_rate, float loudness_headroom_db,
                   int32_t loudness_compressor, void* d_workspace, int16_t* d_pcm16, float* d_wav_out,
                   float* d_lkfs_gain, void* stream);
/* mvb_audio_post over n signals with one launch set per 32 signals (mvb_audio_post is the same launch set over one).
 * d_wav fp32 and d_pcm16 / d_wav_out: signal i at off_i = n_0 + ... + n_{i-1} (n_samples: HOST int32 [n]); d_lkfs_gain
 * optional fp32 [n][2].  Signal i's PCM, LKFS and gain are bit-identical to mvb_audio_post on it alone, edge cases
 * included, and no signal's values affect another's.  d_workspace:
 * mvb_audio_post_batch_workspace_bytes(max_batch, max_total_samples) bytes, passed with the capacities it was sized for.
 * MVB_ERR_ARG unless 1 <= n <= max_batch, every n_i >= 1 and sum n_i <= max_total_samples; MVB_ERR_UNSUPPORTED when a
 * signal exceeds 15,996 gating blocks; both before anything is launched. */
size_t mvb_audio_post_batch_workspace_bytes(int32_t max_batch, int32_t max_total_samples);
int mvb_audio_post_batch(const float* d_wav, int32_t n, const int32_t* n_samples, int32_t sample_rate, float loudness_headroom_db,
                         int32_t loudness_compressor, void* d_workspace, int32_t max_batch, int32_t max_total_samples,
                         int16_t* d_pcm16, float* d_wav_out, float* d_lkfs_gain, void* stream);

#define MVB_OK 0
#define MVB_ERR_CUDA 1
#define MVB_ERR_ARG 2
#define MVB_ERR_PROMPT_TOO_LONG 3
#define MVB_ERR_UNSUPPORTED 4

#ifdef __cplusplus
}
#endif
#endif /* MVB200_H */

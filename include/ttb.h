/* tortoise-b200: C-ABI of the sm_90a kernel library (libttb.so).
 *
 * The reference (neonbjb/tortoise-tts) has no FFI layer: its hot path is PyTorch modules calling
 * ATen/cuBLAS/cuDNN. This header is the boundary a maintainer would bind instead (ctypes stub in
 * INTEGRATION.md): every entry point takes raw device pointers, sizes and a cudaStream_t (as void*),
 * returns 0 on success or a negative code (message via ttb_last_error()), and never throws.
 * Each function cites the reference computation (file:line under /root/reference/tortoise) it replaces.
 *
 * Conventions: activations are TOKEN-MAJOR ([tokens, channels], channels contiguous) unless noted;
 * "bf16" pointers are passed as void* to keep this header free of CUDA types; all kernels are enqueued
 * on `stream` and do not synchronise.
 */
#ifndef TTB_H
#define TTB_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* ttb_last_error(void);
int ttb_version(void);
/* 1 if the current device is compute capability 9.0 (sm_90a, the only supported target), else 0 */
int ttb_device_ok(void);

/* ---------------------------------------------------------------- dense contraction (wgmma) */
enum { TTB_ACT_NONE = 0, TTB_ACT_GELU_NEW = 1, TTB_ACT_SILU = 2, TTB_ACT_GEGLU = 3, TTB_ACT_LRELU02 = 4, TTB_ACT_TANH = 5,
       TTB_ACT_GELU_ERF = 6 /* exact 0.5 x (1 + erf(x / sqrt 2)): HF ACT2FN['gelu'] of the wav2vec2 aligner */ };

typedef struct TtbGemmArgs {
  const void* A;        /* bf16 [batch, rows, lda] activations (K contiguous) */
  const void* W;        /* bf16 [N, taps*K] weights */
  const float* bias;    /* [N] or NULL */
  const float* residual;/* fp32 [batch, M, ldr] or NULL (added after the activation) */
  float* out_f32;       /* fp32 [batch, M, ldo] or NULL */
  void* out_bf16;       /* bf16 [batch, M, ldob] or NULL */
  long long a_bstride, res_bstride, outf_bstride, outb_bstride; /* batch strides, in elements */
  int lda, ldr, ldo, ldob;
  int rows;             /* valid rows of A per batch item (conv zero-padding boundary) */
  int M, N, K;          /* output rows per batch item, output columns, reduction per tap */
  int taps, pad;        /* Conv1d kernel size (1 = plain GEMM) and left padding */
  int batch;
  int act;              /* TTB_ACT_* ; GEGLU expects W rows interleaved (u0,g0,u1,g1,..) and writes N/2 columns */
  float alpha;          /* accumulator scale */
  int tile_n;           /* 0 = auto, 32, 64 or 128 */
  int force_ref;        /* 1 = SIMT checker kernel (tests only) */
  int splitk;           /* > 1: split the reduction over grid.z; writes raw fp32 partials out_f32[split][M][ldo]
                           (outf_bstride = stride between splits); batch must be 1, no epilogue fusion */
  int cluster;          /* 2 or 4: CTAs adjacent in N form a cluster and share the activation tile by TMA multicast
                           (tile_n picks the tile width: 32, 64, else 128); 0/1 = off */
  int variant;          /* 0 = auto; 1 = one tile per CTA; 2 = persistent kernel; with tile_n = 32 also 3 / 4 = one tile
                           per CTA with a 5- / 4-stage pipeline (tools/gemm_sweep.py, tools/gemm_diag.py).
                           7 = persistent warp-specialised 128x256 kernel, no split-K (the default, unless TTB_GEMM_WS=0,
                           when tile_n = 0, variant = 0, no split-K / cluster and at least one wave of 128x128 tiles).
                           Experiments not yet validated on hardware (never chosen automatically): 5 = two TMA issuer
                           threads per CTA, 6 = reserved (rejected) */
  float* gn_partials;   /* non-NULL: the epilogue also leaves the GroupNorm statistics of its OUTPUT (after bias, activation
                           and residual) in a ttb_groupnorm scratch buffer: (sum, sum of squares) of every 32-row x 32-column
                           block, i.e. one partial per (batch item, group, row block) for 32 channels per group. Needs
                           N == 32 * gn_groups and ceil(M / 32) <= TTB_GROUPNORM_SPLITS; consumed by ttb_groupnorm_apply. */
  int gn_groups;
  int tap_dilation;     /* > 1: conv taps are tap_dilation rows apart (dilated Conv1d; `pad` stays in rows, e.g.
                           dilation * (k - 1) / 2); 0 / 1 = adjacent rows */
  int w_static;         /* 1 = W is a parameter: no kernel enqueued earlier on the stream writes it. The one-tile kernel
                           may then fetch its weight tiles before it waits for the preceding kernel (programmatic
                           dependent launch); results do not change */
} TtbGemmArgs;

/* nn.Linear / HF Conv1D / nn.Conv1d(k=1,3) as one wgmma GEMM with fused bias/activation/residual.
 * Replaces: GPT2 c_attn/c_proj/c_fc (HF 4.31 modeling_gpt2, via models/autoregressive.py:150-163),
 * mel_head (autoregressive.py:42), CLVP to_q/k/v/to_out/FF (models/xtransformers.py:519-521,429-474),
 * DiffusionTts convs (models/diffusion_decoder.py:83-103, models/arch_util.py:107-111),
 * KernelPredictor.kernel_conv (models/vocoder.py:59-62). */
int ttb_gemm(const TtbGemmArgs* args, void* stream);

/* Development aid (no reference counterpart): when buf != NULL every one-tile-per-CTA ttb_gemm launch writes 8 x u64
 * per CTA into it (globaltimer ns at: start, [1]=SM id, setup done, first operands landed, last MMA issued,
 * accumulator complete, epilogue done, exit). The buffer must hold 8 * grid-size u64. NULL switches tracing off. */
int ttb_debug_gemm_trace(void* buf);

/* ---------------------------------------------------------------- normalisation */
/* y = LN(x) (eps 1e-5), optionally followed by a second LN (gpt.ln_f then final_norm,
 * autoregressive.py:42,174,348). x fp32 [M, D]; writes bf16 and/or fp32. */
int ttb_layernorm(const float* x, int M, int D, const float* g1, const float* b1, const float* g2, const float* b2,
                  void* out_bf16, float* out_f32, void* stream);
/* Residual update fused with the LayerNorm that follows it (and with the split-K reduction of the GEMM before it):
 *   x[m,:] += bias + sum_s partials[s][m,:]   (written back, fp32);   y = LN(x) (optionally chained with a 2nd LN).
 * GPT-2 block glue `h = x + c_proj(...)` -> `ln_2(h)` (HF modeling_gpt2 GPT2Block via autoregressive.py:150-163). */
int ttb_residual_layernorm(float* x, int M, int D, const float* partials, int nsplit, long long split_stride,
                           const float* bias, const float* g1, const float* b1, const float* g2, const float* b2,
                           void* out_bf16, float* out_f32, void* stream);
/* x / max(||x|| * D^-0.5, 1e-8) * g   (xtransformers.py:335-344) */
int ttb_rmsnorm(const float* x, int M, int D, const float* g, void* out_bf16, void* stream);
/* GroupNorm32 over token-major x [B, S, C] (arch_util.py:21-41) fused with the consumers that follow it in
 * ResBlock / AttentionBlock (diffusion_decoder.py:107-120): y = GN(x)*gamma+beta; if scale_shift:
 * y = y*(1+scale[b,c]) + shift[b,c] (scale_shift fp32 [B, 2C] = [scale|shift]; when ss_row != NULL the table
 * row *ss_row (device-side step counter) at stride ss_row_stride is used); if silu: y = SiLU(y).
 * `partials` is a scratch buffer of TTB_GROUPNORM_SCRATCH_FLOATS(B, groups) floats (per-block partial sums between
 * the statistics and the apply kernel; nothing is kept across calls, so one buffer may serve any number of calls on
 * the same stream). Results are bit-reproducible (no atomics). Output bf16 [B, S, ldo] and/or fp32.
 * Channels per group: a multiple of 4, or exactly 2. The 2-per-group form is GN(16 groups, C = 32) of the
 * tortoise-detect classifier's first level (models/classifier.py, normalization() at arch_util.py:26-41); it needs
 * C / 4 a power of two <= 256, no scale_shift, and ldo / ldof multiples of 4 (columns C..ldo-1 are not written).
 * Anything else returns an error. */
#define TTB_GROUPNORM_SPLITS 128
#define TTB_GROUPNORM_SCRATCH_FLOATS(B, groups) ((B) * (groups) * (2 * TTB_GROUPNORM_SPLITS + 2) + 16)
int ttb_groupnorm(const float* x, int B, int S, int C, int groups, const float* gamma, const float* beta,
                  const float* scale_shift, int ss_bstride, const int* ss_row, int ss_row_stride, int silu,
                  float* partials, void* out_bf16, int ldo, float* out_f32, int ldof, void* stream);
/* The apply half of ttb_groupnorm alone, for an x whose statistics the producing ttb_gemm already left in `partials`
 * (TtbGemmArgs.gn_partials, one partial per 32-row block): x is read once instead of twice. 32 channels per group. */
int ttb_groupnorm_apply(const float* x, int B, int S, int C, int groups, const float* gamma, const float* beta,
                        const float* scale_shift, int ss_bstride, const int* ss_row, int ss_row_stride, int silu,
                        const float* partials, void* out_bf16, int ldo, float* out_f32, int ldof, void* stream);

/* ---------------------------------------------------------------- attention */
typedef struct TtbAttnArgs {
  const void* qkv;      /* bf16 [nseq*T, ld]; q at col 0, k at col k_off, v at col v_off; head h at +64h */
  void* out;            /* bf16 [nseq*T, ldo]; head h at col 64h */
  const float* bias;    /* optional additive relative-position table fp32 [H, 2*T-1]: bias[h][j-i+T-1], or NULL */
  int nseq, T, H;
  int ld, ldo, k_off, v_off;
  float scale;          /* applied to q.k */
  int causal;
  /* optional split form (used for the shared-prompt part of the AR decode attention): keys/values from a head-major
   * cache bf16 [H, Tk, 64] shared by all sequences, result written as fp32 normalised rows + log2-sum-exp so that it
   * can be merged with attention over another key range */
  const void* kv;       /* K cache or NULL */
  const void* kv_v;     /* V cache */
  int kv_headmajor;     /* 1 = kv/kv_v are [H, Tk, 64] */
  int Tk;               /* keys per sequence (0 = T) */
  float* out_f32;       /* fp32 [nseq*T, ldo] (with lse) */
  float* lse;           /* fp32 [nseq*T, H], log2 domain, or NULL */
  int bias_sat;         /* > 0: bias[h][r] == bias[h][-(T-1)] for r <= -bias_sat and == bias[h][T-1] for r >= bias_sat
                           (T5 buckets saturate at max_distance); lets far-from-diagonal tiles skip the table. 0 = unknown */
  int head_dim;         /* 0 or 64: heads of 64 (wgmma kernels). 32 / 96 / 128: short sequences, packed form only; head h
                           at column head_dim * h (diffusion contextual embedder: 2048 channels / 16 heads) */
} TtbAttnArgs;
/* softmax(q k^T * scale + bias) v per (sequence, head), head_dim 64. Replaces QKVAttentionLegacy
 * (arch_util.py:44-77), HF GPT2Attention._attn, and xtransformers Attention (xtransformers.py:660-712). */
int ttb_attention(const TtbAttnArgs* args, void* stream);

/* ---------------------------------------------------------------- autoregressive decode (UnifiedVoice) */
typedef struct TtbArState {      /* device-resident, 64 ints */
  int step;                      /* number of tokens already sampled per candidate */
  int all_finished;
  int reserved[62];              /* [0]: != 0 after a decode step = an internal wait of ar_step_kernel timed out;
                                    [1]: block ticket of ttb_ar_sample (0 between launches) */
} TtbArState;

/* emb[b] = mel_embedding[tok[b]] + mel_pos_embedding[pos(step)] (autoregressive.py:145-149). pos_mode 0 =
 * train-consistent (j), 1 = reference kv-cache rule (j+1). tokens = codes[b, step-1]. */
int ttb_ar_embed_step(const int* codes, int ld_codes, const TtbArState* state, const float* mel_emb,
                      const float* mel_pos, int B, int D, int pos_mode, float* x, void* stream);
/* One-query attention over [shared prefix | candidate KV] for every (candidate, head); appends the new K/V.
 * prefix_k/v: bf16 [H, P, 64]; cand_k/v: bf16 [B, H, Nmax, 64]; qkv bf16 [B, 3*H*64]. */
int ttb_ar_decode_attention(const void* qkv, const void* prefix_k, const void* prefix_v, void* cand_k, void* cand_v,
                            const TtbArState* state, int B, int H, int P, int Nmax, void* out, float* scratch_o,
                            float* scratch_lse, void* stream);   /* scratch: fp32 [2, B, H*64] and [2, B, H] */
/* copy K/V of the prompt from a qkv buffer [P, 3*H*64] into the prefix cache [H, P, 64] */
int ttb_ar_store_prefix(const void* qkv, int P, int H, void* prefix_k, void* prefix_v, void* stream);
/* HF sample() step, fused: repetition penalty over the ids seen (incl. fake prompt ids 1 and 8192), temperature,
 * top-k, top-p, softmax, inverse-CDF draw with the supplied uniform, stop-token bookkeeping
 * (in-tree copy of HF 4.31: models/stream_generator.py:943-1000). logits fp32 [B or 1, V] (ld_logits = 0
 * broadcasts row 0); uniforms [B, ld_u] indexed by state->step; seen: bitmask [B, ceil(V/32)];
 * codes int32 [B, ld_codes]; finished int32 [B]. Advances state->step when `advance` != 0. */
int ttb_ar_sample(const float* logits, int ld_logits, int V, int B, const float* uniforms, int ld_u, uint32_t* seen,
                  int* codes, int ld_codes, int* finished, TtbArState* state, float temperature, int top_k, float top_p,
                  float rep_penalty, int stop_token, int advance, void* stream);
/* ttb_ar_sample with the reference's TypicalLogitsWarper(mass=typical_mass) (utils/typical_sampling.py:11-33) between
 * the repetition penalty and the temperature: only the typical set T of the penalised scores can be drawn (top-k keeps
 * min(top_k, |T|) tokens). typical_mass in (0, 1], else -1. Where the cumulative mass never reaches typical_mass
 * (mass 1 under rounding) every token is kept; the reference raises an IndexError there. */
int ttb_ar_sample_typical(const float* logits, int ld_logits, int V, int B, const float* uniforms, int ld_u,
                          uint32_t* seen, int* codes, int ld_codes, int* finished, TtbArState* state, float temperature,
                          int top_k, float top_p, float rep_penalty, int stop_token, int advance, float typical_mass,
                          void* stream);
/* fix_autoregressive_output (api.py:87-114) for every row + calm-token trim length (api.py:547-556) */
int ttb_ar_fix_codes(int* codes, int B, int L, int stop_token, int* trim_len, void* stream);
/* rows of an embedding table + optional positional table -> fp32 [n, D]; ids int32, pos int32 (or NULL) */
int ttb_embed(const int* ids, const int* pos, int n, int D, const float* table, const float* pos_table, float* out,
              void* stream);

/* ---- whole decode step as ONE persistent kernel (csrc/ar_step.cu) ----
 * GPT2InferenceModel.forward for one new token of every candidate (models/autoregressive.py:108-186 + the HF GPT2Block
 * stack + final_norm + mel_head): embed -> L x {ln_1, c_attn, attention over [shared prompt | own KV] with KV append,
 * c_proj, ln_2, c_fc + gelu_new, mlp.c_proj} -> ln_f -> final_norm -> mel_head, written to `logits`. The sampler
 * (ttb_ar_sample) consumes `logits` as before. KV layout differs from ttb_ar_decode_attention: K and V of a position are
 * adjacent, prefix_kv bf16 [L][H][P][2][64] (ttb_ar_step_store_prefix), cand_kv bf16 [L][B][H][Nmax][2][64]. */
typedef struct TtbArStepLayer {      /* device pointers of one GPT-2 block; weights bf16 K-major [out, in] */
  const void *wqkv, *wproj, *wfc, *wproj2;
  const float *ln1_g, *ln1_b, *bqkv, *bproj, *ln2_g, *ln2_b, *bfc, *bproj2;
} TtbArStepLayer;
typedef struct TtbArStepArgs {
  int B, D, H, L, V, P, Nmax, pos_mode;    /* candidates (<= 256), width (= 64 H, <= 1024), heads, layers, vocab, prompt
                                              positions (<= 352), KV slots per candidate, position rule (ttb_ar_embed_step) */
  const TtbArStepLayer* layers;            /* HOST array [L]; read by ttb_ar_step_setup only */
  const void* w_head; const float* b_head; /* mel_head bf16 [V, D], fp32 [V] */
  const float *lnf_g, *lnf_b, *fn_g, *fn_b;
  const float *mel_emb, *mel_pos;          /* fp32 tables */
  const int* codes; int ld_codes;          /* sampled tokens [B, ld_codes]; the token fed is codes[b, step-1] */
  TtbArState* state;                       /* state->reserved[0] != 0 after a launch = internal time-out (protocol error) */
  float* x;                                /* fp32 [B, D] residual stream (workspace) */
  void *a, *qkv, *o, *h, *hn;              /* bf16 workspaces [B, D], [B, 3D], [B, D], [B, 4D], [B, D] */
  float* part;                             /* fp32 split-K scratch, ttb_ar_step_workspace() floats */
  float* logits;                           /* fp32 [B, V] */
  const void* prefix_kv; void* cand_kv;
  void* tables;                            /* device, ttb_ar_step_workspace() bytes; filled by ttb_ar_step_setup */
  void* sync;                              /* device, ttb_ar_step_workspace() bytes; zeroed by ttb_ar_step_setup */
  int debug_layer_begin, debug_layer_end;  /* debug_layer_end > 0: run layers [begin, end) only */
  int debug_phase_mask;                    /* != 0: subset of phases (bit 0 embed+ln_1, 1 c_attn, 2 attention, 3 c_proj, 4 ln_2,
                                              5 c_fc, 6 mlp.c_proj, 7 next ln_1 / final norms, 8 mel_head) - tests and probes */
  int attn_compact;                        /* 1: the attention-only launch (debug_phase_mask = 4, one layer) runs in 8-warp CTAs
                                              whose shared memory is sized to the prompt (~118 KB at P = 174), so that CTAs of
                                              another stream fit beside them (two decode chains); same results */
} TtbArStepArgs;
int ttb_ar_step_workspace(const TtbArStepArgs* args, long long* part_floats, long long* table_bytes, long long* sync_bytes);
int ttb_ar_step_setup(const TtbArStepArgs* args, void* stream);      /* synchronous; once per (weights, workspace, B) */
int ttb_ar_decode_step(const TtbArStepArgs* args, void* stream);     /* one launch; CUDA-graph capturable */
int ttb_ar_step_store_prefix(const void* qkv, int P, int H, void* prefix_kv, void* stream);

/* ---------------------------------------------------------------- CLVP */
/* rotary (dim 32) on the first 32 dims of every head of q, k AND v (xtransformers.py:625-629,264-286);
 * qkv bf16 [nseq*T, 3*H*64] in place. */
int ttb_clvp_rotary(void* qkv, int nseq, int T, int H, void* stream);
/* LayerNorm + mean over the sequence (xtransformers.py:1234, clvp.py:15-17,123-124): x fp32 [nseq*T, D] -> [nseq, D] */
int ttb_clvp_pool(const float* x, int nseq, int T, int D, const float* g, const float* b, float* out, void* stream);
/* latent = normalize(pooled @ W^T) ; score[b] = <latent[b], text_latent> * exp(temperature) (clvp.py:126-135).
 * If text_latent == NULL only the normalised latents are written. */
int ttb_clvp_project(const float* pooled, int n, int D, const float* W, float* latents, const float* text_latent,
                     float temp_exp, float* scores, void* stream);

/* ---------------------------------------------------------------- diffusion */
/* timestep_embedding(t, C) (diffusion_decoder.py:21-39) for n timesteps -> fp32 [n, C] */
int ttb_timestep_embedding(const int* t, int n, int C, float* out, void* stream);
/* y[m, :] = act_in(x[m, :]) @ W^T + b for small M (emb layers / time_embed); fp32 SIMT */
int ttb_linear_small(const float* x, int M, int K, const float* W, const float* b, int N, int silu_in, int silu_out,
                     float* out, void* stream);
/* nearest-neighbour upsample along tokens (F.interpolate(mode='nearest'), diffusion_decoder.py:249) fused with the
 * conditioning scale/shift: out[s, c] = x[floor(s*N/S), c] ; x fp32 [N, C] -> bf16/fp32 [S, ld] */
int ttb_interp_nearest(const float* x, int N, int S, int C, void* out_bf16, int ldo, float* out_f32, int ldof, void* stream);
typedef struct TtbDiffStepArgs {
  const float* model_out;   /* fp32 [nb, S, ld_out]: batch 0 = conditional (eps | var), batch 1 = unconditional */
  long long out_bstride; int ld_out;
  float* x;                 /* fp32 [S, C] current sample, updated in place */
  void* x_bf16; int ld_xb;  /* bf16 copy [S, ld_xb] (zero-padded channels) for the next inp_block conv, or NULL */
  const float* noise;       /* fp32 [iters, S, C] pre-drawn, indexed by call order */
  const float* tables;      /* fp32 [6, iters]: sqrt_recip_ac, sqrt_recipm1_ac, post_logvar_clipped, log_betas, coef1, coef2 */
  const int* step;          /* device counter: call index (0 .. iters-1); spaced index i = iters-1-call */
  int S, C, iters;
  int cond_free; float cond_free_k;
  float* mel_out;           /* optional fp32 [C, S] channel-major denormalised mel written when i == 0 */
  long long parity_stride;  /* != 0: model_out is the double-buffered exchange area of ttb_pair_exchange; this call reads
                               model_out + (call & 1) * parity_stride */
} TtbDiffStepArgs;
/* p_mean_variance + p_sample epilogue (utils/diffusion.py:340-418,487-531): CFG mix with linear ramp,
 * learned-range variance, eps->x0 clamp, posterior mean, ancestral noise; denormalize_tacotron_mel on the
 * last step (utils/audio.py:63-64). */
int ttb_diffusion_step(const TtbDiffStepArgs* args, void* stream);
/* CFG branch pair on two GPUs (no reference counterpart: the reference runs both branches on one device,
 * utils/diffusion.py:340-342): copies this rank's branch output `src` (n floats) into slot (call & 1, branch_off) of the
 * local AND the partner's exchange area (peer memory mapped through CUDA IPC), publishes epoch + call + 1 in the
 * partner's flag word of that parity and waits for the partner's. One launch, CUDA-graph capturable. *err is set to 1
 * if the partner does not answer within 5 s. */
int ttb_pair_exchange(const float* src, float* local_area, float* peer_area, long long n, long long parity_stride,
                      long long branch_off, int* peer_flags, int* my_flags, const int* counter, const int* epoch,
                      unsigned int* done_ctr, int* err, void* stream);
int ttb_enable_peer_access(int peer_device);
/* exchange buffers for ttb_pair_exchange: own cudaMalloc allocation + its 64-byte CUDA-IPC handle; the partner process maps
 * it with ttb_peer_open (call with ITS device current: peer access is enabled for the mapping) */
int ttb_peer_alloc(long long bytes, void** ptr, void* handle64);
int ttb_peer_open(const void* handle64, void** ptr);
int ttb_peer_close(void* ptr);
int ttb_peer_free(void* ptr);
/* ---------------------------------------------------------------- HiFiGAN decoder of the api_fast path (token-major) */
/* v = leaky_relu((a + b + c) * scale, slope) for fp32 [R, C] inputs (b, c may be NULL; slope 1 = identity) written as the
 * error-compensated bf16 triple [hi | lo | hi] (3C columns, zero-filled up to ldo) that a GEMM contracts with weights
 * packed [Wh | Wh | Wl]: fp32-grade products from bf16 tensor-core operands (as ttb_voc_to_tokens_bf16 split != 0).
 * Serves F.leaky_relu before every HiFiGAN convolution and the mean over the three ResBlocks
 * (hifigan_decoder.py:92-95,254-265). */
int ttb_act_split_cast(const float* a, const float* b, const float* c, float scale, float slope, int R, int C, void* out,
                       int ldo, void* stream);
/* F.interpolate(mode='linear', align_corners=False, scale_factor=1/rscale) along tokens: x fp32 [N, C] -> [S, C]
 * (hifigan_decoder.py:283-292). src = (s + 0.5) * rscale - 0.5 clamped at 0, neighbours clamped at N - 1. */
int ttb_interp_linear(const float* x, int N, int C, float rscale, int S, float* out, void* stream);
/* misc small device helpers */
int ttb_counter_add(int* counter, int delta, void* stream);
int ttb_transpose_f32(const float* in, int R, int Cc, float* out, void* stream);           /* [R, C] -> [C, R] */
/* fp32 [R, Cc] (row stride ld_in) -> bf16 [R, ncols_out] (row stride ldo), columns >= Cc zero-filled */
int ttb_cast_pad_bf16(const float* in, int R, int Cc, int ld_in, void* out, int ldo, int ncols_out, void* stream);
int ttb_broadcast_rows(const float* row, int R, int Cc, float* out_f32, void* out_bf16, int ldo, void* stream);

/* ---------------------------------------------------------------- conditioning front-end (get_conditioning_latents) */
/* torchaudio.functional.resample (api.py:284): polyphase FIR. kernels fp32 [up, klen] built on the host
 * (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99); out[i*up + j] = sum_k xpad[i*down + k] * kernels[j][k],
 * xpad = x preceded by `width` zeros. m = number of output samples wanted. */
int ttb_audio_resample(const float* x, int n, const float* kernels, int down, int up, int klen, int width, float* out,
                       int m, void* stream);
/* STFT (center = True, reflect padding, hop) -> |.|^power -> mel filterbank -> log(max(., floor)) [/ div[c]].
 * power 2 + div = mel_norms: TorchMelSpectrogram (arch_util.py:295-331); power 1 + clip: TacotronSTFT.mel_spectrogram
 * (utils/audio.py:177-191, utils/stft.py:133-157). window fp32 [n_fft], twiddle fp32 [n_fft][2] = (cos, sin)(2 pi i / n_fft),
 * fb fp32 [n_mels, n_fft/2+1]. Frames = 1 + n / hop. out_bf16 token-major [frames, ldo] (columns >= n_mels zeroed),
 * out_f32 channel-major [n_mels, frames]; either may be NULL. */
int ttb_audio_stft_mel(const float* x, int n, int n_fft, int hop, const float* window, const float* twiddle,
                       const float* fb, int n_mels, int power, int clip, float floor_v, const float* div, void* out_bf16,
                       int ldo, float* out_f32, void* stream);
/* out[c] = (accumulate ? out[c] : 0) + scale * sum_r x[r*ld + c]  (means over positions / clips, autoregressive.py:451,
 * diffusion_decoder.py:228-229) */
int ttb_mean_rows(const float* x, int R, int C, int ld, float scale, int accumulate, float* out, void* stream);
/* one row: out = leaky_relu(x @ (W*wscale)^T + b*bscale, slope) * gain  (EqualLinear / nn.Linear of RandomLatentConverter,
 * random_latent_generator.py:21-50) */
int ttb_equal_linear(const float* x, int K, const float* W, const float* b, int N, float wscale, float bscale, float slope,
                     float gain, float* out, void* stream);

/* ---------------------------------------------------------------- UnivNet vocoder (channel-major fp32 [C, L]) */
/* Conv1d, small channel counts, zero or reflect padding, optional LeakyReLU on input/output, optional residual add
 * (vocoder.py:40-64 KernelPredictor convs, 146-153 dilated conv, 245-265 conv_pre/conv_post). tanh_out for conv_post. */
int ttb_voc_conv1d(const float* x, int Cin, int L, const float* w, const float* b, int Cout, int ksize, int dilation,
                   int reflect, float lrelu_in, float lrelu_out, int tanh_out, const float* residual, float* out,
                   void* stream);
/* LeakyReLU + ConvTranspose1d(k = 2*stride, stride, padding = stride/2 + stride%2, output_padding = stride%2)
 * (vocoder.py:138-142). w: [Cin, Cout, 2*stride]. x [C, L] -> [C, L*stride] */
int ttb_voc_convt(const float* x, int C, int L, const float* w, const float* b, int stride, float lrelu_in, float* out,
                  void* stream);
/* location-variable convolution + gated activation, fused (vocoder.py:169-178,182-216):
 *   o[oc, f*hop+s] = sum_{i,k} ypad[i, f*hop+s+k] * K[f][i][k][oc] + Bias[f][oc];  x += sigmoid(o[:C]) * tanh(o[C:])
 * y [C, L] (L = F*hop); kernels fp32 [F, ldk] with this layer's block at column koff laid out [i][k][oc];
 * bias fp32 [F, ldb] at column boff laid out [oc]. */
int ttb_voc_lvc_gate(const float* y, int C, int L, int hop, const float* kernels, int ldk, int koff, const float* bias,
                     int ldb, int boff, float* x, void* stream);
/* channel-major fp32 [C, L] -> token-major bf16 [L, ldo] (feeds the kernel-predictor GEMM). split != 0 writes the
 * error-compensated triple [hi | lo | hi] (ldo >= 3C) to be contracted with weights packed as [Wh | Wh | Wl]. */
int ttb_voc_to_tokens_bf16(const float* x, int C, int L, void* out, int ldo, int split, void* stream);

/* ---------------------------------------------------------------- wav2vec2 CTC aligner (prompt redaction) */
/* Wav2Vec2ForCTC forward of Wav2VecAlignment.align (utils/wav2vec_alignment.py:58-70); the projections, strided convs,
 * grouped positional conv (TTB_ACT_GELU_ERF epilogue), encoder LayerNorms and attention run on ttb_gemm, ttb_layernorm
 * and ttb_attention. */
/* clip_norm = (x - mean) / sqrt(var + 1e-7) over the whole 16 kHz clip, var unbiased (wav2vec_alignment.py:65),
 * deterministic (no atomics), fused with feature-extractor conv layer 0 (Conv1d(1, C, 10, stride 5) + bias), LayerNorm
 * over the C channels (eps 1e-5) and exact GELU (HF Wav2Vec2LayerNormConvLayer). x fp32 [n]; w fp32 [C, 10]; b, g, beta
 * fp32 [C]; C a multiple of 32, <= 512. stats: device scratch of 2 floats (mean, sqrt(var + 1e-7) are left there).
 * Writes bf16 token-major [(n - 10) / 5 + 1, ldo]. */
int ttb_wav2vec_conv0(const float* x, int n, const float* w, const float* b, const float* g, const float* beta, int C,
                      float* stats, void* out_bf16, int ldo, void* stream);
/* y = LN(x) * g + b (eps 1e-5), then exact GELU if gelu != 0, over fp32 rows x [M, D] (D a multiple of 128, <= 1024);
 * writes bf16 and/or fp32 [M, D]. The LayerNorm + GELU after feature-extractor conv layers 1-6
 * (HF Wav2Vec2LayerNormConvLayer). */
int ttb_layernorm_act(const float* x, int M, int D, const float* g, const float* b, int gelu, void* out_bf16,
                      float* out_f32, void* stream);
/* out[t] = argmax_j x[t, j] over fp32 [T, V] (logits.argmax(-1), wav2vec_alignment.py:70,97): the first index on ties and
 * NaN above every number, as torch.argmax. out int32 [T]. */
int ttb_argmax_rows(const float* x, int T, int V, int* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif

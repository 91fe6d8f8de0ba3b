/*
 * satb200 - C ABI of the GPU-native (H100, sm_90a) Stable Audio denoising hot path.
 *
 * The reference (yukara-ikemiya/friendly-stable-audio-tools) is pure Python/PyTorch and has
 * no FFI of its own; the boundary it offers for this path is a Python object contract
 * (SURVEY.md 8b).  These entry points are what the drop-in Python modules bind through
 * ctypes (INTEGRATION.md shows the stub) and each one names the reference interface it
 * replaces.  Conventions:
 *   - every pointer argument documented as "device" is a CUDA device pointer in
 *     caller-owned storage (e.g. torch.Tensor.data_ptr()); fp32 unless stated;
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream); all work is
 *     enqueued asynchronously on it;
 *   - return value: 0 = ok, negative = error (message: satb_last_error());
 *   - handles are not re-entrant; use one handle per (device, model).
 */
#ifndef SATB200_H_
#define SATB200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define SATB_ABI_VERSION 3

typedef struct SatbDit SatbDit;
typedef struct SatbOobleck SatbOobleck;
typedef struct SatbPqmf SatbPqmf;

/* Mirrors the constructor kwargs of DiffusionTransformer
 * (reference stable_audio_tools/models/dit.py:15-30) for the continuous_transformer backbone. */
typedef struct SatbDitConfig {
  int io_channels;
  int embed_dim;
  int depth;
  int num_heads;
  int cond_token_dim;       /* 0 = no cross-attention */
  int global_cond_dim;      /* 0 = no global conditioning */
  int project_cond_tokens;  /* dit.py:54 */
  int project_global_cond;  /* dit.py:65 */
  int global_cond_type;     /* 0 = "prepend", 1 = "adaLN" (dit.py:29,185-204) */
  int patch_size;           /* must be 1 */
  int operand_dtype;        /* 0 = fp16 (the reference's autocast dtype), 1 = bf16, 2 = fp8: e4m3 operands with
                               power-of-two row scales for the self-attention QKV, cross-attention q and feed-forward
                               input GEMMs, fp16 everywhere else; any other value is refused */
  int qk_norm;              /* 1 = L2-normalise q and k per head before RoPE / attention
                               (attn_kwargs.qk_norm, models/transformer.py:298,433-436) */
  int input_concat_dim;     /* extra input channels concatenated to x before the 1x1 pre-conv (dit.py:38,163-168); the
                               caller passes x with io_channels + input_concat_dim channels */
  int prepend_cond_dim;     /* width of the prepend conditioning tokens (dit.py:75-81), 0 = none */
} SatbDitConfig;

/* Mirrors OobleckEncoder/OobleckDecoder kwargs (models/autoencoders.py:119-194). */
#define SATB_MAX_STAGES 8
typedef struct SatbOobleckConfig {
  int in_channels;          /* encoder input / decoder output channels: 1 or 2 (audio), or a multiple of 8 up to 128
                               (the channels * num_bands sub-bands of a PQMF pretransform) */
  int channels;
  int latent_dim;           /* decoder input channels / encoder output channels */
  int n_stages;             /* len(c_mults) == len(strides) */
  int c_mults[SATB_MAX_STAGES];
  int strides[SATB_MAX_STAGES];
  int final_tanh;           /* decoder only */
  int is_decoder;           /* 1 = OobleckDecoder, 0 = OobleckEncoder */
  int operand_dtype;        /* 0 = fp16, 1 = bf16 (conv operands; accumulation is fp32), 2 = fp16 split hi + lo:
                             * three MMAs per product, ~fp32 accuracy (the reference's own precision for this path) */
} SatbOobleckConfig;

/* ---- library ---------------------------------------------------------------------- */
const char* satb_last_error(void);
int satb_abi_version(void);
unsigned long long satb_launch_count(void);   /* kernels launched by this library so far */
void satb_reset_launch_count(void);
/* Replaying a captured CUDA graph launches kernels this library cannot count: the caller adds the number recorded
 * while the graph was captured. */
void satb_add_launch_count(unsigned long long n);

/* ---- DiT: replaces DiffusionTransformer (models/dit.py:14-364) + ContinuousTransformer
 *      (models/transformer.py:705-809) behind DiTWrapper.forward (models/diffusion.py:491-529) */
int satb_dit_create(const SatbDitConfig* cfg, SatbDit** out);
void satb_dit_destroy(SatbDit* h);
/* conformer=True models (ContinuousTransformer / TransformerBlock kwarg, models/transformer.py:557-591,645,680-681,
 * 697-698): enable != 0 adds the conformer branch x += conformer(x) between cross-attention and the feed-forward of
 * every block.  Call after satb_dit_create and before the first satb_dit_load_weight; embed_dim <= 1536.  finalize then
 * requires the nine "transformer.layers.{i}.conformer.*" tensors of every layer.  Its GEMMs take 16-bit operands in
 * every operand_dtype (fp16 in the fp8 mode).  A handle that never calls this runs the model without the branch. */
int satb_dit_set_conformer(SatbDit* h, int enable);
/* Feed-forward options (FeedForward kwargs via ff_kwargs, models/transformer.py:238-287,643): inner_dim = int(dim *
 * mult); glu 1 = SwiGLU (FF-in "ff.ff.0.proj" Linear(dim, 2 inner), always biased), 0 = "ff.ff.0.1" then SiLU;
 * conv_kernel_size 0 = Linear layers, else use_conv with that odd kernel size and padding k / 2: FF-out "ff.ff.2" becomes
 * Conv1d(inner, dim, k) over the tokens, and so does a non-GLU FF-in (Conv1d(dim, inner, k)); the GLU projection stays
 * a Linear.  bias 0 = no_bias (FF-out and a non-GLU FF-in lose their bias).  A convolution runs over each item's
 * tokens (prepended ones included), zero-padded at the item's ends, every CFG row its own item; it takes 16-bit
 * operands in every operand_dtype (fp16 in the fp8 mode, whose e4m3 FF-in is the Linear one).  The inner width is
 * padded with zeros to a multiple of 64 at load time (exact).  Call after satb_dit_create and before the first
 * satb_dit_load_weight; bad values (inner_dim < 1, an even or negative kernel size) and late calls are refused.
 * finalize then requires the variant's keys and names the missing ones.  The default is (4 * embed_dim, 1, 0, 1): a
 * handle that never calls this runs the default feed-forward. */
int satb_dit_set_feedforward(SatbDit* h, int inner_dim, int glu, int conv_kernel_size, int bias);
/* Positional options (ContinuousTransformer kwargs, models/transformer.py:50-96,737-785): rotary 1 = rotary_pos_emb
 * (the "transformer.rotary_pos_emb.inv_freq" key), 0 = no RoPE (no inv_freq key; q and k are not rotated).  pos_type
 * 0 = none, 1 = use_sinusoidal_emb (ScaledSinusoidalEmbedding: keys "transformer.pos_emb.scale" [1] and, since the
 * reference keeps it out of the state dict, its inv_freq buffer [embed_dim / 2] under "transformer.pos_emb.inv_freq"),
 * 2 = use_abs_pos_emb (AbsolutePositionalEmbedding: "transformer.pos_emb.emb.weight" [abs_max_len, embed_dim]).
 * abs_max_len: abs_pos_emb_max_length with pos_type 2, else 0.  The embedding is added to every row after the prepend
 * concat: positions count the prepended tokens (global-conditioning and prepend-conditioning ones) and, with patching,
 * patched tokens.  Forwards whose latent + prepended tokens exceed abs_max_len are refused.  Call after
 * satb_dit_create and before the first satb_dit_load_weight; bad values and late calls are refused.  finalize then
 * requires the variant's keys and names the missing ones.  The default is (1, 0, 0): a handle that never calls this
 * runs rotary positions only. */
int satb_dit_set_positions(SatbDit* h, int rotary, int pos_type, int abs_max_len);
/* FP8 self-attention (DiffusionTransformer attention_dtype "fp8"; DESIGN.md section 5): enable 1 runs every block's
 * self-attention on e4m3 q, k, v and probabilities (power-of-two scales per (token, head) for q and k, per (item, head,
 * channel) for v), with an fp32 accumulator and the 16-bit output of the operand mode; cross-attention stays 16-bit.
 * Head dim 64 only; works with every operand_dtype.  Call before satb_dit_finalize; a later call, another head dim
 * with enable 1, and an enable other than 0 or 1 are refused.  Default 0. */
int satb_dit_set_attention_fp8(SatbDit* h, int enable);
/* FP8 FF-out (DiffusionTransformer ff_out_dtype "fp8"; DESIGN.md sections 3-5): enable 1 runs every block's FF-out GEMM
 * on e4m3 operands.  FF-in's epilogue then stores the SwiGLU (or plain SiLU) output as e4m3 with one power-of-two scale
 * per (row, 128 columns) instead of 16 bits, and ff.ff.2.weight is kept only as an e4m3 copy with one scale per row;
 * each 128-wide k-block's partial product is scaled by its activation block scale before it is accumulated.  Needs
 * operand_dtype 2 (fp8), a Linear feed-forward (no conv_kernel_size) and an inner width that, padded to a multiple of 64,
 * is a multiple of 128.  Call after satb_dit_set_feedforward and before the first satb_dit_load_weight (the option
 * decides how ff.ff.2.weight is stored), so before satb_dit_finalize; a later call, a null handle, an enable other than
 * 0 or 1, and enable 1 on any other model are refused before any CUDA call.  Default 0. */
int satb_dit_set_ff_out_fp8(SatbDit* h, int enable);
/* One state-dict entry (key relative to DiffusionTransformer, e.g.
 * "transformer.layers.0.self_attn.to_qkv.weight"); src: device fp32, contiguous.
 * Replaces nn.Module.load_state_dict for this module (models/pretrained.py:24). */
int satb_dit_load_weight(SatbDit* h, const char* name, const float* src, long long numel, void* stream);
int satb_dit_finalize(SatbDit* h, void* stream);
/* Pre-allocate activations for `rows` transformer rows (2*B under CFG) of L latent tokens. */
int satb_dit_reserve(SatbDit* h, int rows, int L);
/* Step-invariant conditioning (dit.py:149-154 to_cond_embed / to_global_embed, and every
 * layer's cross-attention to_kv, transformer.py:425): cross [B, Mctx, cond_token_dim],
 * neg_cross (same shape, or NULL), global [B, global_cond_dim] (or NULL); device fp32. */
/* Prepend conditioning for the NEXT satb_dit_prepare_cond (dit.py:157-161,185-195,309-311): prepend [B, n_tokens,
 * prepend_cond_dim] device fp32 (NULL / 0 tokens = none).  Its to_prepend_embed tokens go in front of the
 * global-conditioning token; the unconditional CFG rows get zeros.  "prepend" global_cond_type only. */
int satb_dit_set_prepend_cond(SatbDit* h, const float* prepend, int B, int n_tokens, void* stream);
int satb_dit_prepare_cond(SatbDit* h, const float* cross, const float* neg_cross, const float* global, int B,
                          int Mctx, int use_cfg, void* stream);
/* One denoiser call = DiffusionTransformer.forward (dit.py:228-364): x [B, C, L], t [B] ->
 * out [B, C, L]; CFG combine and rescale (dit.py:338-347) included when use_cfg was set. */
int satb_dit_forward(SatbDit* h, const float* x, const float* t, float* out, int B, int L, float cfg_scale,
                     float scale_phi, void* stream);
/* Same, additionally copying the residual stream after the last block
 * ([rows * (L + prepend), embed_dim]; = info["hidden_states"][-1], transformer.py:804-805). */
int satb_dit_forward_debug(SatbDit* h, const float* x, const float* t, float* out, float* hidden, int B, int L,
                           float cfg_scale, float scale_phi, void* stream);

/* ---- Token-sharded (context-parallel) DiT forward: one process drives `world` ranks (1 .. 8), each a finalized handle
 * with a full copy of the weights on its device; several ranks may share one device.  Rank r holds tokens
 * token_begin[r] .. token_begin[r + 1] - 1 of every item (positions after the prepend concat, N = n_prepend + L), the
 * n_prepend prepended tokens (the global-conditioning token and any prepend-conditioning tokens) on rank 0.  Once per
 * layer each rank gathers every rank's self-attention k / v into one full-sequence buffer and attends its own queries
 * against all of them; everything else runs per token on the rank's own rows. */
typedef struct SatbDitGroup SatbDitGroup;
/* The split, in token_begin[world + 1]: boundaries on multiples of 128 tokens when N >= 128 * world, as even as possible
 * otherwise; rank 0 holds at least the prepended tokens; no rank is empty.  world > N is refused.  Host only. */
int satb_dit_group_plan(int world, int n_prepend, int L, int* token_begin);
/* handles[world]: finalized handles of one model (identical configs and options, checked), one per rank, each its own;
 * devices[world]: their device ids.  Conformer blocks, use_conv feed-forwards and FP8 self-attention are refused with
 * -5.  Ranks on distinct devices need peer access between them (refused with a message when missing); it is enabled
 * for this process.  Each handle keeps its own conditioning: call satb_dit_set_prepend_cond / satb_dit_prepare_cond on
 * every handle, with the same conditioning, before satb_dit_group_forward.  The handles outlive the group, which must
 * be destroyed explicitly. */
int satb_dit_group_create(SatbDit* const* handles, const int* devices, int world, SatbDitGroup** out);
/* The CFG-split group: two rows of `world` ranks (1 .. 8 each), handles[2 world] and devices[2 world] holding row 0's
 * ranks, then row 1's.  A CFG call (the handles' conditioning prepared with use_cfg) runs its conditional rows on row
 * 0 and its unconditional rows on row 1, each row token-sharded over its own ranks by satb_dit_group_plan(world, ...),
 * so the two halves exchange nothing until the combine: row-0 rank j reads row-1 rank j's project_out output (same
 * tokens) through a peer pointer and writes the guided output; row 1 writes none.  Every rank keeps the conditioning
 * of the batched CFG forward and uses the rows of its half (cross-attention K / V, prepend tokens, adaLN rows), so each
 * half computes what the batched forward computes for those rows.  A call without CFG runs row 0 only, as the group of
 * satb_dit_group_create(row 0's handles) would.  Conformer blocks, use_conv feed-forwards and FP8 self-attention are
 * refused with -5 only when world > 1 (a row of one rank holds every token).  Peer access is needed, and enabled,
 * between every pair of distinct devices.  The group takes the same forward, graph, reset, stats and destroy calls as
 * a satb_dit_group_create group; its graph is captured again when any of the 2 world handles changes. */
int satb_dit_group_create_cfg(SatbDit* const* handles, const int* devices, int world, SatbDitGroup** out);
void satb_dit_group_destroy(SatbDitGroup* g);
/* One denoiser call over the ranks: x[r] [B, C, L_r] and out[r] [B, io_channels, L_r], rank r's latent tokens (L_r =
 * token_begin[r + 1] - token_begin[r], less n_prepend on rank 0), and t[r] [B], all on rank r's device; streams[r] is
 * rank r's stream.  Enqueues only (ranks are ordered with events); the caller's current device is restored.  On a
 * satb_dit_group_create_cfg group, x, t and streams hold 2 world entries (row 0's ranks, then row 1's; row 1's x and t
 * are read by CFG calls only and may be null otherwise) and out holds world entries, row 0's. */
int satb_dit_group_forward(SatbDitGroup* g, const float* const* x, const float* const* t, float* const* out, int B,
                           int L, float cfg_scale, float scale_phi, void* const* streams);
/* The same call replayed from one CUDA graph whose nodes live on every rank's device: one cudaGraphLaunch on
 * home_stream.  x [B, C, L], t [B] and out [B, io_channels, L] are whole tensors on rank 0's device, at addresses the
 * caller keeps fixed; rank_streams[r] (created streams, on rank r's device; 2 world of them for a CFG group) are used
 * while capturing.  The graph copies
 * each rank's slice of x and t in, runs the group forward and copies each rank's slice of out back.  The first call,
 * and every call after the key (x, t, out, B, L, cfg_scale, scale_phi) changed or after any handle's weights,
 * conditioning or workspaces may have moved (satb_dit_finalize, satb_dit_set_prepend_cond, satb_dit_prepare_cond, a
 * workspace reserve), runs one eager group forward at the shape and then captures and instantiates the graph.  Graph
 * launches and satb_dit_group_forward calls may alternate: the library orders them with events.  Refused while
 * profiling is on; a failed capture or instantiation returns the CUDA error with its message.  Each launch adds the
 * kernel launches it replays to satb_launch_count. */
int satb_dit_group_graph_forward(SatbDitGroup* g, const float* x, const float* t, float* out, int B, int L,
                                 float cfg_scale, float scale_phi, void* const* rank_streams, void* home_stream);
/* Drops the group's graph (satb_dit_group_destroy does too); the next graph call captures again. */
int satb_dit_group_graph_reset(SatbDitGroup* g);
/* Graphs captured and launched so far, and the kernel launches of the current graph (0: none). */
int satb_dit_group_graph_stats(const SatbDitGroup* g, long long* captures, long long* replays,
                               unsigned long long* launches);
/* The group forward's K/V gather on its own (tests and timing): kv [R, N, 2 D] 16-bit = the columns D .. 3 D - 1 of
 * every rank's qkv[s] [R, n_s, 3 D], rank s's rows at tokens token_begin[s] .. token_begin[s + 1] - 1 of each item
 * (N = token_begin[world], token_begin[0] = 0).  qkv[s] may be a peer device's pointer. */
int satb_kv_gather(const void* const* qkv, const int* token_begin, int world, void* kv, int R, int D, void* stream);

/* Per-kernel-class CUDA-event timing used by bench.py's roofline line: enable, run forwards,
 * then read ms[8]/count[8] (0 ff_in GEMM, 1 ff_out GEMM, 2 qkv GEMM, 3 self-attention core,
 * 4 attention out GEMM, 5 cross-attention, 6 LayerNorm, 7 conformer branch (conformer models only)). */
int satb_dit_profile(SatbDit* h, int enable);
int satb_dit_profile_read(SatbDit* h, float* ms, int* count);

/* ---- primitives exposed for the drop-in modules and the parity tests ---------------- */
/* SnakeBeta.forward (models/blocks.py:330-358): x, y [B, C, T]; alpha, beta [C]. */
int satb_snake_beta(const float* x, const float* alpha, const float* beta, float* y, int B, int C, long long T,
                    int logscale, void* stream);
/* LayerNorm.forward (models/transformer.py:188-206) with 16-bit output (fp16/bf16 bits). */
int satb_layernorm(const float* x, const float* gamma, const float* beta, void* out16, int rows, int D, int bf16,
                   void* stream);
/* Test entry point: the LayerNorm of the FP8 mode, out8 [rows, D] e4m3 and row_scale [rows] fp32 with
 * out8[r, :] = e4m3_rn(y[r, :] / row_scale[r]), row_scale[r] = 2^e, e the smallest integer (>= -126) with
 * max |y[r, :]| <= 448 * 2^e (1 for an all-zero row).  y = LayerNorm(x) (* (1 + mod_scale) + mod_shift when mod_scale is
 * given: adaLN, item = (r / rows_per_item) % n_items, row stride mod_stride; else mod_* are ignored). */
int satb_layernorm_fp8(const float* x, const float* gamma, const float* beta, const float* mod_scale,
                       const float* mod_shift, long long mod_stride, int rows_per_item, int n_items, void* out8,
                       float* row_scale, int rows, int D, void* stream);
/* C[M, N] (fp32) = A[M, K] * W[N, K]^T, A and W 16-bit (fp16/bf16 bits) row-major: nn.Linear
 * without bias (F.linear call sites transformer.py:422-430,548). */
int satb_linear_f32out(const void* a16, const void* w16, float* c, int M, int N, int K, int bf16, void* stream);
/* Test entry point (no product path calls it): C = A[M, K] * W[N, K]^T through ONE of the fused-epilogue GEMM
 * instances the DiT forward launches, chosen by `epi`, `bn` and `bf16`.  The instances: store32 BN 64 / 256;
 * store16, head_norm16 and residual BN 128 / 256; qkv_rope, swiglu and store32_pos BN 256; anything else returns an
 * error.  The
 * remaining fields are the epilogue's parameters (csrc/gemm.cuh); all pointers are device pointers, 16-byte aligned;
 * fields an epilogue does not use are ignored. */
#define SATB_EPI_STORE32 0      /* out fp32 = acc (+ bias) */
#define SATB_EPI_STORE16 1      /* out 16-bit = act(acc (+ bias)) */
#define SATB_EPI_HEAD_NORM16 2  /* 64-wide heads, L2-normalised below norm_cols, rotary (nf 16) below rope_cols */
#define SATB_EPI_QKV_ROPE 3     /* partial rotary of every head below rope_cols */
#define SATB_EPI_SWIGLU 4       /* out[:, N / 2] = value * silu(gate), 32 / 32 interleaved columns */
#define SATB_EPI_RESIDUAL 5     /* h += (acc (+ bias)) (* gate) */
/* 6 was the LayerNorm-fold residual epilogue, since removed: it is refused, and the number is not reused. */
#define SATB_EPI_STORE32_POS 7  /* out fp32 = acc (+ bias) + pos_tab[row % seq_len, :] (BN 256: DiT project_in with a
                                   positional embedding) */
/* e4m3 QKV epilogues of FP8 self-attention (satb_gemm_probe_qk8 only; the other probes refuse them): */
#define SATB_EPI_QKV_ROPE_E4M3 8   /* qkv_rope at head dim 64 (nf 16), q / k columns stored e4m3 (SatbQkE4m3), v 16-bit */
#define SATB_EPI_HEAD_NORM_E4M3 9  /* head_norm16 with norm_cols = 128 heads, q / k stored e4m3 (SatbQkE4m3), v 16-bit */
/* The GEMMs of the FP8 FF-out option (satb_gemm_probe_ff8 only; the other probes refuse them): */
#define SATB_EPI_SWIGLU_E4M3 13    /* swiglu, the N / 2 outputs stored as e4m3 blocks of 128 columns with their scales */
#define SATB_EPI_SILU_E4M3 14      /* silu(acc (+ bias)), stored as e4m3 blocks of 128 columns with their scales */
#define SATB_EPI_RESIDUAL_A8 15    /* residual, A e4m3 with one scale per (row, 128-wide k-block) */
typedef struct SatbGemmProbe {
  int epi, bn, bf16, b_static;      /* b_static 1: weight prefetch before the dependency wait, as the forward runs */
  void* out;                        /* store32 (fp32), store16, head_norm16, qkv_rope, swiglu (16-bit) */
  int ld;                           /* row pitch in elements of out, or of h */
  const float* bias;                /* [N] or NULL */
  int act;                          /* store16: 0 none, 1 SiLU */
  float* h;                         /* residual: fp32 [M, ld] updated in place */
  const float* gate;                /* residual: [*, gate_ld] or NULL; row item = (row / rows_per_item) % n_items */
  int rows_per_item, gate_ld, n_items;
  int rope_cols, seq_len, head_dim, nf;   /* rotary: position = row % seq_len; tables [seq_len, nf] */
  const float* cos_tab;
  const float* sin_tab;
  int norm_cols;                    /* head_norm16 */
  const float* pos_tab;             /* store32_pos: [seq_len, N] fp32 */
} SatbGemmProbe;
int satb_gemm_probe(const void* a16, const void* w16, int M, int N, int K, const SatbGemmProbe* p, void* stream);
/* Test entry point: the same through ONE of the FP8-mode instances of the DiT forward: a8 [M, K] and w8 [N, K] e4m3
 * with one fp32 scale per row (a_scale [M], w_scale [N]); C = (a_scale[m] w_scale[n] sum_k a8[m, k] w8[n, k]) through
 * the epilogue.  Instances: qkv_rope and swiglu BN 256, store16 BN 128 / 256, head_norm16 BN 128; bf16 must be 0
 * (fp16 outputs) and K a multiple of 128. */
int satb_gemm_probe_fp8(const void* a8, const void* w8, const float* a_scale, const float* w_scale, int M, int N, int K,
                        const SatbGemmProbe* p, void* stream);
/* Test entry point: the feed-forward's token convolution (satb_dit_set_feedforward with conv_kernel_size k), through
 * the GEMM launch the DiT forward makes:
 *   C[r * n_seq + l, n] = sum_t sum_c a16[r, l + t - k / 2, c] * w16[t * N + n, c]   (rows outside 0..n_seq-1: zero)
 * a16: 16-bit [R, item_stride, K] (item_stride >= n_seq rows; rows n_seq.. of an item are never read); w16: tap-major
 * [k * N, K]; C goes through p's epilogue: SATB_EPI_STORE16 (out [R * n_seq, ld], bias, act) or SATB_EPI_RESIDUAL (h,
 * bias, gate).  p->bn: 0 = the N tile the forward picks for this shape, or 128 / 256; p->bf16 selects the instance.
 * k odd, K % 8 == 0, N % 32 == 0; pointers 16-byte aligned. */
int satb_token_conv_probe(const void* a16, long long item_stride, const void* w16, int R, int n_seq, int K, int N, int k,
                          const SatbGemmProbe* p, void* stream);
/* Test entry point: the DiT forward's token-row kernel (the project_in GEMM's A operand).  x [B_src, C, L] fp32 ->
 * a16 [R * (P + L), lda] 16-bit (bf16 or fp16) with lda >= C, lda % 8 == 0: row r * (P + L) + P + l, column c holds
 * x[r % B_src, c, l]; the P leading rows of every item and the columns C .. lda-1 of every row are written as zeros. */
int satb_dit_pre_probe(const float* x, void* a16, int R, int B_src, int C, int lda, int L, int P, int bf16, void* stream);
/* Test entry points (no product path calls them): the DiT forward's small kernels, each through the launch function the
 * forward itself calls.  Every one checks its arguments before any CUDA call; device pointers are fp32 unless stated.
 *
 * satb_layernorm_mod: satb_layernorm with the adaLN modulation of satb_layernorm_fp8: out16[r, :] = 16-bit of
 * LayerNorm(x[r, :]) * (1 + mod_scale[item, :]) + mod_shift[item, :], item = (r / rows_per_item) % n_items, vector of
 * item i at mod_scale + i * mod_stride (mod_scale NULL: no modulation, mod_* ignored).  x, gamma, beta, mod_* 16-byte
 * aligned, out16 8-byte aligned; D a multiple of 128, <= 2048. */
int satb_layernorm_mod(const float* x, const float* gamma, const float* beta, const float* mod_scale,
                       const float* mod_shift, long long mod_stride, int rows_per_item, int n_items, void* out16,
                       int rows, int D, int bf16, void* stream);
/* Timestep features (models/blocks.py:95-97): t [B], w [F] -> out [B, 2 F] = [cos(2 pi t w) | sin(2 pi t w)]. */
int satb_fourier_probe(const float* t, const float* w, float* out, int B, int F, void* stream);
/* out[r, n] = act(sum_k in[r, k] W[n, k] (+ bias[n]) (+ add[r, n])), act = SiLU when silu_out: in [R, K], W [N, K] (both
 * 16-byte aligned), bias [N] / add [R, N] may be NULL.  1 <= R <= 4096, K a multiple of 4, 4 <= K <= 6400. */
int satb_skinny_linear_probe(const float* in, const float* W, const float* bias, const float* add, float* out, int R,
                             int K, int N, int silu_out, void* stream);
/* The prepended rows of the residual stream h [R, N_seq, D]: rows j < Pp of item r get pre[r, j, :] (r < B and pre given;
 * else zeros), row Pp gets tok[r % B, :]; pos [N_seq, D] (may be NULL) adds pos[j, :].  Rows past Pp are not written. */
int satb_write_prepend_probe(const float* tok, const float* pre, const float* pos, float* h, int R, int B, int N_seq,
                             int D, int Pp, void* stream);
/* ssg [rows, depth * 6 D], in place: g -> sigmoid(1 - g) on chunks 2 and 5 of every 6 D-wide layer block. */
int satb_gate_sigmoid_probe(float* ssg, int rows, int depth, int D, void* stream);
/* y [R * N_seq, ldy] (R = B, or 2 B with cfg: conditional rows first; only columns < C are read) -> out [B, C, L]:
 * the P leading rows of every item dropped, the CFG combine and std rescale of models/dit.py:338-347 when cfg != 0. */
int satb_dit_post_probe(const float* y, int ldy, float* out, int B, int C, int L, int N_seq, int P, int cfg,
                        float cfg_scale, float scale_phi, void* stream);
/* dst16[r, c] = 16-bit (fp16 / bf16, round to nearest even) of src[perm ? perm[r] : r, c], c < cols, at row pitches
 * src_ld / dst_ld (elements); perm: device int32 [rows] or NULL.  Any number of rows. */
int satb_cast_rows_probe(const float* src, void* dst16, const int* perm, int rows, int cols, long long src_ld,
                         long long dst_ld, int bf16, void* stream);
/* The FP8 mode's weight quantiser: dst8[r, :] = e4m3_rn(src[perm ? perm[r] : r, :] / row_scale[r]) with the row-scale
 * rule of satb_layernorm_fp8.  src [*, cols] 16-byte aligned, dst8 4-byte aligned, cols a multiple of 4. */
int satb_quant_rows_fp8_probe(const float* src, void* dst8, float* row_scale, const int* perm, int rows, int cols,
                              void* stream);
/* C [M, N] = A [M, K] B [K, N], fp32 row-major, float64 products and sums (the conformer weight fold). */
int satb_matmul_f64_probe(const float* A, const float* B, float* C, int M, int N, int K, void* stream);
/* One step of the v-objective k-diffusion samplers in a single pass over the latents (replaces the
 * ~20 elementwise torch kernels of K.external.VDenoiser.forward + sample_dpmpp_{2m,3m}_sde's update,
 * reference call sites inference/sampling.py:159,225-228): with v = model(x * c_in, t),
 *   den = c_out v + c_skip x;  x_next = a x + b den + c den_1 + d den_2 + s noise;  x_in_next = x_next * c_in_next.
 * den_1, den_2, noise, x_in_next may be NULL; all tensors fp32 with n elements (n % 4 == 0). */
int satb_sampler_update(const float* x, const float* v, const float* den_1, const float* den_2, const float* noise,
                        float* den, float* x_next, float* x_in_next, long long n, float c_skip, float c_out, float a,
                        float b, float c, float d, float s, float c_in_next, void* stream);
/* One step of the v-diffusion DDIM sampler (reference inference/sampling.py:64-118) in a single pass, with the
 * reference's fp32 rounding (every product and sum rounded on its own, in its order):
 *   pred = x alpha - v sigma;  eps = x sigma + v alpha;  x_next = pred alpha_next + eps adj_sigma + noise ddim_sigma.
 * noise may be NULL (no noise term); x_next and pred may each be NULL (the last step writes pred only), not both.
 * All tensors fp32 with n >= 1 elements; outputs must not overlap the inputs. */
int satb_vdiffusion_update(const float* x, const float* v, const float* noise, float* x_next, float* pred, long long n,
                           float alpha, float sigma, float alpha_next, float adj_sigma, float ddim_sigma, void* stream);
/* One model call's worth of sampler arithmetic for every fixed-step sampler of inference/sampling.py (Euler for
 * rectified flow, Heun, DPM-2, linear multistep, DPM-Solver++(2S) ancestral, and the multistep SDE samplers with a
 * callback or inpainting) in a single pass over the latents.  Each of them is linear in x (the state the model was
 * called at), y (the model output), a few stored tensors and the noise, so one kernel serves all of them with
 * host-computed scalars:
 *   den    = c_out y + c_skip x                                     (VDenoiser.forward; c_out = 1, c_skip = 0 passes a
 *                                                                    den computed earlier through as y)
 *   x      = mask[l] <= blend_thr ? init + renoise * blend_sigma : x (the inpainting callback, written back into x;
 *                                                                    only when mask is given; l = index % L)
 *   d      = (x - den) * inv_sigma                                  (the Karras ODE derivative)
 *   x_next = a x + b den + g d + sum_k c[k] buf[k] + s noise;  x_in_next = x_next * c_in_next.
 * den, d, x_next and x_in_next are written when non-NULL (at least one must be); buf[k] is read when non-NULL, noise
 * when non-NULL.  All tensors fp32, n elements (n % 4 == 0), 16-byte aligned, no output overlapping an input; mask
 * is [L] fp32 and the blend rounds init + renoise * blend_sigma like the fp32 torch expression. */
#define SATB_SAMPLER_STEP_BUFS 4
typedef struct SatbSamplerStep {
  float* x;                                   /* read; written back only with a mask */
  const float* y;
  const float* buf[SATB_SAMPLER_STEP_BUFS];
  const float* noise;
  const float* mask;                          /* [L] */
  const float* init;
  const float* renoise;
  float* den;
  float* d;
  float* x_next;
  float* x_in_next;
  long long n;
  int L;
  float c_skip, c_out, inv_sigma, a, b, g, c[SATB_SAMPLER_STEP_BUFS], s, c_in_next, blend_sigma, blend_thr;
} SatbSamplerStep;
int satb_sampler_step(const SatbSamplerStep* p, void* stream);
/* softmax(q k^T / sqrt(64)) v (transformer.py:496-536): q [B, Nq, H*64], k/v [B, Nk, Hkv*64],
 * out [B, Nq, H*64]; 16-bit, contiguous. */
int satb_attention(const void* q16, const void* k16, const void* v16, void* o16, int B, int H, int Hkv, int Nq, int Nk,
                   int bf16, void* stream);
/* The same for any supported head dim d (32, 64, 96 or 128; transformer.py:290-352 takes dim_heads from the model):
 * softmax(q k^T / sqrt(d)) v with q [B, Nq, H*d], k/v [B, Nk, Hkv*d], out [B, Nq, H*d]; 16-bit, contiguous.
 * Head h uses kv head h / (H / Hkv).  head_dim 64 gives the bits of satb_attention. */
int satb_attention_hd(const void* q16, const void* k16, const void* v16, void* o16, int B, int H, int Hkv, int Nq,
                      int Nk, int head_dim, int bf16, void* stream);
/* Test entry point (no product path calls it): the same attention on strided operands, through the launch the DiT
 * forward makes (the fused [rows, N, 3 H d] QKV buffer of self-attention, the [rows, Mctx, 2 Hkv d] KV buffer of
 * cross-attention).  q / k / v / o are 16-bit [B, rows, ld*] with batch strides *_bs (elements); head h of q starts
 * at column q_col + h d, kv head h / (H / Hkv) of k and v at k_col + (h / (H / Hkv)) d, v_col + ...; o's head h at
 * column h d.  q_cols / k_cols / v_cols are the widths (from column 0) the operand holds: head dim 64 reads it through
 * a tensor map that spans exactly these columns and Nq / Nk rows per item.  Pointers, strides and column offsets
 * must be multiples of 16 bytes; strides and column offsets must not be negative. */
typedef struct SatbAttentionProbe {
  int B, H, Hkv, Nq, Nk, head_dim, bf16;
  const void* q;
  const void* k;
  const void* v;
  void* o;
  long long ldq, ldk, ldv, ldo;
  long long q_bs, k_bs, v_bs, o_bs;
  int q_cols, k_cols, v_cols;
  int q_col, k_col, v_col;
} SatbAttentionProbe;
int satb_attention_probe(const SatbAttentionProbe* p, void* stream);

/* Test entry points of the FP8 self-attention (satb_dit_set_attention_fp8), head dim 64, one kv head per head.
 * pad(n) = n rounded up to a multiple of 128; buffers device, 16-byte aligned (sv 8-byte).  Operand layouts:
 *   q8, k8 [B, N, H*64] e4m3 = e4m3_rn(x / s), s = 2^e per (token, head), e the smallest integer with amax <= 448 * 2^e,
 *   e >= -126, s = 1 for an all-zero head (x: the 16-bit values the QKV epilogue would store); sq, sk [B*H, pad(N)]
 *   those s at [item * H + head, token];
 *   vt8 [B*H, 64, pad(N)] e4m3 of v^T / sv per (item, head, channel) over the item's N tokens, same rule; within every
 *   32-key group, stored position j holds key 16 (j/16) + 8 ((j%4)/2) + 2 ((j/4)%4) + j%2; zero past N;  sv [B*H, 64].
 * satb_attention_fp8_vt: v16 [B, N, H*64] 16-bit -> vt8, sv.
 * satb_attention_fp8_core: o16 [B, Nq, H*64] = softmax((q8 sq)(k8 sk)^T / 8) (vt8^T sv) with P in e4m3 (see the
 *   header comment of csrc/attention_fp8.cu) on operands of that layout (q8 / sq with Nq rows, k8 / sk / vt8 with Nk).
 * satb_gemm_probe_qk8: the QKV GEMM with SATB_EPI_QKV_ROPE_E4M3 (bn 256) or SATB_EPI_HEAD_NORM_E4M3 (bn 256; 128 with
 *   FP8 operands) as the forward runs it: A [M, K], W [N, K] 16-bit (a_scale NULL) or e4m3 with row scales a_scale [M],
 *   w_scale [N] (fp16 out only); p gives out / ld (v columns >= 128 heads, 16-bit), bf16, b_static, rope_cols,
 *   seq_len, cos_tab / sin_tab ([seq_len, 16]); q columns [0, 64 heads) -> o->q8, k columns -> o->k8 (row pitch
 *   64 heads), scales at (row / seq_len * heads + head) * scale_ld + row % seq_len.  N a multiple of 64. */
typedef struct SatbQkE4m3 {
  void* q8;
  void* k8;
  float* sq;
  float* sk;
  int heads, scale_ld;
} SatbQkE4m3;
int satb_attention_fp8_vt(const void* v16, void* vt8, float* sv, int B, int H, int N, int bf16, void* stream);
int satb_attention_fp8_core(const void* q8, const void* k8, const float* sq, const float* sk, const void* vt8,
                            const float* sv, void* o16, int B, int H, int Nq, int Nk, int bf16, void* stream);
int satb_gemm_probe_qk8(const void* a, const void* w, const float* a_scale, const float* w_scale, int M, int N, int K,
                        const SatbGemmProbe* p, const SatbQkE4m3* o, void* stream);
/* Test entry point of the FP8 FF-out option (satb_dit_set_ff_out_fp8), through the instances the DiT forward launches;
 * a8 [M, K] and w8 [N, K] e4m3, w_scale [N], K a multiple of 128, bf16 0.
 *   SATB_EPI_SWIGLU_E4M3 (bn 256) and SATB_EPI_SILU_E4M3 (bn 128 / 256): FF-in, a_scale [M] (one per row).  The epilogue's
 *     fp32 outputs (N / 2 SwiGLU columns or N SiLU columns, bias as in swiglu / store16) are stored as ff8 [M, ld] e4m3
 *     and ff_scale [M, ld / 128]: for every row and 128-column block, scale = 2^e with e the smallest integer (>= -126)
 *     with max |y| <= 448 * 2^e (1 for an all-zero block), ff8 = e4m3_rn(y / scale).  ld a multiple of 128.
 *   SATB_EPI_RESIDUAL_A8 (bn 128): FF-out, a_scale [M, K / 128] (the scale of a8[m, k] is a_scale[m, k / 128]);
 *     C[m, n] = w_scale[n] sum_kb a_scale[m, kb] sum_{k in kb} a8[m, k] w8[n, k] goes through the residual epilogue (h, ld,
 *     bias, gate).  ff8 and ff_scale are ignored. */
int satb_gemm_probe_ff8(const void* a8, const void* w8, const float* a_scale, const float* w_scale, int M, int N, int K,
                        const SatbGemmProbe* p, void* ff8, float* ff_scale, void* stream);

/* Test entry point: the kernel of the conformer branch, out = silu(LayerNorm(depthwise_conv(g))) per item
 * (transformer.py:583-586): g, out [items * n_seq, D] 16-bit (fp16/bf16 bits), 16-byte aligned; the convolution runs
 * over the n_seq rows of each item with 17 taps and 8 zero rows of padding at both ends; w [D, 1, 17] fp32 (device),
 * gamma, beta [D] fp32 (beta may be NULL), eps 1e-5.  D a multiple of 128, <= 1536. */
int satb_conformer_dwconv(const void* g16, const float* w, const float* gamma, const float* beta, void* out16, int items,
                          int n_seq, int D, int bf16, void* stream);

/* ---- Oobleck VAE: replaces OobleckDecoder / OobleckEncoder.forward
 *      (models/autoencoders.py:119-194) behind AudioAutoencoder.encode/decode (:268-343) */
int satb_oobleck_create(const SatbOobleckConfig* cfg, SatbOobleck** out);
/* The same for the blocks' other options (models/autoencoders.py:29-116):
 *   activation        SATB_OOB_ACT_SNAKE (use_snake=True: SnakeBeta, "alpha" / "beta" keys) or SATB_OOB_ACT_ELU
 *                     (use_snake=False: nn.ELU(), no parameters, so finalize looks up no alpha / beta keys);
 *   nearest_upsample  1: every decoder block upsamples by nearest-neighbour x s followed by a bias-free weight-normed
 *                     Conv1d k = 2s, padding 'same' ("layers.{b}.layers.1.1.weight_g / weight_v"; use_nearest_upsample)
 *                     instead of a ConvTranspose1d.  Any decoder stride >= 2 is accepted, odd ones included.  The conv
 *                     runs as a 3-tap convolution of the low-rate input; finalize folds its weights (fp64 sums).
 *                     Refused for an encoder.
 * Unknown values are refused.  satb_oobleck_create(cfg, out) is satb_oobleck_create_variant(cfg, SNAKE, 0, out).  The
 * options are fixed for the handle's lifetime: they decide which weights finalize expects. */
#define SATB_OOB_ACT_SNAKE 0
#define SATB_OOB_ACT_ELU 1
int satb_oobleck_create_variant(const SatbOobleckConfig* cfg, int activation, int nearest_upsample, SatbOobleck** out);
void satb_oobleck_destroy(SatbOobleck* h);
/* State-dict entry relative to the encoder/decoder module ("layers.1.layers.1.weight_v" ...). */
int satb_oobleck_load_weight(SatbOobleck* h, const char* name, const float* src, long long numel, void* stream);
int satb_oobleck_finalize(SatbOobleck* h, void* stream);
/* Decoder: z [B, latent_dim, L] -> audio [B, in_channels, L * prod(strides)]. */
int satb_oobleck_decode(SatbOobleck* h, const float* z, float* audio, int B, int L, void* stream);
/* Encoder: audio [B, in_channels, T] -> pre-bottleneck [B, latent_dim, T / prod(strides)]
 * (the deterministic mean|scale tensor; the VAE sampling stays in PyTorch, bottleneck.py:46-62). */
int satb_oobleck_encode(SatbOobleck* h, const float* audio, float* latents, int B, long long T, void* stream);

/* ---- Time-sharded Oobleck decode / encode: one process drives `world` ranks (1 .. 8), each a finalized handle with a
 * full copy of the weights on its device; several ranks may share one device.  Rank r runs the ordinary decode (encode)
 * of latents ext[2r] .. ext[2r + 1] - 1 (their samples for the encoder): its own range begin[r] .. begin[r + 1] - 1 plus
 * a recompute margin on each interior side, clipped to the item.  The home device (rank 0's) then gathers every rank's
 * own range, read through peer pointers, into the whole output.  The margin covers the receptive field, and no
 * convolution route depends on where a position falls in a tile, so the result is bit-identical to the single-device
 * call. */
typedef struct SatbOobleckGroup SatbOobleckGroup;
/* The split of an item of L latents for a handle of config cfg (is_decoder picks the decoder or the encoder) and
 * nearest_upsample (as satb_oobleck_create_variant): begin[world + 1] (an even split, begin[0] = 0, begin[world] = L),
 * ext[2 world] (rank r's extended range [ext[2r], ext[2r + 1]) in latents) and *margin, the receptive field of one latent
 * in latents on either side, derived from the layer list.  world > L is refused, and so is, for world > 1, a rank range
 * shorter than the margin.  Host only. */
int satb_oobleck_group_plan(int world, int L, const SatbOobleckConfig* cfg, int nearest_upsample, int* begin, int* ext,
                            int* margin);
/* handles[world]: finalized handles of one model (same config and block options, checked), one per rank, each its own;
 * devices[world]: their device ids, devices[0] the home device.  Ranks on a device other than the home device need peer
 * access in both directions with it (refused with a message when missing); it is enabled for this process.  The group
 * owns one stream per rank; the handles outlive the group, which must be destroyed explicitly. */
int satb_oobleck_group_create(SatbOobleck* const* handles, const int* devices, int world, SatbOobleckGroup** out);
void satb_oobleck_group_destroy(SatbOobleckGroup* g);
/* As satb_oobleck_decode / satb_oobleck_encode over the ranks: z, audio (and audio, latents) are whole tensors on the
 * home device, stream a stream there.  Each rank copies its extended input slice from the home device on its own
 * stream after the work already on `stream`, then decodes (encodes); the gather kernel runs on `stream` after every
 * rank, and each rank's next call waits for it.  Enqueues only; the caller's current device is restored.  The per-rank
 * slices are allocated at their extended shapes and grow when needed (after the last gather). */
int satb_oobleck_group_decode(SatbOobleckGroup* g, const float* z, float* audio, int B, int L, void* stream);
int satb_oobleck_group_encode(SatbOobleckGroup* g, const float* audio, float* latents, int B, long long T, void* stream);

/* Test entry points (no product path calls them).
 * satb_oobleck_probe runs ONE step of a finalized handle's decode or encode on caller-owned device buffers, through
 * the same host function (and so the same kernel instances, route, next Snake and raw-stream choice) as the product
 * loop.  Steps, with the buffers each one reads and writes ("16-bit": [B, L, C] channels-last in the operand type; in
 * fp16x3 mode every 16-bit buffer has its lo half at byte offset lo_off; "raw": [B, L, C] fp16 in fp16 mode, fp32
 * otherwise):
 *   DEC_IN    in: fp32 NCL latents [B, latent_dim, L]; scratch: their 16-bit copy; out16
 *   DEC_UP    block b: in (16-bit, L positions) -> raw_out, out16 (L * stride positions)
 *   DEC_RES   unit (b, j): in (16-bit), raw_in -> raw_out (if wrote_raw), the result in `in` or `scratch`
 *   DEC_OUT   in (16-bit) -> out32 (NCL fp32 audio)
 *   ENC_IN    in: fp32 NCL audio [B, in_channels, L] -> raw_out, out16; with in_channels > 2, scratch: its 16-bit copy
 *   ENC_RES   unit (b, j), as DEC_RES
 *   ENC_DOWN  block b: in (16-bit, L positions, a multiple of the stride) -> raw_out (if wrote_raw), out16
 *   ENC_OUT   in (16-bit) -> out32 (NCL fp32 pre-bottleneck)
 * A ResidualUnit updates its raw stream in place: the probe first copies raw_in to raw_out (when they differ).  Its
 * 16-bit result lands in `in` (two-launch route, which also uses scratch) or in `scratch` (fused route):
 * result_in_scratch says which.  Blocks and units count as in the state dict: b = 1 .. n_stages, j = 0 .. 2.  Every
 * pointer a step uses must be 16-byte aligned. */
#define SATB_OOB_DEC_IN 0
#define SATB_OOB_DEC_UP 1
#define SATB_OOB_DEC_RES 2
#define SATB_OOB_DEC_OUT 3
#define SATB_OOB_ENC_IN 4
#define SATB_OOB_ENC_RES 5
#define SATB_OOB_ENC_DOWN 6
#define SATB_OOB_ENC_OUT 7
/* routes (bits of SatbOobleckProbe.routes): the kernels one step launched */
#define SATB_OOB_ROUTE_GEMM 1           /* implicit-GEMM conv, general EpiConv epilogue */
#define SATB_OOB_ROUTE_GEMM_LEAN 2      /* implicit-GEMM conv, lean EpiConv epilogue */
#define SATB_OOB_ROUTE_FUSED 4          /* fused ResidualUnit (conv_halo, FUSE), general epilogue */
#define SATB_OOB_ROUTE_FUSED_LEAN 8     /* fused ResidualUnit, lean epilogue */
#define SATB_OOB_ROUTE_HALO_NCL 16      /* halo-tile conv with the NCL fp32 store */
#define SATB_OOB_ROUTE_GEMM_NCL 32      /* implicit-GEMM conv with the NCL fp32 store */
#define SATB_OOB_ROUTE_CUDA_CORE 64     /* encoder input conv on CUDA cores */
typedef struct SatbOobleckProbe {
  int step, block, unit, B, L;      /* L: input positions per item */
  void* in;                         /* 16-bit input (overwritten by a two-launch ResidualUnit), or fp32 NCL */
  const void* raw_in;
  void* raw_out;
  void* out16;
  void* scratch;
  float* out32;
  long long lo_off;                 /* fp16x3 only */
  /* set by the call */
  int result_in_scratch, wrote_raw, routes;
} SatbOobleckProbe;
int satb_oobleck_probe(SatbOobleck* h, SatbOobleckProbe* p, void* stream);
/* The stored weights of the finalized conv `prefix` ("layers.1.layers.1."): the 16-bit [tap][n][k] block (and, in
 * fp16x3 mode, its lo block right after it), or the fp32 [cout][cin][k] weights of a CUDA-core conv.  *bytes gets
 * the size; dst (device, may be NULL to ask for the size) receives the data. */
int satb_oobleck_weights(SatbOobleck* h, const char* prefix, void* dst, long long* bytes, void* stream);

/* ---- PQMF filterbank: replaces PQMF.forward / PQMF.inverse (models/pqmf.py) behind PQMFPretransform.encode / decode
 *      (models/pretransforms.py:114-133), fp32 on the CUDA cores.
 * num_bands: a power of 2 in [2, 256]; taps: the filter bank's length (the reference pads it to a power of two), a
 * multiple of 2 * num_bands, at most 16384.  Every call checks its arguments before any CUDA call. */
int satb_pqmf_create(int num_bands, int taps, SatbPqmf** out);
void satb_pqmf_destroy(SatbPqmf* h);
/* filter_bank: device [num_bands, taps] (the "pqmf.filter_bank" buffer).  Builds the handle's polyphase weights on
 * `stream`; call it again after the buffer changes. */
int satb_pqmf_load_filter(SatbPqmf* h, const float* filter_bank, void* stream);
/* audio [B, C, T] -> bands [B, C * num_bands, ceil(T / num_bands)] (band k of channel c at row c * num_bands + k):
 * the signal zero-padded to a multiple of num_bands, polyphase analysis, alias cancellation (PQMF.forward + the
 * pretransform's "b c n t -> b (c n) t"). */
int satb_pqmf_analysis(SatbPqmf* h, const float* audio, float* bands, int B, int C, long long T, void* stream);
/* bands [B, C * num_bands, frames] -> audio [B, C, frames * num_bands] (PQMF.inverse). */
int satb_pqmf_synthesis(SatbPqmf* h, const float* bands, float* audio, int B, int C, int frames, void* stream);

/* ---- T5 encoder: replaces Hugging Face T5EncoderModel.forward (transformers models/t5/modeling_t5.py) behind
 *      T5Conditioner.forward (models/conditioners.py).  Prompts are packed (sum of lengths rows, nothing computed for
 *      padding); fp32 residual stream, 16-bit GEMM operands; csrc/t5.cu describes the launches.
 * Mirrors the T5Config fields the encoder uses.  Refused by satb_t5_create: d_kv other than 64 or 128, feed_forward_proj
 * other than relu / gated-gelu, d_model not a multiple of 128 or above 4096, d_ff not a multiple of 32. */
#define SATB_T5_FF_RELU 0          /* "relu": DenseReluDense.wi, ReLU, wo */
#define SATB_T5_FF_GATED_GELU 1    /* "gated-gelu": gelu_new(wi_0 x) * (wi_1 x), wo */
typedef struct SatbT5Config {
  int vocab_size;
  int d_model;
  int d_kv;
  int num_heads;
  int d_ff;
  int num_layers;
  int relative_attention_num_buckets;
  int relative_attention_max_distance;   /* informational: the buckets come from satb_t5_set_buckets */
  int feed_forward_proj;                 /* SATB_T5_FF_* */
  float layer_norm_epsilon;
  int operand_dtype;                     /* 0 = fp16 (the reference's dtype), 1 = bf16 */
} SatbT5Config;
typedef struct SatbT5 SatbT5;
int satb_t5_create(const SatbT5Config* cfg, SatbT5** out);
void satb_t5_destroy(SatbT5* h);
/* One T5EncoderModel state-dict entry by its HF key ("shared.weight" or "encoder.embed_tokens.weight",
 * "encoder.block.{i}.layer.0.SelfAttention.{q,k,v,o}.weight", block 0's "...SelfAttention.relative_attention_bias.weight",
 * "encoder.block.{i}.layer.1.DenseReluDense.{wi | wi_0, wi_1, wo}.weight", "encoder.block.{i}.layer.{0,1}.layer_norm.weight",
 * "encoder.final_layer_norm.weight"); src: device fp32, contiguous. */
int satb_t5_load_weight(SatbT5* h, const char* name, const float* src, long long numel, void* stream);
/* buckets (host) [1023]: the bucket of relative position j - i = k - 511 at index k, as
 * T5Attention._relative_position_bucket(bidirectional=True, num_buckets, max_distance) gives it; each in
 * [0, num_buckets).  Required before satb_t5_finalize. */
int satb_t5_set_buckets(SatbT5* h, const int* buckets, int n);
/* Optional output projection (the conditioner's proj_out Linear): W [out_dim, d_model], b [out_dim], device fp32;
 * out_dim a multiple of 8.  Without it the encoder writes d_model columns. */
int satb_t5_set_proj_out(SatbT5* h, const float* W, const float* b, int out_dim, void* stream);
/* Checks that every weight and the buckets are there and builds the bias table (synchronous). */
int satb_t5_finalize(SatbT5* h, void* stream);
/* ids_dev [B, L] int64 (device), lengths_host [B]: item b is the right-padded prefix ids[b, :lengths[b]] (0 <= length
 * <= L); 1 <= L <= 512.  out_dev [B, L, out_dim or d_model] fp32: the encoder's last hidden state (projected when
 * proj_out is set) at valid positions, exact zeros at padded ones.  Ids outside [0, vocab_size) are clamped to the table
 * (the Python layer refuses them). */
int satb_t5_encode(SatbT5* h, const long long* ids_dev, const int* lengths_host, int B, int L, float* out_dev,
                   void* stream);
/* Test entry points (no product path calls them), through the launches the encode makes:
 * satb_t5_rmsnorm_probe: out[r, :] = w * (x[r, :] * rsqrt(mean(x[r, :]^2) + eps)); x [rows, D] fp32; out_kind 0 = fp16
 *   (saturating at +-65504), 1 = bf16, 2 = fp32; D a multiple of 4, at most 4096; pointers 16-byte aligned.
 * satb_t5_attention_probe: qkv16 [M, 3 H d_kv] packed rows (M = sum of lengths_host[B], each at most 512): q of head h
 *   at column h d_kv, k at (H + h) d_kv, v at (2 H + h) d_kv; bias_tab [H, 1023] fp32, entry k the bias of key j for
 *   query i with k = j - i + 511; o16 [M, H d_kv] = softmax(q k^T + bias) v per item and head (no scale).
 * satb_t5_gemm_probe: C = A[M, K] W[N, K]^T through one of the encoder's own FF-in epilogues (p->epi, p->bn 128 / 256,
 *   p->bf16, p->out, p->ld); the other GEMM probes refuse these ids and this one refuses theirs. */
#define SATB_EPI_RELU16 10    /* out 16-bit = max(acc, 0), saturating in fp16 */
#define SATB_EPI_GEGLU16 11   /* out[:, N / 2] = value * gelu_new(gate), 32 / 32 interleaved columns, saturating in fp16 */
int satb_t5_rmsnorm_probe(const float* x, const float* w, void* out, int rows, int D, float eps, int out_kind,
                          void* stream);
int satb_t5_attention_probe(const void* qkv16, const float* bias_tab, const int* lengths_host, int B, int H, int d_kv,
                            int bf16, void* o16, void* stream);
int satb_t5_gemm_probe(const void* a16, const void* w16, int M, int N, int K, const SatbGemmProbe* p, void* stream);
/* satb_t5_linear_probe: C = A[M, K] W[N, K]^T through the encoder's own GEMM launch with the parameters an encode
 *   passes: SATB_EPI_STORE16 (QKV; out, ld), SATB_EPI_RESIDUAL (o-projection and FF-out: h[M, ld] += C, no bias, no
 *   gate), SATB_EPI_STORE32 (proj_out: out = C + bias, bias required), SATB_EPI_RELU16 / SATB_EPI_GEGLU16 (FF-in).
 *   A's tensor map spans a_rows >= M rows, as the encoder's spans its workspace; the tiles cover M.  p->bn: 128, 256,
 *   or 0 for the tile the encoder picks at this (M, N).  p->bf16 selects the operand type.
 * satb_t5_bias_table: copies the finalized relative-position bias table [H, 1023] fp32 (entry k of head h: the bias of
 *   relative position k - 511, rel[bucket, h]) to the device buffer dst (synchronous). */
int satb_t5_linear_probe(const void* a16, int a_rows, const void* w16, int M, int N, int K, const SatbGemmProbe* p,
                         void* stream);
int satb_t5_bias_table(SatbT5* h, float* dst, void* stream);

/* ---- RoBERTa encoder: replaces Hugging Face RobertaModel(output_hidden_states=True).hidden_states[n] (transformers
 *      models/roberta/modeling_roberta.py), the text branch behind the CLAP text conditioner's features
 *      (models/conditioners.py CLAPTextConditioner).  All B L rows are computed, keys limited to each item's valid
 *      prefix; fp32 residual stream, 16-bit GEMM operands; csrc/roberta.cu describes the launches.
 * Mirrors the RobertaConfig fields the encoder uses, with num_layers the number of layers an encode runs (n: index n of
 * hidden_states, 0 = the embedding output).  Refused by satb_roberta_create: hidden_size not a multiple of 128 or above
 * 1024, head dim (hidden_size / num_heads) other than 64, intermediate_size not a multiple of 32. */
typedef struct SatbRobertaConfig {
  int vocab_size;
  int hidden_size;
  int num_heads;
  int intermediate_size;
  int num_layers;                 /* layers run */
  int max_position_embeddings;
  int type_vocab_size;
  int pad_token_id;               /* also the padding_idx of the position ids */
  float layer_norm_eps;
  int operand_dtype;              /* 0 = fp16, 1 = bf16 */
} SatbRobertaConfig;
typedef struct SatbRoberta SatbRoberta;
int satb_roberta_create(const SatbRobertaConfig* cfg, SatbRoberta** out);
void satb_roberta_destroy(SatbRoberta* h);
/* One RobertaModel state-dict entry by its HF key ("embeddings.{word,position,token_type}_embeddings.weight",
 * "embeddings.LayerNorm.{weight,bias}", "encoder.layer.{i}.attention.self.{query,key,value}.{weight,bias}",
 * "encoder.layer.{i}.attention.output.{dense,LayerNorm}.{weight,bias}", "encoder.layer.{i}.intermediate.dense.{weight,bias}",
 * "encoder.layer.{i}.output.{dense,LayerNorm}.{weight,bias}", i < num_layers); src: device fp32, contiguous. */
int satb_roberta_load_weight(SatbRoberta* h, const char* name, const float* src, long long numel, void* stream);
/* Optional output projection (the conditioner's proj_out Linear): W [out_dim, hidden_size], b [out_dim], device fp32;
 * out_dim a multiple of 8.  Without it the encoder writes hidden_size columns. */
int satb_roberta_set_proj_out(SatbRoberta* h, const float* W, const float* b, int out_dim, void* stream);
/* Checks that every weight is there (synchronous). */
int satb_roberta_finalize(SatbRoberta* h, void* stream);
/* ids_dev [B, L] int64 (device), lengths_host [B]: the keys of item b are positions [0, lengths[b]) (1 <= length <= L);
 * 1 <= L <= 512 and L + pad_token_id < max_position_embeddings.  out_dev [B, L, out_dim or hidden_size] fp32: hidden
 * state n (projected when proj_out is set) at every position, padded ones included.  Ids outside [0, vocab_size) are
 * clamped to the table (the Python layer refuses them). */
int satb_roberta_encode(SatbRoberta* h, const long long* ids_dev, const int* lengths_host, int B, int L, float* out_dev,
                        void* stream);
/* Test entry points (no product path calls them), through the launches the encode makes:
 * satb_roberta_embed_probe: y[b L + t] = LayerNorm(word[ids[b, t]] + tok[0] + pos[p]) with p the position id of
 *   create_position_ids_from_input_ids (padding_idx pad); y32 fp32 and y16 16-bit (fp16 saturating, or bf16) [B L, D].
 * satb_roberta_layernorm_probe: y = LayerNorm(x) (gamma, beta) of x [rows, D] fp32 into y32 (may be x) and y16.
 * satb_roberta_attention_probe: qkv16 [B L, 3 H 64] (q of head h at column 64 h, k at 64 (H + h), v at 64 (2 H + h));
 *   o16 [B L, H 64] = softmax(q k^T / 8) v over keys [0, lengths_host[b]) of item b, for every one of its L rows.
 * satb_roberta_linear_probe: C = A[M, K] W[N, K]^T through the encoder's GEMM launch with the parameters an encode
 *   passes (bias required, ld == N): SATB_EPI_STORE16 (QKV), SATB_EPI_RESIDUAL (out-proj and FF-out: h += C + bias),
 *   SATB_EPI_STORE32 (proj_out), SATB_EPI_BIAS_GELU16 (FF-in); p->bf16 selects the operand type. */
#define SATB_EPI_BIAS_GELU16 12   /* out 16-bit = gelu(acc + bias) with the erf GELU, saturating in fp16 */
int satb_roberta_embed_probe(const long long* ids, int B, int L, const float* word, int vocab, const float* pos,
                             int max_pos, const float* tok, const float* gamma, const float* beta, int D, int pad,
                             float eps, float* y32, void* y16, int bf16, void* stream);
int satb_roberta_layernorm_probe(const float* x, const float* gamma, const float* beta, int rows, int D, float eps,
                                 float* y32, void* y16, int bf16, void* stream);
int satb_roberta_attention_probe(const void* qkv16, const int* lengths_host, int B, int L, int H, int bf16, void* o16,
                                 void* stream);
int satb_roberta_linear_probe(const void* a16, const void* w16, int M, int N, int K, const SatbGemmProbe* p,
                              void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SATB200_H_ */

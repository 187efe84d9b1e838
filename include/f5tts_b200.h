/*
 * f5tts_b200 — C ABI of the H100-native F5-TTS / E2-TTS ODE-sampling hot path.
 *
 * Plain C symbols, raw device pointers + explicit sizes, a CUDA stream, `int` return (0 = ok, < 0 = error;
 * f5_last_error() returns the message for the calling thread).  No ownership transfer: every buffer, including
 * the scratch workspace, belongs to the caller.  The only library-owned object is the opaque f5_engine, which
 * stores architecture constants and POINTERS to the caller's re-packed weights (see f5_weights).  Calls on
 * distinct (stream, workspace) pairs may run concurrently (the reference samples from a ThreadPoolExecutor,
 * infer/utils_infer.py:540-541).
 *
 * Each entry point names the reference interface it replaces (paths relative to /root/reference/src/f5_tts).
 * The reference has no native FFI on this path (it is pure PyTorch); the binding a maintainer adds is the ctypes
 * stub shown in INTEGRATION.md / f5_tts_b200/_lib.py.
 *
 * Requires an sm_90a device (wgmma / TMA).  There is no CPU or non-Hopper fallback.
 */
#ifndef F5TTS_B200_H
#define F5TTS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* f5_stream_t; /* cudaStream_t */

int f5_version(void);
const char* f5_last_error(void);
/* number of kernels this library has launched in this process (bench.py reports it as gpu_launches) */
unsigned long long f5_launch_count(void);

/* ------------------------------------------------------------------------------------------------------------
 * Kernel-level entry points (used by the parity tests and by the Python operator mirrors)
 * ------------------------------------------------------------------------------------------------------------ */

enum { F5_ACT_NONE = 0, F5_ACT_GELU_TANH = 1, F5_ACT_GELU_ERF = 2, F5_ACT_MISH = 3 };
/* F5_EPI_QKV_NORM_ROPE: F5_EPI_QKV_ROPE with the reference's qk_norm="rms_norm" (model/modules.py:402-409, 492-496;
 * RMSNorm modules.py:286-305) on every q and k head before RoPE: v * rsqrt(mean_head(v^2) + 1e-6) * gain[c % 64], in
 * fp32, v = acc + bias.  Needs q_norm, k_norm, rope tables, seq and inner % 64 == 0.  Since f5_version() 105. */
enum { F5_EPI_F16 = 0, F5_EPI_F32 = 1, F5_EPI_RESID = 2, F5_EPI_QKV_ROPE = 3, F5_EPI_QKV_NORM_ROPE = 4 };

/* Fused linear: C = epilogue(A[M,K] . W[N,K]^T) — replaces nn.Linear (aten::addmm) call sites
 * model/modules.py:317,338,360-361,398-400 and, with conv_taps != 0, the grouped Conv1d(k=taps, groups=N/k,
 * padding=taps/2) of ConvPositionEmbedding (model/modules.py:175-201), k channels per group.
 *   A fp16 [batches*rows, lda]; W fp16 [N, ldw] (conv: [taps][N][k]); fp32 accumulation. */
typedef struct {
  int rows;      /* valid rows per batch entry (plain GEMM: M, batches = 1) */
  int batches;
  int n_out;
  int k;         /* reduction length (plain) ; conv: channels per group, 0 = 64 (a multiple of 8, <= 64, dividing
                    n_out; anything else is rejected) */
  int lda, ldw;  /* elements */
  int bn;        /* output tile width: 64 | 128 | 192 | 256 (0 = the planner picks the width) */
  int epi, act;
  int conv_taps; /* 0 = plain GEMM */
  int cta_pair;  /* must be 0 (there are no cluster-pair tiles); kept so the struct layout does not change */
  const float* bias;
  void* out;               /* fp16 (F16 / QKV_ROPE) or fp32 (F32) [batches*rows, ldo] */
  void* out16b;            /* optional fp16 masked copy for F32 */
  float* resid;            /* RESID: in/out fp32 */
  int ldo;
  const float* gate;       /* RESID: per-column gate (NULL = 1) */
  const int* step_ptr;     /* device step counter used to index gate (NULL = 0) */
  long long gate_step_stride;
  const int* row_len;      /* per-sample valid rows (NULL = all) */
  int seq;                 /* rows per sample */
  const float* rope_cos;   /* [seq, dim_head / 2] */
  const float* rope_sin;
  int inner, pe_heads;
  int weights_static;      /* 1 = W was NOT written by the kernel preceding this call on the stream (model weights):
                              its first tiles are fetched ahead of the programmatic-dependent-launch wait */
  /* Packed / variable-length execution: 1 = output tiles whose rows all lie past row_len of their sample are skipped
   * entirely (not loaded, multiplied or stored: their output rows keep whatever the buffer held).  Needs row_len and
   * seq.  The reference's counterpart is its masked mode (flash_attn_varlen / attn_mask, modules.py:513-540). */
  int skip_padded_tiles;
  const float* q_norm;     /* QKV_NORM_ROPE: fp32 [dim_head] RMSNorm gain of the q heads (attn.q_norm.weight) */
  const float* k_norm;     /* QKV_NORM_ROPE: fp32 [dim_head] RMSNorm gain of the k heads (attn.k_norm.weight) */
  /* QKV epilogues: columns per head, 0 (= 64), 64 or 128.  At 128, rope tables are [seq, 64], the RMSNorm gains
   * [128], inner and n_out multiples of 128, and QKV_NORM_ROPE runs with bn 128 only (the planner picks it).  Any
   * other epilogue takes 0 or 64.  Since f5_version() 106. */
  int dim_head;
} f5_gemm_args;
int f5_gemm(const void* A, const void* W, const f5_gemm_args* args, f5_stream_t stream);
/* Tile shape f5_gemm would run `args` with (after bn = 0 resolution): *bn tile width, *cta_pair always 0. */
int f5_gemm_tile(const f5_gemm_args* args, int* bn, int* cta_pair);

/* Non-causal attention over the fused QKV buffer — replaces F.scaled_dot_product_attention at
 * model/modules.py:519 (attn_mask=None, or the key mask of modules.py:513-517 via kv_len).
 *   qkv fp16 [batches*seq, 3*heads*64]; out fp16 [batches*seq, heads*64]. dim_head is 64. */
int f5_attention(const void* qkv, void* out, int batches, int seq, int heads, const int* kv_len, float scale,
                 f5_stream_t stream);
/* f5_attention with the head width as an argument: dim_head 64 or 128 (anything else returns -1).
 *   qkv fp16 [batches*seq, 3*heads*dim_head]; out fp16 [batches*seq, heads*dim_head]; the reference's scale is
 *   1/sqrt(dim_head).  f5_attention(...) is f5_attention_dh(..., 64, ...).  Since f5_version() 106. */
int f5_attention_dh(const void* qkv, void* out, int batches, int seq, int heads, int dim_head, const int* kv_len,
                    float scale, f5_stream_t stream);

/* Joint attention of MMDiT (model/modules.py:563-705, JointAttnProcessor): one softmax over the keys [audio | text]
 * for the queries [audio | text].  The two segments are separate fused QKV buffers:
 *   qkv   fp16 [batches*seq,   3*heads*dim_head]   out   fp16 [batches*seq,   heads*dim_head]
 *   qkv_c fp16 [batches*seq_c, 3*heads*dim_head]   out_c fp16 [batches*seq_c, heads*dim_head]
 * kv_len [batches] valid audio keys (>= 1) or NULL (= seq); c_len [batches] valid text keys (0 = the text segment adds no
 * key) or NULL (= seq_c); both device int32.  text_q = 0 computes the audio queries only and leaves out_c unwritten
 * (the last MMDiT block discards its text output).  dim_head 64 or 128.  Since f5_version() 107. */
int f5_attention_joint(const void* qkv, const void* qkv_c, void* out, void* out_c, int batches, int seq, int seq_c,
                       int heads, int dim_head, const int* kv_len, const int* c_len, int text_q, float scale,
                       f5_stream_t stream);

/* f5_attention_dh and f5_attention_joint with the query rows per CTA given: qwg consumer warpgroups of 64 rows, 2 or
 * (dim_head 64) 4; anything else returns -1.  qwg = 0 is the planner's choice, which the two calls above always make.
 * Both widths give the same output bit for bit; the choice only changes the grid (and so the speed). */
int f5_attention_qwg(const void* qkv, void* out, int batches, int seq, int heads, int dim_head, const int* kv_len,
                     float scale, int qwg, f5_stream_t stream);
int f5_attention_joint_qwg(const void* qkv, const void* qkv_c, void* out, void* out_c, int batches, int seq, int seq_c,
                           int heads, int dim_head, const int* kv_len, const int* c_len, int text_q, float scale,
                           int qwg, f5_stream_t stream);
/* the qwg that f5_attention_dh picks for this problem on the current device (-1 for invalid arguments) */
int f5_attention_qwg_choice(int batches, int seq, int heads, int dim_head);

/* Row normalisation + modulation -> fp16 (model/modules.py:312-326,333-347,753; x_transformers RMSNorm unett.py:154)
 *   mode 0: LN(eps) * (1 + a[c]) + b[c]   mode 1: LN(eps) * a[c] + b[c]   mode 2: x/||x|| * sqrt(D) * a[c] */
int f5_row_norm(const float* x, void* out_f16, int rows, int D, int mode, float eps, const float* a, const float* b,
                f5_stream_t stream);

/* Vocos mel front-end — replaces MelSpec.forward / get_vocos_mel_spectrogram (model/modules.py:80-151).
 *   wav fp32 [B, nw]; fb fp32 [513, n_mels]; out fp32 [B, n_mels, T] (or [B, T, n_mels] if out_btc), T = 1 + nw/256 */
int f5_mel_spectrogram(const float* wav, int B, int nw, const float* fb, int n_mels, float* out, int out_btc,
                       f5_stream_t stream);

/* Vocos back-end — replaces vocos.Vocos.decode as used at infer/utils_infer.py:511 (VocosBackbone + ISTFTHead). */
typedef struct {
  const void* embed_w;   /* fp16 [512, 704]  im2col-packed Conv1d(100,512,7) weight, K padded 700 -> 704 */
  const float* embed_b;
  const float* norm_w; const float* norm_b;
  const float* dw_w[8]; const float* dw_b[8];        /* [512, 7], [512] */
  const float* ln_w[8]; const float* ln_b[8];
  const void* pw1_w[8]; const float* pw1_b[8];       /* fp16 [1536, 512] */
  const void* pw2_w[8]; const float* pw2_b[8];       /* fp16 [512, 1536] */
  const float* gamma[8];
  const float* final_w; const float* final_b;
  const void* head_w; const float* head_b;           /* fp16 [1026, 512] */
  int dim, inter, layers, n_mels;
} f5_vocos_weights;
/* workspace of either decode entry point below */
size_t f5_vocos_workspace_bytes(int B, int T);
/* mel fp32 [B, 100, T] -> wav fp32 [B, 256*(T-1)] */
int f5_vocos_decode(const f5_vocos_weights* w, const float* mel, int B, int T, void* workspace, size_t ws_bytes,
                    float* wav, f5_stream_t stream);
/* Variable-length batch decode.  lengths: HOST int32 [B] valid frames per sample, each in [2, T], or NULL (= exactly
 * f5_vocos_decode).  Sample b's first 256*(lengths[b]-1) output samples are bit-identical to f5_vocos_decode of
 * mel[b, :, :lengths[b]] alone, and the rest of its row is 0; mel frames at or past lengths[b] are never read (NaN or
 * inf there has no effect).  Out-of-range lengths return -1 before anything is launched.  The lengths are copied into
 * the workspace, so calls that differ only in lengths replay one captured graph.  Since f5_version() 104. */
int f5_vocos_decode_varlen(const f5_vocos_weights* w, const float* mel, int B, int T, const int* lengths,
                           void* workspace, size_t ws_bytes, float* wav, f5_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * Engine: the whole CFM.sample NFE loop (model/cfm.py:160-223) for a DiT (backbones/dit.py:319-370), UNetT
 * (backbones/unett.py:244-307) or MMDiT (backbones/mmdit.py:198-246) backbone.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  /* 0 = DiT, 1 = UNetT, 2 = MMDiT (since f5_version() 107).  MMDiT needs text_dim = conv_layers = long_skip =
   * text_avg_upsample = 0 and pe_attn_head = -1 (rope on every head), and f5_weights.ctx_layers. */
  int backbone;
  /* dim_head: 64, or since f5_version() 106 also 128 (rope over the full head, softmax scale 1/sqrt(dim_head));
   * heads * dim_head must be a multiple of 128 and at most 1024 at dim_head 128 */
  int dim, depth, heads, dim_head, ff_inner, mel_dim, text_dim, text_num_embeds, conv_layers;
  int text_mask_padding; /* yaml arch.text_mask_padding */
  int pe_attn_head;      /* -1 = all heads */
  int attn_mask_enabled;
  /* Since f5_version() 105; all 0 reproduce the earlier engine exactly. */
  int qk_norm;           /* 1 = qk_norm="rms_norm": per-head RMSNorm of q and k before RoPE (modules.py:402-409,
                            492-496); needs q_norm_w / k_norm_w in every layer */
  int long_skip;         /* DiT long_skip_connection (backbones/dit.py:228, 354-365): x = long_skip_w .
                            cat(x after the last block, x after the input embedding) before norm_out */
  int text_avg_upsample; /* DiT text_embedding_average_upsampling (backbones/dit.py:41-84, 131-137): each sample's
                            valid text tokens spread evenly over its audio length; needs text_mask_padding */
  /* Since f5_version() 108.  UNetT skip_connect_type (backbones/unett.py:127, 290-297): how each later-half layer
   * combines x with the x its mirror first-half layer saved.  0 = "concat": x = w_skip . cat(x, skip), w_skip needed in
   * every later-half layer; 1 = "add": x = x + skip; 2 = "none": the saved x is not used.  1 and 2 take no w_skip and
   * need an even depth.  Non-zero only for UNetT; a zeroed struct gets 0, the engine before this field. */
  int skip_type;
} f5_arch;

typedef struct {
  const void* w_qkv; const float* b_qkv;   /* fp16 [3*inner, D] (to_q | to_k | to_v), fp32 [3*inner] */
  const void* w_out; const float* b_out;   /* fp16 [D, inner] */
  const void* w_ff1; const float* b_ff1;   /* fp16 [F, D] */
  const void* w_ff2; const float* b_ff2;   /* fp16 [D, F] */
  const void* w_skip;                      /* UNetT later half with skip_type 0: fp16 [D, 2D], else NULL */
  const float* g_attn; const float* g_ff;  /* UNetT RMSNorm gains */
  const float* q_norm_w; const float* k_norm_w; /* arch.qk_norm: fp32 [dim_head] attn.q_norm / k_norm weight
                                                   (modules.py:406-407), else NULL */
} f5_layer_weights;

/* MMDiT text-stream ("context") weights of one block (modules.py:763-846; Attention *_c, modules.py:411-432).
 * The last block (context_pre_only) has no to_out_c and no ff_c: w_out_c .. b_ff2_c are NULL there. */
typedef struct {
  const void* w_qkv_c; const float* b_qkv_c;     /* fp16 [3*inner, D] (to_q_c | to_k_c | to_v_c), fp32 [3*inner] */
  const void* w_out_c; const float* b_out_c;     /* fp16 [D, inner] */
  const void* w_ff1_c; const float* b_ff1_c;     /* fp16 [F, D] */
  const void* w_ff2_c; const float* b_ff2_c;     /* fp16 [D, F] */
  const float* q_norm_c; const float* k_norm_c;  /* arch.qk_norm: fp32 [dim_head] attn.c_q_norm / c_k_norm, else NULL */
} f5_ctx_layer_weights;

typedef struct {
  const void* time_w0; const float* time_b0;  /* fp16 [D, 256] */
  const void* time_w1; const float* time_b1;  /* fp16 [D, D] */
  const float* text_table;                    /* fp32 [V+1, Td] */
  struct {
    const float* dw_w; const float* dw_b; const float* ln_w; const float* ln_b;
    const void* pw1_w; const float* pw1_b;    /* fp16 [2Td, Td] */
    const float* grn_gamma; const float* grn_beta;
    const void* pw2_w; const float* pw2_b;    /* fp16 [Td, 2Td] */
  } text_blocks[8];
  const void* proj_w; const float* proj_b;    /* fp16 [D, Kpad] input_embed.proj, K zero-padded to a multiple of 64 */
  int proj_kpad;
  const void* conv_w[2]; const float* conv_b[2]; /* fp16 [31][D][D/16] re-packed grouped conv, fp32 [D] */
  const void* mod_w; const float* mod_b;      /* DiT: fp16 [depth*6D + 2D, D] all AdaLN linears stacked; fp32 bias */
  const f5_layer_weights* layers;             /* [depth] */
  const float* g_out;                         /* UNetT norm_out.g */
  const void* out_w; const float* out_b;      /* fp16 [mel, D] proj_out */
  const void* long_skip_w;                    /* arch.long_skip: fp16 [D, 2D] long_skip_connection.weight
                                                 (backbones/dit.py:228, no bias), else NULL */
  /* MMDiT (backbone 2) only, since f5_version() 107; read only then.
   *   text_table  fp32 [V+1, D] text_embed.text_embed.weight;  proj_w  audio_embed.linear, K = 2*mel zero-padded to
   *   proj_kpad (a multiple of 64);  conv_w / conv_b  audio_embed.conv_pos_embed;  layers[i]  the audio stream (to_q/k/v,
   *   to_out.0, ff_x, q_norm / k_norm);  mod_w  every AdaLN linear stacked, per block [attn_norm_x: 6D | attn_norm_c:
   *   6D, or 2D (scale, shift) in the last block], then norm_out 2D.
   * Text padding must be trailing (as list_str_to_idx pads); the valid text length of each sample is the number of ids
   * that are not -1, counted on the device. */
  const f5_ctx_layer_weights* ctx_layers;     /* [depth] */
} f5_weights;

typedef struct f5_engine f5_engine;
int f5_engine_create(const f5_arch* arch, const f5_weights* weights, f5_engine** out);
void f5_engine_destroy(f5_engine* e);

typedef struct {
  int B, N, nt, steps;
  const long long* text;     /* device int64 [B, nt], padded with -1 (model/utils.py:99-106) */
  const float* step_cond;    /* device fp32 [B, N, mel]  (cfm.py:151-153) */
  float* y;                  /* device fp32 [B, N, mel]  in: y0 (cfm.py:196-201), out: trajectory[-1] */
  const int* duration;       /* device int32 [B] per-sample lengths = `mask` of cfm.py:155-158, or NULL (B == 1) */
  const float* t;            /* HOST fp32 [steps+1] time grid after EPSS / sway (cfm.py:211-216) */
  float cfg_strength;        /* < 1e-5 -> single un-packed forward (cfm.py:166-177) */
  float* trajectory;         /* device fp32 [steps+1, B, N, mel] or NULL: y at the grid points only, for either method */
  int use_graph;             /* capture one backbone evaluation into a CUDA graph and replay it once per evaluation */
  float* v_out;              /* optional device fp32 [Be, N, mel]: raw backbone output of the LAST evaluation (the value
                                transformer(x, cond, text, time, mask, cfg_infer=...) returns, dit.py:367-370) */
  int exact_varlen;          /* with duration != NULL: 1 = every sample is computed exactly as if it were ALONE in the batch
                                with N = duration[b] — text blocks, conv position embedding and attention see nothing past
                                the sample's end, padded tiles are skipped.  This is what a loop of B = 1 sample() calls
                                computes (the reference's per-chunk loop, infer/utils_infer.py:540-541), in one batch.
                                0 = the reference's batched semantics (padded rows computed; attended unless
                                arch.attn_mask_enabled) */
  int method;                /* 0 = euler, 1 = midpoint: torchdiffeq's fixed-grid method (odeint_kwargs, cfm.py:39-43,
                                218).  Euler makes `steps` backbone evaluations, midpoint 2 * steps (at t_k and at
                                t_k + dt_k/2).  Any other value is rejected. */
} f5_sample_args;
/* nfe: backbone evaluations of the call — steps for euler, 2 * steps for midpoint.  For MMDiT this is the workspace of
 * a call with nt = N (an upper bound whenever nt < N, as CFM.sample gives for text from list_str_to_idx). */
size_t f5_sample_workspace_bytes(const f5_engine* e, int B, int N, int nfe, float cfg_strength);
/* The workspace of a call with text length nt; equals f5_sample_workspace_bytes for DiT and UNetT.  f5_sample rejects
 * a workspace smaller than this for its nt.  Since f5_version() 107. */
size_t f5_sample_workspace_bytes_nt(const f5_engine* e, int B, int N, int nt, int nfe, float cfg_strength);
int f5_sample(f5_engine* e, const f5_sample_args* args, void* workspace, size_t ws_bytes, f5_stream_t stream);

/* One f5_sample call with classifier-free guidance split over two engines: side 0 computes the conditional half of every
 * backbone evaluation, side 1 the unconditional half, and after each evaluation each side copies the other's half of
 * the flow (B * N * mel fp32 values) into its own workspace and runs the same fused CFG + ODE update.  Both sides then
 * hold the same y; the final y, trajectory and v_out are bit for bit those of f5_sample(e0, a0, ...).
 *   e1 may be e0 (two workspaces on one device) or an engine over the same weights on another device, each workspace
 *   on its engine's device (the device is read from the workspace pointer).  a0 and a1 describe the same problem (B, N,
 *   nt, steps, t, cfg_strength >= 1e-5, method, use_graph, exact_varlen, durations given or not); a1's text, step_cond,
 *   y and duration are copies on side 1's device, its y a buffer of its own, its trajectory and v_out NULL.
 *   stream0 and stream1 must differ; the call is ordered after earlier work on each stream and completes on both: each
 *   stream waits for the other side's last read of its workspace.  Peer access between the two devices is enabled
 *   once per process where the hardware allows it.  Since f5_version() 109. */
int f5_sample_cfg_split(f5_engine* e0, const f5_sample_args* a0, void* ws0, size_t ws0_bytes, f5_stream_t stream0,
                        f5_engine* e1, const f5_sample_args* a1, void* ws1, size_t ws1_bytes, f5_stream_t stream1);
/* workspace of either side of f5_sample_cfg_split (nfe as for f5_sample_workspace_bytes).  Since f5_version() 109. */
size_t f5_sample_cfg_split_workspace_bytes(const f5_engine* e, int B, int N, int nt, int nfe);

/* One backbone evaluation: the reference's operator transformer(x, cond, text, time, mask, drop_audio_cond, drop_text,
 * cfg_infer, cache) (backbones/dit.py:319-370, unett.py:244-307, mmdit.py:198-246) with a time per sample, for samplers
 * outside f5_sample (another ODE method, a solver of the caller's, samples at different times).  Since f5_version() 110.
 *   mode F5_FORWARD_COND: the conditional flow [B, N, mel]; F5_FORWARD_CFG: cond rows then uncond rows [2B, N, mel]
 *   (cfg_infer=True); F5_FORWARD_UNCOND: the unconditional flow [B, N, mel] (drop_audio_cond = drop_text = True).
 *   Each sample's time embedding, AdaLN rows and UNetT time token come from its own time[b]; the cond and uncond rows of
 *   a sample share them.
 *   use_graph: the evaluation runs as one CUDA graph, captured once per (workspace, B, N, nt for MMDiT, mode, duration
 *   given or not) and replayed.  Before it, outside the graph, x and step_cond are packed into the workspace's input
 *   operand and the time embedding and AdaLN rows of `time` are computed there, so new values replay the same graph.
 *   reuse_text: skip the text embeddings and rotary tables and use those the previous f5_forward call on this workspace
 *   computed, even if `text` changed since (the reference's cache=True).  That call must have had the same B, N, nt, mode
 *   and durations given or not, and no f5_sample call may have used the workspace since; otherwise the call fails. */
enum { F5_FORWARD_COND = 0, F5_FORWARD_CFG = 1, F5_FORWARD_UNCOND = 2 };
typedef struct {
  int B, N, nt;
  const float* x;          /* device fp32 [B, N, mel]: the noisy state */
  const float* step_cond;  /* device fp32 [B, N, mel]: the masked cond audio */
  const long long* text;   /* device int64 [B, nt], padded with -1 */
  const int* duration;     /* device int32 [B] = mask.sum(1) (the reference's batched mask semantics), or NULL */
  const float* time;       /* device fp32 [B] */
  int mode;                /* F5_FORWARD_* */
  float* v_out;            /* device fp32 [2B, N, mel] for F5_FORWARD_CFG, else [B, N, mel] */
  int use_graph;
  int reuse_text;
} f5_forward_args;
size_t f5_forward_workspace_bytes(const f5_engine* e, int B, int N, int nt, int mode);
/* number of captured CUDA graphs the engine holds (f5_sample and f5_forward; at most 16).  Since f5_version() 110. */
int f5_engine_graph_count(f5_engine* e);
int f5_forward(f5_engine* e, const f5_forward_args* args, void* workspace, size_t ws_bytes, f5_stream_t stream);

/* algorithmic FLOPs of one f5_sample call making nfe backbone evaluations (SURVEY.md §8d formula) — used by bench.py
 * for the roofline */
double f5_sample_flops(const f5_engine* e, int B, int N, int nfe, float cfg_strength);
/* f5_sample_flops at text length nt: for MMDiT it counts the text stream and the joint attention over N + nt keys;
 * for DiT and UNetT it equals f5_sample_flops.  f5_sample_flops of an MMDiT engine is this at nt = N.  Since
 * f5_version() 107. */
double f5_sample_flops_nt(const f5_engine* e, int B, int N, int nt, int nfe, float cfg_strength);

#ifdef __cplusplus
}
#endif
#endif /* F5TTS_B200_H */

// Engine: the CFM.sample NFE loop (model/cfm.py:160-223) over a DiT (backbones/dit.py:319-370), UNetT
// (backbones/unett.py:244-307) or MMDiT (backbones/mmdit.py:198-246) backbone, expressed as a fixed kernel schedule over a
// caller-owned workspace.
//
// The ODE solver is torchdiffeq's fixed-grid Euler (one backbone evaluation per grid interval, at t_k) or midpoint
// (two: at t_k, then at t_k + dt_k/2 from the half-step state).  `evals` below counts backbone evaluations (NFE):
// steps for Euler, 2 * steps for midpoint.
// Per sample() call (hoisted out of the NFE loop because it is evaluation- or batch-invariant):
//   * text embeddings, cond + uncond variants (dit.py:284-314 caches them the same way)
//   * time embedding of every evaluation time and — DiT — the AdaLN modulation vectors of every (evaluation, block)
//     as one [evals, depth*6D + 2D] table: 22 weight-streaming GEMVs per evaluation become one GEMM per call
//   * the per-evaluation solver table (OdeStage: update coefficient, trajectory row or -1)
//   * rotary cos/sin table, static columns of the packed input projection operand
// Per evaluation: input projection -> grouped conv position embedding x2 (tensor-core implicit GEMM) -> depth x
// {norm+modulate, fused QKV+RoPE GEMM, flash attention, out-proj (+gate, +mask, +residual), norm+modulate,
//  FF1+GELU, FF2 (+gate, +residual)} -> final norm -> proj_out -> fused CFG + ODE stage update.
// MMDiT keeps a second residual stream for the text (c, [Be*nt, D]): per block both streams are normalised and projected
// to QKV, one joint attention runs over [audio | text], and each stream has its own gated out-projection and FF pair (the
// last block computes only the text QKV its audio queries attend to).
// Every kernel reads the evaluation index from a device counter, so one captured CUDA graph serves all evaluations
// of either method: the method reaches the graph only through the tables the prologue writes.
#include <cmath>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <vector>

#include "internal.h"

namespace f5 {

static inline size_t al256(size_t x) { return (x + 255) & ~size_t(255); }

struct Bump {
  uint8_t* base;
  size_t off = 0;
  explicit Bump(void* p) : base(reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 255) & ~uintptr_t(255))) {}
  template <typename T>
  T* take(size_t count) {
    T* r = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += al256(count * sizeof(T));
    return r;
  }
};

// One residual stream of the backbone: the audio rows, or MMDiT's text rows.  Every transformer block runs the same
// norm -> QKV -> attention -> out-projection -> norm -> FF1 -> FF2 sequence over it.
struct TokenStream {
  float* res;                // residual [rows, D]
  __half *a, *qkv, *ao, *g;  // normalised copy, QKV, attention output, FF hidden
  long long rows;            // Be * seq
  int seq;                   // tokens per sample
  float *rope_cos, *rope_sin;  // [seq, dim_head / 2]
  const int* out_len;   // [Be] valid rows of the out-projection (padded rows are zeroed), or null
  const int* skip_len;  // [Be] valid rows when every GEMM skips tiles of padding only, or null
};

struct Layout {
  // sizes
  int B, Be, N, evals, packed;  // evals: backbone evaluations per call (steps, or 2 * steps for midpoint)
  // CFG split (f5_sample_cfg_split): -1 = both halves stacked on the batch axis (f5_sample); 0 / 1 = this workspace
  // computes only the conditional / unconditional half: Be = B rows of work, while xin, v and the MMDiT text embedding
  // keep both halves (Bx = 2B samples) so that the unchanged update kernel runs over the full v
  int half, Bx;
  // f5_forward: the time and modulation tables hold one row per sample (evals = B), and every reader takes the row of
  // its sample (b % B: the cond and uncond rows of a sample share it) instead of the evaluation counter's
  bool per_sample;
  long long M;  // Be * N mel frames (the audio stream's rows without the UNetT time token)
  // common
  int* step_ptr;    // [0]: evaluation counter
  SampleIo* io;     // caller tensors + cfg scale of THIS call, read by the step kernels through the workspace
  OdeStage* stage;  // [evals]
  float* t_dev;     // [evals] evaluation times
  int* row_len;     // [Be] or unused
  int* kv_len;      // [Be] or unused
  int* frame_len;   // [Be] valid mel frames per sample (row_len without the UNetT time token)
  int* valid_len;   // [B]
  float *tfeat, *th1, *temb;
  __half* temb_silu;
  float* mod;
  // text
  float* tx;
  uint8_t* filler;
  __half *ta, *tg;
  float *sumsq, *nx;
  // step buffers
  __half* xin;      // this half's rows of xin_all (= xin_all unless split)
  __half* xin_all;  // [Bx*N, kin]
  float* h0;
  __half *h0h, *c1;
  // audio stream: seq = N (+1 for the UNetT time token); residual is the UNetT residual, DiT / MMDiT: alias of h0.
  // Its row lengths depend on the call's arguments and are set when the plans are built.
  TokenStream x;
  std::vector<float*> skips;
  __half* cat;
  float* v;      // this half's rows of v_all (= v_all unless split)
  float* v_all;  // [Bx*seq, mel]: cond rows, then uncond rows
  float* x_embed;  // DiT long_skip_connection: x after the input embedding [M1, D] (cat(...) goes to `cat`), else null
  float* txu;      // text_embedding_average_upsampling: upsampled text [2B, N, Td], else null
  // MMDiT text stream (all null for DiT / UNetT): nt tokens per sample; out_len = c_len, no tile skipping
  TokenStream c;
  float* c0;      // [Be*nt, D] the text embedding the residual restarts from at every evaluation
  float* c0_all;  // [Bx*nt, D] text embedding of both CFG variants (c0 points at this half's rows)
  int* c_len;     // [Be] valid text tokens per sample (this half's entries of c_len_all [Bx])
  int* c_len_all;
  size_t bytes;
};

}  // namespace f5

using namespace f5;

// One instantiated step graph.  The graph touches only the workspace: the caller's tensors (y, trajectory) and the CFG
// scale reach the kernels through the SampleIo block the prologue writes into the workspace, so the cache key is the
// workspace address plus the shape parameters the layout / kernel plans depend on — a fresh `y` or `trajectory`
// allocation per call no longer forces a re-capture.  The ODE method is not in the key: it only changes the contents
// of the time, modulation and OdeStage tables, which every call's prologue rewrites, while `evals` fixes where those
// tables sit in the workspace.  So Euler over 2S steps and midpoint over S steps replay the same graph, each with its
// own tables, and an Euler and a midpoint call with different `evals` never share one.  Entries are reference-counted:
// a launch in flight on one thread keeps its graph alive while another thread evicts it.
struct GraphHolder {
  cudaGraphExec_t exec = nullptr;
  int nodes = 0;  // kernel/memcpy nodes per replay (for the launch counter)
  ~GraphHolder() {
    if (exec) cudaGraphExecDestroy(exec);
  }
};
struct GraphKey {
  const void* ws;
  int B, N, evals, packed, masked;  // masked: 0 = no lengths, 1 = lengths (reference batched semantics), 2 = exact_varlen
  int nt;  // MMDiT: the text length sets the text-stream layout and plans.  0 for DiT / UNetT, whose graphs do not
           // depend on it (keying them on it would re-capture whenever text lengths differ)
  int half;  // Layout::half: -1 for f5_sample's graph (the whole evaluation), 0 / 1 for one CFG half of a split call
             // (the evaluation up to proj_out: the exchange and the update run outside the graph)
  int forward;  // 1: an f5_forward graph (one evaluation up to proj_out with per-sample modulation rows)
  bool operator==(const GraphKey& o) const {
    return ws == o.ws && B == o.B && N == o.N && evals == o.evals && packed == o.packed && masked == o.masked &&
           nt == o.nt && half == o.half && forward == o.forward;
  }
};
struct GraphEntry {
  GraphKey key;
  std::shared_ptr<GraphHolder> g;
};

// The problem whose text embeddings an f5_forward call left in a workspace (f5_forward_args.reuse_text checks it)
struct TextHeld {
  const void* ws;
  int B, N, nt, mode, masked;
  bool operator==(const TextHeld& o) const {
    return ws == o.ws && B == o.B && N == o.N && nt == o.nt && mode == o.mode && masked == o.masked;
  }
};

struct f5_engine {
  f5_arch arch;
  f5_weights w;
  std::vector<f5_layer_weights> layers;
  std::vector<f5_layer_weights> ctx;  // MMDiT text stream (the f5_ctx_layer_weights in the same slots)
  int inner, modW, kin;
  std::mutex mu;
  std::vector<GraphEntry> graphs;
  std::vector<TextHeld> text_held;  // under mu
};

static constexpr int kDiT = 0, kUNetT = 1, kMMDiT = 2;  // f5_arch.backbone
static constexpr int kSkipConcat = 0, kSkipAdd = 1, kSkipNone = 2;  // f5_arch.skip_type (UNetT skip_connect_type)

// MMDiT: first row of block i's modulation vectors in the AdaLN table ([x: 6D | c: 6D] per block, the last block's c
// part 2D, then norm_out 2D); DiT: [6D] per block, then norm_out
static size_t mod_block(const f5_arch& A, int i) { return (size_t)i * (A.backbone == kMMDiT ? 12 : 6) * A.dim; }

static void take_stream_bufs(const f5_engine* e, Bump& bp, TokenStream& st) {
  st.a = bp.take<__half>((size_t)st.rows * e->arch.dim);
  st.qkv = bp.take<__half>((size_t)st.rows * 3 * e->inner);
  st.ao = bp.take<__half>((size_t)st.rows * e->inner);
  st.g = bp.take<__half>((size_t)st.rows * e->arch.ff_inner);
}

static void plan_layout(const f5_engine* e, Layout& L, void* ws, int B, int N, int nt, int evals, float cfg,
                        int half = -1) {
  const f5_arch& A = e->arch;
  Bump bp(ws);
  L.B = B;
  L.N = N;
  L.evals = evals;
  L.half = half;
  L.per_sample = false;
  L.packed = (cfg < 1e-5f && half < 0) ? 0 : 1;
  L.Be = (L.packed && half < 0) ? 2 * B : B;
  L.Bx = L.packed ? 2 * B : B;
  L.M = (long long)L.Be * N;
  TokenStream& X = L.x;
  X = TokenStream{};
  X.seq = A.backbone == kUNetT ? N + 1 : N;
  X.rows = (long long)L.Be * X.seq;
  const long long M1 = X.rows;
  const int D = A.dim, Td = A.text_dim;
  L.step_ptr = bp.take<int>(64);
  L.io = bp.take<SampleIo>(1);
  L.stage = bp.take<OdeStage>(evals);
  L.t_dev = bp.take<float>(evals);
  X.rope_cos = bp.take<float>((size_t)X.seq * (A.dim_head / 2));
  X.rope_sin = bp.take<float>((size_t)X.seq * (A.dim_head / 2));
  L.row_len = bp.take<int>(L.Be);
  L.kv_len = bp.take<int>(L.Be);
  L.frame_len = bp.take<int>(L.Be);
  L.valid_len = bp.take<int>(B);
  L.tfeat = bp.take<float>((size_t)evals * 256);
  L.th1 = bp.take<float>((size_t)evals * D);
  L.temb = bp.take<float>((size_t)evals * D);
  L.temb_silu = bp.take<__half>((size_t)evals * D);
  L.mod = bp.take<float>((size_t)evals * (e->modW > 0 ? e->modW : 1));
  L.tx = bp.take<float>((size_t)2 * B * N * Td);
  L.filler = bp.take<uint8_t>((size_t)B * N);
  L.ta = bp.take<__half>((size_t)2 * B * N * Td);
  L.tg = bp.take<__half>((size_t)2 * B * N * 2 * Td);
  L.sumsq = bp.take<float>((size_t)2 * B * ((N + kGrnRows - 1) / kGrnRows) * 2 * Td);
  L.nx = bp.take<float>((size_t)2 * B * 2 * Td);
  L.xin_all = bp.take<__half>((size_t)L.Bx * N * e->kin);
  L.xin = L.xin_all + (half > 0 ? (size_t)B * N * e->kin : 0);
  L.h0 = bp.take<float>((size_t)L.M * D);
  L.h0h = bp.take<__half>((size_t)L.M * D);
  L.c1 = bp.take<__half>((size_t)L.M * D);
  L.skips.clear();
  if (A.backbone == kUNetT) {
    // concat and add keep the depth/2 saved rows; only concat has the [x | skip] operand of its combiner GEMM
    X.res = bp.take<float>((size_t)M1 * D);
    if (A.skip_type != kSkipNone)
      for (int i = 0; i < A.depth / 2; ++i) L.skips.push_back(bp.take<float>((size_t)M1 * D));
    L.cat = A.skip_type == kSkipConcat ? bp.take<__half>((size_t)M1 * 2 * D) : nullptr;
  } else {
    X.res = L.h0;
    L.cat = nullptr;
  }
  take_stream_bufs(e, bp, X);
  L.v_all = bp.take<float>((size_t)L.Bx * X.seq * A.mel_dim);
  L.v = L.v_all + (half > 0 ? (size_t)B * X.seq * A.mel_dim : 0);
  // buffers of the architecture options last: with the options off the layout is the one above
  L.x_embed = nullptr;
  if (A.long_skip) {
    L.x_embed = bp.take<float>((size_t)M1 * D);
    L.cat = bp.take<__half>((size_t)M1 * 2 * D);
  }
  L.txu = A.text_avg_upsample ? bp.take<float>((size_t)2 * B * N * Td) : nullptr;
  TokenStream& C = L.c;
  C = TokenStream{};
  L.c0 = L.c0_all = nullptr;
  L.c_len = L.c_len_all = nullptr;
  if (A.backbone == kMMDiT) {
    C.seq = nt;
    C.rows = (long long)L.Be * nt;
    C.res = bp.take<float>((size_t)C.rows * D);
    L.c0_all = bp.take<float>((size_t)L.Bx * nt * D);
    L.c0 = L.c0_all + (half > 0 ? (size_t)B * nt * D : 0);
    take_stream_bufs(e, bp, C);
    C.rope_cos = bp.take<float>((size_t)nt * (A.dim_head / 2));
    C.rope_sin = bp.take<float>((size_t)nt * (A.dim_head / 2));
    L.c_len_all = bp.take<int>(L.Bx);
    L.c_len = L.c_len_all + (half > 0 ? B : 0);
    C.out_len = L.c_len;
  }
  L.bytes = bp.off + 512;
}

extern "C" {

int f5_engine_create(const f5_arch* arch, const f5_weights* weights, f5_engine** out) {
  if (!arch || !weights || !out) {
    set_error("engine_create: null argument");
    return -1;
  }
  if (arch->dim_head != 64 && arch->dim_head != 128) {
    set_error("engine_create: dim_head must be 64 or 128 (got %d)", arch->dim_head);
    return -1;
  }
  if (arch->dim_head == 128 && arch->heads * 128 > 1024) {  // inner = heads * 128 is a multiple of 128
    set_error("engine_create: at dim_head 128, heads * dim_head must be at most 1024 (heads=%d)", arch->heads);
    return -1;
  }
  if (arch->dim % 128 || arch->dim > 1024 || (arch->ff_inner % 64)) {
    set_error("engine_create: dim must be a multiple of 128 and <= 1024, ff_inner a multiple of 64 (dim=%d ff=%d)",
              arch->dim, arch->ff_inner);
    return -1;
  }
  if (arch->conv_layers > 8 || (arch->conv_layers > 0 && (arch->text_dim % 64 || arch->text_dim > 512))) {
    set_error("engine_create: text conv blocks need text_dim %% 64 == 0, <= 512, at most 8 layers");
    return -1;
  }
  if (arch->backbone < kDiT || arch->backbone > kMMDiT) {
    set_error("engine_create: backbone must be 0 (DiT), 1 (UNetT) or 2 (MMDiT), got %d", arch->backbone);
    return -1;
  }
  if (arch->backbone == kMMDiT) {
    if (arch->text_dim || arch->conv_layers || arch->long_skip || arch->text_avg_upsample || arch->pe_attn_head >= 0) {
      set_error("engine_create: MMDiT takes no text_dim, conv_layers, long_skip or text_avg_upsample and applies rope "
                "to every head (pe_attn_head -1); got text_dim=%d conv_layers=%d long_skip=%d text_avg_upsample=%d "
                "pe_attn_head=%d", arch->text_dim, arch->conv_layers, arch->long_skip, arch->text_avg_upsample,
                arch->pe_attn_head);
      return -1;
    }
    if (arch->depth < 1 || weights->ctx_layers == nullptr) {
      set_error("engine_create: MMDiT needs depth >= 1 and ctx_layers");
      return -1;
    }
    for (int i = 0; i < arch->depth; ++i) {
      const f5_ctx_layer_weights& c = weights->ctx_layers[i];
      const bool last = i == arch->depth - 1;
      if (!c.w_qkv_c || !c.b_qkv_c || (!last && (!c.w_out_c || !c.b_out_c || !c.w_ff1_c || !c.b_ff1_c || !c.w_ff2_c ||
                                                 !c.b_ff2_c)) ||
          (arch->qk_norm && (!c.q_norm_c || !c.k_norm_c))) {
        set_error("engine_create: MMDiT text-stream weights missing in layer %d", i);
        return -1;
      }
    }
  }
  if ((arch->long_skip || arch->text_avg_upsample) && arch->backbone != kDiT) {
    set_error("engine_create: long_skip and text_avg_upsample are DiT options");
    return -1;
  }
  if (arch->text_avg_upsample && !arch->text_mask_padding) {
    set_error("engine_create: text_avg_upsample needs text_mask_padding (backbones/dit.py:41-43)");
    return -1;
  }
  if (arch->long_skip && weights->long_skip_w == nullptr) {
    set_error("engine_create: long_skip needs long_skip_w");
    return -1;
  }
  if (arch->skip_type < kSkipConcat || arch->skip_type > kSkipNone || (arch->skip_type && arch->backbone != kUNetT)) {
    set_error("engine_create: skip_type must be 0 (concat), 1 (add) or 2 (none), and non-zero only for UNetT "
              "(backbone %d, skip_type %d)", arch->backbone, arch->skip_type);
    return -1;
  }
  if (arch->backbone == kUNetT && arch->skip_type != kSkipConcat) {
    // every first-half layer pushes x and every later-half layer pops one (unett.py:286-294): an odd depth pops more
    // than it pushed
    if (arch->depth % 2) {
      set_error("engine_create: UNetT skip_type add / none needs an even depth (got %d)", arch->depth);
      return -1;
    }
    for (int i = 0; i < arch->depth; ++i)
      if (weights->layers[i].w_skip != nullptr) {
        set_error("engine_create: UNetT skip_type add / none has no skip projection, but layer %d has w_skip", i);
        return -1;
      }
  }
  if (arch->backbone == kUNetT && arch->skip_type == kSkipConcat)
    for (int i = arch->depth / 2; i < arch->depth; ++i)
      if (weights->layers[i].w_skip == nullptr) {
        set_error("engine_create: UNetT skip_type concat needs w_skip in every later-half layer (layer %d)", i);
        return -1;
      }
  if (arch->qk_norm)
    for (int i = 0; i < arch->depth; ++i)
      if (weights->layers[i].q_norm_w == nullptr || weights->layers[i].k_norm_w == nullptr) {
        set_error("engine_create: qk_norm needs q_norm_w and k_norm_w in every layer (layer %d)", i);
        return -1;
      }
  if (int rc = configure_kernels()) return rc;
  f5_engine* e = new f5_engine();
  e->arch = *arch;
  // ctx_layers is read only for MMDiT: callers built before it existed pass a struct that ends before it
  std::memcpy(&e->w, weights, offsetof(f5_weights, ctx_layers));
  e->w.ctx_layers = nullptr;
  e->layers.assign(weights->layers, weights->layers + arch->depth);
  e->w.layers = e->layers.data();
  e->inner = arch->heads * arch->dim_head;
  e->modW = arch->backbone == kDiT ? arch->depth * 6 * arch->dim + 2 * arch->dim : 0;
  if (arch->backbone == kMMDiT) {
    for (int i = 0; i < arch->depth; ++i) {
      const f5_ctx_layer_weights& c = weights->ctx_layers[i];
      f5_layer_weights lw{};
      lw.w_qkv = c.w_qkv_c, lw.b_qkv = c.b_qkv_c, lw.w_out = c.w_out_c, lw.b_out = c.b_out_c;
      lw.w_ff1 = c.w_ff1_c, lw.b_ff1 = c.b_ff1_c, lw.w_ff2 = c.w_ff2_c, lw.b_ff2 = c.b_ff2_c;
      lw.q_norm_w = c.q_norm_c, lw.k_norm_w = c.k_norm_c;
      e->ctx.push_back(lw);
    }
    e->modW = (int)mod_block(*arch, arch->depth - 1) + 8 * arch->dim + 2 * arch->dim;
  }
  e->kin = weights->proj_kpad;
  if (e->kin % 64 || e->kin < 2 * arch->mel_dim + arch->text_dim) {
    set_error("engine_create: proj_kpad must be a multiple of 64 covering 2*mel + text_dim");
    delete e;
    return -1;
  }
  *out = e;
  return 0;
}

void f5_engine_destroy(f5_engine* e) {
  if (!e) return;
  delete e;  // graph holders destroy their executables
}

size_t f5_sample_workspace_bytes_nt(const f5_engine* e, int B, int N, int nt, int nfe, float cfg_strength) {
  Layout L;
  plan_layout(e, L, nullptr, B, N, nt, nfe, cfg_strength);
  return L.bytes;
}

size_t f5_sample_workspace_bytes(const f5_engine* e, int B, int N, int nfe, float cfg_strength) {
  return f5_sample_workspace_bytes_nt(e, B, N, N, nfe, cfg_strength);
}

double f5_sample_flops_nt(const f5_engine* e, int B, int N, int nt, int nfe, float cfg_strength) {
  const f5_arch& A = e->arch;
  const double D = A.dim, mel = A.mel_dim, Td = A.text_dim, F = A.ff_inner, Ld = A.depth;
  // attention width heads * dim_head: QKV 6 n D I + out-projection 2 n I D, QK^T + PV 4 n^2 I.  At dim_head 64 the
  // DiT / UNetT count keeps the form it always had (I = D, as in every shipped config), so figures reported before stay
  // comparable.
  const double I = A.backbone != kMMDiT && A.dim_head == 64 ? D : double(e->inner);
  const double Be = cfg_strength < 1e-5f ? B : 2.0 * B;
  double per;  // one sample-forward
  if (A.backbone == kMMDiT) {
    const double n = N, m = nt;
    // every block: audio QKV + out + FF; text QKV; joint attention (QK^T + PV) of the audio queries over N + nt keys.
    // Every block but the last: text out + FF and the text queries' attention.
    per = Ld * (8.0 * n * D * I + 4.0 * n * D * F + 6.0 * m * D * I + 4.0 * n * (n + m) * I) +
          (Ld - 1.0) * (2.0 * m * I * D + 4.0 * m * D * F + 4.0 * m * (n + m) * I);
    per += 2.0 * n * (2 * mel) * D + 2.0 * (2.0 * n * D * (D / 16.0) * 31.0) + 2.0 * n * D * mel;
  } else if (A.backbone == kDiT) {
    const double n = N;
    per = Ld * (8.0 * n * D * I + 4.0 * n * D * F + 4.0 * n * n * I) + 2.0 * n * (2 * mel + Td) * D +
          2.0 * (2.0 * n * D * (D / 16.0) * 31.0) + 2.0 * n * D * mel;
    if (A.long_skip) per += 2.0 * n * D * (2.0 * D);  // long_skip_connection: Linear(2D -> D)
  } else {
    const double n1 = N + 1.0, n = N;
    // concat: the combiner Linear(2D -> D) of every later-half layer; add and none have no GEMM there
    const double combiner = A.skip_type == kSkipConcat ? (Ld / 2.0) * 4.0 * n1 * D * D : 0.0;
    per = Ld * (8.0 * n1 * D * I + 4.0 * n1 * D * F + 4.0 * n1 * n1 * I) + combiner +
          2.0 * n * (2 * mel + Td) * D + 2.0 * (2.0 * n * D * (D / 16.0) * 31.0) + 2.0 * n1 * D * mel;
  }
  double total = nfe * Be * per;
  // text embedding, once per sample and CFG branch: conv_layers x (2 pointwise GEMMs); none in MMDiT
  total += 2.0 * B * A.conv_layers * (2.0 * 2.0 * N * Td * 2.0 * Td);
  // conditioning: time MLP + AdaLN table, one row per evaluation, computed once per call
  total += nfe * (2.0 * 256 * D + 2.0 * D * D + 2.0 * D * (double)e->modW);
  return total;
}

double f5_sample_flops(const f5_engine* e, int B, int N, int nfe, float cfg_strength) {
  return f5_sample_flops_nt(e, B, N, N, nfe, cfg_strength);
}

}  // extern "C"

// -------------------------------------------------------------------------------------------------------------
namespace {

struct BlockPlans {
  GemmPlan qkv, oproj, ff1, ff2;
  GemmPlan skip;  // UNetT later-half layers with skip_type concat: the combiner GEMM
};

struct StepPlans {
  GemmPlan proj, conv1, conv2, out_proj, long_skip;
  std::vector<BlockPlans> x, c;  // per layer: the audio stream, the MMDiT text stream
  std::vector<AttnPlan> attn;  // identical per layer, kept once (MMDiT: one with text queries, one for the last block)
};

#define RC(x)                \
  do {                       \
    int _rc = (x);           \
    if (_rc) return _rc;     \
  } while (0)

f5_gemm_args base_args(long long rows, int n_out, int k, int lda, int ldw, int bn, int epi, int act) {
  f5_gemm_args a{};
  a.weights_static = 1;  // every W the engine multiplies by is a packed model weight
  a.rows = (int)rows;
  a.batches = 1;
  a.n_out = n_out;
  a.k = k;
  a.lda = lda;
  a.ldw = ldw;
  a.bn = bn;
  a.epi = epi;
  a.act = act;
  return a;
}

constexpr int kAutoTile = 0;  // bn = 0: the GEMM planner picks the tile shape per problem (gemm.cu: pick_tile)

// f5_forward: a gated residual GEMM reads the AdaLN gate row of each output row's sample (EPI_RESID_SAMPLE).  The tile
// width stays the one the planner picked for EPI_RESID, so each output element is computed exactly as in f5_sample.
void gate_per_sample(const Layout& L, const TokenStream& st, GemmPlan& pl) {
  if (!L.per_sample || pl.p.gate == nullptr) return;
  pl.epi = EPI_RESID_SAMPLE;
  pl.p.gate_seq = st.seq;
  pl.p.gate_samples = L.B;
}

// The four GEMMs of one block of one stream: QKV (+ per-head RMSNorm) + RoPE on the first pe_heads heads, out-projection
// (+ gate, + zeroed padded rows, + residual), FF1 + GELU, FF2 (+ gate, + residual).  m: the block's AdaLN vectors of
// this stream (gates at 2D and 5D), or null (UNetT: no gates).  qkv_only: MMDiT's last text block (context_pre_only).
// The MMDiT text stream (modules.py:783-846 with context_dim = dim) ropes text positions 0..nt-1 on every head, zeroes
// its padded rows in the out-projection (c_mask, modules.py:700-703) and computes every row.
int plan_block(const f5_engine* e, const Layout& L, const TokenStream& st, const f5_layer_weights& lw, const float* m,
               int pe_heads, bool qkv_only, BlockPlans& P) {
  const f5_arch& A = e->arch;
  const int D = A.dim, F = A.ff_inner, inner = e->inner;
  auto varlen = [&](f5_gemm_args& a) {
    if (!st.skip_len) return;
    a.row_len = st.skip_len;
    a.seq = st.seq;
    a.skip_padded_tiles = 1;
  };
  auto gate = [&](f5_gemm_args& a, int off) {
    if (!m) return;
    a.gate = m + off * D;
    a.step_ptr = L.step_ptr;
    a.gate_step_stride = e->modW;
  };
  {
    f5_gemm_args a = base_args(st.rows, 3 * inner, D, D, D, kAutoTile, A.qk_norm ? F5_EPI_QKV_NORM_ROPE : F5_EPI_QKV_ROPE,
                               F5_ACT_NONE);
    a.q_norm = lw.q_norm_w;
    a.k_norm = lw.k_norm_w;
    a.bias = lw.b_qkv;
    a.out = st.qkv;
    a.ldo = 3 * inner;
    a.seq = st.seq;
    a.rope_cos = st.rope_cos;
    a.rope_sin = st.rope_sin;
    a.inner = inner;
    a.pe_heads = pe_heads;
    a.dim_head = A.dim_head;
    varlen(a);
    RC(gemm_plan(&P.qkv, st.a, lw.w_qkv, &a));
  }
  if (qkv_only) return 0;
  {
    f5_gemm_args a = base_args(st.rows, D, inner, inner, inner, kAutoTile, F5_EPI_RESID, F5_ACT_NONE);
    a.bias = lw.b_out;
    a.resid = st.res;
    a.ldo = D;
    a.seq = st.seq;
    a.row_len = st.out_len;
    gate(a, 2);
    varlen(a);
    RC(gemm_plan(&P.oproj, st.ao, lw.w_out, &a));
    gate_per_sample(L, st, P.oproj);
  }
  {
    f5_gemm_args a = base_args(st.rows, F, D, D, D, kAutoTile, F5_EPI_F16, F5_ACT_GELU_TANH);
    a.bias = lw.b_ff1;
    a.out = st.g;
    a.ldo = F;
    varlen(a);
    RC(gemm_plan(&P.ff1, st.a, lw.w_ff1, &a));
  }
  {
    f5_gemm_args a = base_args(st.rows, D, F, F, F, kAutoTile, F5_EPI_RESID, F5_ACT_NONE);
    a.bias = lw.b_ff2;
    a.resid = st.res;
    a.ldo = D;
    gate(a, 5);
    varlen(a);
    RC(gemm_plan(&P.ff2, st.g, lw.w_ff2, &a));
    gate_per_sample(L, st, P.ff2);
  }
  return 0;
}

int build_step_plans(f5_engine* e, const Layout& L, const f5_sample_args* sa, StepPlans& P) {
  const f5_arch& A = e->arch;
  const f5_weights& W = e->w;
  const int D = A.dim;
  const long long M1 = L.x.rows;
  const bool mmdit = A.backbone == kMMDiT;
  const bool masked = sa->duration != nullptr;
  const bool strict = masked && sa->exact_varlen;  // every sample exactly as if alone in the batch (f5_sample_args)
  // input projection / conv position embedding see per-sample lengths (MMDiT's AudioEmbedding takes no mask,
  // backbones/mmdit.py:67-78: only exact_varlen confines it)
  const bool mask_in = (A.backbone == kDiT && masked) || strict;

  {  // input projection: h0 = xin . proj_w^T + b ; h0h = fp16(mask(h0))
    f5_gemm_args a = base_args(L.M, D, e->kin, e->kin, e->kin, 128, F5_EPI_F32, F5_ACT_NONE);
    a.bias = W.proj_b;
    a.out = L.h0;
    a.out16b = L.h0h;
    a.ldo = D;
    a.seq = L.N;
    a.row_len = mask_in ? L.frame_len : nullptr;
    a.skip_padded_tiles = (mask_in && (A.attn_mask_enabled || strict)) ? 1 : 0;
    RC(gemm_plan(&P.proj, L.xin, W.proj_w, &a));
  }
  for (int c = 0; c < 2; ++c) {  // grouped conv position embedding
    f5_gemm_args a{};
    a.weights_static = 1;
    a.rows = L.N;
    a.batches = L.Be;
    a.n_out = D;
    a.k = D / 16;  // ConvPositionEmbedding(groups=16): channels per group
    a.lda = D;
    a.conv_taps = 31;
    a.act = F5_ACT_MISH;
    a.bias = W.conv_b[c];
    a.ldo = D;
    a.seq = L.N;
    a.row_len = mask_in ? L.frame_len : nullptr;
    a.skip_padded_tiles = (mask_in && (A.attn_mask_enabled || strict)) ? 1 : 0;
    if (c == 0) {
      a.epi = F5_EPI_F16;
      a.out = L.c1;
      RC(gemm_plan(&P.conv1, L.h0h, W.conv_w[0], &a));
    } else {
      a.epi = F5_EPI_RESID;
      a.resid = L.h0;
      RC(gemm_plan(&P.conv2, L.c1, W.conv_w[1], &a));
    }
  }
  // Variable-length execution (SURVEY.md §8f-1): in the reference's key-masked mode (attn_mask_enabled, modules.py:
  // 513-518) padded rows influence nothing, so every GEMM / conv / attention tile that holds only padding is skipped.
  // In the default "faithful" mode padded keys ARE attended (SURVEY.md §0.5) and every row must be computed.
  const int key_mask = (masked && (A.attn_mask_enabled || strict)) ? 1 : 0;
  // MMDiT's conv position embedding reads padded audio rows (no mask, mmdit.py:67-78), and those rows evolve with the
  // ODE like any other: outside exact_varlen they must be computed in full.  UNetT's conv is unmasked too
  // (unett.py:90-102); add and none compute every row the same way, concat keeps the tile skipping it always had.
  const bool unmasked_conv = mmdit || (A.backbone == kUNetT && A.skip_type != kSkipConcat);
  const int skip = unmasked_conv ? (strict ? 1 : 0) : key_mask;
  TokenStream X = L.x;
  X.out_len = masked ? L.row_len : nullptr;
  X.skip_len = skip ? L.row_len : nullptr;
  const int pe_heads = A.pe_attn_head < 0 ? A.heads : A.pe_attn_head;
  P.x.resize(A.depth);
  for (int i = 0; i < A.depth; ++i) {
    const f5_layer_weights& lw = e->layers[i];
    if (A.backbone != kDiT && lw.w_skip) {
      f5_gemm_args a = base_args(M1, D, 2 * D, 2 * D, 2 * D, 128, F5_EPI_F32, F5_ACT_NONE);
      a.out = X.res;
      a.ldo = D;
      RC(gemm_plan(&P.x[i].skip, L.cat, lw.w_skip, &a));  // (EPI_F32 direct-store path: not tile-skipped)
    }
    const float* m = A.backbone == kUNetT ? nullptr : L.mod + mod_block(A, i);  // DiT and MMDiT: AdaLN gates
    RC(plan_block(e, L, X, lw, m, pe_heads, false, P.x[i]));
  }
  if (A.long_skip) {  // x = cat(x, x_embed) . long_skip_w^T, no bias (backbones/dit.py:228, 363-364)
    f5_gemm_args a = base_args(M1, D, 2 * D, 2 * D, 2 * D, 128, F5_EPI_F32, F5_ACT_NONE);
    a.out = X.res;
    a.ldo = D;
    RC(gemm_plan(&P.long_skip, L.cat, W.long_skip_w, &a));
  }
  {
    f5_gemm_args a = base_args(M1, A.mel_dim, D, D, D, 128, F5_EPI_F32, F5_ACT_NONE);
    a.bias = W.out_b;
    a.out = L.v;
    a.ldo = A.mel_dim;
    RC(gemm_plan(&P.out_proj, X.a, W.out_w, &a));
  }
  P.attn.resize(1);
  if (mmdit) {
    P.c.resize(A.depth);
    for (int i = 0; i < A.depth; ++i)
      RC(plan_block(e, L, L.c, e->ctx[i], L.mod + mod_block(A, i) + 6 * D, A.heads, i == A.depth - 1, P.c[i]));
    // joint attention: [0] for the blocks with text queries, [1] for the last block, whose text output is discarded
    P.attn.resize(2);
    for (int last = 0; last < 2; ++last)
      RC(attn_joint_plan(&P.attn[last], X.qkv, L.c.qkv, X.ao, L.c.ao, L.Be, X.seq, L.c.seq, A.heads, A.dim_head,
                         key_mask ? L.kv_len : nullptr, key_mask ? L.c_len : nullptr, last ? 0 : 1,
                         1.0f / sqrtf((float)A.dim_head)));
    return 0;
  }
  RC(attn_plan(&P.attn[0], X.qkv, X.ao, L.Be, X.seq, A.heads, A.dim_head, key_mask ? L.kv_len : nullptr,
               1.0f / sqrtf((float)A.dim_head)));
  return 0;
}

// Instrumented build (make TRACE=1) only: F5_DIAG_SKIP="norm,attn,qkv,out,ff1,ff2,conv" removes kernels from the step
// schedule (timing decomposition; results are wrong).  The production library has no such switch.
#ifdef F5_TRACE
static bool diag_skip(const char* what) {
  static const char* v = getenv("F5_DIAG_SKIP");
  return v != nullptr && strstr(v, what) != nullptr;
}
#else
static constexpr bool diag_skip(const char*) { return false; }
#endif

int norm_mod(const f5_engine* e, const Layout& L, const TokenStream& st, int mode, const float* a, const float* b,
             bool step_indexed, cudaStream_t s, const float* skip = nullptr) {
  NormParams p{};
  p.skip = skip;
  p.x = st.res;
  p.out = st.a;
  p.rows = (int)st.rows;
  p.D = e->arch.dim;
  p.eps = 1e-6f;
  p.a = a;
  p.b = b;
  p.step_ptr = step_indexed && !L.per_sample ? L.step_ptr : nullptr;
  p.step_stride = step_indexed ? e->modW : 0;
  if (step_indexed && L.per_sample) {  // AdaLN (mode 0) with the row of each row's sample
    mode = 4;
    p.sample_seq = st.seq;
    p.samples = L.B;
  }
  p.params_static = 1;  // modulation table / gains: complete long before the GEMM that produces x
  if (diag_skip("norm")) return 0;
  return run_row_norm(mode, p, s);
}

int gemm_step(const GemmPlan& plan, const char* what, cudaStream_t s) {
  return diag_skip(what) ? 0 : gemm_run(plan, s);
}

// Norm -> FF1 -> FF2 of one stream: AdaLN with the block's vectors m (scale_mlp, shift_mlp), or, m null, UNetT's
// RMSNorm with gain g
int run_ff(const f5_engine* e, const Layout& L, const TokenStream& st, const BlockPlans& bp, const float* m,
           const float* g, cudaStream_t s) {
  const int D = e->arch.dim;
  RC(m ? norm_mod(e, L, st, 0, m + 4 * D, m + 3 * D, true, s) : norm_mod(e, L, st, 2, g, nullptr, false, s));
  RC(gemm_step(bp.ff1, "ff1", s));
  return gemm_step(bp.ff2, "ff2", s);
}

// One transformer block.  MMDiT (modules.py:806-846) runs the text stream beside the audio stream: both streams' AdaLN
// and QKV, one joint attention, then the text stream's gated out-projection and FF pair before the audio stream's FF
// pair (the last block computes only the text QKV).
int run_block(f5_engine* e, const Layout& L, const StepPlans& P, int i, cudaStream_t s) {
  const f5_arch& A = e->arch;
  const int D = A.dim;
  const bool mmdit = A.backbone == kMMDiT, last = i == A.depth - 1;
  const f5_layer_weights& lw = e->layers[i];
  const float* mx = A.backbone == kUNetT ? nullptr : L.mod + mod_block(A, i);
  const float* mc = mmdit ? mx + 6 * D : nullptr;
  if (mx) {
    RC(norm_mod(e, L, L.x, 0, mx + D, mx, true, s));  // scale_msa, shift_msa
  } else if (A.skip_type == kSkipAdd && i >= A.depth / 2) {
    // x += skip and attn_norm in one pass over the rows (row norm mode 3)
    RC(norm_mod(e, L, L.x, 3, lw.g_attn, nullptr, false, s, L.skips[A.depth - 1 - i]));
  } else {
    if (A.skip_type != kSkipNone && i < A.depth / 2) {
      RC(check_cuda(cudaMemcpyAsync(L.skips[i], L.x.res, sizeof(float) * L.x.rows * D, cudaMemcpyDeviceToDevice, s),
                    "skip copy"));
    } else if (A.skip_type == kSkipConcat) {
      RC(run_concat_half(L.x.res, L.skips[A.depth - 1 - i], L.cat, L.x.rows, D, s));
      RC(gemm_run(P.x[i].skip, s));
    }
    RC(norm_mod(e, L, L.x, 2, lw.g_attn, nullptr, false, s));
  }
  if (mmdit)  // last: AdaLayerNorm_Final (scale, shift)
    RC(last ? norm_mod(e, L, L.c, 0, mc, mc + D, true, s) : norm_mod(e, L, L.c, 0, mc + D, mc, true, s));
  RC(gemm_step(P.x[i].qkv, "qkv", s));
  if (mmdit) RC(gemm_step(P.c[i].qkv, "qkv", s));
  if (!diag_skip("attn")) RC(attn_run(P.attn[mmdit && last ? 1 : 0], s));
  RC(gemm_step(P.x[i].oproj, "out", s));
  if (mmdit && !last) {
    RC(gemm_step(P.c[i].oproj, "out", s));
    RC(run_ff(e, L, L.c, P.c[i], mc, nullptr, s));
  }
  return run_ff(e, L, L.x, P.x[i], mx, lw.g_ff, s);
}

// One backbone evaluation up to and including proj_out: v (this layout's half of it when split) holds the flow
int run_body(f5_engine* e, const Layout& L, const StepPlans& P, cudaStream_t s) {
  const f5_arch& A = e->arch;
  const int D = A.dim;
  RC(gemm_run(P.proj, s));
  if (!diag_skip("conv")) {
    RC(gemm_run(P.conv1, s));
    RC(gemm_run(P.conv2, s));
  }
  if (A.backbone == kUNetT)
    RC(L.per_sample ? run_prepend_time_token_per_sample(L.x.res, L.h0, L.temb, L.B, L.N, D, L.x.rows, s)
                    : run_prepend_time_token(L.x.res, L.h0, L.temb, L.step_ptr, L.N, D, L.x.rows, s));
  if (A.backbone == kMMDiT) {
    // the text stream restarts from its embedding at every evaluation (get_input_embed, mmdit.py:177-196)
    RC(check_cuda(cudaMemcpyAsync(L.c.res, L.c0, sizeof(float) * L.c.rows * D, cudaMemcpyDeviceToDevice, s),
                  "text stream copy"));
  }
  if (A.long_skip)
    RC(check_cuda(cudaMemcpyAsync(L.x_embed, L.x.res, sizeof(float) * L.x.rows * D, cudaMemcpyDeviceToDevice, s),
                  "long skip copy"));
  for (int i = 0; i < A.depth; ++i) RC(run_block(e, L, P, i, s));
  if (A.long_skip) {
    RC(run_concat_half(L.x.res, L.x_embed, L.cat, L.x.rows, D, s));
    RC(gemm_run(P.long_skip, s));
  }
  if (A.backbone == kUNetT) {
    RC(norm_mod(e, L, L.x, 2, e->w.g_out, nullptr, false, s));
  } else {
    const float* m = L.mod + (e->modW - 2 * D);
    RC(norm_mod(e, L, L.x, 0, m, m + D, true, s));  // AdaLayerNorm_Final: scale, shift (modules.py:342-347)
  }
  return gemm_run(P.out_proj, s);
}

// The fused CFG + ODE stage update over the full v (both halves), rewriting the x columns of every row of xin
int run_update(const f5_engine* e, const Layout& L, cudaStream_t s) {
  const f5_arch& A = e->arch;
  EulerParams ep{};
  ep.io = L.io;
  ep.v = L.v_all;
  ep.xin = L.xin_all;
  ep.stage = L.stage;
  ep.step_ptr = L.step_ptr;
  ep.BN = L.B * L.N;
  ep.mel = A.mel_dim;
  ep.Kpad = e->kin;
  ep.packed = L.packed;
  ep.N = L.N;
  ep.seq_tok = L.x.seq;
  ep.tok_off = A.backbone == kUNetT ? 1 : 0;
  ep.B = L.B;
  return run_cfg_euler(ep, s);
}

int run_step(f5_engine* e, const Layout& L, const StepPlans& P, cudaStream_t s) {
  RC(run_body(e, L, P, s));
  return run_update(e, L, s);
}

// Per-sample lengths of a call with durations (device int32 [B]): row, key, frame and valid lengths, and the buffer clears
// that tile skipping relies on
int set_lengths(f5_engine* e, const Layout& L, const int* duration, bool exact_varlen, cudaStream_t s) {
  const f5_arch& A = e->arch;
  const int D = A.dim, B = L.B;
  // row_len[Be] = duration (+1 for the UNetT time token, unett.py:274-275); kv_len likewise
  std::vector<int> hd(B);
  RC(check_cuda(cudaMemcpyAsync(hd.data(), duration, sizeof(int) * B, cudaMemcpyDeviceToHost, s), "dur d2h"));
  RC(check_cuda(cudaStreamSynchronize(s), "dur sync"));
  std::vector<int> rl(L.Be);
  for (int i = 0; i < L.Be; ++i) rl[i] = hd[i % B] + (A.backbone == kUNetT ? 1 : 0);
  RC(check_cuda(cudaMemcpyAsync(L.row_len, rl.data(), sizeof(int) * L.Be, cudaMemcpyHostToDevice, s), "row_len"));
  RC(check_cuda(cudaMemcpyAsync(L.kv_len, rl.data(), sizeof(int) * L.Be, cudaMemcpyHostToDevice, s), "kv_len"));
  RC(check_cuda(cudaMemcpyAsync(L.valid_len, hd.data(), sizeof(int) * B, cudaMemcpyHostToDevice, s), "valid_len"));
  std::vector<int> fl(L.Be);
  for (int i = 0; i < L.Be; ++i) fl[i] = hd[i % B];
  RC(check_cuda(cudaMemcpyAsync(L.frame_len, fl.data(), sizeof(int) * L.Be, cudaMemcpyHostToDevice, s), "frame_len"));
  RC(check_cuda(cudaStreamSynchronize(s), "len sync"));
  if (A.attn_mask_enabled || exact_varlen) {
    // tile skipping leaves padded rows of these buffers unwritten for the whole call: the conv inputs must read as
    // zero there (= the conv's padding), and q/k/v rows next to a sample's end are multiplied by P = 0 (must be finite)
    RC(check_cuda(cudaMemsetAsync(L.h0h, 0, sizeof(__half) * L.M * D, s), "h0h clear"));
    RC(check_cuda(cudaMemsetAsync(L.c1, 0, sizeof(__half) * L.M * D, s), "c1 clear"));
    RC(check_cuda(cudaMemsetAsync(L.x.qkv, 0, sizeof(__half) * L.x.rows * 3 * e->inner, s), "qkv clear"));
  }
  return 0;
}

// Time embedding of the L.evals times in t_dev (modules.py:852-862) and, DiT / MMDiT, their rows of the AdaLN table
int run_time_embed(f5_engine* e, const Layout& L, cudaStream_t s) {
  const f5_arch& A = e->arch;
  const f5_weights& W = e->w;
  const int D = A.dim, S = L.evals;
  RC(run_time_features(L.t_dev, L.tfeat, S, 256, s));
  RC(run_small_linear(1, L.tfeat, reinterpret_cast<const __half*>(W.time_w0), W.time_b0, L.th1, S, 256, D, s));
  RC(run_small_linear(0, L.th1, reinterpret_cast<const __half*>(W.time_w1), W.time_b1, L.temb, S, D, D, s));
  if (A.backbone == kDiT || A.backbone == kMMDiT) {
    RC(run_silu_to_half(L.temb, L.temb_silu, (long long)S * D, s));
    f5_gemm_args a = base_args(S, e->modW, D, D, D, 128, F5_EPI_F32, F5_ACT_NONE);
    a.bias = W.mod_b;
    a.out = L.mod;
    a.ldo = e->modW;
    GemmPlan pl;
    RC(gemm_plan(&pl, L.temb_silu, W.mod_w, &a));
    RC(gemm_run(pl, s));
  }
  return 0;
}

// Text embedding of both CFG variants (dit.py:86-139 / unett.py:55-84; MMDiT: mmdit.py:42-60 and its rope table).
// masked: durations were given (set_lengths wrote valid_len); strict: exact_varlen.
int run_text_embed(f5_engine* e, const Layout& L, const long long* text, int nt, bool masked, bool strict,
                   cudaStream_t s) {
  const f5_arch& A = e->arch;
  const f5_weights& W = e->w;
  const int D = A.dim, Td = A.text_dim, B = L.B, N = L.N;
  const bool dit = A.backbone == kDiT;
  const bool mmdit = A.backbone == kMMDiT;
  if (mmdit) {  // text embedding of both CFG variants and the text rope table; no text columns in the input projection
    RC(run_mmdit_text_embed(text, B, L.Bx, L.c.seq, D, W.text_table, A.text_num_embeds + 1, A.text_mask_padding,
                            L.c0_all, L.c_len_all, s));
    RC(run_rope_table(L.c.rope_cos, L.c.rope_sin, L.c.seq, A.dim_head / 2, s));
  }
  TextGatherParams tp{};
  tp.ids = text;
  tp.B = B;
  tp.nt = nt;
  tp.N = N;
  tp.Td = Td;
  tp.valid_len = (dit && masked) ? L.valid_len : nullptr;
  tp.table = W.text_table;
  tp.num_embeds = A.text_num_embeds + 1;
  tp.add_pos = A.conv_layers > 0;
  tp.out = L.tx;
  tp.filler = L.filler;
  if (!mmdit) RC(run_text_gather(tp, s));
  const int R2 = 2 * B * N;
  for (int i = 0; i < A.conv_layers; ++i) {
    if (A.text_mask_padding) RC(run_mask_rows(L.tx, L.filler, B * N, R2, Td, s));
    DwConvLnParams dp{};
    dp.x = L.tx;
    dp.out = L.ta;
    dp.B = 2 * B;
    dp.N = N;
    dp.C = Td;
    dp.w = W.text_blocks[i].dw_w;
    dp.wb = W.text_blocks[i].dw_b;
    dp.ln_w = W.text_blocks[i].ln_w;
    dp.ln_b = W.text_blocks[i].ln_b;
    dp.eps = 1e-6f;
    RC(run_dwconv7_ln(dp, s));
    f5_gemm_args g1 = base_args(R2, 2 * Td, Td, Td, Td, 128, F5_EPI_F16, F5_ACT_GELU_ERF);
    g1.bias = W.text_blocks[i].pw1_b;
    g1.out = L.tg;
    g1.ldo = 2 * Td;
    RC(f5_gemm(L.ta, W.text_blocks[i].pw1_w, &g1, s));
    // exact_varlen: the sequence ends at the sample's own length — rows past it take no part in GRN's norm over the
    // sequence (modules.py:243) and are cleared again after the block (= the zero padding a B = 1 call would see)
    if (strict) RC(run_mask_rows_len_half(L.tg, L.valid_len, B, N, R2, 2 * Td, s));
    RC(run_grn(L.tg, L.sumsq, L.nx, W.text_blocks[i].grn_gamma, W.text_blocks[i].grn_beta, 2 * B, N, 2 * Td, s));
    f5_gemm_args g2 = base_args(R2, Td, 2 * Td, 2 * Td, 2 * Td, 64, F5_EPI_RESID, F5_ACT_NONE);
    g2.bias = W.text_blocks[i].pw2_b;
    g2.resid = L.tx;
    g2.ldo = Td;
    RC(f5_gemm(L.tg, W.text_blocks[i].pw2_w, &g2, s));
    if (strict) RC(run_mask_rows_len(L.tx, L.valid_len, B, N, R2, Td, s));
  }
  if (A.conv_layers > 0 && A.text_mask_padding) RC(run_mask_rows(L.tx, L.filler, B * N, R2, Td, s));
  if (A.text_avg_upsample)  // audio lengths: duration (the reference's seq_len = mask.sum), else N
    RC(run_text_avg_upsample(L.tx, L.txu, L.filler, masked ? L.valid_len : nullptr, B, N, nt, Td, s));
  return 0;
}

// xin = [x | cond or 0 | text embedding | 0] of every packed row
int run_pack(f5_engine* e, const Layout& L, const float* y, const float* step_cond, cudaStream_t s) {
  const f5_arch& A = e->arch;
  PackParams pp{};
  pp.xin = L.xin_all;
  pp.B = L.B;
  pp.N = L.N;
  pp.mel = A.mel_dim;
  pp.Td = A.text_dim;
  pp.Kpad = e->kin;
  pp.packed = L.packed;
  pp.y = y;
  pp.step_cond = step_cond;
  pp.text = A.text_avg_upsample ? L.txu : L.tx;
  return run_pack_input(pp, s);
}

int run_prologue(f5_engine* e, const Layout& L, const f5_sample_args* sa, cudaStream_t s) {
  const f5_arch& A = e->arch;
  const int N = L.N, S = L.evals;
  const bool masked = sa->duration != nullptr;
  const bool strict = masked && sa->exact_varlen;
  // small host -> device control data (pageable source: cudaMemcpyAsync stages it before returning).
  // Per grid interval k (torchdiffeq's fixed-grid solvers): Euler evaluates at t_k and commits y + dt_k * g; midpoint
  // evaluates at t_k, forms y + half_dt_k * g as the next evaluation's input only, then evaluates at t_k + half_dt_k
  // and commits y + dt_k * g.  Times are fp32 (the reference builds the grid in the parameter dtype).
  std::vector<OdeStage> stage;
  std::vector<float> te;
  stage.reserve(S);
  te.reserve(S);
  for (int k = 0; k < sa->steps; ++k) {
    const float dt = sa->t[k + 1] - sa->t[k];
    if (sa->method == 1) {
      const float half_dt = 0.5f * dt;
      te.push_back(sa->t[k]);
      stage.push_back(OdeStage{half_dt, -1});
      te.push_back(sa->t[k] + half_dt);
      stage.push_back(OdeStage{dt, k + 1});
    } else {
      te.push_back(sa->t[k]);
      stage.push_back(OdeStage{dt, k + 1});
    }
  }
  RC(check_cuda(cudaMemcpyAsync(L.stage, stage.data(), sizeof(OdeStage) * S, cudaMemcpyHostToDevice, s), "stage h2d"));
  RC(check_cuda(cudaMemcpyAsync(L.t_dev, te.data(), sizeof(float) * S, cudaMemcpyHostToDevice, s), "t h2d"));
  RC(check_cuda(cudaMemsetAsync(L.step_ptr, 0, sizeof(int) * 64, s), "step memset"));
  SampleIo io{sa->y, sa->trajectory, sa->cfg_strength};
  RC(check_cuda(cudaMemcpyAsync(L.io, &io, sizeof(io), cudaMemcpyHostToDevice, s), "io h2d"));
  if (masked) RC(set_lengths(e, L, sa->duration, sa->exact_varlen != 0, s));
  RC(run_rope_table(L.x.rope_cos, L.x.rope_sin, L.x.seq, A.dim_head / 2, s));
  RC(run_time_embed(e, L, s));  // every evaluation time
  RC(run_text_embed(e, L, sa->text, sa->nt, masked, strict, s));
  RC(run_pack(e, L, sa->y, sa->step_cond, s));
  if (sa->trajectory)
    RC(check_cuda(cudaMemcpyAsync(sa->trajectory, sa->y, sizeof(float) * L.B * N * A.mel_dim, cudaMemcpyDeviceToDevice, s),
                  "trajectory[0]"));
  return 0;
}

int copy_v_out(const f5_engine* e, const Layout& L, const f5_sample_args* sa, cudaStream_t s) {
  if (!sa->v_out) return 0;
  const int mel = e->arch.mel_dim;
  const int off = e->arch.backbone == kUNetT ? 1 : 0;
  for (int b = 0; b < L.Bx; ++b)
    RC(check_cuda(cudaMemcpyAsync(sa->v_out + (size_t)b * L.N * mel, L.v_all + ((size_t)b * L.x.seq + off) * mel,
                                  sizeof(float) * L.N * mel, cudaMemcpyDeviceToDevice, s),
                  "v_out copy"));
  return 0;
}

// The graph of `key`: from the engine's cache, or captured now on the current device.  plan(P) builds the plans the
// captured work runs, run(P, stream) issues that work.
template <typename Plan, typename Run>
int cached_graph(f5_engine* e, const GraphKey& key, Plan&& plan, Run&& run, std::shared_ptr<GraphHolder>* out) {
  std::shared_ptr<GraphHolder> g;
  {
    std::lock_guard<std::mutex> lk(e->mu);
    for (auto& en : e->graphs)
      if (en.key == key) g = en.g;
  }
  if (!g) {
    // Capture outside the engine mutex (thread-local capture mode: concurrent sample() calls capture independently)
    // on a private stream — the caller's stream may be the legacy default stream, which cannot capture.
    StepPlans P;
    RC(plan(P));
    cudaStream_t cs;
    RC(check_cuda(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking), "capture stream"));
    if (int brc = check_cuda(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal), "begin capture")) {
      cudaStreamDestroy(cs);
      return brc;
    }
    const unsigned long long before = f5_launch_count();
    const int rc = run(P, cs);
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(cs, &graph);
    cudaStreamDestroy(cs);
    count_launch(-(int)(f5_launch_count() - before));  // captured, not launched
    if (rc || ce != cudaSuccess) {
      if (graph) cudaGraphDestroy(graph);
      return rc ? rc : check_cuda(ce, "end capture");
    }
    g = std::make_shared<GraphHolder>();
    size_t nn = 0;
    cudaGraphGetNodes(graph, nullptr, &nn);
    g->nodes = (int)nn;
    const cudaError_t ie = cudaGraphInstantiate(&g->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ie != cudaSuccess) {
      g->exec = nullptr;
      return check_cuda(ie, "graph instantiate");
    }
    std::lock_guard<std::mutex> lk(e->mu);
    if (e->graphs.size() >= 16) e->graphs.erase(e->graphs.begin());  // holder is freed when its last user is done
    e->graphs.push_back(GraphEntry{key, g});
  }
  *out = std::move(g);
  return 0;
}

// The step graph of this (workspace, shapes, half)
int step_graph(f5_engine* e, const Layout& L, const f5_sample_args* sa, const void* ws,
               std::shared_ptr<GraphHolder>* out) {
  const GraphKey key{ws, sa->B, sa->N, L.evals, L.packed, sa->duration == nullptr ? 0 : (sa->exact_varlen ? 2 : 1),
                     e->arch.backbone == kMMDiT ? sa->nt : 0, L.half, 0};
  return cached_graph(
      e, key, [&](StepPlans& P) { return build_step_plans(e, L, sa, P); },
      [&](const StepPlans& P, cudaStream_t cs) { return L.half < 0 ? run_step(e, L, P, cs) : run_body(e, L, P, cs); },
      out);
}

// A workspace written by f5_sample no longer holds the text embeddings of an earlier f5_forward call
void forget_text(f5_engine* e, const void* ws) {
  std::lock_guard<std::mutex> lk(e->mu);
  for (size_t i = 0; i < e->text_held.size();)
    if (e->text_held[i].ws == ws) e->text_held.erase(e->text_held.begin() + i);
    else ++i;
}

int check_problem(const char* fn, const f5_sample_args* sa) {
  if (sa->B <= 0 || sa->N <= 0 || sa->steps <= 0 || sa->nt <= 0) {
    set_error("%s: empty problem (B=%d N=%d steps=%d nt=%d)", fn, sa->B, sa->N, sa->steps, sa->nt);
    return -1;
  }
  if (sa->method != 0 && sa->method != 1) {
    set_error("%s: method must be 0 (euler) or 1 (midpoint), got %d", fn, sa->method);
    return -1;
  }
  return 0;
}

// One side of a call: the whole call of f5_sample, or one CFG half of f5_sample_cfg_split (below)
struct Side {
  f5_engine* e;
  const f5_sample_args* sa;
  void* ws;
  size_t bytes;
  cudaStream_t s;
  int dev = -1;
  Layout L;
  StepPlans P;                      // without use_graph
  std::shared_ptr<GraphHolder> g;  // with use_graph
  cudaEvent_t ready = nullptr, pulled = nullptr;  // CFG split only
};

// The workspace layout of one side (half -1: f5_sample; 0 / 1: that CFG half) and the check that it fits
int side_layout(Side& sd, int half) {
  const f5_sample_args* sa = sd.sa;
  const int evals = sa->method == 1 ? 2 * sa->steps : sa->steps;
  plan_layout(sd.e, sd.L, sd.ws, sa->B, sa->N, sa->nt, evals, sa->cfg_strength, half);
  if (sd.bytes >= sd.L.bytes) return 0;
  if (half < 0)
    set_error("f5_sample: workspace too small (%zu < %zu)", sd.bytes, sd.L.bytes);
  else
    set_error("f5_sample_cfg_split: workspace %d too small (%zu < %zu)", half, sd.bytes, sd.L.bytes);
  return -1;
}

// The prologue of one side, then its step graph (use_graph) or its plans
int side_prepare(Side& sd) {
  forget_text(sd.e, sd.ws);
  RC(run_prologue(sd.e, sd.L, sd.sa, sd.s));
  if (sd.sa->use_graph) return step_graph(sd.e, sd.L, sd.sa, sd.ws, &sd.g);
  return build_step_plans(sd.e, sd.L, sd.sa, sd.P);
}

}  // namespace

extern "C" int f5_sample(f5_engine* e, const f5_sample_args* sa, void* workspace, size_t ws_bytes, f5_stream_t stream) {
  if (!e || !sa || !workspace) {
    set_error("f5_sample: null argument");
    return -1;
  }
  RC(check_problem("f5_sample", sa));
  Side sd{e, sa, workspace, ws_bytes, reinterpret_cast<cudaStream_t>(stream)};
  RC(side_layout(sd, -1));
  RC(side_prepare(sd));
  const int evals = sd.L.evals;
  if (sd.g) {
    for (int k = 0; k < evals; ++k) RC(check_cuda(cudaGraphLaunch(sd.g->exec, sd.s), "graph launch"));
    count_launch(sd.g->nodes * evals);
  } else {
    for (int k = 0; k < evals; ++k) RC(run_step(e, sd.L, sd.P, sd.s));
  }
  return copy_v_out(e, sd.L, sa, sd.s);
}

// -------------------------------------------------------------------------------------------------------------
// CFG split (f5_sample_cfg_split): the conditional half of the packed batch on one workspace, the unconditional half on
// another, usually on another device.  The halves share nothing inside a backbone evaluation; they meet only in the
// update g = pred + (pred - null) * cfg.  So per evaluation k each side runs its half up to proj_out (run_body), pulls
// the other side's half of v into its own full v, and runs the unchanged update kernel over the full v: both sides
// then hold the same y and the same x columns of xin, and the next evaluation starts from identical inputs.
//
// Ordering, with s_d the stream of side d and o the other side.  Per evaluation k, host order:
//   pass 1, each d:  [k > 0] s_d waits pulled_o       (o's pull of d's v from evaluation k-1 is done)
//                    run_body on s_d                   (writes d's half of v_d)
//                    record ready_d on s_d
//   pass 2, each d:  s_d waits ready_o                 (o's half of v_o is complete)
//                    copy o's half of v_o -> v_d       (on s_d)
//                    record pulled_d on s_d
//                    run_update on s_d                 (reads both halves of v_d)
// Each buffer is written on one stream only; the cross-stream hazards are the copy's source, v_o's half on o: read
// after o wrote it (ready_o) and before o overwrites it at k+1 (o waits pulled_d before its next run_body).  The copy's
// destination is d's own v, read only by d's update, later on s_d.  At the end each stream waits for the other's last
// pull, so neither workspace is reused while the other side still reads it.  Every wait is enqueued after the record it
// refers to (pass 1 of k waits on pass 2 of k-1, pass 2 on pass 1 of k), so a wait never refers to work that was not
// issued: if a side fails partway and the host stops, a wait on an event whose record was never issued refers to the
// previous record or none, and does not block.  No kernel waits on a flag written by the other side.
namespace {

int pointer_device(const void* p, const char* what, int* dev) {
  cudaPointerAttributes at{};
  RC(check_cuda(cudaPointerGetAttributes(&at, p), what));
  if (at.type != cudaMemoryTypeDevice) {
    set_error("f5_sample_cfg_split: %s is not device memory", what);
    return -1;
  }
  *dev = at.device;
  return 0;
}

// Direct copies between the two devices where the hardware allows it (a per-process context setting, made once per
// ordered pair); otherwise cudaMemcpyPeerAsync stages through the host.
int enable_peer_access(int dev, int peer) {
  static std::mutex mu;
  static std::vector<std::pair<int, int>> done;
  std::lock_guard<std::mutex> lk(mu);
  for (auto& p : done)
    if (p.first == dev && p.second == peer) return 0;
  int can = 0;
  RC(check_cuda(cudaDeviceCanAccessPeer(&can, dev, peer), "cudaDeviceCanAccessPeer"));
  if (can) {
    RC(check_cuda(cudaSetDevice(dev), "cudaSetDevice"));
    const cudaError_t err = cudaDeviceEnablePeerAccess(peer, 0);
    if (err == cudaErrorPeerAccessAlreadyEnabled)
      cudaGetLastError();  // enabled before (by this library or by the caller): not an error
    else
      RC(check_cuda(err, "cudaDeviceEnablePeerAccess"));
  }
  done.emplace_back(dev, peer);
  return 0;
}

int split_check(const Side* sd) {
  const f5_sample_args *a = sd[0].sa, *b = sd[1].sa;
  if (a->B != b->B || a->N != b->N || a->nt != b->nt || a->steps != b->steps || a->method != b->method ||
      a->use_graph != b->use_graph || a->exact_varlen != b->exact_varlen || a->cfg_strength != b->cfg_strength ||
      (a->duration == nullptr) != (b->duration == nullptr)) {
    set_error("f5_sample_cfg_split: the two argument blocks must describe the same problem (B, N, nt, steps, method, "
              "use_graph, exact_varlen, cfg_strength, duration given or not)");
    return -1;
  }
  for (int k = 0; k <= a->steps; ++k)
    if (a->t[k] != b->t[k]) {
      set_error("f5_sample_cfg_split: the two time grids differ at %d", k);
      return -1;
    }
  if (a->cfg_strength < 1e-5f) {
    set_error("f5_sample_cfg_split: cfg_strength %g has no unconditional half to split off", a->cfg_strength);
    return -1;
  }
  if (b->trajectory || b->v_out) {
    set_error("f5_sample_cfg_split: only the first side writes trajectory and v_out");
    return -1;
  }
  if (a->y == b->y || sd[0].s == sd[1].s) {
    set_error("f5_sample_cfg_split: each side needs its own y and its own stream");
    return -1;
  }
  if (std::memcmp(&sd[0].e->arch, &sd[1].e->arch, sizeof(f5_arch)) != 0) {
    set_error("f5_sample_cfg_split: the two engines have different architectures");
    return -1;
  }
  const uint8_t *w0 = static_cast<const uint8_t*>(sd[0].ws), *w1 = static_cast<const uint8_t*>(sd[1].ws);
  if (w0 < w1 + sd[1].bytes && w1 < w0 + sd[0].bytes) {
    set_error("f5_sample_cfg_split: the two workspaces overlap");
    return -1;
  }
  return 0;
}

int split_loop(Side* sd, int evals) {
  const size_t half_floats = (size_t)sd[0].L.B * sd[0].L.x.seq * sd[0].e->arch.mel_dim;
  for (int k = 0; k < evals; ++k) {
    for (int d = 0; d < 2; ++d) {
      Side &me = sd[d], &o = sd[1 - d];
      RC(check_cuda(cudaSetDevice(me.dev), "cudaSetDevice"));
      if (k > 0) RC(check_cuda(cudaStreamWaitEvent(me.s, o.pulled, 0), "wait pulled"));
      if (me.g) {
        RC(check_cuda(cudaGraphLaunch(me.g->exec, me.s), "graph launch"));
        count_launch(me.g->nodes);
      } else {
        RC(run_body(me.e, me.L, me.P, me.s));
      }
      RC(check_cuda(cudaEventRecord(me.ready, me.s), "record ready"));
    }
    for (int d = 0; d < 2; ++d) {
      Side &me = sd[d], &o = sd[1 - d];
      RC(check_cuda(cudaSetDevice(me.dev), "cudaSetDevice"));
      RC(check_cuda(cudaStreamWaitEvent(me.s, o.ready, 0), "wait ready"));
      RC(check_cuda(cudaMemcpyPeerAsync(me.L.v_all + (o.L.v - o.L.v_all), me.dev, o.L.v, o.dev,
                                        sizeof(float) * half_floats, me.s),
                    "v exchange"));
      RC(check_cuda(cudaEventRecord(me.pulled, me.s), "record pulled"));
      RC(run_update(me.e, me.L, me.s));
    }
  }
  return 0;
}

int split_run(Side* sd) {
  for (int d = 0; d < 2; ++d) RC(side_layout(sd[d], d));
  if (sd[0].dev != sd[1].dev) {
    RC(enable_peer_access(sd[0].dev, sd[1].dev));
    RC(enable_peer_access(sd[1].dev, sd[0].dev));
  }
  for (int d = 0; d < 2; ++d) {
    Side& me = sd[d];
    RC(check_cuda(cudaSetDevice(me.dev), "cudaSetDevice"));
    RC(check_cuda(cudaEventCreateWithFlags(&me.ready, cudaEventDisableTiming), "event create"));
    RC(check_cuda(cudaEventCreateWithFlags(&me.pulled, cudaEventDisableTiming), "event create"));
    RC(side_prepare(me));
  }
  return split_loop(sd, sd[0].L.evals);
}

}  // namespace

extern "C" size_t f5_sample_cfg_split_workspace_bytes(const f5_engine* e, int B, int N, int nt, int nfe) {
  Layout L;
  plan_layout(e, L, nullptr, B, N, nt, nfe, 1.0f, 0);  // both halves have the same layout
  return L.bytes;
}

extern "C" int f5_sample_cfg_split(f5_engine* e0, const f5_sample_args* a0, void* ws0, size_t ws0_bytes,
                                   f5_stream_t stream0, f5_engine* e1, const f5_sample_args* a1, void* ws1,
                                   size_t ws1_bytes, f5_stream_t stream1) {
  if (!e0 || !a0 || !ws0 || !e1 || !a1 || !ws1) {
    set_error("f5_sample_cfg_split: null argument");
    return -1;
  }
  RC(check_problem("f5_sample_cfg_split", a0));
  Side sd[2] = {{e0, a0, ws0, ws0_bytes, reinterpret_cast<cudaStream_t>(stream0)},
                {e1, a1, ws1, ws1_bytes, reinterpret_cast<cudaStream_t>(stream1)}};
  RC(split_check(sd));
  RC(pointer_device(ws0, "workspace 0", &sd[0].dev));
  RC(pointer_device(ws1, "workspace 1", &sd[1].dev));
  int caller_dev = 0;
  RC(check_cuda(cudaGetDevice(&caller_dev), "cudaGetDevice"));
  int rc = split_run(sd);
  // Also after a failure: each stream waits for the other side's last pull (a no-op for an event never recorded), so
  // neither workspace is handed back while the other side may still read it.  Then the events go (destroying an event
  // with work pending is allowed: its resources are released once that work completes).
  for (int d = 0; d < 2; ++d) {
    Side &me = sd[d], &o = sd[1 - d];
    if (!me.ready || !o.pulled) continue;
    const cudaError_t err = cudaSetDevice(me.dev) != cudaSuccess ? cudaErrorInvalidDevice
                                                                  : cudaStreamWaitEvent(me.s, o.pulled, 0);
    if (!rc) rc = check_cuda(err, "final wait");
  }
  if (!rc) {
    cudaSetDevice(sd[0].dev);
    rc = copy_v_out(e0, sd[0].L, a0, sd[0].s);
  }
  for (int d = 0; d < 2; ++d) {
    cudaSetDevice(sd[d].dev);
    if (sd[d].ready) cudaEventDestroy(sd[d].ready);
    if (sd[d].pulled) cudaEventDestroy(sd[d].pulled);
  }
  cudaSetDevice(caller_dev);
  return rc;
}

// -------------------------------------------------------------------------------------------------------------
// One backbone evaluation (f5_forward): the reference's transformer(x, cond, text, time, mask, ...) operator, with a
// time per sample.  The layout is f5_sample's with one row of the time and AdaLN tables per sample (evals = B) and
// L.per_sample set: the norm, gated-residual GEMM (EPI_RESID_SAMPLE) and UNetT time-token kernels read the row of their
// sample.  Per call:
//   eager:  time -> t_dev, lengths (with durations), time MLP + AdaLN table of the B times, [text embeddings and rotary
//           tables unless reuse_text], input pack
//   graph:  the evaluation up to proj_out (captured once per workspace, shapes, mode and mask given or not; it reads
//           only the workspace, so new x, cond or times replay it)
//   eager:  v -> v_out
// The order is f5_sample's prologue order, for the same reason: the norm kernels fetch their modulation rows before the
// programmatic-launch wait, so the AdaLN table must be complete before the evaluation's first kernel starts.  The pack
// kernel, a plain launch, sits between the two and ends only after everything before it.
namespace {

void forward_layout(const f5_engine* e, Layout& L, void* ws, int B, int N, int nt, int mode) {
  // cond: un-packed (B rows); CFG: cond | uncond stacked (2B rows); uncond: the unconditional half alone, as one side
  // of f5_sample_cfg_split computes it
  plan_layout(e, L, ws, B, N, nt, B, mode == F5_FORWARD_COND ? 0.0f : 1.0f, mode == F5_FORWARD_UNCOND ? 1 : -1);
  L.per_sample = true;
}

int forward_check(const f5_forward_args* fa) {
  if (fa->B <= 0 || fa->N <= 0 || fa->nt <= 0) {
    set_error("f5_forward: empty problem (B=%d N=%d nt=%d)", fa->B, fa->N, fa->nt);
    return -1;
  }
  if (fa->mode < F5_FORWARD_COND || fa->mode > F5_FORWARD_UNCOND) {
    set_error("f5_forward: mode must be 0 (cond), 1 (cfg) or 2 (uncond), got %d", fa->mode);
    return -1;
  }
  if (!fa->x || !fa->step_cond || !fa->text || !fa->time || !fa->v_out) {
    set_error("f5_forward: x, step_cond, text, time and v_out are required");
    return -1;
  }
  return 0;
}

int forward_run(f5_engine* e, const f5_forward_args* fa, void* ws, size_t ws_bytes, cudaStream_t s) {
  const f5_arch& A = e->arch;
  const int B = fa->B, N = fa->N, nt = fa->nt;
  Layout L;
  forward_layout(e, L, ws, B, N, nt, fa->mode);
  if (ws_bytes < L.bytes) {
    set_error("f5_forward: workspace too small (%zu < %zu)", ws_bytes, L.bytes);
    return -1;
  }
  const bool masked = fa->duration != nullptr;
  const TextHeld held{ws, B, N, nt, fa->mode, masked ? 1 : 0};
  {
    std::lock_guard<std::mutex> lk(e->mu);
    bool found = false;
    for (size_t i = 0; i < e->text_held.size();)
      if (e->text_held[i].ws != ws) {
        ++i;
      } else if (fa->reuse_text && e->text_held[i] == held) {
        found = true;
        ++i;
      } else {
        e->text_held.erase(e->text_held.begin() + i);  // about to be overwritten, or of another problem
      }
    if (fa->reuse_text && !found) {
      set_error("f5_forward: reuse_text, but the workspace holds no text embeddings of this problem (B=%d N=%d nt=%d "
                "mode %d, durations %s)", B, N, nt, fa->mode, masked ? "given" : "not given");
      return -1;
    }
  }
  RC(check_cuda(cudaMemcpyAsync(L.t_dev, fa->time, sizeof(float) * B, cudaMemcpyDeviceToDevice, s), "time copy"));
  if (masked) RC(set_lengths(e, L, fa->duration, false, s));
  RC(run_time_embed(e, L, s));
  if (!fa->reuse_text) {
    RC(run_rope_table(L.x.rope_cos, L.x.rope_sin, L.x.seq, A.dim_head / 2, s));
    RC(run_text_embed(e, L, fa->text, nt, masked, false, s));
    std::lock_guard<std::mutex> lk(e->mu);
    if (e->text_held.size() >= 64) e->text_held.erase(e->text_held.begin());
    e->text_held.push_back(held);
  }
  RC(run_pack(e, L, fa->x, fa->step_cond, s));
  f5_sample_args sa{};  // the fields build_step_plans reads
  sa.B = B;
  sa.N = N;
  sa.nt = nt;
  sa.duration = fa->duration;
  auto run = [&](const StepPlans& P, cudaStream_t cs) { return run_body(e, L, P, cs); };
  if (fa->use_graph) {
    const GraphKey key{ws, B, N, L.evals, L.packed, masked ? 1 : 0, A.backbone == kMMDiT ? nt : 0, L.half, 1};
    std::shared_ptr<GraphHolder> g;
    RC(cached_graph(e, key, [&](StepPlans& P) { return build_step_plans(e, L, &sa, P); }, run, &g));
    RC(check_cuda(cudaGraphLaunch(g->exec, s), "graph launch"));
    count_launch(g->nodes);
  } else {
    StepPlans P;
    RC(build_step_plans(e, L, &sa, P));
    RC(run(P, s));
  }
  // v (this layout's rows: Be samples of seq rows) -> v_out [Be, N, mel], without the UNetT time token
  const int mel = A.mel_dim, off = A.backbone == kUNetT ? 1 : 0;
  RC(check_cuda(cudaMemcpy2DAsync(fa->v_out, sizeof(float) * N * mel, L.v + (size_t)off * mel,
                                  sizeof(float) * L.x.seq * mel, sizeof(float) * N * mel, L.Be,
                                  cudaMemcpyDeviceToDevice, s),
                "v_out copy"));
  return 0;
}

}  // namespace

extern "C" int f5_engine_graph_count(f5_engine* e) {
  if (!e) return 0;
  std::lock_guard<std::mutex> lk(e->mu);
  return (int)e->graphs.size();
}

extern "C" size_t f5_forward_workspace_bytes(const f5_engine* e, int B, int N, int nt, int mode) {
  Layout L;
  forward_layout(e, L, nullptr, B, N, nt, mode);
  return L.bytes;
}

extern "C" int f5_forward(f5_engine* e, const f5_forward_args* args, void* workspace, size_t ws_bytes,
                          f5_stream_t stream) {
  if (!e || !args || !workspace) {
    set_error("f5_forward: null argument");
    return -1;
  }
  RC(forward_check(args));
  return forward_run(e, args, workspace, ws_bytes, reinterpret_cast<cudaStream_t>(stream));
}

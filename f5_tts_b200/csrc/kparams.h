// Kernel parameter blocks and tile constants shared by device code and the host planners.
#pragma once
#include <cuda_fp16.h>
#include <stddef.h>
#include <stdint.h>

namespace f5 {

enum : int { ACT_NONE = 0, ACT_GELU_TANH = 1, ACT_GELU_ERF = 2, ACT_MISH = 3 };
enum : int {
  EPI_F16 = 0,       // out16[m,n] = mask(act(acc + bias))
  EPI_F32 = 1,       // out32[m,n] = acc + bias ; optional out16b[m,n] = mask(acc + bias) (fp16 copy)
  EPI_RESID = 2,     // resid32[m,n] += gate[n] * mask(act(acc + bias))
  EPI_QKV_ROPE = 3,  // out16[m,n] = rope(acc + bias) for the first pe_heads heads of q,k; plain for the rest
  // as EPI_QKV_ROPE, with a per-head RMSNorm(64, eps 1e-6, gain q_norm / k_norm) on every q and k head before RoPE
  EPI_QKV_NORM_ROPE = 4,
  // EPI_QKV_ROPE / EPI_QKV_NORM_ROPE over 128-column heads.  Kernel-internal: the C ABI selects them with
  // f5_gemm_args.dim_head = 128.
  EPI_QKV_ROPE_DH128 = 5,
  EPI_QKV_NORM_ROPE_DH128 = 6,
  // EPI_RESID with the gate row of each output row's sample: gate + ((row / gate_seq) % gate_samples) *
  // gate_step_stride.  Engine-internal (f5_forward, gemm.cu: kGemmSampleKernels), so the kernels of f5_sample keep
  // their step-indexed gate.
  EPI_RESID_SAMPLE = 7,
};

struct GemmParams {
  int rows;      // valid rows per batch entry
  int n_out;     // output columns
  int num_kb;    // 64-wide K blocks (plain) or taps (conv)
  int batches;   // gridDim.z
  const float* bias;
  void* out;     // fp16 (EPI_F16/QKV) or fp32 (EPI_F32)
  __half* out16b;  // optional fp16 copy for EPI_F32
  float* resid;  // EPI_RESID in/out
  int ldo;       // leading dimension of out / resid (elements)
  const float* gate;  // [n_out] at gate + (*step_ptr) * gate_step_stride, or null (gate = 1)
  const int* step_ptr;
  long long gate_step_stride;
  const int* row_len;  // per-sample valid length (sample = global_row / seq), or null
  int seq;             // rows per sample
  const float* rope_cos;  // [seq, dh/2]
  const float* rope_sin;
  int inner;     // heads * dim_head
  int pe_heads;  // heads that get rotary (q and k sections)
  int conv_pad;  // CONV: taps/2
  int skip_pad;    // 1: 128-row tiles whose rows all lie past their sample's row_len are not computed
  int w_prefetch;  // W tiles may be loaded before griddepcontrol.wait (weights are not produced by the predecessor)
  int conv_g;      // CONV: channels per group (<= 64); one output tile computes one group
#ifdef F5_TRACE
  int diag_no_epi;  // instrumented build: skip the epilogue (nothing is stored) to time the main loop alone
#endif
  // EPI_QKV_NORM_ROPE: fp32 [dim_head] RMSNorm gains of the q and k heads.  Last, so the other epilogues' kernels keep their
  // parameter offsets.
  const float* q_norm;
  const float* k_norm;
  // EPI_RESID_SAMPLE: rows per sample, and the number of gate rows (the samples of the call; the conditional and
  // unconditional rows of a sample share one).  Last, so every other field keeps its parameter offset.
  int gate_seq;
  int gate_samples;
};

constexpr int kBM = 128;
constexpr int kBK = 64;


struct AttnParams {
  int seq;            // tokens per sample
  int heads;
  int batches;        // packed batch Be
  int inner;          // heads * dim_head
  const int* kv_len;  // [Be] valid keys per sample, or null (= seq)
  float scale_log2;   // softmax scale * log2(e)
  __half* out;        // [Be*seq, inner]
};

// Second key / query segment of the joint (MMDiT) attention kernel
struct AttnJointParams {
  int seq_c;          // text tokens per sample
  const int* c_len;   // [Be] valid text keys per sample (0 allowed), or null (= seq_c)
  __half* out_c;      // [Be*seq_c, inner]
  int q_blocks_a;     // audio query blocks, ceil(seq / (64 qwg)); grid.x beyond them are text query blocks
};

// qwg softmax / MMA warpgroups (64 query rows each, 64 qwg query rows per CTA): qwg = 2, or 4 at head width 64
// (attn.cu: attn_choose_qwg).  qwg = 2 adds a TMA producer warp.  qwg = 4 has none: 17 warps would put five warps on
// one of the SM's four register-file quarters (16384 registers each) and cap every thread at 96 registers, where the
// consumer spills; 16 warps leave it the 128 it needs, so consumer warp 0 issues the loads (attn.cuh).
constexpr int attn_threads(int qwg) { return qwg == 4 ? 512 : 128 * qwg + 32; }
constexpr int kAttnBKV = 128;       // keys per tile
constexpr int kAttnStages = 3;      // K and V rings
constexpr uint32_t kAttnTile = 128 * 64 * 2;  // 16 KB: one 128-row x 64-column TMA box
// Q (qwg / 2 tiles of 128 rows) + K,V rings + alignment slack + barriers, for head width dh (dh / 64 boxes per tile).
// dh = 128 with three stages is 7 x 32 KB + 1.25 KB = 225.25 KB of the 227 KB an H100 CTA may have (DESIGN.md §4);
// dh = 64 at qwg = 4 is 8 x 16 KB + 1.25 KB.
constexpr size_t attn_smem_bytes(int dh, int qwg = 2) {
  return size_t(kAttnTile) * (dh / 64) * (qwg / 2 + 2 * kAttnStages) + 1024 + 256;
}
constexpr size_t kAttnSmem = attn_smem_bytes(64);
static_assert(attn_smem_bytes(128) <= 227 * 1024, "dim_head 128 attention tiles exceed shared memory");
static_assert(attn_smem_bytes(64, 4) <= 227 * 1024, "4-warpgroup attention tiles exceed shared memory");

}  // namespace f5

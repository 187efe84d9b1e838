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
};

constexpr int kBM = 128;
constexpr int kBK = 64;


struct AttnParams {
  int seq;            // tokens per sample
  int heads;
  int batches;        // packed batch Be
  int inner;          // heads * 64
  const int* kv_len;  // [Be] valid keys per sample, or null (= seq)
  float scale_log2;   // softmax scale * log2(e)
  __half* out;        // [Be*seq, inner]
};

constexpr int kAttnThreads = 288;   // two softmax / MMA warpgroups (64 query rows each) + one TMA producer warp
constexpr int kAttnBQ = 128;        // query rows per CTA
constexpr int kAttnBKV = 128;       // keys per tile
constexpr int kAttnStages = 3;      // K and V rings
constexpr uint32_t kAttnTile = 128 * 64 * 2;  // 16 KB
// Q + K,V rings + alignment slack + barriers
constexpr size_t kAttnSmem = size_t(kAttnTile) * (1 + 2 * kAttnStages) + 1024 + 256;

}  // namespace f5

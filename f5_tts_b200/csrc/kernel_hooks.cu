// Test entry points of libf5tts_b200_kernels.so: one extern "C" wrapper per launcher of ops.cu, so the kernel tests run
// the product's own object code and launch configurations one kernel at a time.  Linked with the same objects as
// libf5tts_b200.so; the product library does not contain this file and exports none of these symbols.
// Every wrapper returns 0 or the launcher's error code (message: f5k_last_error()).
#include "internal.h"

using namespace f5;

namespace {
inline cudaStream_t st(void* s) { return reinterpret_cast<cudaStream_t>(s); }
}  // namespace

extern "C" {

const char* f5k_last_error() { return f5_last_error(); }

int f5k_row_norm(int mode, const float* x, void* out, int rows, int D, float eps, const float* a, const float* b,
                 const int* step_ptr, long long step_stride, int params_static, void* s) {
  NormParams p{};
  p.x = x;
  p.out = reinterpret_cast<__half*>(out);
  p.rows = rows;
  p.D = D;
  p.eps = eps;
  p.a = a;
  p.b = b;
  p.step_ptr = step_ptr;
  p.step_stride = step_stride;
  p.params_static = params_static;
  return run_row_norm(mode, p, st(s));
}

int f5k_dwconv7_ln(const float* x, void* out, int B, int N, int C, const float* w, const float* wb, const float* ln_w,
                   const float* ln_b, float eps, void* s) {
  DwConvLnParams p{};
  p.x = x;
  p.out = reinterpret_cast<__half*>(out);
  p.B = B;
  p.N = N;
  p.C = C;
  p.w = w;
  p.wb = wb;
  p.ln_w = ln_w;
  p.ln_b = ln_b;
  p.eps = eps;
  return run_dwconv7_ln(p, st(s));
}

int f5k_text_gather(const long long* ids, int B, int nt, int N, int Td, const int* valid_len, const float* table,
                    int num_embeds, int add_pos, float* out, uint8_t* filler, void* s) {
  TextGatherParams p{};
  p.ids = ids;
  p.B = B;
  p.nt = nt;
  p.N = N;
  p.Td = Td;
  p.valid_len = valid_len;
  p.table = table;
  p.num_embeds = num_embeds;
  p.add_pos = add_pos;
  p.out = out;
  p.filler = filler;
  return run_text_gather(p, st(s));
}

int f5k_mask_rows(float* x, const uint8_t* filler, int BN, int rows, int C, void* s) {
  return run_mask_rows(x, filler, BN, rows, C, st(s));
}

int f5k_mask_rows_len(void* x, int is_half, const int* valid_len, int B, int N, int rows, int C, void* s) {
  if (is_half) return run_mask_rows_len_half(reinterpret_cast<__half*>(x), valid_len, B, N, rows, C, st(s));
  return run_mask_rows_len(reinterpret_cast<float*>(x), valid_len, B, N, rows, C, st(s));
}

int f5k_grn_rows() { return kGrnRows; }

int f5k_grn(void* g, float* partial, float* nx, const float* gamma, const float* beta, int B, int N, int C, void* s) {
  return run_grn(reinterpret_cast<__half*>(g), partial, nx, gamma, beta, B, N, C, st(s));
}

int f5k_pack_input(void* xin, int B, int N, int mel, int Td, int Kpad, int packed, const float* y,
                   const float* step_cond, const float* text, void* s) {
  PackParams p{};
  p.xin = reinterpret_cast<__half*>(xin);
  p.B = B;
  p.N = N;
  p.mel = mel;
  p.Td = Td;
  p.Kpad = Kpad;
  p.packed = packed;
  p.y = y;
  p.step_cond = step_cond;
  p.text = text;
  return run_pack_input(p, st(s));
}

// io: device SampleIo {float* y; float* traj; float cfg}; stage: device OdeStage[evals] {float coef; int traj_row};
// step_ptr: device int[2] (evaluation counter, CTA done counter)
int f5k_cfg_euler(const void* io, const float* v, void* xin, const void* stage, int* step_ptr, int BN, int mel,
                  int Kpad, int packed, int N, int seq_tok, int tok_off, int B, void* s) {
  EulerParams p{};
  p.io = reinterpret_cast<const SampleIo*>(io);
  p.v = v;
  p.xin = reinterpret_cast<__half*>(xin);
  p.stage = reinterpret_cast<const OdeStage*>(stage);
  p.step_ptr = step_ptr;
  p.BN = BN;
  p.mel = mel;
  p.Kpad = Kpad;
  p.packed = packed;
  p.N = N;
  p.seq_tok = seq_tok;
  p.tok_off = tok_off;
  p.B = B;
  return run_cfg_euler(p, st(s));
}

int f5k_small_linear(int act, const float* in, const void* W, const float* bias, float* out, int S, int K, int Nout,
                     void* s) {
  return run_small_linear(act, in, reinterpret_cast<const __half*>(W), bias, out, S, K, Nout, st(s));
}

int f5k_time_features(const float* t, float* feat, int S, int dim, void* s) {
  return run_time_features(t, feat, S, dim, st(s));
}

int f5k_silu_to_half(const float* in, void* out, long long n, void* s) {
  return run_silu_to_half(in, reinterpret_cast<__half*>(out), n, st(s));
}

int f5k_rope_table(float* cs, float* sn, int seq, int half, void* s) { return run_rope_table(cs, sn, seq, half, st(s)); }

int f5k_prepend_time_token(float* dst, const float* src, const float* t_emb, const int* step_ptr, int N, int D,
                           long long rows_out, void* s) {
  return run_prepend_time_token(dst, src, t_emb, step_ptr, N, D, rows_out, st(s));
}

int f5k_concat_half(const float* x, const float* skip, void* out, long long rows, int D, void* s) {
  return run_concat_half(x, skip, reinterpret_cast<__half*>(out), rows, D, st(s));
}

int f5k_vocos_im2col(const float* mel, int B, int C, int T, void* A, int Kpad, void* s) {
  return run_vocos_im2col(mel, B, C, T, reinterpret_cast<__half*>(A), Kpad, st(s));
}

int f5k_ln_affine_f32(const float* x, float* out, int rows, int D, float eps, const float* w, const float* b, void* s) {
  return run_ln_affine_f32(x, out, rows, D, eps, w, b, st(s));
}

int f5k_istft(const float* head, int ld, float* frames, float* wav, int B, int T, void* s) {
  FftTables tab;
  if (int rc = fft_tables(&tab, st(s))) return rc;
  return run_istft(head, ld, frames, wav, B, T, tab, st(s));
}

}  // extern "C"

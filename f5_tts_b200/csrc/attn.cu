// Host side of the wgmma attention kernels + C entry points f5_attention (dim_head 64), f5_attention_dh and
// f5_attention_joint.
#include "attn.cuh"
#include "internal.h"

namespace f5 {

int attn_plan(AttnPlan* pl, const void* qkv, void* out, int batches, int seq, int heads, int dim_head,
              const int* kv_len, float scale) {
  if (batches <= 0 || seq <= 0 || heads <= 0) {
    set_error("attention: empty problem");
    return -1;
  }
  if (dim_head != 64 && dim_head != 128) {
    set_error("attention: dim_head must be 64 or 128 (got %d)", dim_head);
    return -1;
  }
  const int inner = heads * dim_head;
  const uint64_t dims[3] = {(uint64_t)3 * inner, (uint64_t)seq, (uint64_t)batches};
  const uint64_t strides[2] = {(uint64_t)3 * inner * 2, (uint64_t)seq * 3 * inner * 2};
  const uint32_t box[3] = {64, 128, 1};
  int rc = encode_tmap_f16(&pl->tm, qkv, 3, dims, strides, box);
  if (rc) return rc;
  pl->p.seq = seq;
  pl->p.heads = heads;
  pl->p.batches = batches;
  pl->p.inner = inner;
  pl->p.kv_len = kv_len;
  pl->p.scale_log2 = scale * 1.4426950408889634f;
  pl->p.out = reinterpret_cast<__half*>(out);
  pl->grid = dim3((seq + kAttnBQ - 1) / kAttnBQ, heads, batches);
  pl->dh = dim_head;
  return 0;
}

int attn_joint_plan(AttnPlan* pl, const void* qkv, const void* qkv_c, void* out, void* out_c, int batches, int seq,
                    int seq_c, int heads, int dim_head, const int* kv_len, const int* c_len, int text_q, float scale) {
  if (seq_c <= 0) {
    set_error("joint attention: empty text segment (seq_c=%d)", seq_c);
    return -1;
  }
  if (int rc = attn_plan(pl, qkv, out, batches, seq, heads, dim_head, kv_len, scale)) return rc;
  const int inner = heads * dim_head;
  const uint64_t dims[3] = {(uint64_t)3 * inner, (uint64_t)seq_c, (uint64_t)batches};
  const uint64_t strides[2] = {(uint64_t)3 * inner * 2, (uint64_t)seq_c * 3 * inner * 2};
  const uint32_t box[3] = {64, 128, 1};
  if (int rc = encode_tmap_f16(&pl->tmC, qkv_c, 3, dims, strides, box)) return rc;
  pl->joint = 1;
  pl->jp.seq_c = seq_c;
  pl->jp.c_len = c_len;
  pl->jp.out_c = reinterpret_cast<__half*>(out_c);
  pl->jp.q_blocks_a = (seq + kAttnBQ - 1) / kAttnBQ;
  pl->grid.x = pl->jp.q_blocks_a + (text_q ? (seq_c + kAttnBQ - 1) / kAttnBQ : 0);
  return 0;
}

template <typename K>
static int attn_configure_kernel(K* kernel, int dh) {
  if (int rc = check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)attn_smem_bytes(dh)),
                          "cudaFuncSetAttribute(attn smem)"))
    return rc;
  cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
  return 0;
}

template <int DH>
static int attn_configure_dh() {
  if (int rc = attn_configure_kernel(attn_fwd_wgmma_kernel<DH>, DH)) return rc;
  return attn_configure_kernel(attn_joint_wgmma_kernel<DH>, DH);
}

int attn_configure() {
  if (int rc = attn_configure_dh<64>()) return rc;
  return attn_configure_dh<128>();
}

int attn_run(const AttnPlan& pl, cudaStream_t s) {
  if (int rc = configure_kernels()) return rc;
  PdlLaunch L(pl.grid, dim3(kAttnThreads), attn_smem_bytes(pl.dh), s);
  cudaError_t e;
  if (pl.joint)
    e = pl.dh == 128 ? cudaLaunchKernelEx(&L.cfg, attn_joint_wgmma_kernel<128>, pl.tm, pl.tmC, pl.p, pl.jp)
                     : cudaLaunchKernelEx(&L.cfg, attn_joint_wgmma_kernel<64>, pl.tm, pl.tmC, pl.p, pl.jp);
  else
    e = pl.dh == 128 ? cudaLaunchKernelEx(&L.cfg, attn_fwd_wgmma_kernel<128>, pl.tm, pl.p)
                     : cudaLaunchKernelEx(&L.cfg, attn_fwd_wgmma_kernel<64>, pl.tm, pl.p);
  if (int rc = check_cuda(e, "attention launch")) return rc;
  count_launch();
  return check_launch("attn_fwd_wgmma_kernel launch");
}

}  // namespace f5

extern "C" int f5_attention_dh(const void* qkv, void* out, int batches, int seq, int heads, int dim_head,
                               const int* kv_len, float scale, f5_stream_t stream) {
  f5::AttnPlan pl;
  if (int rc = f5::attn_plan(&pl, qkv, out, batches, seq, heads, dim_head, kv_len, scale)) return rc;
  return f5::attn_run(pl, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int f5_attention(const void* qkv, void* out, int batches, int seq, int heads, const int* kv_len, float scale,
                            f5_stream_t stream) {
  return f5_attention_dh(qkv, out, batches, seq, heads, 64, kv_len, scale, stream);
}

extern "C" int f5_attention_joint(const void* qkv, const void* qkv_c, void* out, void* out_c, int batches, int seq,
                                  int seq_c, int heads, int dim_head, const int* kv_len, const int* c_len, int text_q,
                                  float scale, f5_stream_t stream) {
  f5::AttnPlan pl;
  if (int rc = f5::attn_joint_plan(&pl, qkv, qkv_c, out, out_c, batches, seq, seq_c, heads, dim_head, kv_len, c_len,
                                   text_q, scale))
    return rc;
  return f5::attn_run(pl, reinterpret_cast<cudaStream_t>(stream));
}

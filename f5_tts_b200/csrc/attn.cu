// Host side of the wgmma attention kernel + C entry point f5_attention.
#include "attn.cuh"
#include "internal.h"

namespace f5 {

int attn_plan(AttnPlan* pl, const void* qkv, void* out, int batches, int seq, int heads, const int* kv_len,
              float scale) {
  if (batches <= 0 || seq <= 0 || heads <= 0) {
    set_error("attention: empty problem");
    return -1;
  }
  const int inner = heads * 64;
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
  return 0;
}

int attn_configure() {
  if (int rc = check_cuda(cudaFuncSetAttribute(attn_fwd_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)kAttnSmem),
                          "cudaFuncSetAttribute(attn smem)"))
    return rc;
  cudaFuncSetAttribute(attn_fwd_wgmma_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
  return 0;
}

int attn_run(const AttnPlan& pl, cudaStream_t s) {
  if (int rc = configure_kernels()) return rc;
  PdlLaunch L(pl.grid, dim3(kAttnThreads), kAttnSmem, s);
  if (int rc = check_cuda(cudaLaunchKernelEx(&L.cfg, attn_fwd_wgmma_kernel, pl.tm, pl.p), "attention launch")) return rc;
  count_launch();
  return check_launch("attn_fwd_wgmma_kernel launch");
}

}  // namespace f5

extern "C" int f5_attention(const void* qkv, void* out, int batches, int seq, int heads, const int* kv_len, float scale,
                            f5_stream_t stream) {
  f5::AttnPlan pl;
  if (int rc = f5::attn_plan(&pl, qkv, out, batches, seq, heads, kv_len, scale)) return rc;
  return f5::attn_run(pl, reinterpret_cast<cudaStream_t>(stream));
}

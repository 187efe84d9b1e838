// Host side of the wgmma attention kernels + C entry points f5_attention (dim_head 64), f5_attention_dh,
// f5_attention_joint, and f5_attention_qwg / f5_attention_joint_qwg (the same with the query warpgroups per CTA given).
#include "attn.cuh"
#include "internal.h"

namespace f5 {

static int attn_q_blocks(int seq, int qwg) { return (seq + 64 * qwg - 1) / (64 * qwg); }

// Query warpgroups per CTA.  A 4-warpgroup CTA (256 queries) puts twice the rows on an SM's tensor cores as a
// 2-warpgroup one (128 queries), and the SM holds one CTA of either kind, so 4 pays whenever the 128-query grid needs
// more than one wave: its SMs then run two or more 128-query blocks one after the other anyway.  When the 128-query
// grid fits in one wave (blocks128 CTAs <= SMs), 4 would halve the CTAs and leave SMs idle that the 128-query grid
// uses: keep 2.  Head width 128 stays at 2 (its consumer needs 163 registers; 544 threads leave 120).
// On 132 SMs, 16 heads: Be 2, N 938 -> 256 CTAs of 128 queries, two waves -> 4 (128 CTAs of 256, one wave);
// Be 2, N 469 -> 128 CTAs, one wave -> 2; Be 16 at N 938 / 1875 -> 4.
static int attn_choose_qwg(int dim_head, long long blocks128) {
  return dim_head == 64 && blocks128 > num_sms() ? 4 : 2;
}

int attn_plan(AttnPlan* pl, const void* qkv, void* out, int batches, int seq, int heads, int dim_head,
              const int* kv_len, float scale, int qwg) {
  if (batches <= 0 || seq <= 0 || heads <= 0) {
    set_error("attention: empty problem");
    return -1;
  }
  if (dim_head != 64 && dim_head != 128) {
    set_error("attention: dim_head must be 64 or 128 (got %d)", dim_head);
    return -1;
  }
  if (qwg != 0 && qwg != 2 && !(qwg == 4 && dim_head == 64)) {
    set_error("attention: query warpgroups must be 0 (chosen by the planner), 2, or 4 at dim_head 64 (got %d at %d)",
              qwg, dim_head);
    return -1;
  }
  if (qwg == 0) qwg = attn_choose_qwg(dim_head, (long long)attn_q_blocks(seq, 2) * heads * batches);
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
  pl->grid = dim3(attn_q_blocks(seq, qwg), heads, batches);
  pl->dh = dim_head;
  pl->qwg = qwg;
  return 0;
}

int attn_joint_plan(AttnPlan* pl, const void* qkv, const void* qkv_c, void* out, void* out_c, int batches, int seq,
                    int seq_c, int heads, int dim_head, const int* kv_len, const int* c_len, int text_q, float scale,
                    int qwg) {
  if (seq_c <= 0) {
    set_error("joint attention: empty text segment (seq_c=%d)", seq_c);
    return -1;
  }
  if (qwg == 0 && heads > 0 && batches > 0 && seq > 0)
    qwg = attn_choose_qwg(dim_head, (long long)(attn_q_blocks(seq, 2) + (text_q ? attn_q_blocks(seq_c, 2) : 0)) *
                                        heads * batches);
  if (int rc = attn_plan(pl, qkv, out, batches, seq, heads, dim_head, kv_len, scale, qwg)) return rc;
  const int inner = heads * dim_head;
  const uint64_t dims[3] = {(uint64_t)3 * inner, (uint64_t)seq_c, (uint64_t)batches};
  const uint64_t strides[2] = {(uint64_t)3 * inner * 2, (uint64_t)seq_c * 3 * inner * 2};
  const uint32_t box[3] = {64, 128, 1};
  if (int rc = encode_tmap_f16(&pl->tmC, qkv_c, 3, dims, strides, box)) return rc;
  pl->joint = 1;
  pl->jp.seq_c = seq_c;
  pl->jp.c_len = c_len;
  pl->jp.out_c = reinterpret_cast<__half*>(out_c);
  pl->jp.q_blocks_a = attn_q_blocks(seq, pl->qwg);
  pl->grid.x = pl->jp.q_blocks_a + (text_q ? attn_q_blocks(seq_c, pl->qwg) : 0);
  return 0;
}

template <typename K>
static int attn_configure_kernel(K* kernel, int dh, int qwg) {
  if (int rc = check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)attn_smem_bytes(dh, qwg)),
                          "cudaFuncSetAttribute(attn smem)"))
    return rc;
  cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
  return 0;
}

template <int DH, int QWG>
static int attn_configure_dh() {
  if (int rc = attn_configure_kernel(attn_fwd_wgmma_kernel<DH, QWG>, DH, QWG)) return rc;
  return attn_configure_kernel(attn_joint_wgmma_kernel<DH, QWG>, DH, QWG);
}

int attn_configure() {
  if (int rc = attn_configure_dh<64, 2>()) return rc;
  if (int rc = attn_configure_dh<64, 4>()) return rc;
  return attn_configure_dh<128, 2>();
}

int attn_run(const AttnPlan& pl, cudaStream_t s) {
  if (int rc = configure_kernels()) return rc;
  PdlLaunch L(pl.grid, dim3(attn_threads(pl.qwg)), attn_smem_bytes(pl.dh, pl.qwg), s);
  cudaError_t e;
  if (pl.joint)
    e = pl.dh == 128 ? cudaLaunchKernelEx(&L.cfg, attn_joint_wgmma_kernel<128, 2>, pl.tm, pl.tmC, pl.p, pl.jp)
        : pl.qwg == 4 ? cudaLaunchKernelEx(&L.cfg, attn_joint_wgmma_kernel<64, 4>, pl.tm, pl.tmC, pl.p, pl.jp)
                      : cudaLaunchKernelEx(&L.cfg, attn_joint_wgmma_kernel<64, 2>, pl.tm, pl.tmC, pl.p, pl.jp);
  else
    e = pl.dh == 128 ? cudaLaunchKernelEx(&L.cfg, attn_fwd_wgmma_kernel<128, 2>, pl.tm, pl.p)
        : pl.qwg == 4 ? cudaLaunchKernelEx(&L.cfg, attn_fwd_wgmma_kernel<64, 4>, pl.tm, pl.p)
                      : cudaLaunchKernelEx(&L.cfg, attn_fwd_wgmma_kernel<64, 2>, pl.tm, pl.p);
  if (int rc = check_cuda(e, "attention launch")) return rc;
  count_launch();
  return check_launch("attn_fwd_wgmma_kernel launch");
}

}  // namespace f5

extern "C" int f5_attention_qwg(const void* qkv, void* out, int batches, int seq, int heads, int dim_head,
                                const int* kv_len, float scale, int qwg, f5_stream_t stream) {
  f5::AttnPlan pl;
  if (int rc = f5::attn_plan(&pl, qkv, out, batches, seq, heads, dim_head, kv_len, scale, qwg)) return rc;
  return f5::attn_run(pl, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int f5_attention_qwg_choice(int batches, int seq, int heads, int dim_head) {
  if (batches <= 0 || seq <= 0 || heads <= 0 || (dim_head != 64 && dim_head != 128)) return -1;
  return f5::attn_choose_qwg(dim_head, (long long)f5::attn_q_blocks(seq, 2) * heads * batches);
}

extern "C" int f5_attention_dh(const void* qkv, void* out, int batches, int seq, int heads, int dim_head,
                               const int* kv_len, float scale, f5_stream_t stream) {
  return f5_attention_qwg(qkv, out, batches, seq, heads, dim_head, kv_len, scale, 0, stream);
}

extern "C" int f5_attention(const void* qkv, void* out, int batches, int seq, int heads, const int* kv_len, float scale,
                            f5_stream_t stream) {
  return f5_attention_dh(qkv, out, batches, seq, heads, 64, kv_len, scale, stream);
}

extern "C" int f5_attention_joint_qwg(const void* qkv, const void* qkv_c, void* out, void* out_c, int batches,
                                      int seq, int seq_c, int heads, int dim_head, const int* kv_len, const int* c_len,
                                      int text_q, float scale, int qwg, f5_stream_t stream) {
  f5::AttnPlan pl;
  if (int rc = f5::attn_joint_plan(&pl, qkv, qkv_c, out, out_c, batches, seq, seq_c, heads, dim_head, kv_len, c_len,
                                   text_q, scale, qwg))
    return rc;
  return f5::attn_run(pl, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int f5_attention_joint(const void* qkv, const void* qkv_c, void* out, void* out_c, int batches, int seq,
                                  int seq_c, int heads, int dim_head, const int* kv_len, const int* c_len, int text_q,
                                  float scale, f5_stream_t stream) {
  return f5_attention_joint_qwg(qkv, qkv_c, out, out_c, batches, seq, seq_c, heads, dim_head, kv_len, c_len, text_q,
                                scale, 0, stream);
}

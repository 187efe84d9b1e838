// Non-causal flash-attention forward on wgmma for dim_head DH = 64 or 128 (reference: model/modules.py:471-556,
// F.scaled_dot_product_attention(q, k, v, attn_mask=None | key mask), scale 1/sqrt(DH)).
//
// One CTA = one (sample, head, block of 64 QWG queries), QWG = 2 or (DH = 64 only) 4 consumer warpgroups.  q/k/v are
// read in place from the fused QKV projection output [Be*seq, 3*inner] (fp16) through ONE 3-D TMA tensor map (cols,
// seq rows, sample): no head-split transpose ever touches HBM, and rows past the end of a sample are zero-filled by
// TMA instead of leaking the next sample.  A 128B-swizzled box
// is at most 64 fp16 wide, so a 128-row tile of a head is DH / 64 boxes of 128 x 64 (16 KB each), one after the other.
// Warp roles: warps 0..4 QWG - 1 = QWG consumer warpgroups, warpgroup g owns query rows [64 g, 64 g + 64).  The TMA
// loads (Q once, then a kAttnStages-deep ring of K and V tiles of 128 keys) come from warp 8, a producer warp of its
// own, at QWG = 2 (288 threads), and from consumer warp 0 at QWG = 4 (512 threads; see attn_threads).
//   S = Q K^T   : wgmma m64n128k16 x DH / 16, both operands K-major in shared memory, fp32 in registers
//   softmax     : online max / sum in fp32 on the accumulator fragment (a row is spread over the four threads of a
//                 quad: two shuffles per row max); exponentials with MUFU.EX2 in log2 units
//   O += P V    : P is converted to packed fp16 in registers — the accumulator fragment of S has exactly the layout of
//                 wgmma's register A operand, so P never touches shared memory — times V consumed MN-major straight
//                 from its TMA layout (wgmma m64nDHk16, transposed B; at DH = 128 the two 64-column boxes of V are the
//                 two 64-wide MN blocks of the operand, kAttnTile bytes apart)
// The warpgroups run independently, so one's exponentials overlap another's tensor-core work.  Every query row goes
// through the same instructions whatever QWG is, so both widths give the same output bit for bit; QWG = 4 (one CTA
// per SM) puts twice the rows on each SM's tensor cores and halves the K/V loads per query.
#pragma once
#include "common.cuh"
#include "kparams.h"
#include "wgmma.cuh"

namespace f5 {

__device__ __forceinline__ float ex2_approx(float x) {  // one MUFU.EX2; -inf -> 0
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// JOINT (MMDiT joint attention, reference model/modules.py:563-705): queries and keys are [audio | text], the audio
// segment read through tmQKV ([Be, seq, 3 inner]) and the text segment through tmC ([Be, jp.seq_c, 3 inner]).  Query
// blocks [0, jp.q_blocks_a) are audio, the rest text; each writes its own segment's output.  The producer streams the
// audio key tiles, then the text key tiles, through the same ring; the tail of each segment is masked on its own, so
// every tile still holds at least one valid key.  A text segment with no valid keys contributes no tile.
template <int DH, bool JOINT, int QWG>
__device__ __forceinline__ void attn_fwd_body(const CUtensorMap* tmQKV, const CUtensorMap* tmC, const AttnParams& p,
                                              const AttnJointParams& jp) {
  static_assert(DH == 64 || DH == 128, "head width");
  static_assert(QWG == 2 || (QWG == 4 && DH == 64), "4 query warpgroups only at head width 64 (register budget)");
  constexpr int BOXES = DH / 64;                   // 64-column TMA boxes per tile row
  constexpr uint32_t TILE = kAttnTile * BOXES;     // one 128-row tile of q, k or v
  constexpr int QBOXES = QWG / 2;                  // 128-row tiles of q
  constexpr int BQ = 64 * QWG;                     // query rows per CTA
  constexpr int PRODUCER = QWG == 2 ? 8 : 0;       // warp that issues the TMA loads (at QWG = 4 a consumer warp)
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - smem_u32(smem_raw));
  uint8_t* sQ = smem;                              // QBOXES tiles: warpgroup g's 64 rows start at g * 8 KB
  uint8_t* sK = sQ + QBOXES * TILE;                // kAttnStages tiles
  uint8_t* sV = sK + kAttnStages * TILE;           // kAttnStages tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kAttnStages * TILE);
  uint64_t* q_full = bars;                         // [1]
  uint64_t* k_full = q_full + 1;                   // [stages]
  uint64_t* k_empty = k_full + kAttnStages;        // [stages]
  uint64_t* v_full = k_empty + kAttnStages;        // [stages]
  uint64_t* v_empty = v_full + kAttnStages;        // [stages]

  const int warp = threadIdx.x >> 5;
  const int qb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  bool text_q = false;  // JOINT: this CTA's queries are text rows
  int q0 = qb * BQ;
  if constexpr (JOINT) {
    text_q = qb >= jp.q_blocks_a;
    if (text_q) q0 = (qb - jp.q_blocks_a) * BQ;
  }
  const CUtensorMap* tmQ = text_q ? tmC : tmQKV;
  const int col_q = h * DH, col_k = p.inner + h * DH, col_v = 2 * p.inner + h * DH;

  if (warp == PRODUCER && elect_one()) {
    tma_prefetch_desc(tmQKV);
    if constexpr (JOINT) tma_prefetch_desc(tmC);
    mbar_init(q_full, 1);
    for (int s = 0; s < kAttnStages; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&k_empty[s], 4 * QWG);  // one arrival per consumer warp
      mbar_init(&v_full[s], 1);
      mbar_init(&v_empty[s], 4 * QWG);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();
  // a sample always has at least one key: kv_len < 1 (caller error on the public entry point) is treated as 1
  const int kv_len = p.kv_len ? max(1, min(p.kv_len[b], p.seq)) : p.seq;
  int n_kv = (kv_len + kAttnBKV - 1) / kAttnBKV;
  const int n_kv_a = n_kv;  // JOINT: tiles [n_kv_a, n_kv) are text keys
  int kv_len_c = 0;
  if constexpr (JOINT) {
    kv_len_c = jp.c_len ? max(0, min(jp.c_len[b], jp.seq_c)) : jp.seq_c;
    n_kv += (kv_len_c + kAttnBKV - 1) / kAttnBKV;
  }

  // QWG = 4 (BOXES = 1): K and V of key tile j into ring slot j % kAttnStages, once that slot is free
  auto load_kv = [&](int j) {
    const int s = j % kAttnStages;
    bool text_kv = false;
    if constexpr (JOINT) text_kv = j >= n_kv_a;
    const CUtensorMap* tmKV = text_kv ? tmC : tmQKV;
    const int k0 = (text_kv ? j - n_kv_a : j) * kAttnBKV;
    mbar_expect_tx(&k_full[s], TILE);
    tma_load_3d(sK + s * TILE, tmKV, &k_full[s], col_k, k0, b);
    mbar_expect_tx(&v_full[s], TILE);
    tma_load_3d(sV + s * TILE, tmKV, &v_full[s], col_v, k0, b);
  };
  if constexpr (QWG == 4) {
    if (warp == PRODUCER && lane_id() == 0) {  // q tiles that hold no query row of the sample are not loaded
      const int seq_q = text_q ? jp.seq_c : p.seq;
      const int nq = min(QBOXES, (seq_q - q0 + 127) / 128);
      mbar_expect_tx(q_full, nq * TILE);
      for (int t = 0; t < nq; ++t) tma_load_3d(sQ + t * TILE, tmQ, q_full, col_q, q0 + 128 * t, b);
      for (int j = 0; j < min(n_kv, kAttnStages); ++j) load_kv(j);  // the empty ring; later tiles: consumer loop
    }
  } else if (warp == PRODUCER) {
    if (elect_one()) {
      mbar_expect_tx(q_full, TILE);
#pragma unroll
      for (int c = 0; c < BOXES; ++c) tma_load_3d(sQ + c * kAttnTile, tmQ, q_full, col_q + 64 * c, q0, b);
      if constexpr (JOINT) {
        for (int j = 0; j < n_kv; ++j) {
          const int s = j % kAttnStages;
          const uint32_t ph = (j / kAttnStages) & 1;
          const bool text_kv = j >= n_kv_a;
          const CUtensorMap* tmKV = text_kv ? tmC : tmQKV;
          const int k0 = (text_kv ? j - n_kv_a : j) * kAttnBKV;
          mbar_wait(&k_empty[s], ph ^ 1);
          mbar_expect_tx(&k_full[s], TILE);
#pragma unroll
          for (int c = 0; c < BOXES; ++c)
            tma_load_3d(sK + s * TILE + c * kAttnTile, tmKV, &k_full[s], col_k + 64 * c, k0, b);
          mbar_wait(&v_empty[s], ph ^ 1);
          mbar_expect_tx(&v_full[s], TILE);
#pragma unroll
          for (int c = 0; c < BOXES; ++c)
            tma_load_3d(sV + s * TILE + c * kAttnTile, tmKV, &v_full[s], col_v + 64 * c, k0, b);
        }
      } else {
        for (int j = 0; j < n_kv; ++j) {
          const int s = j % kAttnStages;
          const uint32_t ph = (j / kAttnStages) & 1;
          mbar_wait(&k_empty[s], ph ^ 1);
          mbar_expect_tx(&k_full[s], TILE);
#pragma unroll
          for (int c = 0; c < BOXES; ++c)
            tma_load_3d(sK + s * TILE + c * kAttnTile, tmQKV, &k_full[s], col_k + 64 * c, j * kAttnBKV, b);
          mbar_wait(&v_empty[s], ph ^ 1);
          mbar_expect_tx(&v_full[s], TILE);
#pragma unroll
          for (int c = 0; c < BOXES; ++c)
            tma_load_3d(sV + s * TILE + c * kAttnTile, tmQKV, &v_full[s], col_v + 64 * c, j * kAttnBKV, b);
        }
      }
    }
    return;
  }

  // ===== consumer warpgroup g: query rows r and r + 8 of its 64, columns 8 j + c2 (+1) of each fragment =====
  const int g = warp >> 2;
  const int lane = int(lane_id());
  const int r = 64 * g + 16 * (warp & 3) + (lane >> 2);
  const int c2 = 2 * (lane & 3);
  const uint64_t qdesc = make_wgmma_desc_sw128(smem_u32(sQ + g * (64 * 128)));
  if constexpr (QWG > 2) {
    const int seq_q = text_q ? jp.seq_c : p.seq;
    if (q0 + 64 * g >= seq_q) {  // no query row of the sample: no MMA, but every ring slot is waited on and released
      for (int j = 0; j < n_kv; ++j) {
        const int s = j % kAttnStages;
        const uint32_t ph = (j / kAttnStages) & 1;
        mbar_wait(&k_full[s], ph);
        __syncwarp();
        if (lane == 0) mbar_arrive(&k_empty[s]);
        mbar_wait(&v_full[s], ph);
        __syncwarp();
        if (lane == 0) mbar_arrive(&v_empty[s]);
      }
      return;
    }
  }
  float o[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.0f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.0f, 0.0f};  // l: this thread's partial row sums
  mbar_wait(q_full, 0);
  for (int j = 0; j < n_kv; ++j) {
    const int s = j % kAttnStages;
    const uint32_t ph = (j / kAttnStages) & 1;
    if constexpr (QWG == 4) {
      // warp 0 refills the slot of tile j - 1 with tile j + 2 once every warp has released it.  Warpgroup 0 itself
      // released it last iteration, and the other warpgroups may run up to two tiles ahead of it, so in steady state
      // it finds the slot free and the load is issued two tiles before it is needed.  (Warpgroup 0 always has a
      // query row, so it never takes the no-MMA path above.)
      if (warp == PRODUCER && j >= 1 && j + 2 < n_kv) {
        if (lane == 0) {
          const int sf = (j + 2) % kAttnStages;
          const uint32_t phf = ((j - 1) / kAttnStages) & 1;
          mbar_wait(&k_empty[sf], phf);
          mbar_wait(&v_empty[sf], phf);
          load_kv(j + 2);
        }
        __syncwarp();
      }
    }
    int kv_rem = kv_len - j * kAttnBKV;  // valid keys in this tile (>= 1)
    if constexpr (JOINT) {
      if (j >= n_kv_a) kv_rem = kv_len_c - (j - n_kv_a) * kAttnBKV;
    }
    float sc[64];
    mbar_wait(&k_full[s], ph);
    const uint64_t kdesc = make_wgmma_desc_sw128(smem_u32(sK + s * TILE));
    wgmma_fence();
    // k-step k: 16 columns of the head, in box k / 4 (kAttnTile bytes = kAttnTile >> 4 descriptor units further on)
#pragma unroll
    for (int k = 0; k < DH / 16; ++k) {
      const uint64_t off = uint64_t((k >> 2) * (kAttnTile >> 4) + 2 * (k & 3));
      wgmma_ss_n128(sc, qdesc + off, kdesc + off, k != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&k_empty[s]);
    if (kv_rem < kAttnBKV) {  // last tile of the sample: keys at or past the end get a score of -inf
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (8 * (i >> 2) + c2 + (i & 1) >= kv_rem) sc[i] = -INFINITY;
    }
    float alpha[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {  // fragment row hr: sc[4 j + 2 hr], sc[4 j + 2 hr + 1]
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(sc[4 * jj + 2 * hr], sc[4 * jj + 2 * hr + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[hr], mx * p.scale_log2);  // finite: every tile holds at least one valid key
      alpha[hr] = ex2_approx(m_run[hr] - m_new);                // first tile: exp2(-inf) = 0
      m_run[hr] = m_new;
      float sum = 0.0f;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const float e0 = ex2_approx(fmaf(sc[4 * jj + 2 * hr], p.scale_log2, -m_new));
        const float e1 = ex2_approx(fmaf(sc[4 * jj + 2 * hr + 1], p.scale_log2, -m_new));
        sc[4 * jj + 2 * hr] = e0;
        sc[4 * jj + 2 * hr + 1] = e1;
        sum += e0 + e1;
      }
      l_run[hr] = l_run[hr] * alpha[hr] + sum;
    }
#pragma unroll
    for (int jj = 0; jj < DH / 8; ++jj) {
      o[4 * jj + 0] *= alpha[0];
      o[4 * jj + 1] *= alpha[0];
      o[4 * jj + 2] *= alpha[1];
      o[4 * jj + 3] *= alpha[1];
    }
    // P as wgmma A fragments: keys [16 kk, 16 kk + 16) are S fragment columns 2 kk and 2 kk + 1
    uint32_t pa[8][4];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      pa[kk][0] = pack_half2(sc[8 * kk + 0], sc[8 * kk + 1]);
      pa[kk][1] = pack_half2(sc[8 * kk + 2], sc[8 * kk + 3]);
      pa[kk][2] = pack_half2(sc[8 * kk + 4], sc[8 * kk + 5]);
      pa[kk][3] = pack_half2(sc[8 * kk + 6], sc[8 * kk + 7]);
    }
    mbar_wait(&v_full[s], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {  // B = 16 key rows of V (2 KB apart), MN-major
      if constexpr (DH == 64)
        wgmma_rs_n64_bt(o, pa[kk], make_wgmma_desc_sw128(smem_u32(sV + s * TILE + kk * 16 * 128)), 1);
      else
        wgmma_rs_n128_bt(o, pa[kk], make_wgmma_desc_sw128_mn(smem_u32(sV + s * TILE + kk * 16 * 128), kAttnTile), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&v_empty[s]);
  }
  // epilogue: O / l -> fp16 (the row sum is spread over the quad)
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    float l = l_run[hr];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv_l = 1.0f / l;
    const int qrow = q0 + r + 8 * hr;
    const int seq_o = text_q ? jp.seq_c : p.seq;
    if (qrow < seq_o) {
      __half* out = (text_q ? jp.out_c : p.out) + ((long long)b * seq_o + qrow) * p.inner + h * DH + c2;
#pragma unroll
      for (int jj = 0; jj < DH / 8; ++jj)
        *reinterpret_cast<uint32_t*>(out + 8 * jj) = pack_half2(o[4 * jj + 2 * hr] * inv_l, o[4 * jj + 2 * hr + 1] * inv_l);
    }
  }
}

template <int DH, int QWG>
__global__ void __launch_bounds__(attn_threads(QWG), 1)
attn_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQKV, const AttnParams p) {
  attn_fwd_body<DH, false, QWG>(&tmQKV, &tmQKV, p, AttnJointParams{});
}

template <int DH, int QWG>
__global__ void __launch_bounds__(attn_threads(QWG), 1)
attn_joint_wgmma_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmC,
                        const AttnParams p, const AttnJointParams jp) {
  attn_fwd_body<DH, true, QWG>(&tmQKV, &tmC, p, jp);
}

}  // namespace f5

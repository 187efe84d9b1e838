// Persistent, warp-specialised wgmma GEMM / grouped-conv-as-GEMM for sm_90a.
//
//   C[m, n] = epilogue( sum_k A[m, k] * W[n, k] )        A, W fp16, K-major; fp32 accumulation in registers.
//
// grid = min(#tiles, #SMs); every CTA walks tiles t = blockIdx.x, +gridDim.x, ... (n fastest, so CTAs that run
// together share the A row-panel in L2 and sweep W once).  Warp roles (288 threads):
//   warps 0..7    two consumer warpgroups: warpgroup g computes rows [64 g, 64 g + 64) of the 128 x BN tile with
//                 wgmma m64nBNk16 (both operands read from shared memory), then runs the fused bias / activation /
//                 qk RMSNorm / RoPE (64- or 128-column heads) / gate / mask epilogue straight from its accumulator
//                 registers
//   warp 8        TMA producer (one elected lane): STAGES-deep ring of {A 128x64, W BNx64} fp16 tiles, SWIZZLE_128B.  It
//                 runs ahead into the next tile's k-blocks while the consumers are in the epilogue.
// Pipeline: smem full / empty mbarriers (TMA <-> wgmma); every consumer warp releases a slot once its MMAs retired.
// Tails in M, N and K come from TMA out-of-bounds zero fill plus guarded stores.
//
// CONV mode computes the reference's grouped Conv1d(k=31, groups=16, padding=15) (model/modules.py:175-201) with
// G = conv_g channels per group (a multiple of 8, at most 64; G = dim / 16) as 31 accumulated 128x64x64 GEMMs per
// (row tile, group): tap t multiplies the activation tile shifted by (t - 15) rows — the shift is just the TMA row
// coordinate, and rows outside [0, seq) of the SAME sample are zero-filled by the 4-D tensor map {G, groups, rows,
// batches}, which is exactly the conv's zero padding.  Columns G..63 of the A and W tiles are zero-filled too, so a
// group never reads its neighbours' channels; at G < 64 the tensor cores do 64 / G times the algorithmic work.
// Output columns n0 + G.. of a tile are never stored.
#pragma once
#include "common.cuh"
#include "kparams.h"
#include "wgmma.cuh"

namespace f5 {

constexpr int kGemmThreads = 288;  // two consumer warpgroups + one producer warp
constexpr int kGemmEmptyArrivals = 8;  // consumer warps per CTA

// depth of the {A, W} k-block ring for a BN-wide tile
__host__ __device__ constexpr int gemm_stages(int bn) { return bn == 64 ? 7 : bn == 128 ? 5 : bn == 192 ? 4 : 3; }

constexpr size_t gemm_smem_bytes(int bn) {
  return size_t(gemm_stages(bn)) * (kBM * kBK * 2 + bn * kBK * 2) + 1024 /*align slack*/ + 256 /*barriers*/;
}

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t da, uint64_t db, int scale_d) {
  if constexpr (BN == 64) wgmma_ss_n64(d, da, db, scale_d);
  else if constexpr (BN == 128) wgmma_ss_n128(d, da, db, scale_d);
  else if constexpr (BN == 192) wgmma_ss_n192(d, da, db, scale_d);
  else wgmma_ss_n256(d, da, db, scale_d);
}

// Packed / variable-length execution (SURVEY.md §8f-1; reference masked mode modules.py:513-540): with skip_pad, a tile
// whose rows ALL lie past the end of their sample is never loaded, multiplied or stored.  Every warp role evaluates the
// same predicate, so the smem ring and the tile order stay in step.  m0 = first row of the tile;
// CONV: rows are per sample (bz), plain: rows are the flattened [samples x seq] axis.
template <bool CONV>
__device__ __forceinline__ bool tile_is_padding(const GemmParams& p, int m0, int bz) {
  if (!p.skip_pad) return false;
  if (CONV) return m0 >= p.row_len[bz];
  const int last = min(m0 + kBM, p.rows) - 1;
  const int b0 = m0 / p.seq;
  if (b0 != last / p.seq) return false;  // the tile reaches into the next sample, whose first rows are valid
  return m0 - b0 * p.seq >= p.row_len[b0];
}

// Fused epilogue of one thread's accumulator fragment: rows row0 and row0 + 8 (half h = 0, 1), columns
// n0 + 8 j + c2 (+ 1) in acc[4 j + 2 h] (+ 1), up to n_end().  It runs over chunks of 8 to 64 columns, and every global
// load of a chunk (bias, gate, RoPE cos / sin, residual) is issued before the first store of the chunk.  Stores may
// alias those inputs as far as the compiler knows, so a loop that loads and stores per column pair waits one full
// memory latency per pair; here a chunk waits about once.
template <int BN, int EPI, int ACT, bool CONV>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, float* acc, int n0, int c2, int row0, int bz,
                                              const float* gate) {
  // first column not stored: a CONV tile ends with its group.  Evaluated at each use, so the plain kernels compile
  // exactly as when they compared with p.n_out directly.
  auto n_end = [&]() { return CONV ? n0 + p.conv_g : p.n_out; };
  constexpr bool NORM = EPI == EPI_QKV_NORM_ROPE || EPI == EPI_QKV_NORM_ROPE_DH128;
  // per-sample gate rows (EPI_RESID_SAMPLE): each of the thread's two rows may lie in another sample
  constexpr bool PS = EPI == EPI_RESID_SAMPLE;
  constexpr bool RESID = EPI == EPI_RESID || PS;
  constexpr bool QKV = EPI == EPI_QKV_ROPE || EPI == EPI_QKV_ROPE_DH128 || NORM;
  // head width of the QKV epilogues (columns of one q, k or v head)
  constexpr int DH = (EPI == EPI_QKV_ROPE_DH128 || EPI == EPI_QKV_NORM_ROPE_DH128) ? 128 : 64;
  constexpr int LOG_DH = DH == 128 ? 7 : 6;
  // chunk width: the widest whose loads fit beside the BN / 2 accumulators without spilling (ptxas caps a 288-thread
  // CTA at 168 registers per thread).  QKV_NORM_ROPE adds its bias before the chunks, which frees the bias registers.
  // RESID_SAMPLE keeps a second row of gates: half the RESID chunk at 128 and 256.
  constexpr int CW = NORM ? (BN <= 128 ? 64 : BN == 192 ? 32 : 8)
                   : PS   ? (BN == 256 ? 8 : 32)
                   : BN <= 128 ? (QKV ? 32 : 64)
                     : BN == 192 ? (QKV ? 16 : 32)
                                 : (EPI == EPI_F16 ? 32 : RESID ? 16 : 8);
  constexpr int J = CW / 8;  // column pairs of one thread in a chunk
  bool in[2], valid[2];
  long long grow[2];
  int pos[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = row0 + 8 * h;
    in[h] = r < p.rows;
    grow[h] = (long long)bz * p.rows + r;
    valid[h] = true;
    pos[h] = 0;
    if (in[h] && p.seq > 0) {
      pos[h] = int(grow[h] % p.seq);
      if (p.row_len != nullptr) valid[h] = pos[h] < p.row_len[grow[h] / p.seq];
    }
    if (RESID) in[h] = in[h] && valid[h];  // masked rows keep their residual
  }
  const float* gate_row[2] = {gate, gate};
  if (PS && gate != nullptr) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (in[h]) gate_row[h] = gate + (long long)((grow[h] / p.gate_seq) % p.gate_samples) * p.gate_step_stride;
  }
  // qk_norm shuffles within quads: every lane of the warp has to reach them, so no lane leaves early
  if (!NORM && !in[0] && !in[1]) return;
  float rinv[2];  // qk_norm: 1 / RMS of rows row0, row0 + 8 of the current head
#pragma unroll
  for (int cc = 0; cc < BN / CW; ++cc) {
    const int nb = n0 + CW * cc;
    if (nb >= n_end()) break;
    // qk_norm, at the first chunk of a head: the bias goes into the head's accumulators here (the chunks below add none),
    // then, for a q or k head, 1 / RMS over its DH columns in fp32.  The head lies in this tile (BN, n0 and CW divide
    // into DH-column heads: at DH = 128 only the 128-wide tile is instantiated); one row of it is spread over the
    // 4 lanes of a quad, DH / 4 values each, so one pass over the head's registers and two quad shuffles give the sum of
    // squares.  Kept per head, not per tile: 16 live values for a 256-wide tile spill.
    if (NORM && ((CW * cc) & (DH - 1)) == 0) {
      const int hb = (CW * cc) >> 3;  // first 8-column group of the head
      const bool qk = nb / p.inner < 2;  // the same for the whole warp
      float ss[2] = {0.0f, 0.0f};
#pragma unroll
      for (int j = 0; j < DH / 8; ++j) {
        float2 b = make_float2(0.0f, 0.0f);
        if (p.bias != nullptr) b = __ldg(reinterpret_cast<const float2*>(p.bias + nb + 8 * j + c2));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float& v0 = acc[4 * (hb + j) + 2 * h];
          float& v1 = acc[4 * (hb + j) + 2 * h + 1];
          v0 += b.x;
          v1 += b.y;
          if (qk) ss[h] += v0 * v0 + v1 * v1;
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        ss[h] += __shfl_xor_sync(0xffffffffu, ss[h], 1);
        ss[h] += __shfl_xor_sync(0xffffffffu, ss[h], 2);
        rinv[h] = rsqrtf(ss[h] * (1.0f / float(DH)) + 1e-6f);
      }
    }
    if (NORM && !in[0] && !in[1]) continue;
    // ---- loads ----
    float2 b[J], g[J], gs[2][J];  // gs: PS only, the gates of rows row0 and row0 + 8
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int nc = nb + 8 * j + c2;
      b[j] = make_float2(0.0f, 0.0f);
      g[j] = make_float2(1.0f, 1.0f);
      gs[0][j] = gs[1][j] = g[j];
      if (nc >= n_end()) continue;
      const bool pair_ok = nc + 1 < n_end();
      if (!NORM && p.bias != nullptr) {
        if (pair_ok) b[j] = __ldg(reinterpret_cast<const float2*>(p.bias + nc));
        else b[j].x = __ldg(p.bias + nc);
      }
      if (EPI == EPI_RESID && gate != nullptr) {
        g[j].x = gate[nc];
        if (pair_ok) g[j].y = gate[nc + 1];
      }
      if (PS && gate != nullptr) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!in[h]) continue;
          gs[h][j].x = gate_row[h][nc];
          if (pair_ok) gs[h][j].y = gate_row[h][nc + 1];
        }
      }
    }
    bool rope = false, nrm = false;
    float rc[2][J], rs[2][J];
    float2 gn[J];
    if (QKV) {  // inner % DH == 0 and CW divides DH: a chunk lies in one head of one section
      const int sec = nb / p.inner, head = (nb - sec * p.inner) >> LOG_DH;
      rope = sec < 2 && head < p.pe_heads;
      if (NORM) {
        nrm = sec < 2;
        if (nrm) {
          const float* gw = sec == 0 ? p.q_norm : p.k_norm;
#pragma unroll
          for (int j = 0; j < J; ++j) gn[j] = __ldg(reinterpret_cast<const float2*>(gw + (nb & (DH - 1)) + 8 * j + c2));
        }
      }
      if (rope) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < J; ++j) {
            const int pr = ((nb & (DH - 1)) >> 1) + 4 * j + (c2 >> 1);
            rc[h][j] = in[h] ? __ldg(p.rope_cos + (long long)pos[h] * (DH / 2) + pr) : 0.0f;
            rs[h][j] = in[h] ? __ldg(p.rope_sin + (long long)pos[h] * (DH / 2) + pr) : 0.0f;
          }
      }
    }
    float2 x[2][J];
    if (RESID) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < J; ++j) {
          const int nc = nb + 8 * j + c2;
          const float* o = p.resid + grow[h] * p.ldo + nc;
          x[h][j] = make_float2(0.0f, 0.0f);
          if (!in[h] || nc >= n_end()) continue;
          if (nc + 1 < n_end()) x[h][j] = *reinterpret_cast<const float2*>(o);  // ldo % 4 == 0, nc even: aligned
          else x[h][j].x = o[0];
        }
    }
    // ---- math and stores ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!in[h]) continue;
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int nc = nb + 8 * j + c2;
        if (nc >= n_end()) continue;
        const bool pair_ok = nc + 1 < n_end();
        float v0 = acc[4 * (J * cc + j) + 2 * h], v1 = acc[4 * (J * cc + j) + 2 * h + 1];
        if (!NORM && p.bias != nullptr) {
          v0 += b[j].x;
          if (pair_ok) v1 += b[j].y;
        }
        if (NORM && nrm) {
          const float r = rinv[h];
          v0 = v0 * r * gn[j].x;
          v1 = v1 * r * gn[j].y;
        }
        if (QKV && rope) {
          const float c = rc[h][j], s = rs[h][j];
          const float x0 = v0, x1 = v1;
          v0 = x0 * c - x1 * s;
          v1 = x1 * c + x0 * s;
        }
        if (ACT == ACT_GELU_TANH) {
          v0 = gelu_tanh(v0);
          v1 = gelu_tanh(v1);
        } else if (ACT == ACT_GELU_ERF) {
          v0 = gelu_erf(v0);
          v1 = gelu_erf(v1);
        } else if (ACT == ACT_MISH) {
          v0 = mish(v0);
          v1 = mish(v1);
        }
        if (EPI == EPI_F16 || QKV) {
          __half* o = reinterpret_cast<__half*>(p.out) + grow[h] * p.ldo + nc;
          if (!valid[h]) v0 = v1 = 0.0f;
          if (pair_ok) *reinterpret_cast<uint32_t*>(o) = pack_half2(v0, v1);
          else *o = __float2half_rn(v0);
        } else if (EPI == EPI_F32) {
          float* o = reinterpret_cast<float*>(p.out) + grow[h] * p.ldo + nc;
          if (pair_ok && !(p.ldo & 1)) {
            *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
          } else {
            o[0] = v0;
            if (pair_ok) o[1] = v1;
          }
          if (p.out16b != nullptr) {
            __half* o2 = p.out16b + grow[h] * p.ldo + nc;
            if (!valid[h]) v0 = v1 = 0.0f;
            if (pair_ok && !(p.ldo & 1)) {
              *reinterpret_cast<uint32_t*>(o2) = pack_half2(v0, v1);
            } else {
              o2[0] = __float2half_rn(v0);
              if (pair_ok) o2[1] = __float2half_rn(v1);
            }
          }
        } else if (RESID) {
          float* o = p.resid + grow[h] * p.ldo + nc;
          float2 xv = x[h][j];
          const float2 gg = PS ? gs[h][j] : g[j];
          if (pair_ok) {
            xv.x += gg.x * v0;
            xv.y += gg.y * v1;
            *reinterpret_cast<float2*>(o) = xv;
          } else {
            o[0] = xv.x + gg.x * v0;
          }
        }
      }
    }
  }
}

template <int BN, int EPI, int ACT, bool CONV>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  static_assert(BN == 64 || BN == 128 || BN == 192 || BN == 256, "BN");
  constexpr int STAGES = gemm_stages(BN);
  constexpr uint32_t A_BYTES = kBM * kBK * 2;
  constexpr uint32_t B_BYTES = BN * kBK * 2;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base - smem_u32(smem_raw));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(sB + STAGES * B_BYTES);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5;
  const int cta_id = int(blockIdx.x);
  const int cta_step = int(gridDim.x);
  // CONV: one output tile per group of conv_g channels; the tile's columns past conv_g are computed, never stored
  const int tile_w = CONV ? p.conv_g : BN;
  const int tiles_n = CONV ? p.n_out / p.conv_g : (p.n_out + BN - 1) / BN;
  const int tiles_m = (p.rows + kBM - 1) / kBM;
  const int num_tiles = tiles_n * tiles_m * p.batches;

  if (warp == 8 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kGemmEmptyArrivals);
    }
    fence_mbar_init();
  }
  __syncthreads();
  // Programmatic dependent launch: everything above overlapped the predecessor's tail.  The producer goes one step
  // further (below): W tiles are weights, not produced by the predecessor, so their TMA loads are issued BEFORE the
  // dependency wait and the DRAM latency of the first STAGES k-blocks hides under the predecessor too.
  if (warp != 8) pdl_wait();  // predecessor kernel finished: its outputs (our A operand, residual, ...) are visible
  pdl_launch_dependents();    // let the next kernel's prologue overlap our tail

  if (warp == 8) {
    if (elect_one()) {
      // ===== TMA producer =====
      uint32_t it = 0;  // running k-block counter across tiles -> stage / phase
      auto load_w = [&](int s, int kb, int n0) {
        if (CONV) tma_load_2d(sB + s * B_BYTES, &tmB, &full[s], 0, kb * p.n_out + n0);  // [tap][out_channel][in G]
        else tma_load_2d(sB + s * B_BYTES, &tmB, &full[s], kb * kBK, n0);
      };
      // weights of the first tile's first k-blocks: in flight before the dependency wait (slots are free at start)
      uint32_t pre = 0;
      if (cta_id < num_tiles && p.w_prefetch) {
        pre = uint32_t(p.num_kb < STAGES ? p.num_kb : STAGES);
        for (uint32_t kb = 0; kb < pre; ++kb) {
          mbar_expect_tx(&full[kb], A_BYTES + B_BYTES);
          load_w(int(kb), int(kb), (cta_id % tiles_n) * tile_w);
        }
      }
      pdl_wait();
      for (int t = cta_id; t < num_tiles; t += cta_step) {
        const int n0 = (t % tiles_n) * tile_w;
        const int m0 = ((t / tiles_n) % tiles_m) * kBM;
        const int bz = t / (tiles_n * tiles_m);
        if (tile_is_padding<CONV>(p, m0, bz)) continue;
        for (int kb = 0; kb < p.num_kb; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          if (it >= pre) {
            mbar_wait(&empty[s], ph ^ 1);
            mbar_expect_tx(&full[s], A_BYTES + B_BYTES);
            load_w(s, kb, n0);
          }
          if (CONV) tma_load_4d(sA + s * A_BYTES, &tmA, &full[s], 0, t % tiles_n, m0 + kb - p.conv_pad, bz);  // tap shift
          else tma_load_3d(sA + s * A_BYTES, &tmA, &full[s], kb * kBK, m0, bz);
        }
      }
    }
  } else {
    // ===== consumers: warpgroup g owns rows [64 g, 64 g + 64) of the tile =====
    const int g = warp >> 2;
    const int lane = int(lane_id());
    const int r_in_tile = 64 * g + 16 * (warp & 3) + (lane >> 2);  // fragment rows r_in_tile and r_in_tile + 8
    const int c2 = 2 * (lane & 3);
    const float* gate = nullptr;
    if (EPI == EPI_RESID && p.gate != nullptr)
      gate = p.gate + (p.step_ptr ? (long long)(*p.step_ptr) : 0) * p.gate_step_stride;
    if (EPI == EPI_RESID_SAMPLE) gate = p.gate;  // the row of each output row's sample is picked in the epilogue
    float acc[BN / 2];
    uint32_t it = 0;
    auto release = [&](int s) {
      if (lane == 0) mbar_arrive(&empty[s]);
    };
    for (int t = cta_id; t < num_tiles; t += cta_step) {
      const int n0 = (t % tiles_n) * tile_w;
      const int m0 = ((t / tiles_n) % tiles_m) * kBM;
      const int bz = t / (tiles_n * tiles_m);
      if (tile_is_padding<CONV>(p, m0, bz)) continue;
      int prev = -1;
      for (int kb = 0; kb < p.num_kb; ++kb, ++it) {
        const int s = it % STAGES;
        mbar_wait(&full[s], (it / STAGES) & 1);
        const uint64_t adesc = make_wgmma_desc_sw128(smem_u32(sA + s * A_BYTES + g * (64 * 128)));
        const uint64_t bdesc = make_wgmma_desc_sw128(smem_u32(sB + s * B_BYTES));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k)  // +32 bytes (16 fp16) along K inside the 128B swizzle atom = +2
          wgmma_tile<BN>(acc, adesc + uint64_t(2 * k), bdesc + uint64_t(2 * k), (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs retired: its slot goes back to the producer
        wgmma_fence_regs(acc);
        if (prev >= 0) release(prev);
        prev = s;
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      release(prev);
#ifdef F5_TRACE
      if (p.diag_no_epi) continue;  // main loop alone (F5_GEMM_EPI=none)
#endif
      epilogue_tile<BN, EPI, ACT, CONV>(p, acc, n0, c2, m0 + r_in_tile, bz, gate);
    }
  }
}

}  // namespace f5

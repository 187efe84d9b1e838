// Host side of the wgmma GEMM: tensor-map encoding, instantiation table, launch, C entry point f5_gemm.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <atomic>
#include <mutex>

#include "gemm.cuh"
#include "internal.h"

namespace f5 {

static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add((unsigned long long)(long long)n, std::memory_order_relaxed); }
int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return 0;
  set_error("%s: %s", what, cudaGetErrorString(e));
  return -2;
}
int check_launch(const char* what) { return check_cuda(cudaGetLastError(), what); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int encode_tmap_f16(CUtensorMap* m, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides,
                    const uint32_t* box) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver / not a TMA-capable device)");
    return -3;
  }
  bool aligned = !(reinterpret_cast<uintptr_t>(ptr) & 15);
  for (int i = 0; i + 1 < rank; ++i) aligned = aligned && !(strides[i] & 15);
  if (!aligned) {
    set_error("tensor map: pointer/strides must be 16-byte aligned (ptr=%p s1=%llu)", ptr,
              (unsigned long long)strides[0]);
    return -4;
  }
  cuuint64_t gd[4];
  cuuint64_t gs[3];
  cuuint32_t bx[4];
  cuuint32_t estr[4] = {1, 1, 1, 1};
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    if (i + 1 < rank) gs[i] = strides[i];
  }
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), gd, gs, bx, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed: %d (rank %d dims %llu,%llu box %u,%u)", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    return -5;
  }
  return 0;
}

// Every instantiated GEMM kernel.  configure_kernels sets them all up, gemm_run launches the entry that matches a plan,
// and pick_tile only considers widths that have an entry for the epilogue.
struct GemmKernel {
  int bn, epi, act;
  bool conv;
  void (*fn)(CUtensorMap, CUtensorMap, GemmParams);
};
#define F5_GEMM_KERNEL(BN, EPI, ACT, CONV) {BN, EPI, ACT, CONV, gemm_wgmma_kernel<BN, EPI, ACT, CONV>}
static const GemmKernel kGemmKernels[] = {
    F5_GEMM_KERNEL(64, EPI_F16, ACT_NONE, false),
    F5_GEMM_KERNEL(64, EPI_F16, ACT_GELU_TANH, false),
    F5_GEMM_KERNEL(64, EPI_F16, ACT_GELU_ERF, false),
    F5_GEMM_KERNEL(64, EPI_F32, ACT_NONE, false),
    F5_GEMM_KERNEL(64, EPI_RESID, ACT_NONE, false),
    F5_GEMM_KERNEL(128, EPI_F16, ACT_NONE, false),
    F5_GEMM_KERNEL(128, EPI_F16, ACT_GELU_TANH, false),
    F5_GEMM_KERNEL(128, EPI_F16, ACT_GELU_ERF, false),
    F5_GEMM_KERNEL(128, EPI_F32, ACT_NONE, false),
    F5_GEMM_KERNEL(128, EPI_RESID, ACT_NONE, false),
    F5_GEMM_KERNEL(256, EPI_F16, ACT_NONE, false),
    F5_GEMM_KERNEL(256, EPI_F16, ACT_GELU_TANH, false),
    F5_GEMM_KERNEL(256, EPI_F16, ACT_GELU_ERF, false),
    F5_GEMM_KERNEL(256, EPI_F32, ACT_NONE, false),
    F5_GEMM_KERNEL(256, EPI_RESID, ACT_NONE, false),
    F5_GEMM_KERNEL(128, EPI_QKV_ROPE, ACT_NONE, false),
    F5_GEMM_KERNEL(192, EPI_QKV_ROPE, ACT_NONE, false),
    F5_GEMM_KERNEL(192, EPI_F16, ACT_NONE, false),
    F5_GEMM_KERNEL(192, EPI_F16, ACT_GELU_TANH, false),
    F5_GEMM_KERNEL(192, EPI_RESID, ACT_NONE, false),
    F5_GEMM_KERNEL(256, EPI_QKV_ROPE, ACT_NONE, false),
    F5_GEMM_KERNEL(64, EPI_F16, ACT_MISH, true),
    F5_GEMM_KERNEL(64, EPI_RESID, ACT_MISH, true),
    F5_GEMM_KERNEL(128, EPI_QKV_NORM_ROPE, ACT_NONE, false),
    F5_GEMM_KERNEL(192, EPI_QKV_NORM_ROPE, ACT_NONE, false),
    F5_GEMM_KERNEL(256, EPI_QKV_NORM_ROPE, ACT_NONE, false),
    // 128-column heads (f5_gemm_args.dim_head = 128).  QKV_NORM_ROPE is 128 wide only: a 192-wide tile would split a
    // head, and the 256-wide one spills (24 bytes; DESIGN.md §4).
    F5_GEMM_KERNEL(128, EPI_QKV_ROPE_DH128, ACT_NONE, false),
    F5_GEMM_KERNEL(192, EPI_QKV_ROPE_DH128, ACT_NONE, false),
    F5_GEMM_KERNEL(256, EPI_QKV_ROPE_DH128, ACT_NONE, false),
    F5_GEMM_KERNEL(128, EPI_QKV_NORM_ROPE_DH128, ACT_NONE, false),
};
#undef F5_GEMM_KERNEL

// Engine-internal instantiations that no f5_gemm_args selects: the per-sample gate of f5_forward's gated residual GEMMs
// (EPI_RESID_SAMPLE), at the widths pick_tile chooses from for EPI_RESID.  The engine plans such a GEMM as EPI_RESID and
// then switches the plan's epilogue, so the width is the one f5_sample runs the same problem with.
// tests/test_gpu_gemm_resid_sample.py checks each entry element by element against per-sample EPI_RESID launches.
template <int BN>
constexpr GemmKernel sample_gate_kernel() {
  return GemmKernel{BN, EPI_RESID_SAMPLE, ACT_NONE, false, gemm_wgmma_kernel<BN, EPI_RESID_SAMPLE, ACT_NONE, false>};
}
static const GemmKernel kGemmSampleKernels[] = {sample_gate_kernel<128>(), sample_gate_kernel<192>(),
                                                sample_gate_kernel<256>()};

static const GemmKernel* find_kernel(int bn, int epi, int act, bool conv) {
  for (const GemmKernel& k : kGemmKernels)
    if (k.bn == bn && k.epi == epi && k.act == act && k.conv == conv) return &k;
  for (const GemmKernel& k : kGemmSampleKernels)
    if (k.bn == bn && k.epi == epi && k.act == act && k.conv == conv) return &k;
  return nullptr;
}

// cudaFuncSetAttribute is per device: the configured flag and the SM count are tracked per device ordinal, so one
// process may drive engines on several GPUs (ADVICE r1).
namespace {
constexpr int kMaxDevices = 64;
struct DeviceState {
  bool configured = false;
  int sms = 0;
};
DeviceState g_dev[kMaxDevices];
std::mutex g_dev_mu;
int current_device() {
  int d = 0;
  cudaGetDevice(&d);
  return (d >= 0 && d < kMaxDevices) ? d : 0;
}
}  // namespace

int configure_kernels() {
  const int dev = current_device();
  std::lock_guard<std::mutex> lk(g_dev_mu);
  if (g_dev[dev].configured) return 0;
  auto setup = [](const GemmKernel& k) {
    const int rc = check_cuda(cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   (int)gemm_smem_bytes(k.bn)),
                              "cudaFuncSetAttribute(gemm smem)");
    if (rc == 0) cudaFuncSetAttribute(k.fn, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    return rc;
  };
  for (const GemmKernel& k : kGemmKernels)
    if (int rc = setup(k)) return rc;
  for (const GemmKernel& k : kGemmSampleKernels)
    if (int rc = setup(k)) return rc;
  if (int rc = attn_configure()) return rc;
  g_dev[dev].configured = true;
  return 0;
}

bool pdl_enabled() {
#ifdef F5_TRACE  // diagnostic build only: F5_PDL=0 launches without programmatic dependent launch
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("F5_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
#else
  return true;
#endif
}

int num_sms() {
  const int dev = current_device();
  int n = g_dev[dev].sms;  // written once per device; a racing first call computes the same value
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    g_dev[dev].sms = n;
  }
  return n;
}

int gemm_run(const GemmPlan& pl, cudaStream_t s) {
  const GemmKernel* k = find_kernel(pl.bn, pl.epi, pl.act, pl.conv != 0);
  if (!k) {
    set_error("gemm: no kernel instantiated for bn=%d epi=%d act=%d conv=%d", pl.bn, pl.epi, pl.act, pl.conv);
    return -6;
  }
  if (int rc = configure_kernels()) return rc;
  PdlLaunch L(pl.grid, dim3(kGemmThreads), gemm_smem_bytes(pl.bn), s);
  if (int rc = check_cuda(cudaLaunchKernelEx(&L.cfg, k->fn, pl.tmA, pl.tmB, pl.p), "gemm launch")) return rc;
  count_launch();
  return check_launch("gemm_wgmma_kernel launch");
}

// Tile width of a GEMM whose caller left bn = 0.  Cost model in SM clocks of the H100 (132 SMs, 4096 dense fp16
// FLOP / clk / SM): the wgmma main loop of a 128 x BN tile takes k-blocks x (4 BN + 96) clk (tensor-core time plus the
// per-k-block barrier and issue overhead), the register epilogue BN x {20 plain / RoPE, 24 reduce-add, 32 GELU} clk.
// Tiles run in rounds over the SMs; the producer streams the next tile's operands during the epilogue, so a round
// costs main + epilogue.  Checked against the graph-timed sweep of tools/gemm_sweep.py with the chunked epilogue (H100
// SXM 80 GB, 700 W limit): the pick is the fastest width at M = 1876 and within 11 % of it at M = 3752 - 15008.
// QKV + RMSNorm + RoPE is costed as QKV + RoPE: its norm pass added 4 % at M = 1876 at every width but 256, where the
// 128 x 192 pick stays the fastest (tools/qkv_epilogue_time.py, same card).
// Diagnostic build (make TRACE=1) only: F5_BN_<n_out>=<bn> overrides the choice.
static int pick_tile(long long rows, int batches, int n_out, int k, int epi, int act) {
#ifdef F5_TRACE
  char key[32];
  snprintf(key, sizeof key, "F5_BN_%d", n_out);
  if (const char* e = getenv(key)) {
    const int bn = atoi(e);
    if (bn == 64 || bn == 128 || bn == 192 || bn == 256) return bn;
  }
#endif
  const int sms = num_sms();
  const double kb = double((k + 63) / 64);
  const double epi_col = (act == F5_ACT_GELU_TANH || act == F5_ACT_GELU_ERF) ? 32.0 : (epi == F5_EPI_RESID ? 24.0 : 20.0);
  int best = 128;
  double best_cost = 1e30;
  const int cand[3] = {128, 192, 256};
  for (const int bn : cand) {
    if (!find_kernel(bn, epi, act, false)) continue;
    if (bn > 128 && n_out < bn) continue;
    const long long tiles = ((rows + 127) / 128) * ((n_out + bn - 1) / bn) * batches;
    const double rounds = double((tiles + sms - 1) / sms);
    const double cost = rounds * (kb * (4.0 * bn + 96.0) + epi_col * bn);
    if (cost < best_cost) {
      best_cost = cost;
      best = bn;
    }
  }
  return best;
}

// Epilogue of the kernel that runs `a`: the QKV epilogues over 128-column heads are instantiations of their own.
static int kernel_epi(const f5_gemm_args* a) {
  if (a->dim_head != 128) return a->epi;
  return a->epi == F5_EPI_QKV_ROPE ? EPI_QKV_ROPE_DH128 : a->epi == F5_EPI_QKV_NORM_ROPE ? EPI_QKV_NORM_ROPE_DH128 : a->epi;
}

// Tile width f5_gemm runs `a` with: conv tiles are 64 wide, bn = 0 leaves the width to the planner.
static int resolve_tile(const f5_gemm_args* a, int* bn) {
  if (a->cta_pair != 0) {
    set_error("gemm: cta_pair must be 0 (there are no cluster-pair tiles)");
    return -1;
  }
  *bn = a->conv_taps > 0 ? 64
        : a->bn != 0    ? a->bn
                        : pick_tile(a->rows, a->batches, a->n_out, a->k, kernel_epi(a), a->act);
  return 0;
}

int gemm_plan(GemmPlan* pl, const void* A, const void* W, const f5_gemm_args* a) {
  memset(pl, 0, sizeof(*pl));
  const bool conv = a->conv_taps > 0;
  int bn;
  if (int rc = resolve_tile(a, &bn)) return rc;
  if (bn != 64 && bn != 128 && bn != 192 && bn != 256) {
    set_error("gemm: bn must be 64, 128, 192 or 256");
    return -1;
  }
  if (a->rows <= 0 || a->batches <= 0 || a->n_out <= 0) {
    set_error("gemm: empty problem (rows=%d batches=%d n_out=%d)", a->rows, a->batches, a->n_out);
    return -1;
  }
  const bool qkv_epi = a->epi == F5_EPI_QKV_ROPE || a->epi == F5_EPI_QKV_NORM_ROPE;
  if (a->dim_head != 0 && a->dim_head != 64 && !(qkv_epi && a->dim_head == 128)) {
    set_error("gemm: dim_head must be 0 (= 64), 64 or, with a QKV epilogue, 128 (got %d)", a->dim_head);
    return -1;
  }
  if (a->dim_head == 128) {
    if (a->inner <= 0 || a->inner % 128 || a->n_out % 128 || a->rope_cos == nullptr || a->rope_sin == nullptr ||
        a->seq <= 0 || conv) {
      set_error("gemm: QKV epilogues at dim_head 128 need inner %% 128 == 0, n_out %% 128 == 0, rope tables and seq");
      return -1;
    }
    if (a->epi == F5_EPI_QKV_NORM_ROPE && bn != 128) {
      set_error("gemm: QKV_NORM_ROPE at dim_head 128 runs with bn 128 only (got %d)", bn);
      return -1;
    }
  }
  if (a->epi == F5_EPI_QKV_ROPE && (a->inner % 64 || a->rope_cos == nullptr || a->seq <= 0)) {
    set_error("gemm: QKV_ROPE needs inner %% 64 == 0, rope tables and seq");
    return -1;
  }
  if (a->epi == F5_EPI_QKV_NORM_ROPE &&
      (a->inner <= 0 || a->inner % 64 || a->n_out % 64 || a->rope_cos == nullptr || a->rope_sin == nullptr ||
       a->seq <= 0 || a->q_norm == nullptr || a->k_norm == nullptr || conv)) {
    set_error("gemm: QKV_NORM_ROPE needs q_norm and k_norm, inner %% 64 == 0, n_out %% 64 == 0, rope tables and seq");
    return -1;
  }
  pl->bn = bn;
  pl->epi = kernel_epi(a);
  pl->act = a->act;
  pl->conv = conv ? 1 : 0;
  GemmParams& p = pl->p;
  p.rows = a->rows;
  p.n_out = a->n_out;
  p.batches = a->batches;
  p.bias = a->bias;
  p.out = a->out;
  p.out16b = reinterpret_cast<__half*>(a->out16b);
  p.resid = a->resid;
  p.ldo = a->ldo;
  p.gate = a->gate;
  p.step_ptr = a->step_ptr;
  p.gate_step_stride = a->gate_step_stride;
  p.row_len = a->row_len;
  p.seq = a->seq;
  p.rope_cos = a->rope_cos;
  p.rope_sin = a->rope_sin;
  p.inner = a->inner > 0 ? a->inner : 64;
  p.pe_heads = a->pe_heads;
  p.q_norm = a->q_norm;
  p.k_norm = a->k_norm;
  p.conv_pad = a->conv_taps / 2;
  p.skip_pad = (a->skip_padded_tiles && a->row_len != nullptr && a->seq > 0 && (conv || a->batches == 1)) ? 1 : 0;
  // a prefetched W tile belongs to the CTA's first tile: not known to be computed when padded tiles are skipped
  p.w_prefetch = (a->weights_static && !p.skip_pad) ? 1 : 0;
#ifdef F5_TRACE  // diagnostic build only: F5_GEMM_EPI=none runs the main loop without the epilogue
  {
    const char* e = getenv("F5_GEMM_EPI");
    p.diag_no_epi = (e && strcmp(e, "none") == 0) ? 1 : 0;
  }
#endif
  int rc;
  if (conv) {
    const int G = a->k == 0 ? 64 : a->k;  // channels per group
    if (G <= 0 || G % 8 || G > 64 || a->n_out % G || a->lda < a->n_out) {
      set_error("conv gemm: channels per group must be a multiple of 8, at most 64, and divide the channel count "
                "(got %d per group, %d channels, lda %d)", G, a->n_out, a->lda);
      return -1;
    }
    p.num_kb = a->conv_taps;
    p.conv_g = G;
    // activations [batches][rows][lda] viewed as {G, groups, rows, batches}: a 64-wide box at group g holds the G
    // channels of g and zeros past them, so a group never reads another group's channels
    const uint64_t dA[4] = {(uint64_t)G, (uint64_t)(a->n_out / G), (uint64_t)a->rows, (uint64_t)a->batches};
    const uint64_t sA[3] = {(uint64_t)G * 2, (uint64_t)a->lda * 2, (uint64_t)a->rows * a->lda * 2};
    const uint32_t bA[4] = {64, 1, 128, 1};
    if ((rc = encode_tmap_f16(&pl->tmA, A, 4, dA, sA, bA))) return rc;
    // weights [taps][n_out][G]: input columns past G are zero-filled; box rows past the group's G output channels
    // only feed accumulator columns that are never stored
    const uint64_t dW[2] = {(uint64_t)G, (uint64_t)a->conv_taps * a->n_out};
    const uint64_t sW[1] = {(uint64_t)G * 2};
    const uint32_t bW[2] = {64, 64};
    if ((rc = encode_tmap_f16(&pl->tmB, W, 2, dW, sW, bW))) return rc;
  } else {
    if (a->k <= 0 || a->lda < a->k || a->ldw < a->k) {
      set_error("gemm: bad k/lda/ldw (%d, %d, %d)", a->k, a->lda, a->ldw);
      return -1;
    }
    p.num_kb = (a->k + kBK - 1) / kBK;
    const uint64_t dA[3] = {(uint64_t)a->k, (uint64_t)a->rows, (uint64_t)a->batches};
    const uint64_t sA[2] = {(uint64_t)a->lda * 2, (uint64_t)a->rows * a->lda * 2};
    const uint32_t bA[3] = {64, 128, 1};
    if ((rc = encode_tmap_f16(&pl->tmA, A, 3, dA, sA, bA))) return rc;
    const uint64_t dW[2] = {(uint64_t)a->k, (uint64_t)a->n_out};
    const uint64_t sW[1] = {(uint64_t)a->ldw * 2};
    const uint32_t bW[2] = {64, (uint32_t)bn};
    if ((rc = encode_tmap_f16(&pl->tmB, W, 2, dW, sW, bW))) return rc;
  }
  if (a->epi == F5_EPI_RESID && (a->ldo % 4 || a->resid == nullptr)) {
    set_error("gemm: RESID epilogue needs resid != NULL and ldo %% 4 == 0 (ldo=%d)", a->ldo);
    return -1;
  }
  if ((a->epi == F5_EPI_F16 || a->epi == F5_EPI_QKV_ROPE || a->epi == F5_EPI_QKV_NORM_ROPE) &&
      (a->ldo % 8 || a->out == nullptr)) {
    set_error("gemm: fp16 epilogue needs out != NULL and ldo %% 8 == 0 (ldo=%d)", a->ldo);
    return -1;
  }
  const long long tiles_n = conv ? a->n_out / p.conv_g : (a->n_out + bn - 1) / bn;
  const long long tiles = tiles_n * ((a->rows + kBM - 1) / kBM) * a->batches;
  pl->grid = dim3((unsigned)(tiles < num_sms() ? tiles : num_sms()), 1, 1);  // persistent: one CTA per SM
  return 0;
}

}  // namespace f5

extern "C" {

int f5_version(void) { return 110; }
const char* f5_last_error(void) { return f5::g_err; }
unsigned long long f5_launch_count(void) { return f5::g_launches.load(); }

int f5_gemm_tile(const f5_gemm_args* args, int* bn, int* cta_pair) {
  if (!args || !bn || !cta_pair) return -1;
  *cta_pair = 0;
  return f5::resolve_tile(args, bn);
}

int f5_gemm(const void* A, const void* W, const f5_gemm_args* args, f5_stream_t stream) {
  f5::GemmPlan pl;
  if (int rc = f5::gemm_plan(&pl, A, W, args)) return rc;
  return f5::gemm_run(pl, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"

// Shared-memory radix-2 FFT kernels for the Vocos mel front-end (STFT -> |.| -> mel -> log) and the Vocos
// ISTFT head (exp/clip/cos/sin -> inverse real FFT -> window -> overlap-add -> envelope normalise).
// n_fft = 1024, hop = 256, hann(periodic) — the only configuration the reference ships
// (infer/utils_infer.py:52-57; configs/*.yaml mel_spec).  One CTA (256 threads) per frame; the whole transform
// lives in shared memory (8 KB data + 4 KB twiddles); global traffic is the algorithmic minimum.
#pragma once
#include "common.cuh"
#include "ew_params.h"

namespace f5 {

constexpr int kNfft = 1024;
constexpr int kHop = 256;
constexpr int kBins = kNfft / 2 + 1;

__device__ __forceinline__ int bitrev10(int i) { return int(__brev(unsigned(i)) >> 22); }

// in-place forward DFT (e^{-i...}) of 1024 complex points held bit-reversed in (re, im); 256 threads.
__device__ __forceinline__ void fft1024_inplace(float* re, float* im, const float* twc, const float* tws) {
#pragma unroll 1
  for (int s = 1; s <= 10; ++s) {
    const int half = 1 << (s - 1);
    const int stride = kNfft >> s;  // twiddle stride
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int bf = threadIdx.x + u * 256;  // butterfly id 0..511
      const int j = bf & (half - 1);
      const int k = (bf >> (s - 1)) << s;
      const int i0 = k + j, i1 = i0 + half;
      const float wr = twc[j * stride], wi = -tws[j * stride];
      const float xr = re[i1], xi = im[i1];
      const float tr = xr * wr - xi * wi, ti = xr * wi + xi * wr;
      const float ar = re[i0], ai = im[i0];
      re[i0] = ar + tr;
      im[i0] = ai + ti;
      re[i1] = ar - tr;
      im[i1] = ai - ti;
    }
    __syncthreads();
  }
}

// FftTables (twiddles, Hann window): ew_params.h
__global__ void fft_tables_kernel(float2* tw, float* hann) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < kNfft / 2) {
    float s, c;
    sincospif(2.0f * float(i) / float(kNfft), &s, &c);
    tw[i] = make_float2(c, s);
  }
  if (i < kNfft) hann[i] = 0.5f - 0.5f * cospif(2.0f * float(i) / float(kNfft));
}

__device__ __forceinline__ void load_twiddles(float* twc, float* tws, const float2* tw) {
  for (int i = threadIdx.x; i < kNfft / 2; i += blockDim.x) {
    const float2 w = __ldg(tw + i);
    twc[i] = w.x;
    tws[i] = w.y;
  }
}

__device__ __forceinline__ int bitrev9(int i) { return int(__brev(unsigned(i)) >> 23); }

// ---------------------------------------------------------------------------------------------------------
// mel front-end (model/modules.py:80-109 -> torchaudio MelSpectrogram(power=1, center=True, norm=None, htk))
// wav [B, nw] -> mel; frame t covers reflect-padded samples [t*256 - 512, t*256 + 512).
// out_btc != 0 : out[b, t, m]  (layout CFM.sample wants, cfm.py:106-109), else out[b, m, t] (MelSpec.forward).
//
// Real-input FFT: the 1024 windowed samples are packed as 512 complex points z[m] = x[2m] + i x[2m+1], ONE 512-point
// complex radix-2 FFT (9 stages, one butterfly per thread and stage) is followed by the split
//   X[k] = (Z[k] + conj Z[512-k]) / 2  -  i w_1024^k (Z[k] - conj Z[512-k]) / 2,   k = 0..512,
// i.e. half the butterflies of a 1024-point complex transform.  Twiddles and window come from per-device tables.
// Filterbank: fb is the caller's dense [513, n_mels] matrix, read as it is at launch time (no host-side index keyed
// by its address, so a rewritten or reallocated filterbank is always seen as it is).  Thread m sums all 513 bins in
// ascending order; fb loads are coalesced across m.  The zero entries of a triangular filter add exact zeros, so the
// result equals a sum over the filter's non-zero band only.
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) mel_stft_kernel(const float* wav, int nw, int T, const float* fb, int n_mels,
                                                        FftTables tab, float* out, int out_btc) {
  __shared__ float re[kNfft / 2 + 1], im[kNfft / 2 + 1], twc[kNfft / 2], tws[kNfft / 2], mag[kBins];
  const int t = blockIdx.x, b = blockIdx.y;
  load_twiddles(twc, tws, tab.tw);
  const float* w = wav + (long long)b * nw;
  for (int m = threadIdx.x; m < kNfft / 2; m += 256) {
    float v[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int i = 2 * m + u;
      int s = t * kHop + i - kNfft / 2;
      if (s < 0) s = -s;
      if (s >= nw) s = 2 * (nw - 1) - s;
      v[u] = w[s] * __ldg(tab.hann + i);
    }
    const int d = bitrev9(m);
    re[d] = v[0];
    im[d] = v[1];
  }
  __syncthreads();
  // 512-point forward DFT, in place, input bit-reversed; w_512^j = (twc, -tws)[2 j]
#pragma unroll 1
  for (int s = 1; s <= 9; ++s) {
    const int half = 1 << (s - 1);
    const int stride = kNfft >> s;  // index step in the 1024-table: 2 * (512 >> s)
    const int bf = threadIdx.x;     // 256 butterflies per stage
    const int j = bf & (half - 1);
    const int i0 = ((bf >> (s - 1)) << s) + j, i1 = i0 + half;
    const float wr = twc[j * stride], wi = -tws[j * stride];
    const float xr = re[i1], xi = im[i1];
    const float tr = xr * wr - xi * wi, ti = xr * wi + xi * wr;
    const float ar = re[i0], ai = im[i0];
    re[i0] = ar + tr;
    im[i0] = ai + ti;
    re[i1] = ar - tr;
    im[i1] = ai - ti;
    __syncthreads();
  }
  if (threadIdx.x == 0) {  // Z[512] = Z[0]
    re[kNfft / 2] = re[0];
    im[kNfft / 2] = im[0];
  }
  __syncthreads();
  for (int k = threadIdx.x; k < kBins; k += 256) {
    const float zr = re[k], zi = im[k], yr = re[kNfft / 2 - k], yi = -im[kNfft / 2 - k];  // Z[k], conj Z[512-k]
    const float er = 0.5f * (zr + yr), ei = 0.5f * (zi + yi);                                // even part
    const float dr = 0.5f * (zr - yr), di = 0.5f * (zi - yi);                                // (Z - conj Z') / 2
    const float c = k < kNfft / 2 ? twc[k] : -1.0f, sn = k < kNfft / 2 ? tws[k] : 0.0f;     // w_1024^k = c - i sn
    // -i * (c - i sn) * (dr + i di) = (-sn - i c) (dr + i di)
    const float orr = -sn * dr + c * di, oi = -sn * di - c * dr;
    const float xr = er + orr, xi = ei + oi;
    mag[k] = sqrtf(xr * xr + xi * xi);
  }
  __syncthreads();
  for (int m = threadIdx.x; m < n_mels; m += 256) {
    float acc = 0.f;
    for (int f = 0; f < kBins; ++f) acc += mag[f] * __ldg(fb + f * n_mels + m);
    const float v = logf(fmaxf(acc, 1e-5f));
    if (out_btc) out[((long long)b * T + t) * n_mels + m] = v;
    else out[((long long)b * n_mels + m) * T + t] = v;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Vocos ISTFT head (vocos ISTFTHead + torch.istft(center=True); SURVEY.md §9.3).
// head: [B*T, 1026] fp32 = [log-mag (513) | phase (513)] per frame.
// frames out: [B*T, 1024] windowed time-domain frames; a second kernel overlap-adds (deterministic gather).
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) istft_frames_kernel(const float* head, int ld, float* frames, FftTables tab) {
  __shared__ float re[kNfft], im[kNfft], twc[kNfft / 2], tws[kNfft / 2];
  const long long fr = blockIdx.x;
  load_twiddles(twc, tws, tab.tw);
  const float* h = head + fr * ld;
  // X[k] = mag (cos p + i sin p), Hermitian extension; inverse via conj(FFT(conj(X))) / N.  Load conj(X).
  for (int k = threadIdx.x; k < kNfft; k += 256) {
    const int f = k <= 512 ? k : kNfft - k;
    const float mag = fminf(expf(h[f]), 100.0f);
    float s, c;
    sincosf(h[kBins + f], &s, &c);
    float xr = mag * c, xi = mag * s;
    if (k > 512) xi = -xi;           // Hermitian mirror
    if (f == 0 || f == 512) xi = 0;  // c2r ignores imag of DC / Nyquist
    const int d = bitrev10(k);
    re[d] = xr;
    im[d] = -xi;  // conj
  }
  __syncthreads();
  fft1024_inplace(re, im, twc, tws);
  for (int n = threadIdx.x; n < kNfft; n += 256) frames[fr * kNfft + n] = re[n] * (1.0f / kNfft) * __ldg(tab.hann + n);
}

// wav[b, i] = sum_t frames[b, t, i + 512 - 256 t] / sum_t hann^2[i + 512 - 256 t],  i in [0, 256 (T-1))
__global__ void istft_ola_kernel(const float* frames, int T, float* wav, int B, FftTables tab) {
  const int L = kHop * (T - 1);
  const long long total = (long long)B * L;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int b = int(idx / L), i = int(idx % L);
    const int pos = i + kNfft / 2;
    const int t_hi = min(T - 1, pos / kHop);
    const int t_lo = pos >= kNfft - kHop ? (pos - (kNfft - kHop)) / kHop : 0;  // smallest t with pos - 256 t <= 1023
    float acc = 0.f, env = 0.f;
    for (int t = t_lo; t <= t_hi; ++t) {
      const int n = pos - t * kHop;
      if (n < 0 || n >= kNfft) continue;
      acc += frames[((long long)b * T + t) * kNfft + n];
      const float w = __ldg(tab.hann + n);
      env += w * w;
    }
    wav[idx] = acc / env;
  }
}

// Vocos embed Conv1d(100 -> 512, k=7, pad=3) as im2col: A[b*T + t, tap*C + c] = mel[b, c, t + tap - 3]  (fp16)
__global__ void vocos_im2col_kernel(const float* mel, int B, int C, int T, __half* A, int Kpad) {
  const long long row = blockIdx.x;
  const int b = int(row / T), t = int(row % T);
  for (int k = threadIdx.x; k < Kpad; k += blockDim.x) {
    float v = 0.f;
    if (k < 7 * C) {
      const int tap = k / C, c = k % C;
      const int tt = t + tap - 3;
      if (tt >= 0 && tt < T) v = mel[((long long)b * C + c) * T + tt];
    }
    A[row * Kpad + k] = __float2half_rn(v);
  }
}

}  // namespace f5

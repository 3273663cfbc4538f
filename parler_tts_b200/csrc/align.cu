// align.cu -- token timestamps from an alignment matrix (ptts_align_dtw): openai-whisper's recipe as transformers states it
// (generation_whisper._median_filter, then _dynamic_time_warping of the negated matrix), for one utterance per CTA.
//
// align_median_kernel: the median of 7 along frames with reflect padding (frame -k reads frame k, frame F - 1 + k reads
// F - 1 - k), each key column on its own; an utterance of 3 frames or fewer is copied unchanged, as _median_filter returns its
// input when the length is <= the half width.  The median is a selection, so the values are the fixture's bit for bit.
//
// align_dtw_kernel: the DTW over the utterance's n unmasked keys (in order; masked keys are dropped, not given a cost) and its F
// frames.  cost[i][j] (i keys, j frames) = -y[j - 1][key i - 1] + min(cost[i-1][j-1], cost[i-1][j], cost[i][j-1]) with
// _dynamic_time_warping's comparisons and tie order: diagonal if strictly below both, else up (previous key) if strictly below
// both, else left (previous frame).  The sums are fp32 adds, as the float32 cost array there rounds each one.  Cells of one
// anti-diagonal i + j are independent: the CTA sweeps the n + F + 1 diagonals with three rolling diagonals of cost in shared
// memory and the trace bytes in global memory, then thread 0 walks the trace back from (n, F) and keeps, for each key, the
// smallest frame on the path.
#include "common.cuh"
#include "kernels.h"

namespace ptts {

constexpr int kMedianHalf = 3;   // width 7

__global__ void __launch_bounds__(256) align_median_kernel(const float* x, int T, int P, const int* n_frames, float* y) {
  const int b = blockIdx.y;
  const int F = min(n_frames[b], T);
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= F * P) return;
  const int t = idx / P, p = idx % P;
  const float* xb = x + (size_t)b * T * P;
  float* yb = y + (size_t)b * T * P;
  if (F <= kMedianHalf) { yb[idx] = xb[idx]; return; }
  float v[2 * kMedianHalf + 1];
#pragma unroll
  for (int k = 0; k < 2 * kMedianHalf + 1; k++) {
    int s = t + k - kMedianHalf;
    s = s < 0 ? -s : (s >= F ? 2 * (F - 1) - s : s);
    v[k] = xb[(size_t)s * P + p];
  }
#pragma unroll
  for (int i = 1; i < 2 * kMedianHalf + 1; i++)   // insertion sort of 7
#pragma unroll
    for (int j = i; j > 0; j--)
      if (v[j] < v[j - 1]) { const float tmp = v[j]; v[j] = v[j - 1]; v[j - 1] = tmp; }
  yb[idx] = v[kMedianHalf];
}

__global__ void __launch_bounds__(256) align_dtw_kernel(const float* y, int T, int P, const int* n_frames, const int* key_mask,
                                                        unsigned char* trace, int* jumps) {
  extern __shared__ __align__(16) float smd[];
  float* cost = smd;                                        // [3][P + 1]: diagonals d, d - 1, d - 2 by key index i
  int* keys = reinterpret_cast<int*>(smd + 3 * (P + 1));   // [P] the unmasked keys in order
  __shared__ int n_keys;
  const int b = blockIdx.x;
  const int F = min(n_frames[b], T);
  const float* yb = y + (size_t)b * T * P;
  int* jb = jumps + (size_t)b * P;
  unsigned char* tr = trace + (size_t)b * (P + 1) * (T + 1);   // [i][j], row stride T + 1
  if (threadIdx.x == 0) {
    int n = 0;
    for (int p = 0; p < P; p++) {
      const bool on = key_mask == nullptr || key_mask[(size_t)b * P + p] != 0;
      if (on) keys[n++] = p;
      jb[p] = on ? 0 : -1;   // an utterance without frames puts every key at frame 0
    }
    n_keys = n;
  }
  __syncthreads();
  const int n = n_keys;
  if (F == 0 || n == 0) return;
  for (int d = 0; d <= n + F; d++) {
    float* cur = cost + (d % 3) * (P + 1);
    const float* p1 = cost + ((d + 2) % 3) * (P + 1);
    const float* p2 = cost + ((d + 1) % 3) * (P + 1);
    const int i_lo = d - F > 0 ? d - F : 0, i_hi = d < n ? d : n;
    for (int i = i_lo + threadIdx.x; i <= i_hi; i += blockDim.x) {
      const int j = d - i;
      if (i == 0 || j == 0) { cur[i] = (i == 0 && j == 0) ? 0.f : INFINITY; continue; }
      const float c0 = p2[i - 1], c1 = p1[i - 1], c2 = p1[i];
      float c;
      unsigned char t;
      if (c0 < c1 && c0 < c2) { c = c0; t = 0; }
      else if (c1 < c0 && c1 < c2) { c = c1; t = 1; }
      else { c = c2; t = 2; }
      cur[i] = __fadd_rn(-yb[(size_t)(j - 1) * P + keys[i - 1]], c);
      tr[(size_t)i * (T + 1) + j] = t;
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  int i = n, j = F;
  while (i > 0 || j > 0) {
    if (i > 0) jb[keys[i - 1]] = j - 1;   // walking back: the last write for a key is its first frame
    const int t = i == 0 ? 2 : (j == 0 ? 1 : tr[(size_t)i * (T + 1) + j]);
    if (t == 0) { i--; j--; }
    else if (t == 1) i--;
    else j--;
  }
}

int launch_align_dtw(const float* x, int B, int T, int P, const int* n_frames, const int* key_mask, float* y, unsigned char* trace,
                     int* jumps, cudaStream_t st) {
  PTTS_REQUIRE(B > 0 && T > 0 && P > 0, "align_dtw: bad shape B %d, T %d, P %d", B, T, P);
  const size_t smem = (size_t)(3 * (P + 1) + P) * sizeof(float);
  PTTS_REQUIRE(smem <= 200 * 1024, "align_dtw: %d keys need %zu B of shared memory (> 200 KB)", P, smem);
  static bool attr = false;
  if (!attr) {
    PTTS_CHECK_CUDA(cudaFuncSetAttribute(align_dtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr = true;
  }
  const int64_t cells = (int64_t)T * P;
  align_median_kernel<<<dim3((unsigned)((cells + 255) / 256), B), 256, 0, st>>>(x, T, P, n_frames, y);
  PTTS_CHECK_CUDA(cudaGetLastError());
  align_dtw_kernel<<<B, 256, smem, st>>>(y, T, P, n_frames, key_mask, trace, jumps);
  PTTS_CHECK_CUDA(cudaGetLastError());
  return PTTS_OK;
}

}  // namespace ptts

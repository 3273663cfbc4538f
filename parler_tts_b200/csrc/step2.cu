// step2.cu -- the CLUSTER decode step: one persistent kernel per generated token, 6 device-wide phases per layer (bf16).
//
// Replaces the same reference code as step.cu (ParlerTTSForCausalLM.forward with q_len == 1, modeling_parler_tts.py:1865-1974 /
// :983-1074, plus one iteration of GenerationMixin._sample) for the shapes layout.h::cluster_shape_ok() accepts (Parler-TTS-Mini:
// MHA, 16 heads).  In step.cu's design every CTA (one per SM) needs the WHOLE 32 x H activation tile in every one of the 8
// dependent phases of a layer: each phase pays a device-wide barrier, the pull of the 66 KB tile, LayerNorm statistics over it
// and an 8-warp split-K reduction through shared memory.  This kernel cuts the dependent chain and the per-CTA fixed work:
//
//   * grid = 4 clusters of 2 CTAs per head (cudaLaunchAttributeClusterDimension; the whole grid must be co-resident, which
//     cluster_step_available asks the occupancy API -- a 132-SM H100 holds 66 clusters of 2, one per TPC, and Mini needs 64).
//     Every GEMM is split 8 ways along K as step.cu splits it over its 8 warps (k32 tile kt -> residue class kt mod 8): rank r
//     of a cluster stages the k-tiles of classes 4r .. 4r+3 (half of K: 8-33 KB of activations instead of 66 KB) and warp w
//     reduces class 4 r + (w >> 1) for destination (w & 1).  Every warp owns whole n-tiles (no split-K through shared memory
//     inside a CTA); the eight partial sums meet through DISTRIBUTED SHARED MEMORY: every lane stores its accumulators straight
//     from registers into the peer's receive slots (st.async, bytes completing on the peer's mbarrier; plain stores into its own
//     CTA's slots), and every destination adds them in class order 0..7.
//   * out-proj / cross out-proj / fc1 / fc2: cluster c owns N/(4 nh) output features, rank d finalises half of them
//     (feature-partitioned exchange).  The residual-stream slice a CTA owns (32 rows x 8 features) never leaves its shared memory.
//   * QKV and q_cross: clusters 4h .. 4h+3 own HEAD h for batch rows 8j .. 8j+7 (one m16 tile with 8 live rows); the exchange is
//     ROW-partitioned (rank d receives rows 8j+4d .. 8j+4d+3 of q|k|v), so RoPE, the KV-cache append and the attention of those 4
//     (row, head) items run inside the same phase: QKV -> self-attention and q_cross -> cross-attention need no device-wide barrier
//     between them.  6 barriers per layer instead of 8.  A warp carries 12 QKV n-tiles (4 q_cross) in two passes of 6 (2): the
//     head's 192 KB QKV slice of a rank streams through the 2 x 64 KB weight ring as four jobs.
//   * weights: one contiguous slice per (phase, cluster, rank) (layout.h cluster_phase, built once by ptts_decoder_finalize), streamed by
//     ONE bulk copy per job into a 2 x 64 KB ring two jobs ahead, with an L2 evict-first policy like the K/V rows (1.2 GB per token
//     must not evict the kernel's own instructions and the small reused tensors).  No HBM -> L2 prefetch: the ring already runs two
//     jobs ahead of its consumer, and every cp.async.bulk.prefetch.L2 costs issue time inside a phase.
//   * fc2 (one n-tile per destination, half of F = 128 KB of activations): staged in two quarters of F, one after the other; a
//     warp's accumulators carry its residue class from the first quarter into the second.
//   * attention: the sweep step.cu's attention phase runs (attention_decode_sweep, two warps per item, 32-key chunks).  Every
//     warp's first K/V chunk is requested at the TOP of the head phase into a stage nothing else touches during the phase, so the
//     HBM round trip runs under the weights wait, the MMAs, the exchange and the epilogue instead of after them.
//   * the activation slice of the next phase is requested by the barrier's polling thread the moment the barrier opens; the
//     per-phase cluster barrier that guards buffer reuse arrives .relaxed (its default .release is a gpu-scope MEMBAR per warp).
//   * one launch runs up to StepParams.n_steps tokens: cur_len, the unfinished count and the stop decision advance on the device.
// Reduction orders are fixed and are step.cu's (k-tiles ascending in one accumulator per warp, warp partials 0..7 added from zero;
// the same LayerNorm statistics, attention and lm-head split): the two step kernels produce the same bits, run to run.
#include "attn_core.cuh"
#include "common.cuh"
#include "kernels.h"
#include "ln_stats.cuh"
#include "sample_core.cuh"
#include "ptx.cuh"
#include "step.h"
#include "step_common.cuh"
#include <type_traits>

namespace ptts {
namespace cl {

constexpr int C = 2;            // CTAs per cluster
constexpr int V = 8;            // K residue classes = warps per CTA: warp w reduces class 4 rank + (w >> 1) for destination (w & 1)
constexpr int THREADS = 256;
constexpr int ROWS = 32;        // batch rows (two m16 tiles; the head phases work on 8 rows = one m16 tile with rows 8-15 repeated)
constexpr int HROWS = 8;        // batch rows of a head-phase cluster
constexpr int ATT_SMEM = attn_decode_smem_per_warp<bf16>();   // one attention warp's scratch: two 32-key K/V stages + 192 floats
constexpr int PROF_STRIDE = 16;  // clock64 stamps per phase row of the optional profile buffer (tools/profile_step2.py)
constexpr int QMAX = 6;         // n-tiles per warp and pass (QKV: 24 n-tiles of a head = 2 passes x 2 warp groups x 6)
constexpr int OFF_STATS = 256, OFF_PART = 512, OFF_RES = 2560, OFF_CVEC = 3584;
constexpr int HDR = 5632;       // mbarriers | row stats | stat partials | residual slice | folded-LN vectors c1[256] c2[256]
constexpr int WB_BYTES = 65536; // one weight ring buffer
constexpr int R_OFF = HDR + 2 * WB_BYTES;
// R region: [activation slice | receive slots], split per phase; attention scratch and the lm-head tile alias it.  The receive
// slots, which peers fill while this CTA may still run its MMAs, start right behind the slice.  Largest plans (H = 1024, F = 4096):
//   fc1   : 32.5 KB slice, receive slots 8 x (256 B stats + 32 x 34 floats) = 36 KB: [32.5 KB, 68.5 KB)
//   fc2   : 64.5 KB quarter slice, receive slots 8 x (256 B + 32 x 8 floats): [64.5 KB, 74.5 KB)
//   QKV   : 8.1 KB slice, receive slots 16 x (32 B stats + 4 x 96 floats) = 24.5 KB: [8.1 KB, 32.6 KB), q|k|v at QKV_OFF; the
//           first K/V stage of attention warps 0-5 in [34 KB, 82 KB), idle for the whole phase (warps 6, 7: the last 8 KB of the
//           two weight buffers, which no job of the phase reaches)
//   q_cross: 8.1 KB slice, receive slots 16 x (32 B + 4 x 32 floats) = 8.5 KB: [8.1 KB, 16.6 KB), q at QKV_OFF; the first K/V
//           stage of all eight attention warps in [24 KB, 88 KB)
//   both head phases: the second K/V stage + 192 floats of attention warps 0, 1 from R's start (over the dead slice and slots)
//   lm heads: the whole x image (65 KB)
constexpr int R_BYTES = 92160;
constexpr int QKV_OFF = R_BYTES - 2048;   // [4 rows][192] bf16 q|k|v (or [4][64] q_cross) of this rank's attention items
constexpr int SMEM_BYTES = R_OFF + R_BYTES;
static_assert(SMEM_BYTES + 1024 <= 227 * 1024, "cluster step kernel shared memory");
static_assert(ROWS * (1024 / 2 + 8) * 2 + V * (256 + ROWS * 34 * 4) <= R_BYTES, "fc1 plan");
static_assert(HROWS * (1024 / 2 + 8) * 2 + V * C * (32 + 4 * 96 * 4) <= QKV_OFF, "QKV plan");
// Attention plan of the head phases.  A warp's first K/V stage is requested at the top of the phase and read at its end, so it
// lies where neither the slice, the receive slots, q|k|v, a weight job of the phase (QKV: four of 48 KB and out-proj's 16 KB;
// q_cross fills one buffer, so its stages are all in R) nor the pair-merge scratch reaches.  The rest of a warp's scratch (second
// stage + 192 floats) is first touched when the attention starts: warps 0, 1 at R's start, warps 2-7 in the held weight buffer.
constexpr int ATT_STAGE = 2 * 32 * HD * 2;         // one K/V stage: 32 keys x (K row + V row)
constexpr int ATT_REST = ATT_SMEM - ATT_STAGE;     // second stage + 192 floats
constexpr int ATT_S0_QKV = 34 * 1024;              // R offset of warp 0's first stage, QKV phase (warps 0-5)
constexpr int ATT_S0_QC = QKV_OFF - V * ATT_STAGE; // R offset of warp 0's first stage, q_cross phase (warps 0-7)
constexpr int ATT_S0_WB = WB_BYTES - ATT_STAGE;    // weight-buffer offset of the first stage of warps 6 (buffer 0) and 7 (buffer 1), QKV phase
static_assert(HROWS * (1024 / 2 + 8) * 2 + V * C * (32 + 4 * 96 * 4) <= ATT_S0_QKV && ATT_S0_QKV + 6 * ATT_STAGE <= QKV_OFF, "attention plan: QKV stages in R");
static_assert(HROWS * (1024 / 2 + 8) * 2 + V * C * (32 + 4 * 32 * 4) <= ATT_S0_QC, "attention plan: q_cross stages in R");
static_assert(2 * ATT_REST <= ATT_S0_QC && 2 * ATT_REST <= ATT_S0_QKV && 6 * ATT_REST <= ATT_S0_WB, "attention plan: second stages");
static_assert(6 * 8 * (1024 / 2) * 2 <= ATT_S0_WB && 16384 + 4 * 128 * 4 <= ATT_S0_WB, "attention plan: QKV weight jobs, out-proj job + pair merge");
static_assert(ROWS * (4096 / 4 + 8) * 2 + V * (256 + ROWS * 8 * 4) <= R_BYTES, "fc2 plan");

// ---- PTX helpers used by this kernel only (ptx.cuh has the shared ones) ------------------------------
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int what) {
  uint32_t ok, spins = 0;
  do {
    ok = mbar_try_wait_cluster(bar, parity);
    if (!ok && ++spins > (1u << 22)) { printf("ptts: cluster step mbarrier timeout (cta %d, barrier kind %d)\n", (int)blockIdx.x, what); __trap(); }
  } while (!ok);
}
// registers -> a peer's shared memory (DSMEM): a remote store whose bytes complete on the peer's mbarrier, with no release and no
// acknowledgement round trip.  Both addresses are the peer's (mapa); the PTX ISA leaves st.async to the executing CTA undefined.
// It is a weak store of the memory model, so the receive slots count as written through the generic proxy: every TMA write over
// them later (the next activation slice, the attention's K/V stages) follows a fence.proxy.async on its issuing thread, after that
// thread's exchange wait (request_slice at each device-wide barrier; the attention before its first K/V stage).
__device__ __forceinline__ void st_async(uint32_t dst_cluster_addr, float v, uint32_t bar_cluster_addr) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];"
               ::"r"(dst_cluster_addr), "r"(__float_as_uint(v)), "r"(bar_cluster_addr) : "memory");
}
__device__ __forceinline__ void st_async(uint32_t dst_cluster_addr, float2 v, uint32_t bar_cluster_addr) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];"
               ::"r"(dst_cluster_addr), "f"(v.x), "f"(v.y), "r"(bar_cluster_addr) : "memory");
}
__device__ __forceinline__ uint32_t mapa(uint32_t addr, uint32_t rank) { uint32_t r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank)); return r; }
__device__ __forceinline__ uint32_t cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
// The per-phase cluster barrier only guards buffer REUSE (a peer may overwrite my receive slots once I have consumed the previous
// phase's); the data itself is ordered by the exchange mbarrier.  A write-after-read needs no
// release: the default .release arrive is a gpu-scope MEMBAR per warp (it waits for the epilogue's global stores to be acknowledged,
// a second time before the layer barrier does).
__device__ __forceinline__ void cluster_arrive_reuse() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }

// K-slice layout of the activation images and of the packed weights: rank r holds the k32 tiles kt with (kt & 7) >> 2 == r, in
// ascending order.  Warp e4 of rank r then reduces the k-tiles kt = 4 r + e4 (mod 8): the tiles, in the order, that warp 4 r + e4
// of step.cu's 8-warp K split reduces, and every destination adds the eight partial sums in that warp order -- so both step
// kernels compute the same bits (step.cu serves the shapes and devices this kernel does not cover).
__host__ __device__ __forceinline__ int kslice(int kt) { return (kt & 7) >> 2; }
__host__ __device__ __forceinline__ int klocal(int kt) { return ((kt >> 3) << 2) | (kt & 3); }
__host__ __device__ __forceinline__ int kglobal(int rank, int lk) { return ((lk >> 2) << 3) | (rank << 2) | (lk & 3); }

// One warp's MMA loop: QN n-tiles x MT m-tiles over the local k-tiles kt0, kt0 + 4, ... < kt_end of the staged slice, one
// accumulator per output (the dependent chain of step.cu, whose sums it must reproduce).  ACC: continue from `out` (fc2's second
// quarter of F).  STATS: the warp also accumulates the LayerNorm row sums of its k-tiles from the A fragments it has loaded anyway
// (the two destination groups of a residue class repeat this work: 6 extra MMAs per k-tile and m-tile buy an exchange without any
// CTA-wide synchronisation).
template <int QN, int MT, bool STATS, bool ACC = false>
__device__ __forceinline__ void mma_slice(float (&out)[2][6][4], RowStatFrag& rst, const bf16* xs, int apitch, const uint4* wb, int KT, int kt0,
                                          int kt_end, int lrow, int lcol) {
  float acc[MT][QN][4];
#pragma unroll
  for (int a = 0; a < MT; a++)
#pragma unroll
    for (int j = 0; j < QN; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) acc[a][j][e] = ACC ? out[a][j][e] : 0.f;
  for (int kt = kt0; kt < kt_end; kt += 4) {
    uint32_t a[MT][2][4];
#pragma unroll
    for (int mt = 0; mt < MT; mt++)
#pragma unroll
      for (int j = 0; j < 2; j++) ldmatrix_x4(a[mt][j], xs + (size_t)(mt * 16 + lrow) * apitch + kt * 32 + j * 16 + lcol);
    if (STATS) {   // every k-tile of this warp's residue class: its blocks then carry complete statistics for it
#pragma unroll
      for (int mt = 0; mt < MT; mt++) { row_stat_mma(rst, mt, a[mt][0]); row_stat_mma(rst, mt, a[mt][1]); }
    }
#pragma unroll
    for (int j = 0; j < QN; j++) {
      const uint4 w = wb[((size_t)j * KT + kt) * 32];
#pragma unroll
      for (int mt = 0; mt < MT; mt++) {
        mma_bf16_16816(acc[mt][j], a[mt][0], w.x, w.y);
        mma_bf16_16816(acc[mt][j], a[mt][1], w.z, w.w);
      }
    }
  }
#pragma unroll
  for (int mt = 0; mt < MT; mt++)
#pragma unroll
    for (int j = 0; j < QN; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) out[mt][j][e] = acc[mt][j][e];
}

// phase kinds of a layer
enum { PH_QKV = 0, PH_O = 1, PH_QC = 2, PH_OC = 3, PH_FC1 = 4, PH_FC2 = 5 };
constexpr int JOBS_PER_LAYER = 9;   // weight jobs: QKV (four quarters of 6 n-tiles), O, QC, OC, FC1, FC2
constexpr int QKV_JOBS = 4;

// source of weight job j for this CTA (9 per layer, then this CTA's lm-head tasks)
__device__ __forceinline__ bool weight_job(const StepParams& p, int j, int cta, int rank, const char*& src, uint32_t& bytes) {
  const int nl = JOBS_PER_LAYER * p.L;
  if (j < nl) {
    const int l = j / JOBS_PER_LAYER, jl = j - JOBS_PER_LAYER * l;
    const int ph = jl < QKV_JOBS ? 0 : jl - (QKV_JOBS - 1);
    // the head phases' slices are shared by the four row-block clusters of a head: indexed (head, rank)
    const int64_t idx = (ph == PH_QKV || ph == PH_QC) ? (int64_t)(cta >> 3) * C + rank : (int64_t)cta;
    const int64_t sz = p.lay.cp_slice[ph];
    bytes = (uint32_t)(ph == PH_QKV ? sz / QKV_JOBS : sz);
    src = p.blob + p.lay.layer0 + p.lay.layer_stride * l + p.lay.cp[ph] + idx * sz + (ph == PH_QKV ? jl * (sz / QKV_JOBS) : 0);
    return true;
  }
  const int task = cta + (int)gridDim.x * (j - nl);
  const int ntasks = p.K * p.V / 32;
  if (task >= ntasks) return false;
  bytes = (uint32_t)(4 * p.H * 16);  // 4 n-tiles x K (fragment order: 16 B per (n-tile, k-pair) lane row)
  src = p.blob + p.lay.heads + (int64_t)task * bytes;
  return true;
}

template <int ITEMS, bool RAGGED>
__global__ void __launch_bounds__(THREADS, 1) decode_step_cluster_kernel(const __grid_constant__ StepParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  Ctrl* ctrl = p.sa.ctrl;
  if (p.prof != nullptr && blockIdx.x == 0 && threadIdx.x == 0) p.prof[(size_t)(6 * p.L + 2) * PROF_STRIDE + 3] = clock64();
  if (ctrl->active == 0) return;  // generation finished: the rest of the enqueued steps are no-ops (uniform over the grid)
  int cur_len = ctrl->cur_len;     // advanced locally when one launch runs several steps
  const unsigned gen = (unsigned)ctrl->launch_gen;
  int pos = p.P + cur_len - 1;  // cache position of the token being fed
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int H = p.H, F = p.F, B = p.B;
  const int rank = (int)cluster_rank(), peer = rank ^ 1;
  const int cta = (int)blockIdx.x;         // = cluster * 2 + rank
  const int cluster = cta >> 1;
  const int head = cluster >> 2, rblk = cluster & 3;   // head phases: this cluster's head and its batch-row block (rows 8 rblk ..)
  const int Ks = H / C, KsF = F / 4;       // K-slice widths: a CTA's half of H, a quarter of F (fc2 stages its half in two)
  const int pitch = Ks + 8, pitchF = KsF + 8;
  const int qe = F / p.nh / 64;            // fc1 n-tiles per destination rank (Mini: 4)
  const int dgrp = warp & 1, e4 = warp >> 1;  // this warp: destination rank (head phases: n-tile group), K class 4 rank + e4

  uint64_t* abar = reinterpret_cast<uint64_t*>(smem);        // activation slice
  uint64_t* wbar = abar + 1;                                  // [2] weight ring
  uint64_t* xbar = abar + 3;                                  // cluster exchange
  uint64_t* attbars = reinterpret_cast<uint64_t*>(smem + 128);  // [8 warps][2] K/V ring stages of the attention
  float* stats = reinterpret_cast<float*>(smem + OFF_STATS);   // [32][2] mean, rstd
  float* part = reinterpret_cast<float*>(smem + OFF_PART);     // [8][32][2]
  float* res_s = reinterpret_cast<float*>(smem + OFF_RES);     // [32][8] residual stream slice owned by this CTA
  float* cvec = reinterpret_cast<float*>(smem + OFF_CVEC);     // c1[256] | c2[256] of the current phase's features
  unsigned char* Rg = smem + R_OFF;
  const uint32_t peer_xbar = mapa(smem_u32(xbar), (uint32_t)peer);
  uint32_t par_a = 0, par_w = 0, par_x = 0, att_parity = 0;

  if (tid == 0) {
    mbar_init<1>(abar); mbar_init<1>(&wbar[0]); mbar_init<1>(&wbar[1]); mbar_init<1>(xbar);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  attention_decode_init_warp(attbars + 2 * warp, lane);
  cluster_arrive(); cluster_wait();   // every peer's mbarriers exist before any remote complete_tx
  unsigned* const bar_ctr = p.bar + (gen & 1u);
  unsigned bar_target = 0u;
  if (cta == 0 && tid == 0) p.bar[(gen + 1u) & 1u] = 0u;  // the counter the NEXT launch will use

  const char* blob = p.blob;
  long long* const prof0 = (p.prof != nullptr && cta == 0) ? p.prof : nullptr;
  long long* prof = prof0;
  prof_mark(prof, 0);

  // weight ring: job j lives in buffer j & 1; jobs 0 and 1 are requested now, job j + 2 when job j's MMA loop has retired
  auto issue_weight_job = [&](int j) {  // ONE thread
    const char* src; uint32_t bytes;
    if (!weight_job(p, j, cta, rank, src, bytes)) return;
    // No proxy fence here: the ring buffers are only ever WRITTEN through the async proxy (weights, K/V stages) and read with
    // generic loads -- a write-after-read across proxies needs none -- and fence.proxy.async waits for every bulk copy the CTA has
    // in flight (a stall wherever one sits behind a 64 KB weight copy).  The one generic-written corner (the attention
    // merge scratch of the q_cross phase) is covered by the fence thread 0 executes at every device-wide barrier (request_slice).
    mbar_expect_tx(&wbar[j & 1], bytes);
    bulk_g2s_evict_first(smem + HDR + (j & 1) * WB_BYTES, src, bytes, &wbar[j & 1]);
  };
  // ---- one launch runs up to p.n_steps tokens (ptts_decode_steps): the gap between dependent cooperative launches, the launch
  // skew in front of the first barrier and the cold instruction fetches of the once-per-token phases are paid once per launch.
  // Nothing below depends on the launch except the barrier counter, which simply keeps counting.
  __shared__ int s_next_active;
  const int n_steps = (p.do_sample_phase && p.n_steps > 1 && prof0 == nullptr) ? p.n_steps : 1;
  int unfinished_prev = 0;   // ctrl->n_unfinished is 0 at launch and only grows inside it (one add per unfinished row and step)
#pragma unroll 1
  for (int it = 0; it < n_steps; it++) {
  pos = p.P + cur_len - 1;
  prof = prof0;
  cluster_arrive_reuse();             // pre-arm: pairs with the first phase's "exchange buffers free" wait
  if (tid == 0) { issue_weight_job(0); issue_weight_job(1); }

  // global activation images, K-sliced for their consumer: [slices][32 rows][slice width + 8] bf16
  bf16* const x_img = p.cl_x;       // 2 slices of H/2 columns (consumers: QKV, q_cross, fc1, lm heads)
  bf16* const a_img = p.cl_attn;    // 2 slices of H/2 columns = 8 heads (consumers: out_proj, cross out_proj)
  bf16* const h_img = p.cl_h;       // 4 slices of F/4 columns (consumer: fc2, two per rank)
  const int x_slice_elems = ROWS * pitch, h_slice_elems = ROWS * pitchF;
  // h feature n -> (quarter 2 kslice + local k-tile / (F / 128), column) of the fc2 image (row 0)
  auto h_offset = [&](int n) {
    const int lk = klocal(n >> 5), kq = KsF >> 5;
    return (size_t)(2 * kslice(n >> 5) + lk / kq) * h_slice_elems + (lk % kq) * 32 + (n & 31);
  };
  // where this CTA's 8 residual / out-proj features live in the x image: feature n = cta * 8 + f (one k32 tile, kslice)
  const int xo_slice = kslice(cta >> 2), xo_col = klocal(cta >> 2) * 32 + (cta & 3) * 8;

  // ---- embeddings: this CTA's 32 x 8 slice of sum_k embed_k[id] (+ position) -> residual slice + x image -----------------
  {
    const int row = tid >> 3, f = tid & 7, n = cta * 8 + f;
    const float v = row < B ? embed_value(p, row, n, row_pos<RAGGED>(p, row, pos)) : 0.f;
    res_s[row * 8 + f] = v;
    x_img[(size_t)xo_slice * x_slice_elems + row * pitch + xo_col + f] = __float2bfloat16_rn(v);
  }
  prof_mark(prof, 6);
  auto request_slice = [&](const bf16* img_slice, uint32_t bytes) {  // thread 0, the moment a device-wide barrier opens
    fence_proxy_async_smem();
    mbar_expect_tx(abar, bytes);
    bulk_g2s(Rg, img_slice, bytes, abar);
  };
  // activation slice of phase kind `sub`: rows of this cluster's row block for the head phases, all 32 rows otherwise; fc2: the
  // first of this rank's two quarters of F (the second is requested when the first one's MMAs have retired)
  auto slice_of = [&](int sub, const bf16*& img, uint32_t& bytes) {
    if (sub == PH_QKV || sub == PH_QC) { img = x_img + (size_t)rank * x_slice_elems + (size_t)(HROWS * rblk) * pitch; bytes = (uint32_t)(HROWS * pitch * 2); }
    else if (sub == PH_O || sub == PH_OC) { img = a_img + (size_t)rank * x_slice_elems; bytes = (uint32_t)(x_slice_elems * 2); }
    else if (sub == PH_FC1) { img = x_img + (size_t)rank * x_slice_elems; bytes = (uint32_t)(x_slice_elems * 2); }
    else { img = h_img + (size_t)(2 * rank) * h_slice_elems; bytes = (uint32_t)(h_slice_elems * 2); }
  };
  {
    const bf16* nimg; uint32_t nbytes;
    slice_of(PH_QKV, nimg, nbytes);
    bar_target = grid_sync(bar_ctr, bar_target, -1, false, nullptr, [&]() { request_slice(nimg, nbytes); });
  }
  prof_mark(prof, 7);

  const int lrow = (lane & 7) + ((lane >> 3) & 1) * 8, lcol = (lane >> 4) * 8;
  const int g = lane >> 2, t4 = lane & 3;
  const int n_phases = 6 * p.L;

  // this warp's attention item: row 8 rblk + 4 rank + (warp >> 1), this cluster's head, whose 64 output features are k-tiles
  // 2 head, 2 head + 1 (adjacent in one K-slice of the attn image)
  const int att_row = HROWS * rblk + 4 * rank + (warp >> 1);
  const int att_slice = kslice(2 * head), att_col = klocal(2 * head) * 32;

#pragma unroll 1
  for (int ph = 0; ph < n_phases; ph++) {
    const int l = ph / 6, sub = ph - 6 * l;
    prof = prof0 ? prof0 + (size_t)(ph + 1) * PROF_STRIDE : nullptr;
    prof_mark(prof, 0);
    const char* lb = blob + p.lay.layer0 + p.lay.layer_stride * l;
    const bool rowpart = (sub == PH_QKV || sub == PH_QC);
    const bool has_ln = (sub == PH_QKV || sub == PH_QC || sub == PH_FC1);
    // n-tiles per warp: head phases per pass (two passes: QKV 2 x 6 of the head's 24, q_cross 2 x 2 of its 8), otherwise per destination
    const int q = (sub == PH_QKV) ? 6 : (sub == PH_QC ? 2 : (sub == PH_FC1 ? qe : 1));
    const int Nc = 4 * q * 8;                                        // head phases: features of the head
    const int KT = (sub == PH_FC2 ? KsF : Ks) >> 5;                  // k32 tiles of a staged slice (fc2: of one quarter of F)
    const int apitch = (sub == PH_FC2) ? pitchF : pitch;
    const int act_bytes = (rowpart ? HROWS : ROWS) * apitch * 2;
    // exchange geometry (receive slots right behind the activation slice).  feature-partitioned: one block per warp, landing in
    // slot (K class) at its destination; row-partitioned: one block per (warp, destination) with the warp's columns of both
    // passes, slot 8 rank + warp
    const int RS = (q == 1) ? 8 : 8 * q + 2;                         // floats per row of a feature-partitioned block
    const int blk = rowpart ? 32 + 4 * 16 * q * 4 : 256 + ROWS * RS * 4;   // one exchanged block: [statistics][rows][columns]
    unsigned char* const recv = Rg + ((act_bytes + 127) & ~127);
    const uint32_t peer_recv = mapa(smem_u32(recv), (uint32_t)peer);
    // bytes the PEER stores into this CTA's slots (its own slots take plain stores); row padding and unread statistics are not sent:
    //   feature-partitioned: V / C slots x (32 rows x 8 q columns, + 32 rows x (S1, S2) with a LayerNorm) x 4 B
    //   row-partitioned    : V slots x 4 rows x 16 q columns + the V / 2 dgrp == 0 warps' 4 rows x (S1, S2), x 4 B
    const uint32_t xbytes = 4u * (rowpart ? V * 4 * 16 * q + V / 2 * 4 * 2 : V / C * (ROWS * 8 * q + (has_ln ? ROWS * 2 : 0)));
    // one value (pair) of this CTA's partial sums -> byte `off` of destination d's receive slots: st.async into the peer, a plain
    // store into this CTA's own slots (published to the epilogue by the CTA barrier in front of the exchange wait)
    auto put = [&](int d, uint32_t off, auto v) {
      if (d == rank) *reinterpret_cast<decltype(v)*>(recv + off) = v;
      else st_async(peer_recv + off, v, peer_xbar);
    };
    const int j0 = JOBS_PER_LAYER * l + (sub == 0 ? 0 : sub + QKV_JOBS - 1);   // first weight job of this phase
    if (tid == 0) mbar_expect_tx(xbar, xbytes);

    // Head phases: this warp's first K/V chunk is requested NOW, so that it lands while the projection runs (the attention at the
    // end of the phase otherwise starts with every warp of the grid waiting for a cold HBM read).  What it reads does not depend
    // on this token: cross-attention rows were written by the prefill; self-attention reads rows < pos, each stored by an earlier
    // token and followed there by fence.proxy.async.global + a device-wide barrier (grid_sync) -- with several tokens per launch
    // too, 6 L barriers lie between a token's append and the next token's request -- and row `pos` comes from shared memory.
    // No fence.proxy.async: thread 0's fence when the last barrier opened (request_slice) is ordered before this by the
    // barrier's closing __syncthreads, and only bulk copies write the stage from then to the end of the attention.
    auto att_stage0 = [&]() -> unsigned char* {   // (computed at each use: nothing more is carried across the MMA loop)
      if (sub == PH_QC) return Rg + ATT_S0_QC + warp * ATT_STAGE;
      return warp < 6 ? Rg + ATT_S0_QKV + warp * ATT_STAGE : smem + HDR + (warp - 6) * WB_BYTES + ATT_S0_WB;
    };
    // The request is sized by the row's own position (row_pos): a ragged continuation's shorter rows never read the slots past it.
    if (rowpart && att_row < B)
      attention_decode_request<bf16>(decode_attn_args(p, l, pos, sub == PH_QC), att_row, head, row_pos<RAGGED>(p, att_row, pos), att_stage0(),
                                     attbars + 2 * warp, lane, warp & 1, 2);

    // folded-LayerNorm vectors of this phase's features: requested now, parked in shared memory after the MMA loop (a global
    // load followed at once by its shared-memory store would park the warp for an L2 round trip in front of the MMAs)
    float cv1 = 0.f, cv2 = 0.f;
    if (has_ln) {
      const float* c1; int ntot;
      if (sub == PH_QKV) { c1 = reinterpret_cast<const float*>(lb + p.lay.c_qkv); ntot = p.qkv_rows; }
      else if (sub == PH_QC) { c1 = reinterpret_cast<const float*>(lb + p.lay.c_qc); ntot = H; }
      else { c1 = reinterpret_cast<const float*>(lb + p.lay.c_fc1); ntot = F; }
      const int nown = rowpart ? Nc : 8 * q;
      if (tid < nown) {
        int n;
        if (sub == PH_QKV) n = (tid >> 6) * (p.nh * HD) + head * HD + (tid & 63);
        else if (sub == PH_QC) n = head * HD + tid;
        else n = cta * 8 * q + tid;
        cv1 = c1[n];
        cv2 = c1[ntot + n];
      }
    }

    // ---- MMA: this warp's n-tiles over its K residue class of the CTA's slice ----
    auto wait_job = [&](int j) {
      mbar_wait(&wbar[j & 1], (par_w >> (j & 1)) & 1u, 1);
      par_w ^= 1u << (j & 1);
    };
    auto ring = [&](int j) { return reinterpret_cast<const uint4*>(smem + HDR + (j & 1) * WB_BYTES) + lane; };
    wait_job(j0);
    if (sub == PH_QKV) wait_job(j0 + 1);
    mbar_wait(abar, par_a, 0);
    par_a ^= 1u;
    prof_mark(prof, 1);
    float acc[2][QMAX][4];
    RowStatFrag rst;
    row_stat_zero(rst);
    {
      const bf16* xs = reinterpret_cast<const bf16*>(Rg);
      if (rowpart) {
        // 8 live rows: the ldmatrix rows 8-15 repeat rows 0-7 (what they produce is never read).  Pass P: warp group dgrp takes
        // unit u = 2 P + dgrp of the head's n-tiles (QKV: weight job j0 + u; q_cross: n-tiles 2 u, 2 u + 1 of job j0).  Each pass's
        // tiles go to their destinations as soon as its MMAs retire, pass 0's with the LayerNorm statistics (complete after it):
        // live row g (fragment elements 0, 1) -> rank g >> 2, row g & 3 of slot 8 rank + warp: [stats 4 x 2][4 rows][16 q]
        auto head_pass = [&](auto pass_tag) {
          constexpr int P = decltype(pass_tag)::value;
          const int u = 2 * P + dgrp;
          float t[2][QMAX][4];
          if (sub == PH_QKV) mma_slice<6, 1, P == 0>(t, rst, xs, apitch, ring(j0 + u), KT, e4, KT, lrow & 7, lcol);
          else mma_slice<2, 1, P == 0>(t, rst, xs, apitch, ring(j0) + (size_t)(2 * u) * KT * 32, KT, e4, KT, lrow & 7, lcol);
          const int d = g >> 2;
          const uint32_t slot = (uint32_t)((8 * rank + warp) * blk);
          if (P == 0) {
            // the peer is past its previous epilogue (it arrived before the device-wide barrier opened): its slots are free
            cluster_wait();
            if (dgrp == 0) {   // the epilogue reads each K class's statistics from its dgrp == 0 warp
              const uint32_t so = slot + 8 * (g & 3);
              if (t4 == 0) put(d, so, rst.s1[0][0]);
              if (t4 == (g >> 1)) put(d, so + 4, (g & 1) ? rst.sq[0][0][1] : rst.sq[0][0][0]);
            }
          }
#pragma unroll
          for (int j = 0; j < QMAX; j++)
            if (j < q) put(d, slot + 32 + 4 * ((g & 3) * 16 * q + P * 8 * q + j * 8 + 2 * t4), make_float2(t[0][j][0], t[0][j][1]));
        };
        head_pass(std::integral_constant<int, 0>{});
        if (sub == PH_QKV) {   // quarters 2 and 3 of the head's QKV slice take the ring buffers of quarters 0 and 1
          prof_mark(prof, 8);
          __syncthreads();
          if (tid == 0) { issue_weight_job(j0 + 2); issue_weight_job(j0 + 3); }
          wait_job(j0 + 2);
          wait_job(j0 + 3);
          prof_mark(prof, 9);
        }
        head_pass(std::integral_constant<int, 1>{});
      } else if (sub == PH_FC2) {
        // quarter 2 rank + qq of F holds local k-tiles [qq KT, (qq + 1) KT) of the weight slice (2 KT per n-tile); the warp's
        // residue class continues from the first quarter into the second in the same accumulators
        auto quarter = [&](auto qq_tag) {
          constexpr int QQ = decltype(qq_tag)::value;
          const uint4* wq = ring(j0) + (size_t)dgrp * 2 * KT * 32 + (size_t)QQ * KT * 32;
          mma_slice<1, 2, false, QQ == 1>(acc, rst, xs, apitch, wq, 2 * KT, (e4 - QQ * KT) & 3, KT, lrow, lcol);
        };
        quarter(std::integral_constant<int, 0>{});
        prof_mark(prof, 8);
        __syncthreads();   // the first quarter is dead: the second one replaces it
        if (tid == 0) request_slice(h_img + (size_t)(2 * rank + 1) * h_slice_elems, (uint32_t)(h_slice_elems * 2));
        mbar_wait(abar, par_a, 0);
        par_a ^= 1u;
        prof_mark(prof, 9);
        quarter(std::integral_constant<int, 1>{});
      } else {
        const uint4* wb = ring(j0) + (size_t)(dgrp * q) * KT * 32;   // this destination's n-tiles
        if (sub == PH_FC1) {
          if (q == 4) mma_slice<4, 2, true>(acc, rst, xs, apitch, wb, KT, e4, KT, lrow, lcol);
          else if (q == 2) mma_slice<2, 2, true>(acc, rst, xs, apitch, wb, KT, e4, KT, lrow, lcol);
          else mma_slice<1, 2, true>(acc, rst, xs, apitch, wb, KT, e4, KT, lrow, lcol);
        } else mma_slice<1, 2, false>(acc, rst, xs, apitch, wb, KT, e4, KT, lrow, lcol);
      }
    }
    prof_mark(prof, 2);
    // ---- exchange: every warp stores its partial block straight into its destination's receive slot, with no CTA-wide
    // synchronisation on the way (the head phases did so inside their passes).  Profile stamps: 12 -> 13 cluster wait, 13 -> 14
    // the stores, 14 -> 15 CTA barrier + weight refill, 15 -> 3 the wait for the peer's bytes ----
    //   feature-partitioned: warp (e4, dgrp) -> rank dgrp, slot 4 rank + e4: [stats 32 x 2][32 rows][RS]
    //   row-partitioned    : warp w -> every rank d, slot 8 rank + w:        [stats 4 x 2][4 rows][16 q]  (rows 4d..4d+3, the warp's columns)
    prof_mark(prof, 12);
    if (!rowpart) cluster_wait();  // the peer is past its previous epilogue: its receive slots are free
    prof_mark(prof, 13);
    if (!rowpart) {
      const uint32_t slot = (uint32_t)((4 * rank + e4) * blk);
#pragma unroll
      for (int mt = 0; mt < 2; mt++)
#pragma unroll
        for (int j = 0; j < QMAX; j++) {
          if (j < q) {
            const uint32_t o = slot + 256 + 4 * ((mt * 16 + g) * RS + j * 8 + 2 * t4);
            put(dgrp, o, make_float2(acc[mt][j][0], acc[mt][j][1]));
            put(dgrp, o + 4 * 8 * RS, make_float2(acc[mt][j][2], acc[mt][j][3]));
          }
        }
      if (has_ln) {   // (S1, S2) of rows g / g+8 of each m-tile over this warp's K class (lane layout: ln_stats.cuh)
#pragma unroll
        for (int mt = 0; mt < 2; mt++) {
          const uint32_t s0 = slot + 8 * (mt * 16 + g), s8 = s0 + 8 * 8;
          if (t4 == 0) { put(dgrp, s0, rst.s1[mt][0]); put(dgrp, s8, rst.s1[mt][2]); }
          if (t4 == (g >> 1)) {
            put(dgrp, s0 + 4, (g & 1) ? rst.sq[mt][0][1] : rst.sq[mt][0][0]);
            put(dgrp, s8 + 4, (g & 1) ? rst.sq[mt][1][3] : rst.sq[mt][1][2]);
          }
        }
      }
    }
    prof_mark(prof, 14);
    if (has_ln && tid < (rowpart ? Nc : 8 * q)) { cvec[tid] = cv1; cvec[256 + tid] = cv2; }   // read in the epilogue, several barriers later
    __syncthreads();  // activation slice and weight buffer(s) are dead; this CTA's stores into its own receive slots are visible
    // The weight ring's refill goes out now, while the partial sums travel (two jobs ahead).  The head phases hold the next head
    // phase's or fc1's weights back until their attention is done (the attention uses that buffer meanwhile), and cross out-proj
    // holds fc2's back: those three go out when the barrier opens (below).
    if (warp == 1 && lane == 0 && !rowpart && sub != PH_OC) issue_weight_job(j0 + 2);
    if (warp == 1 && lane == 0 && sub == PH_QKV) issue_weight_job(j0 + QKV_JOBS);   // out-proj
    prof_mark(prof, 15);
    mbar_wait(xbar, par_x, 2);
    par_x ^= 1u;
    prof_mark(prof, 3);

    // ---- epilogue: sum the partial blocks in a fixed order, LayerNorm fix-up, activation / residual ----
    if (!rowpart) {
      const int row = tid >> 3, f0 = tid & 7;
      float ln_mean = 0.f, ln_rstd = 0.f;
      if (has_ln) {   // (fc1) every thread adds its row's eight partial statistics itself, in block order: broadcast loads instead of a
        float S1 = 0.f, S2 = 0.f;   // 32-thread pass + CTA barrier
#pragma unroll
        for (int v = 0; v < V; v++) { const float2 x = *reinterpret_cast<const float2*>(recv + (size_t)v * blk + row * 8); S1 += x.x; S2 += x.y; }
        ln_mean = S1 / (float)H;
        ln_rstd = rsqrtf(fmaxf(S2 / (float)H - ln_mean * ln_mean, 0.f) + p.eps);
      }
      if (row < B && sub == PH_FC1 && q == 4) {   // 4 consecutive features per thread: 8-byte loads, one 8-byte store
        const int f = 4 * f0;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int sv = 0; sv < V; sv++) {
          const float* bp = reinterpret_cast<const float*>(recv + (size_t)sv * blk + 256) + row * RS + f;
          const float2 a = *reinterpret_cast<const float2*>(bp), b2 = *reinterpret_cast<const float2*>(bp + 2);
          v[0] += a.x; v[1] += a.y; v[2] += b2.x; v[3] += b2.y;
        }
#pragma unroll
        for (int e = 0; e < 4; e++) v[e] = apply_act(DT<bf16>::rnd(ln_rstd * (v[e] - ln_mean * cvec[f + e]) + cvec[256 + f + e]), p.act);
        uint2 pk;
        pk.x = att_pack(v[0], v[1]); pk.y = att_pack(v[2], v[3]);
        *reinterpret_cast<uint2*>(h_img + h_offset(cta * 32 + f) + row * pitchF) = pk;
      } else if (row < B) {
        for (int i = 0; i < q; i++) {
          const int f = f0 + 8 * i;
          float v = 0.f;
#pragma unroll
          for (int sv = 0; sv < V; sv++) v += reinterpret_cast<const float*>(recv + (size_t)sv * blk + 256)[row * RS + f];
          if (sub == PH_FC1) {
            v = ln_rstd * (v - ln_mean * cvec[f]) + cvec[256 + f];
            v = apply_act(DT<bf16>::rnd(v), p.act);
            h_img[h_offset(cta * 8 * q + f) + row * pitchF] = __float2bfloat16_rn(v);
          } else {  // out-proj / cross out-proj / fc2: residual add on the slice this CTA owns
            v = DT<bf16>::rnd(res_s[row * 8 + f] + DT<bf16>::rnd(v));
            res_s[row * 8 + f] = v;
            x_img[(size_t)xo_slice * x_slice_elems + row * pitch + xo_col + f] = __float2bfloat16_rn(v);
          }
        }
      }
    } else {
      bf16* qkv_s = reinterpret_cast<bf16*>(Rg + QKV_OFF);  // [4][Nc]
      auto gather = [&](auto jw_tag) {   // (the column counts are constants of the phase: no run-time divisions)
        constexpr int JW = decltype(jw_tag)::value, NC = 4 * JW, QCW = 2 * JW;   // columns of a unit, of the head, of a warp
        for (int idx = tid; idx < 4 * NC; idx += THREADS) {
          const int r4 = idx / NC, col = idx - r4 * NC;
          const int u = col / JW, cw = (u >> 1) * JW + (col - u * JW);   // unit u = 2 pass + warp group: the warps with dgrp == u & 1
          // row 8 rblk + 4 rank + r4: statistics from the dgrp == 0 warp of every K class, added by every thread itself (broadcast
          // loads: a warp's 32 elements share the row) instead of a 4-thread pass + CTA barrier
          float S1 = 0.f, S2 = 0.f;
#pragma unroll
          for (int e = 0; e < V; e++) {
            const float2 x = *reinterpret_cast<const float2*>(recv + (size_t)(8 * (e >> 2) + 2 * (e & 3)) * blk + r4 * 8);
            S1 += x.x; S2 += x.y;
          }
          const float ln_mean = S1 / (float)H;
          const float ln_rstd = rsqrtf(fmaxf(S2 / (float)H - ln_mean * ln_mean, 0.f) + p.eps);
          float v = 0.f;
#pragma unroll
          for (int e = 0; e < V; e++)   // K classes in order: warp 2 (e & 3) + (u & 1) of rank e >> 2
            v += reinterpret_cast<const float*>(recv + (size_t)(8 * (e >> 2) + 2 * (e & 3) + (u & 1)) * blk + 32)[r4 * QCW + cw];
          v = ln_rstd * (v - ln_mean * cvec[col]) + cvec[256 + col];
          qkv_s[idx] = __float2bfloat16_rn(v);
        }
      };
      if (sub == PH_QKV) gather(std::integral_constant<int, 48>{}); else gather(std::integral_constant<int, 16>{});
      static_assert(HD == 64, "QKV: 2 x 2 units of 6 n-tiles (q|k|v of a head), q_cross: 2 x 2 units of 2 n-tiles");
    }
    prof_mark(prof, 4);
    __syncthreads();   // this CTA's receive slots are consumed (and q|k|v complete): peers may send the next phase's partials
    cluster_arrive_reuse();

    // ---- attention of this rank's 4 (row, head) items: two warps per item, the sweep and the call step.cu's attention phase
    // makes (same key chunks, same split over the two warps, same merge), so the two step kernels agree bit for bit ----
    if (rowpart) {
      if (att_row < B) {
        AttnArgs att = decode_attn_args(p, l, pos, sub == PH_QC);
        const bf16* qkv_s = reinterpret_cast<const bf16*>(Rg + QKV_OFF);
        const int row_base = HROWS * rblk + 4 * rank;
        const bf16* qbase = qkv_s - (size_t)row_base * Nc - (size_t)head * HD;
        att.q = qbase; att.ldq = Nc;
        att.ldo = pitch;
        att.out = a_img + (size_t)att_slice * x_slice_elems + att_col - (size_t)head * HD;
        if (sub == PH_QKV) { att.knew = qbase; att.vnew = qbase; att.ldkv = Nc; att.k_col0 = HD; att.v_col0 = 2 * HD; }
        // the first K/V stage is where the top of the phase asked for it; the rest of a warp's scratch (second stage, then 192
        // floats): warps 0, 1 at R's start, warps 2-7 in the weight buffer whose job is held back; the pair merge in the other
        // buffer behind out-proj's / cross out-proj's 16 KB
        unsigned char* wb0 = smem + HDR;
        unsigned char* held = wb0 + ((sub == PH_QKV ? j0 + 1 : j0) & 1) * WB_BYTES;
        unsigned char* other = wb0 + ((sub == PH_QKV ? j0 : j0 + 1) & 1) * WB_BYTES;
        unsigned char* rest = warp < 2 ? Rg + (size_t)warp * ATT_REST : held + (size_t)(warp - 2) * ATT_REST;
        float* xr = reinterpret_cast<float*>(other + 16384) + (warp >> 1) * 128;
        prof_mark(prof, 10);
        attention_decode_sweep<bf16>(att, att_row, head, row_pos<RAGGED>(p, att_row, pos), att_stage0(), rest, attbars + 2 * warp, lane, att_parity, warp & 1, 2, xr, (warp >> 1) + 1,
                                     true, tid == 0 ? prof : nullptr);
      }
      prof_mark(prof, 5);
    }
    prof_mark(prof, 6);
    if (p.prof != nullptr && l == p.L / 2 && tid == 0) {   // profiling runs: when does EACH CTA reach the barrier of the middle layer's phases
      unsigned long long ns;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns));
      p.prof[(size_t)(n_phases + 4) * PROF_STRIDE + sub * (int)gridDim.x + cta] = (long long)ns;
    }

    // ---- device-wide barrier; the next phase's activation slice is requested the moment it opens ----
    const bool last = (ph + 1 == n_phases);
    const bf16* nimg; uint32_t nbytes;
    if (last) { nimg = x_img; nbytes = (uint32_t)(C * x_slice_elems * 2); }   // lm heads: the whole x image
    else slice_of((sub + 1) % 6, nimg, nbytes);
    // Everything this kernel reads that another CTA wrote during the same launch goes through L2 (TMA bulk copies of the images
    // and the K/V rows, __ldcg of the logits / EOS columns), so the L1 invalidation of an acquire fence protects nothing here and
    // would cost time at every barrier: the per-layer barriers (and the first one) go without it.
    // A 64 KB weight copy issued shortly before the barrier (q_cross's after the self-attention, fc1's after the cross-attention,
    // fc2's during the cross out-proj exchange) is still in flight when the barrier opens; with it there, these barriers took
    // 2-2.5 us longer on an H100.  Those jobs are requested right after the next phase's activation slice instead
    // (request_slice's proxy fence also orders the attention's generic writes into the held buffer before the copy).
    const int held_job = sub == PH_QKV ? j0 + QKV_JOBS + 1 : (sub == PH_QC || sub == PH_OC) ? j0 + 2 : -1;
    bar_target = grid_sync(bar_ctr, bar_target, ph, false, nullptr, [&]() {
      request_slice(nimg, nbytes);
      if (held_job >= 0) issue_weight_job(held_job);
    });
    prof_mark(prof, 7);
  }
  cluster_wait();  // balance the last phase's arrive

  // ---- final LayerNorm + K lm heads: N-split over all CTAs (4 n-tiles per task, full K), no exchange; warp w reduces the
  // k-tiles kt = w (mod 8) and the eight partial tiles are added in warp order, as step.cu's lm-head phase does ----
  prof = prof0 ? prof0 + (size_t)(n_phases + 1) * PROF_STRIDE : nullptr;
  prof_mark(prof, 0);
  {
    const int ntasks = p.K * p.V / 32;
    const float* c1 = reinterpret_cast<const float*>(blob + p.lay.c_heads);
    const float* c2 = c1 + p.K * p.V;
    mbar_wait(abar, par_a, 3);
    par_a ^= 1u;
    const bf16* xs = reinterpret_cast<const bf16*>(Rg);   // [2 slices][32][pitch]
    const int KTH = H >> 5;                                // k32 tiles of the full row
    auto ktile = [&](int kt) { return xs + (size_t)kslice(kt) * x_slice_elems + klocal(kt) * 32; };
    {  // row statistics over the full rows: k-tile kt by warp kt % 8
      RowStatFrag rst;
      row_stat_zero(rst);
      for (int kt = warp; kt < KTH; kt += 8) {
        const bf16* sl = ktile(kt);
#pragma unroll
        for (int mt = 0; mt < 2; mt++)
#pragma unroll
          for (int j = 0; j < 2; j++) {
            uint32_t a[4];
            ldmatrix_x4(a, sl + (size_t)(mt * 16 + lrow) * pitch + j * 16 + lcol);
            row_stat_mma(rst, mt, a);
          }
      }
      row_stat_store(rst, part, warp, lane);
      __syncthreads();
      row_stat_finalize(part, H, ROWS, p.eps, stats);
      __syncthreads();
    }
    prof_mark(prof, 1);
    constexpr int HRS = 40;   // row stride (floats) of the partial tiles [8 warps][32 rows][HRS]: conflict-free epilogue reads
    int job = JOBS_PER_LAYER * p.L;
    for (int task = cta; task < ntasks; task += (int)gridDim.x, job++) {
      mbar_wait(&wbar[job & 1], (par_w >> (job & 1)) & 1u, 4);
      par_w ^= 1u << (job & 1);
      float acc[2][4][4];
#pragma unroll
      for (int a = 0; a < 2; a++)
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
          for (int e = 0; e < 4; e++) acc[a][j][e] = 0.f;
      unsigned char* wbuf = smem + HDR + (job & 1) * WB_BYTES;
      const uint4* wb = reinterpret_cast<const uint4*>(wbuf) + lane;
      for (int kt = warp; kt < KTH; kt += 8) {
        const bf16* sl = ktile(kt);
        uint32_t a[2][2][4];
#pragma unroll
        for (int mt = 0; mt < 2; mt++)
#pragma unroll
          for (int j = 0; j < 2; j++) ldmatrix_x4(a[mt][j], sl + (size_t)(mt * 16 + lrow) * pitch + j * 16 + lcol);
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const uint4 w = wb[((size_t)j * KTH + kt) * 32];
#pragma unroll
          for (int mt = 0; mt < 2; mt++) {
            mma_bf16_16816(acc[mt][j], a[mt][0], w.x, w.y);
            mma_bf16_16816(acc[mt][j], a[mt][1], w.z, w.w);
          }
        }
      }
      __syncthreads();  // the weight buffer is dead: it takes the partial tiles
      float* red = reinterpret_cast<float*>(wbuf);
#pragma unroll
      for (int mt = 0; mt < 2; mt++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
          float* base = red + ((size_t)warp * 32 + mt * 16 + g) * HRS + j * 8 + 2 * t4;
          *reinterpret_cast<float2*>(base) = make_float2(acc[mt][j][0], acc[mt][j][1]);
          *reinterpret_cast<float2*>(base + 8 * HRS) = make_float2(acc[mt][j][2], acc[mt][j][3]);
        }
      __syncthreads();
      {
        const int er = tid >> 3, ec = tid & 7;
        if (er < B) {
          const float mean = stats[2 * er], rstd = stats[2 * er + 1];
#pragma unroll
          for (int j = 0; j < 4; j++) {
            const int cidx = j * 8 + ec, n = task * 32 + cidx;
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < 8; w++) v += red[((size_t)w * 32 + er) * HRS + cidx];
            p.logits[(size_t)er * p.K * p.V + n] = DT<bf16>::rnd(rstd * (v - mean * c1[n]) + c2[n]);
          }
        }
      }
      __syncthreads();  // the partial tiles are consumed: the buffer takes job + 2 (the fence orders their generic writes first)
      if (tid == 32) {
        fence_proxy_async_smem();
        issue_weight_job(job + 2);
      }
    }
  }
  prof_mark(prof, 6);
  bar_target = grid_sync(bar_ctr, bar_target, n_phases, true);
  prof = prof0 ? prof0 + (size_t)(n_phases + 2) * PROF_STRIDE : nullptr;  // tail row: sampling / barrier
  prof_mark(prof, 0);
  if (p.do_sample_phase) {
    const ptts_gen_params gp = *p.sa.gen;
    const int BK = B * p.K;
    sample_phase<ITEMS, RAGGED>(p.sa, gp, BK, cur_len);
    prof_mark(prof, 1);
    // every CTA learns whether any row is still unfinished: thread 0 reads the counter the moment the barrier opens (after its
    // acquire fence); the counter is reset only when the launch ends, so a step's count is the growth since the previous step
    bar_target = grid_sync(bar_ctr, bar_target, n_phases + 1, true, nullptr, [&]() {
      const int tot = *reinterpret_cast<volatile int*>(&ctrl->n_unfinished);
      s_next_active = (tot - unfinished_prev > 0) ? 1 : 0;
      unfinished_prev = tot;
    });
    prof_mark(prof, 2);
  }
  bool go_on = false;
  if (p.do_sample_phase) {
    const int act = s_next_active;   // (written before the barrier's closing __syncthreads)
    if (cta == 0 && tid == 0) {
      ctrl->cur_len = cur_len + 1;
      ctrl->active = act;
      ctrl->steps_run += 1;
    }
    go_on = act != 0;
    cur_len += 1;
  }
  if (!go_on) break;
  }  // steps of this launch
  if (cta == 0 && tid == 0) {
    // (a CTA that is slower out of the last barrier may still read the counter: it then sees a count <= the one it expects and
    // concludes "finished", which is what leaving the loop means anyway)
    if (p.do_sample_phase) ctrl->n_unfinished = 0;
    ctrl->launch_gen = (int)(gen + 1u);
  }
}

// ---- weight repack: fragment-order matrices -> one contiguous slice per (phase, cluster or head, rank) -------------------
// Both layouts are made of the same 512-byte (n8 x k32) tiles, so the repack is a tile gather.
//   head phases (QKV, q_cross): slice (head, rank) = the head's n-tiles x the rank's k-tiles kglobal(rank, 0 .. kts - 1)
//   the others: slice cta = cluster * 2 + rank = the cluster's ntc n-tiles x the rank's k-tiles
__global__ void cluster_pack_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int ph, int nh, int ntc, int kts, int KT_src) {
  const int64_t tile = blockIdx.x;   // dst tile index = (slice * ntc + j) * kts + ktl
  const int ktl = (int)(tile % kts);
  const int j = (int)((tile / kts) % ntc);
  const int slice = (int)(tile / ((int64_t)kts * ntc));
  const int rank = slice & 1, owner = slice >> 1;   // owner = head (head phases) or cluster
  int n_tile;
  if (ph == PH_QKV) n_tile = (j >> 3) * (nh * 8) + owner * 8 + (j & 7);   // q | k | v rows of head `owner` in the fused matrix
  else n_tile = owner * ntc + j;
  const int kt = kglobal(rank, ktl);
  dst[tile * 32 + threadIdx.x] = src[((int64_t)n_tile * KT_src + kt) * 32 + threadIdx.x];
}

}  // namespace cl

// ---- host side ----------------------------------------------------------------------------------
int cluster_pack_layer(const DecoderLayout& L, char* layer, cudaStream_t st) {
  for (int ph = 0; ph < 6; ph++) {
    const ClusterPhase cp = cluster_phase(L, ph);
    const int64_t tiles = (int64_t)cp.owners * cl::C * cp.nt * cp.kt;
    cl::cluster_pack_kernel<<<(unsigned)tiles, 32, 0, st>>>(reinterpret_cast<const uint4*>(layer + cp.mat),
                                                            reinterpret_cast<uint4*>(layer + L.cp[ph]), ph, L.nh, cp.nt, cp.kt, cp.kt_src);
  }
  PTTS_LAUNCH_CHECK();
  return PTTS_OK;
}

static const void* cluster_kernel_fn(const StepParams& p) {
  const bool rg = p.sa.shift != nullptr;
  if (p.sample_items <= 1) return rg ? (const void*)cl::decode_step_cluster_kernel<1, true> : (const void*)cl::decode_step_cluster_kernel<1, false>;
  if (p.sample_items <= 5) return rg ? (const void*)cl::decode_step_cluster_kernel<5, true> : (const void*)cl::decode_step_cluster_kernel<5, false>;
  return rg ? (const void*)cl::decode_step_cluster_kernel<9, true> : (const void*)cl::decode_step_cluster_kernel<9, false>;
}

static void cluster_launch_config(const StepParams& p, cudaLaunchConfig_t& cfg, cudaLaunchAttribute* at, cudaStream_t st) {
  cfg = cudaLaunchConfig_t{};
  cfg.gridDim = dim3((unsigned)(4 * p.nh * cl::C));   // 4 clusters per head
  cfg.blockDim = dim3(cl::THREADS);
  cfg.dynamicSmemBytes = cl::SMEM_BYTES;
  cfg.stream = st;
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = cl::C; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  at[1].id = cudaLaunchAttributeCooperative;   // every CTA spins on the others: co-residency must be guaranteed
  at[1].val.cooperative = 1;
  cfg.attrs = at;
  cfg.numAttrs = 2;
}

// true when the grid of 4 nh clusters of 2 can be co-resident on this device (Mini: 64 of the 66 a 132-SM H100 holds)
bool cluster_step_available(const StepParams& p) {
  const void* fn = cluster_kernel_fn(p);
  static bool told = false;
  auto why = [&](const char* what, cudaError_t e, int n) {
    if (!told) fprintf(stderr, "ptts_b200: cluster step kernel not used (%s: %s, %d co-resident clusters of %d, need %d); the one-CTA-per-SM step kernel runs instead\n",
                       what, cudaGetErrorString(e), n, cl::C, 4 * p.nh);
    told = true;
    cudaGetLastError();
    return false;
  };
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, cl::SMEM_BYTES);
  if (e != cudaSuccess) return why("shared memory attribute", e, 0);
  cudaLaunchConfig_t cfg; cudaLaunchAttribute at[2];
  cluster_launch_config(p, cfg, at, nullptr);
  cfg.numAttrs = 1;  // the occupancy query takes the cluster shape
  int n = 0;
  e = cudaOccupancyMaxActiveClusters(&n, fn, &cfg);
  if (e != cudaSuccess) return why("cluster occupancy query", e, n);
  if (n < 4 * p.nh) return why("too few co-resident clusters", cudaSuccess, n);
  return true;
}

int launch_decode_step_cluster(const StepParams& p, cudaStream_t st) {
  const void* fn = cluster_kernel_fn(p);
  cudaLaunchConfig_t cfg; cudaLaunchAttribute at[2];
  cluster_launch_config(p, cfg, at, st);
  void* args[] = {(void*)&p};
  PTTS_CHECK_CUDA(cudaLaunchKernelExC(&cfg, fn, args));
  return PTTS_OK;
}

}  // namespace ptts

// wgmma.cuh -- the Hopper tensor-core tile pipeline shared by the prefill GEMM (gemm_tc.cu) and the DAC convolutions
// (dac_tc.cu).  One CTA computes a 128 x N tile of D = A B^T with A [rows][K] and B [N][K] both bf16 and K-major:
//   * warp 8 (one thread) is the TMA producer: per K step of 64 it loads a 128 x 64 A box and an N x 64 B box into one of
//     STAGES shared-memory stages with the 128-byte swizzle (TMA zero-fills whatever lies outside the tensor);
//   * warps 0-7 are two consumer warpgroups, each owning 64 rows of the tile: wgmma.mma_async (m64 N k16) reads both operands
//     straight from shared memory and accumulates in fp32 registers; one wgmma group stays in flight while the stage the
//     previous group read is handed back to the producer;
//   * the caller's epilogue then works on the accumulator fragments (frag_row / frag_col give each register's place).
// Stage buffers are 1024-byte aligned (the swizzle atom); full[s] completes on the TMA byte count, empty[s] on one arrival
// per consumer warp.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "ptx.cuh"

namespace ptts {
namespace wg {

constexpr int M_TILE = 128;                          // rows per CTA tile (two consumer warpgroups of wgmma M = 64)
constexpr int K_STAGE = 64;                          // K elements per stage: one 128-byte swizzle row of bf16
constexpr int STAGES = 3;
constexpr int CONSUMER_WARPS = 8;
constexpr int PRODUCER_WARP = CONSUMER_WARPS;
constexpr int THREADS = 32 * (CONSUMER_WARPS + 1);
constexpr int A_BYTES = M_TILE * K_STAGE * 2;

template <int N> constexpr int STAGE_BYTES = (A_BYTES + N * K_STAGE * 2 + 1023) & ~1023;
// dynamic shared memory of a CTA: alignment slack, the stage ring, then 128 B of mbarriers, then `extra` bytes for the caller
template <int N> constexpr size_t smem_bytes(int extra) { return 1024 + (size_t)STAGES * STAGE_BYTES<N> + 128 + extra; }

__device__ __forceinline__ void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory"); }
// A wait that never completes traps (the launch fails) instead of hanging the GPU.  No printf here: a function call inside
// the consumer's K loop would make ptxas serialise the wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
  uint32_t ok, spins = 0;
  do {
    ok = mbar_try_wait(b, parity);
    if (!ok && ++spins > (1u << 24)) __trap();
  } while (!ok);
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)) : "memory");
}

// wgmma shared-memory matrix descriptor, K-major, 128-byte swizzle: 8-row groups 1024 B apart (stride byte offset); the
// leading byte offset is unused in this mode.  16 elements further along K = 32 bytes = +2 in the address field.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t addr) {
  return (uint64_t)((addr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// D[64 x N] (+)= A[64 x 16] B[N x 16]^T, bf16 operands from shared memory, fp32 accumulators; accumulate == 0 overwrites D
__device__ __forceinline__ void mma_n32(float (&d)[16], uint64_t da, uint64_t db, int accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void mma_n64(float (&d)[32], uint64_t da, uint64_t db, int accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void mma_n96(float (&d)[48], uint64_t da, uint64_t db, int accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %50, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, %48, %49, p, 1, 1, 0, 0;\n}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
               : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void mma_n128(float (&d)[64], uint64_t da, uint64_t db, int accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(da), "l"(db), "r"(accumulate));
}

template <int N>
__device__ __forceinline__ void mma(float (&d)[N / 2], uint64_t da, uint64_t db, int accumulate) {
  static_assert(N == 32 || N == 64 || N == 96 || N == 128, "wgmma tile width");
  if constexpr (N == 32) mma_n32(d, da, db, accumulate);
  else if constexpr (N == 64) mma_n64(d, da, db, accumulate);
  else if constexpr (N == 96) mma_n96(d, da, db, accumulate);
  else mma_n128(d, da, db, accumulate);
}

// Accumulator register i of a consumer thread holds tile row frag_row(i) (0..63 inside its warpgroup) and column frag_col(i);
// registers 2j and 2j+1 are adjacent columns of the same row.
__device__ __forceinline__ int frag_row(int i) { return 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int i) { return 8 * (i >> 2) + 2 * (threadIdx.x & 3) + (i & 1); }

struct Pipe {
  unsigned char* stages;
  uint64_t* full;
  uint64_t* empty;
  unsigned char* extra;  // the caller's bytes after the barriers
};

// Carves the dynamic shared memory; thread 0 initialises the barriers.  Call from every thread, then __syncthreads().
template <int N>
__device__ __forceinline__ Pipe pipe_setup(unsigned char* smem_raw) {
  Pipe p;
  p.stages = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  p.full = reinterpret_cast<uint64_t*>(p.stages + STAGES * STAGE_BYTES<N>);
  p.empty = p.full + STAGES;
  p.extra = reinterpret_cast<unsigned char*>(p.full) + 128;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; s++) { mbar_init<1>(&p.full[s]); mbar_init<CONSUMER_WARPS>(&p.empty[s]); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  return p;
}

// The K loop.  load(it, a_dst, b_dst, bar) issues the two TMA loads of K step `it` (producer thread only).  Consumer threads
// return with their 64 x N accumulator fragment in acc; the producer warp returns at once.
template <int N, class Load>
__device__ __forceinline__ void mainloop(const Pipe& p, int n_iter, Load load, float (&acc)[N / 2]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      for (int it = 0; it < n_iter; it++) {
        const int s = it % STAGES, use = it / STAGES;
        if (use > 0) mbar_wait(&p.empty[s], (use - 1) & 1);
        unsigned char* a_dst = p.stages + (size_t)s * STAGE_BYTES<N>;
        mbar_expect_tx(&p.full[s], (uint32_t)(A_BYTES + N * K_STAGE * 2));
        load(it, a_dst, a_dst + A_BYTES, &p.full[s]);
      }
    }
    return;
  }
  const uint32_t a_row0 = (uint32_t)(warp >> 2) * 64 * 128;  // this warpgroup's 64 rows of the A box (a multiple of 1024 B)
  for (int it = 0; it < n_iter; it++) {
    const int s = it % STAGES;
    mbar_wait(&p.full[s], (it / STAGES) & 1);
    const uint32_t a_addr = smem_u32(p.stages + (size_t)s * STAGE_BYTES<N>);
    const uint64_t da = desc_sw128(a_addr + a_row0), db = desc_sw128(a_addr + A_BYTES);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int k = 0; k < K_STAGE / 16; k++) mma<N>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (it > 0 || k > 0) ? 1 : 0);
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    // at most one group in flight: the group of step it-1 has finished reading its stage, hand that stage back
    asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
    if (it > 0 && lane == 0) mbar_arrive(&p.empty[(it - 1) % STAGES]);
  }
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}

}  // namespace wg
}  // namespace ptts

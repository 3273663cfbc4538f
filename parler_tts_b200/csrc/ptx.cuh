// ptx.cuh -- the inline-PTX wrappers more than one kernel file uses: shared-memory addresses, mbarriers, TMA bulk copies,
// L2 prefetches, ldmatrix / mma.sync, and the device-wide barrier of the persistent step kernels (step.cu, step2.cu) with
// the gpu-scope release / relaxed accesses it is built from.
#pragma once
#include "common.cuh"

namespace ptts {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarriers ------------------------------------------------------------------------------------
template <uint32_t COUNT>   // arrivals per phase
__device__ __forceinline__ void mbar_init(uint64_t* bar) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "n"(COUNT));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { mbar_expect_tx(smem_u32(bar), bytes); }
// One probe of phase `parity`: nonzero once it has completed.  Callers loop with their own timeout, which traps.
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
               : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok;
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) { return mbar_try_wait(smem_u32(bar), parity); }
// the same with cluster-scope acquire: also orders what peers of the cluster delivered with complete_tx
__device__ __forceinline__ uint32_t mbar_try_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok;
}

// ---- TMA bulk copies global -> shared memory (completion counted on an mbarrier) ---------------------
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  bulk_g2s(smem_u32(dst), src, bytes, smem_u32(bar));
}
// Streamed-once data (the weights, the K/V rows: ~1.2 GB per token, ten times the L2) is requested with an evict-first policy so
// that it does not push out what IS reused between and inside launches: the kernels' instructions, the folded-LayerNorm vectors,
// the activation images, the logits.
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void bulk_g2s_evict_first(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(l2_evict_first_policy()) : "memory");
}
__device__ __forceinline__ void bulk_g2s_evict_first(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  bulk_g2s_evict_first(smem_u32(dst), src, bytes, smem_u32(bar));
}
// this thread's generic-proxy shared-memory accesses before later async-proxy (TMA) writes
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// HBM -> L2, in pieces of at most 32 KB
__device__ __forceinline__ void l2_prefetch(const void* p, uint32_t bytes) {
  const char* c = reinterpret_cast<const char*>(p);
  while (bytes > 0) {
    const uint32_t n = bytes > 32768u ? 32768u : bytes;
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(c), "r"(n) : "memory");
    c += n;
    bytes -= n;
  }
}

// ---- tensor cores ---------------------------------------------------------------------------------
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* smem_ptr) { ldmatrix_x4(r, smem_u32(smem_ptr)); }
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// D += A B, m16n8k16, bf16 operands, fp32 accumulators
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  mma_bf16_16816(d, a[0], a[1], a[2], a[3], b0, b1);
}

// ---- device-wide barrier of the persistent step kernels --------------------------------------------
__device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

struct NoHook { __device__ __forceinline__ void operator()() const {} };

// Every CTA of the grid adds 1 to a monotonic counter in global memory and waits until it reaches `target` + gridDim.x (the
// returned new target).  Arrive = red.release (cumulative over the CTA's writes ordered by the preceding bar.sync); the spin is a
// RELAXED load (an acquire load would invalidate L1 on every poll); `acq_fence`: one acquire fence after the exit.
//   post:     runs on thread 0 the moment the barrier opens, before the CTA is released (e.g. the next phase's activation copy);
//   side:     runs on thread 32 between the two CTA barriers, i.e. while thread 0 polls: work that needs the whole CTA to be past
//             its shared-memory accesses but not the other CTAs (the next phase's weight copy) costs nothing there;
//   progress: optional [gridDim.x] array of the last phase `ph` each CTA arrived at; a timeout then names the late CTAs.
template <typename Post = NoHook, typename Side = NoHook>
__device__ __forceinline__ unsigned grid_sync(unsigned* ctr, unsigned target, int ph, bool acq_fence, int* progress = nullptr,
                                              Post post = Post(), Side side = Side()) {
  target += gridDim.x;
  // this thread's global writes (generic proxy) -> later TMA reads by other CTAs (async proxy): the proxy fence sits on the
  // writer side of the release/acquire chain, where it overlaps the store drain instead of delaying the next tile copy
  asm volatile("fence.proxy.async.global;" ::: "memory");
  __syncthreads();
  if (threadIdx.x == 0) {
    if (progress) progress[blockIdx.x] = ph;
    red_release_add(ctr, 1u);
    unsigned spins = 0;
    while (ld_relaxed(ctr) < target) {
      if (++spins > (1u << 24)) {
        printf("ptts: grid barrier timeout (cta %d target %u seen %u phase %d)\n", (int)blockIdx.x, target, ld_relaxed(ctr), ph);
        if (progress) for (int i = 0; i < (int)gridDim.x; i++) if (((volatile int*)progress)[i] != ph) printf("ptts:   cta %d is at phase %d\n", i, ((volatile int*)progress)[i]);
        __trap();
      }
    }
    if (acq_fence) asm volatile("fence.acq_rel.gpu;" ::: "memory");
    post();
  } else if (threadIdx.x == 32) {
    side();
  }
  __syncthreads();
  return target;
}

// clock64 stamp of thread 0 into slot `slot` of a profile row (nullptr: profiling off)
__device__ __forceinline__ void prof_mark(long long* prof, int slot) {
  if (prof != nullptr && threadIdx.x == 0) prof[slot] = clock64();
}

}  // namespace ptts

// Hopper (sm_90a) inline-PTX primitives shared by every kernel in this tree:
// mbarrier, TMA (cp.async.bulk.tensor, cluster multicast), wgmma descriptors and fences, clusters, multimem.
// Nothing here comes from the reference operator (it has no GPU code: SURVEY.md §2.6);
// these are the building blocks of the launched workers' hot path.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "wgmma.cuh"

namespace aitj {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Spin on phase parity. A time-bounded spin (~2 s of SM clock) turns a protocol bug into a
// trap (an error the host sees) instead of a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag = 0) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  long long t0 = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) break;
    const long long now = clock64();
    if (t0 == 0) t0 = now;
#ifdef AITJ_MBAR_DEBUG
    else if (now - t0 > 300000000ll) {
      printf("mbar timeout tag=%d parity=%u block=%d thread=%d\n", tag, parity, blockIdx.x, threadIdx.x);
      break;
    }
#else
    else if (now - t0 > 4000000000ll) { __trap(); }
#endif
  }
  (void)tag;
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving reads / writes of accumulator registers across an in-flight wgmma.
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma shared-memory matrix descriptor, 128B swizzle (the layout a SWIZZLE_128B TMA box of 64 bf16 per row leaves):
//   K-major operand:  rows of 64 K-elements (128 B), 8-row groups `sbo` = 1024 B apart, `lbo` unused;
//   MN-major operand: rows of 64 M/N-elements per K index, 8-K-row groups `sbo` = 1024 B apart, successive 64-element
//                     M/N chunks `lbo` bytes apart.
// The tile must start on a 1024-byte boundary (base offset 0); a K step inside a K-major row adds 32 B to the address.
__device__ __forceinline__ uint64_t make_wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;  // SWIZZLE_128B
  return d;
}

// ---------------------------------------------------------------- clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// shared::cluster address of `local_smem_addr` in CTA `cta` of this cluster
__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_smem_addr, uint32_t cta) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(cta));
  return r;
}
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t cta) {
  const uint32_t ra = mapa_u32(smem_u32(bar), cta);
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(ra) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  long long t0 = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) break;
    const long long now = clock64();
    if (t0 == 0) t0 = now;
    else if (now - t0 > 4000000000ll) { __trap(); }
  }
}
// TMA load whose tile lands at the same shared-memory offset of every CTA in `mask` (cluster multicast); each
// destination CTA's mbarrier at the same offset as `bar` receives complete_tx for the bytes delivered to it.
__device__ __forceinline__ void tma_load_2d_mcast(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                  uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], "
      "[%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}

// ---------------------------------------------------------------- NVSwitch multicast (NVLS) reductions
// `p` is an address inside a multicast mapping: the NVSwitch applies the add to the same offset of every
// peer's buffer.  Gradient producers use these instead of local atomics when the gradient buffer is symmetric,
// which turns "compute then all-reduce" into one kernel (the reduction rides on the producer's stores).
__device__ __forceinline__ void mc_red_add_f32(float* p, float v) {
  asm volatile("multimem.red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ void mc_red_add_v4_f32(float* p, float a, float b, float c, float d) {
  asm volatile("multimem.red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a), "f"(b), "f"(c),
               "f"(d)
               : "memory");
}
// ---------------------------------------------------------------- owner-sharded gradients over NVLink peer memory
// Reduce-scatter without a collective: the flat fp32 gradient buffer is a symmetric allocation (same layout on every
// rank, every peer's copy mapped into this process), rank r *owns* the flat range [bound[r], bound[r+1]) and runs the
// optimizer on it, and every gradient-producing kernel adds its contribution straight into the owner's copy with
// `red.global.add` on the peer mapping -- (N-1)/N of the bytes cross NVLink once, nothing is received that the rank
// does not own (multimem.red above delivers every contribution to all N ranks).  One table per translation unit
// (no -rdc): set through aitj_*_set_peers before the first launch, never changed while a CUDA graph that uses it lives.
struct PeerTable {
  const float* base;          // this rank's gradient buffer
  long long delta[8];         // bytes from a local address to the same offset in rank r's buffer (0 for this rank)
  long long bound[9];         // ownership bounds in elements, bound[0] = 0, bound[n] = total
  int n;
};
static __constant__ PeerTable c_peers;

__device__ __forceinline__ int peer_owner(const float* p) {
  const long long e = p - c_peers.base;
  int o = 0;
#pragma unroll
  for (int r = 1; r < 8; ++r) o += (r < c_peers.n && e >= c_peers.bound[r]) ? 1 : 0;
  return o;
}
__device__ __forceinline__ float* peer_ptr(float* p) {
  return reinterpret_cast<float*>(reinterpret_cast<char*>(p) + c_peers.delta[peer_owner(p)]);
}

// gradient accumulation modes of the kernels that produce gradients
enum : int { GRAD_LOCAL = 0, GRAD_MULTICAST = 1, GRAD_PEER = 2 };

__device__ __forceinline__ void red_add_v4_f32(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void grad_add_f32(float* p, float v, int mode) {
  if (mode == GRAD_MULTICAST) mc_red_add_f32(p, v);
  else if (mode == GRAD_PEER) atomicAdd(peer_ptr(p), v);
  else atomicAdd(p, v);
}
__device__ __forceinline__ void grad_add_v4_f32(float* p, float a, float b, float c, float d, int mode) {
  if (mode == GRAD_MULTICAST) mc_red_add_v4_f32(p, a, b, c, d);
  else red_add_v4_f32(mode == GRAD_PEER ? peer_ptr(p) : p, a, b, c, d);
}
// bf16 parameters leave the sharded optimizer through the NVSwitch multicast alias: one store, every rank's copy
__device__ __forceinline__ void mc_store_v2_b32(void* p, uint32_t a, uint32_t b) {
  asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(__uint_as_float(a)),
               "f"(__uint_as_float(b))
               : "memory");
}
__device__ __forceinline__ void mc_store_f32(float* p, float v) {
  asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// ---------------------------------------------------------------- misc math / packing
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
__device__ __forceinline__ float gelu_tanh(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  return 0.5f * x * (1.0f + t);
}
__device__ __forceinline__ float gelu_tanh_grad(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float x2 = x * x;
  float u = k0 * (x + k1 * x * x2);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  float du = k0 * (1.0f + 3.0f * k1 * x2);
  return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * du;
}
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace aitj

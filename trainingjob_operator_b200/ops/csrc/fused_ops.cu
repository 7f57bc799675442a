// Memory-bound fused kernels of the worker training step (sm_90a): LayerNorm fwd/bwd,
// embedding fwd/bwd, softmax-cross-entropy fwd+bwd in one pass, bias-grad column reduce,
// flat-buffer AdamW (fp32 master + bf16 compute copy + grad zeroing in one sweep),
// grad-norm, casts.  All 16-byte vectorised; one HBM read + one write per tensor.
// The reference operator ships no kernels (SURVEY.md §2.6); these serve the launched
// DDP workers that BASELINE.json's samples/sec metric measures.
#include <cstdlib>

#include "ptx.cuh"
#include <string.h>

namespace aitj {

// ------------------------------------------------------------------ LayerNorm forward
// One warp per row; V = C / 256 uint4 vectors per lane (C % 256 == 0).
template <int V>
__global__ void __launch_bounds__(256) layernorm_fwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                            const __nv_bfloat16* __restrict__ gamma,
                                                            const __nv_bfloat16* __restrict__ beta,
                                                            __nv_bfloat16* __restrict__ y, float* __restrict__ mean_out,
                                                            float* __restrict__ rstd_out, int M, float eps) {
  constexpr int C = V * 256;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  float g[V * 8], b[V * 8];
#pragma unroll
  for (int i = 0; i < V; ++i) {
    uint4 gu = *reinterpret_cast<const uint4*>(gamma + (i * 32 + lane) * 8);
    uint4 bu = *reinterpret_cast<const uint4*>(beta + (i * 32 + lane) * 8);
    const uint32_t gw[4] = {gu.x, gu.y, gu.z, gu.w}, bw[4] = {bu.x, bu.y, bu.z, bu.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 gf = unpack_bf16x2(gw[j]), bf = unpack_bf16x2(bw[j]);
      g[i * 8 + 2 * j] = gf.x; g[i * 8 + 2 * j + 1] = gf.y;
      b[i * 8 + 2 * j] = bf.x; b[i * 8 + 2 * j + 1] = bf.y;
    }
  }
  // persistent warps (2 blocks per SM), one row at a time with the NEXT row's loads already in flight: the kernel is a
  // pure stream, so bytes in flight per SM are what sets its bandwidth
  const int stride = gridDim.x * warps_per_block;
  int row = blockIdx.x * warps_per_block + warp;
  uint4 nxt[V];
  if (row < M) {
#pragma unroll
    for (int i = 0; i < V; ++i) nxt[i] = *reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * C + (i * 32 + lane) * 8);
  }
  for (; row < M; row += stride) {
    uint4 cur[V];
#pragma unroll
    for (int i = 0; i < V; ++i) cur[i] = nxt[i];
    if (row + stride < M) {
#pragma unroll
      for (int i = 0; i < V; ++i)
        nxt[i] = *reinterpret_cast<const uint4*>(x + static_cast<size_t>(row + stride) * C + (i * 32 + lane) * 8);
    }
    float v[V * 8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const uint4 u = cur[i];
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 f = unpack_bf16x2(w[j]);
        v[i * 8 + 2 * j] = f.x; v[i * 8 + 2 * j + 1] = f.y;
        s += f.x + f.y;
      }
    }
    const float mean = warp_sum(s) * (1.0f / C);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V * 8; ++i) { float d = v[i] - mean; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / C) + eps);
    __nv_bfloat16* yr = y + static_cast<size_t>(row) * C;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      uint4 o;
      uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float a0 = (v[i * 8 + 2 * j] - mean) * rstd * g[i * 8 + 2 * j] + b[i * 8 + 2 * j];
        float a1 = (v[i * 8 + 2 * j + 1] - mean) * rstd * g[i * 8 + 2 * j + 1] + b[i * 8 + 2 * j + 1];
        ow[j] = pack_bf16x2(a0, a1);
      }
      *reinterpret_cast<uint4*>(yr + (i * 32 + lane) * 8) = o;
    }
    if (lane == 0) { mean_out[row] = mean; rstd_out[row] = rstd; }
  }
}

// Block reduction of one per-thread partial (V*8 columns per lane) to one atomic per column: the upper half of
// the warps hand their partials to the lower half through shared memory, which then publish the partial sums.
constexpr int kLnBwdWarps = 12;
template <int V>
__device__ __forceinline__ void ln_bwd_block_reduce(const float (&acc)[V * 8], float (*red)[V * 256], float* dst, int warp,
                                                    int lane, int mc) {
  constexpr int C = V * 256;
  constexpr int H = kLnBwdWarps / 2;
  __syncthreads();
  if (warp >= H) {
#pragma unroll
    for (int i = 0; i < V; ++i) {
      float* d = &red[warp - H][(i * 32 + lane) * 8];
      *reinterpret_cast<float4*>(d) = make_float4(acc[i * 8], acc[i * 8 + 1], acc[i * 8 + 2], acc[i * 8 + 3]);
      *reinterpret_cast<float4*>(d + 4) = make_float4(acc[i * 8 + 4], acc[i * 8 + 5], acc[i * 8 + 6], acc[i * 8 + 7]);
    }
  }
  __syncthreads();
  if (warp < H) {
#pragma unroll
    for (int i = 0; i < V; ++i) {
      float* d = &red[warp][(i * 32 + lane) * 8];
      const float4 p0 = *reinterpret_cast<const float4*>(d), p1 = *reinterpret_cast<const float4*>(d + 4);
      *reinterpret_cast<float4*>(d) = make_float4(acc[i * 8] + p0.x, acc[i * 8 + 1] + p0.y, acc[i * 8 + 2] + p0.z,
                                                  acc[i * 8 + 3] + p0.w);
      *reinterpret_cast<float4*>(d + 4) = make_float4(acc[i * 8 + 4] + p1.x, acc[i * 8 + 5] + p1.y,
                                                      acc[i * 8 + 6] + p1.z, acc[i * 8 + 7] + p1.w);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < H; ++w) t += red[w][c];
    grad_add_f32(dst + c, t, mc);
  }
}

// ------------------------------------------------------------------ LayerNorm backward
// dx (bf16), dgamma/dbeta accumulated (fp32 atomics) into flat grad buffer. If `dres` != null
// the incoming residual-stream gradient is added to dx (fuses the residual branch add).
template <int V>
__global__ void __launch_bounds__(kLnBwdWarps * 32, 1) layernorm_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                               const __nv_bfloat16* __restrict__ x,
                                                               const __nv_bfloat16* __restrict__ gamma,
                                                               const float* __restrict__ mean_in,
                                                               const float* __restrict__ rstd_in,
                                                               const __nv_bfloat16* __restrict__ dres,
                                                               __nv_bfloat16* __restrict__ dx, float* __restrict__ dgamma,
                                                               float* __restrict__ dbeta, float* __restrict__ dxsum,
                                                               int M, int mc) {
  // dxsum (optional, fp32[C]) += column sums of dx: dx is the gradient of the tensor that fed this LayerNorm,
  // i.e. of "linear output + bias + residual", so its column sum IS that linear's bias gradient -- for free.
  //
  // One warp per row, 12 warps per SM.  The kernel is a pure HBM stream (3 reads + 1 write per element), so what
  // matters is bytes in flight: per-thread state is kept under 168 registers (x / dy / dres stay packed bf16, gamma
  // lives in shared memory) so that 12 warps fit, and all three inputs of a row are requested before any math.
  constexpr int C = V * 256;
  __shared__ float red[kLnBwdWarps / 2][C];
  __shared__ float sgamma[C];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  for (int c = threadIdx.x; c < C; c += blockDim.x) sgamma[c] = __bfloat162float(gamma[c]);
  __syncthreads();
  float dg[V * 8], db[V * 8], ds[V * 8];
#pragma unroll
  for (int i = 0; i < V * 8; ++i) { dg[i] = 0.f; db[i] = 0.f; ds[i] = 0.f; }
  const bool has_res = dres != nullptr;

  for (int row = blockIdx.x * warps_per_block + warp; row < M; row += gridDim.x * warps_per_block) {
    const size_t base = static_cast<size_t>(row) * C;
    uint4 xu[V], du[V], ru[V];
#pragma unroll
    for (int i = 0; i < V; ++i) {
      xu[i] = *reinterpret_cast<const uint4*>(x + base + (i * 32 + lane) * 8);
      du[i] = *reinterpret_cast<const uint4*>(dy + base + (i * 32 + lane) * 8);
    }
#pragma unroll
    for (int i = 0; i < V; ++i)
      ru[i] = has_res ? *reinterpret_cast<const uint4*>(dres + base + (i * 32 + lane) * 8) : make_uint4(0, 0, 0, 0);
    const float mean = mean_in[row], rstd = rstd_in[row];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const uint32_t xw[4] = {xu[i].x, xu[i].y, xu[i].z, xu[i].w}, dw[4] = {du[i].x, du[i].y, du[i].z, du[i].w};
      const float4 g0 = *reinterpret_cast<const float4*>(sgamma + (i * 32 + lane) * 8);
      const float4 g1 = *reinterpret_cast<const float4*>(sgamma + (i * 32 + lane) * 8 + 4);
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 xf = unpack_bf16x2(xw[j]), df = unpack_bf16x2(dw[j]);
        const int k = i * 8 + 2 * j;
        const float h0 = (xf.x - mean) * rstd, h1 = (xf.y - mean) * rstd;
        dg[k] += df.x * h0; dg[k + 1] += df.y * h1;
        db[k] += df.x; db[k + 1] += df.y;
        const float a0 = df.x * gg[2 * j], a1 = df.y * gg[2 * j + 1];
        s1 += a0 + a1;
        s2 += a0 * h0 + a1 * h1;
      }
    }
    s1 = warp_sum(s1) * (1.0f / C);
    s2 = warp_sum(s2) * (1.0f / C);
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const uint32_t xw[4] = {xu[i].x, xu[i].y, xu[i].z, xu[i].w}, dw[4] = {du[i].x, du[i].y, du[i].z, du[i].w};
      const uint32_t rw[4] = {ru[i].x, ru[i].y, ru[i].z, ru[i].w};
      const float4 g0 = *reinterpret_cast<const float4*>(sgamma + (i * 32 + lane) * 8);
      const float4 g1 = *reinterpret_cast<const float4*>(sgamma + (i * 32 + lane) * 8 + 4);
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      uint4 o;
      uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 xf = unpack_bf16x2(xw[j]), df = unpack_bf16x2(dw[j]), rf = unpack_bf16x2(rw[j]);
        const int k = i * 8 + 2 * j;
        const float h0 = (xf.x - mean) * rstd, h1 = (xf.y - mean) * rstd;
        const float a0 = rstd * (df.x * gg[2 * j] - s1 - h0 * s2) + rf.x;
        const float a1 = rstd * (df.y * gg[2 * j + 1] - s1 - h1 * s2) + rf.y;
        ds[k] += a0; ds[k + 1] += a1;
        ow[j] = pack_bf16x2(a0, a1);
      }
      *reinterpret_cast<uint4*>(dx + base + (i * 32 + lane) * 8) = o;
    }
  }
  ln_bwd_block_reduce<V>(dg, red, dgamma, warp, lane, mc);
  ln_bwd_block_reduce<V>(db, red, dbeta, warp, lane, mc);
  if (dxsum != nullptr) ln_bwd_block_reduce<V>(ds, red, dxsum, warp, lane, mc);
}

// ------------------------------------------------------------------ embedding
__global__ void __launch_bounds__(256) embedding_fwd_kernel(const int64_t* __restrict__ tok,
                                                            const __nv_bfloat16* __restrict__ wte,
                                                            const __nv_bfloat16* __restrict__ wpe,
                                                            __nv_bfloat16* __restrict__ out, int M, int T, int C,
                                                            const int64_t* __restrict__ typ = nullptr,
                                                            const __nv_bfloat16* __restrict__ wtt = nullptr) {
  const int vec_per_row = C / 8;
  const size_t total = static_cast<size_t>(M) * vec_per_row;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(i / vec_per_row), c = static_cast<int>(i % vec_per_row) * 8;
    const int64_t t = tok[m];
    uint4 a = *reinterpret_cast<const uint4*>(wte + t * C + c);
    uint4 b = wpe ? *reinterpret_cast<const uint4*>(wpe + static_cast<size_t>(m % T) * C + c) : make_uint4(0, 0, 0, 0);
    // optional third table (BERT's token-type / segment embeddings)
    uint4 d = wtt ? *reinterpret_cast<const uint4*>(wtt + typ[m] * C + c) : make_uint4(0, 0, 0, 0);
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w}, dw[4] = {d.x, d.y, d.z, d.w};
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 fa = unpack_bf16x2(aw[j]), fb = unpack_bf16x2(bw[j]), fd = unpack_bf16x2(dw[j]);
      ow[j] = pack_bf16x2(fa.x + fb.x + fd.x, fa.y + fb.y + fd.y);
    }
    *reinterpret_cast<uint4*>(out + static_cast<size_t>(m) * C + c) = o;
  }
}

__global__ void __launch_bounds__(256) embedding_bwd_kernel(const int64_t* __restrict__ tok,
                                                            const __nv_bfloat16* __restrict__ dx,
                                                            float* __restrict__ dwte, float* __restrict__ dwpe, int M,
                                                            int T, int C, int mc,
                                                            const int64_t* __restrict__ typ = nullptr,
                                                            float* __restrict__ dwtt = nullptr) {
  const int vec_per_row = C / 4;
  const size_t total = static_cast<size_t>(M) * vec_per_row;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(i / vec_per_row), c = static_cast<int>(i % vec_per_row) * 4;
    uint2 u = *reinterpret_cast<const uint2*>(dx + static_cast<size_t>(m) * C + c);
    float2 f0 = unpack_bf16x2(u.x), f1 = unpack_bf16x2(u.y);
    grad_add_v4_f32(dwte + tok[m] * C + c, f0.x, f0.y, f1.x, f1.y, mc);
    if (dwpe) grad_add_v4_f32(dwpe + static_cast<size_t>(m % T) * C + c, f0.x, f0.y, f1.x, f1.y, mc);
    if (dwtt) grad_add_v4_f32(dwtt + typ[m] * C + c, f0.x, f0.y, f1.x, f1.y, mc);
  }
}

// ------------------------------------------------------------------ softmax cross-entropy fwd+bwd
// One block per row. The row (bf16, Vp padded columns, V real) is staged in smem once; the
// kernel writes the per-row loss and overwrites the logits with dlogits = (p - onehot) * gscale.
__global__ void __launch_bounds__(512, 2) softmax_xent_kernel(__nv_bfloat16* __restrict__ logits,
                                                              const int64_t* __restrict__ target,
                                                              float* __restrict__ loss, int V, int Vp, float gscale) {
  // Row staged once in shared memory (2 CTAs / SM so one row loads while the other computes); exp(x - max)
  // overwrites the staged row (bf16), so each element costs one exp and the gradient pass is a scale.
  extern __shared__ uint4 srow4[];
  __shared__ float sred[16];
  __shared__ float sbcast[2];
  const int row = blockIdx.x;
  __nv_bfloat16* g = logits + static_cast<size_t>(row) * Vp;
  const int nvec = Vp / 8, nfull = V / 8;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int tgt = static_cast<int>(target[row]);
  const bool valid = tgt >= 0 && tgt < V;
  const float xt = valid ? __bfloat162float(g[tgt]) : 0.f;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    uint4 u = *reinterpret_cast<const uint4*>(g + i * 8);
    srow4[i] = u;
    float f[8];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) { float2 t = unpack_bf16x2(w[j]); f[2 * j] = t.x; f[2 * j + 1] = t.y; }
    if (i < nfull) {
#pragma unroll
      for (int j = 0; j < 8; ++j) mx = fmaxf(mx, f[j]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) if (i * 8 + j < V) mx = fmaxf(mx, f[j]);
    }
  }
  mx = warp_max(mx);
  if (lane == 0) sred[warp] = mx;
  __syncthreads();
  if (warp == 0) {
    float t = lane < nwarps ? sred[lane] : -INFINITY;
    t = warp_max(t);
    if (lane == 0) sbcast[0] = t;
  }
  __syncthreads();
  mx = sbcast[0];
  const float LOG2E = 1.4426950408889634f;
  const float moff = mx * LOG2E;
  float sum = 0.f;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    uint4 u = srow4[i];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float e[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 t = unpack_bf16x2(w[j]);
      e[2 * j] = exp2f(fmaf(t.x, LOG2E, -moff));
      e[2 * j + 1] = exp2f(fmaf(t.y, LOG2E, -moff));
    }
    if (i >= nfull) {
#pragma unroll
      for (int j = 0; j < 8; ++j) if (i * 8 + j >= V) e[j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) sum += e[j];
    srow4[i] = make_uint4(pack_bf16x2(e[0], e[1]), pack_bf16x2(e[2], e[3]), pack_bf16x2(e[4], e[5]),
                          pack_bf16x2(e[6], e[7]));
  }
  sum = warp_sum(sum);
  __syncthreads();
  if (lane == 0) sred[warp] = sum;
  __syncthreads();
  if (warp == 0) {
    float t = lane < nwarps ? sred[lane] : 0.f;
    t = warp_sum(t);
    if (lane == 0) sbcast[1] = t;
  }
  __syncthreads();
  sum = sbcast[1];
  if (threadIdx.x == 0) loss[row] = valid ? -(xt - mx - logf(sum)) : 0.f;
  const float inv = valid ? gscale / sum : 0.f;
  const float gs = valid ? gscale : 0.f;
  const int tvec = valid ? (tgt >> 3) : -1;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    uint4 u = srow4[i];
    const uint32_t e[4] = {u.x, u.y, u.z, u.w};
    float p[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) { float2 t = unpack_bf16x2(e[j]); p[2 * j] = t.x * inv; p[2 * j + 1] = t.y * inv; }
    if (i == tvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) if (j == (tgt & 7)) p[j] -= gs;
    }
    *reinterpret_cast<uint4*>(g + i * 8) = make_uint4(pack_bf16x2(p[0], p[1]), pack_bf16x2(p[2], p[3]),
                                                      pack_bf16x2(p[4], p[5]), pack_bf16x2(p[6], p[7]));
  }
}

// ------------------------------------------------------------------ cross-entropy from the GEMM's partials (evaluation)
// One warp per row: merge the row's (max, sum of exp) pairs of the EPI_XENT GEMM into its log-sum-exp, loss[row] =
// lse - tgt_logit[row] (0 for a negative target).  acc[0] += the block's sum of losses, acc[1] += its rows with a target,
// in fp64 with one atomic each per block, so micro-batches accumulate on the device without a host synchronisation.
constexpr int kXentWarps = 8;

__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
  if (s2 == 0.f) return;                       // (-inf, 0): a block wholly past the vocabulary
  if (s == 0.f) { m = m2; s = s2; return; }
  const float mn = fmaxf(m, m2);
  s = s * __expf(m - mn) + s2 * __expf(m2 - mn);
  m = mn;
}

__global__ void __launch_bounds__(kXentWarps * 32) xent_finish_kernel(const float2* __restrict__ part,
                                                                      const float* __restrict__ tgt_logit,
                                                                      const int64_t* __restrict__ target,
                                                                      float* __restrict__ loss, double* __restrict__ acc,
                                                                      int M, int nblk) {
  __shared__ double red[kXentWarps][2];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double wsum = 0.0, wcount = 0.0;              // lane 0's running totals of this warp's rows
  for (int row = blockIdx.x * kXentWarps + warp; row < M; row += gridDim.x * kXentWarps) {
    if (target[row] < 0) {
      if (lane == 0) loss[row] = 0.f;
      continue;
    }
    float m = -INFINITY, s = 0.f;
    for (int b = lane; b < nblk; b += 32) {
      const float2 p = part[static_cast<size_t>(row) * nblk + b];
      lse_merge(m, s, p.x, p.y);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
      lse_merge(m, s, m2, s2);
    }
    if (lane == 0) {
      const float l = m + logf(s) - tgt_logit[row];
      loss[row] = l;
      wsum += l;
      wcount += 1.0;
    }
  }
  if (lane == 0) { red[warp][0] = wsum; red[warp][1] = wcount; }
  __syncthreads();
  if (threadIdx.x < 2) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kXentWarps; ++w) t += red[w][threadIdx.x];
    if (t != 0.0) atomicAdd(acc + threadIdx.x, t);
  }
}

// ------------------------------------------------------------------ bias grad: db[N] += colsum(dy[M,N])
__global__ void __launch_bounds__(256) colsum_kernel(const __nv_bfloat16* __restrict__ dy, float* __restrict__ db,
                                                     int M, int N, int rows_per_block, int mc) {
  // block = 32 column-groups(8 cols each => 256 cols) x 8 row lanes
  __shared__ float red[8][256];
  const int cg = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int col0 = blockIdx.x * 256 + cg * 8;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(M, r0 + rows_per_block);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (col0 < N) {
    for (int r = r0 + rl; r < r1; r += 8) {
      uint4 u = *reinterpret_cast<const uint4*>(dy + static_cast<size_t>(r) * N + col0);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 f = unpack_bf16x2(w[j]);
        acc[2 * j] += f.x; acc[2 * j + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[rl][cg * 8 + j] = acc[j];
  __syncthreads();
  const int c = threadIdx.x;
  if (blockIdx.x * 256 + c < N) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][c];
    grad_add_f32(db + blockIdx.x * 256 + c, s, mc);
  }
}

// ------------------------------------------------------------------ attention backward epilogue:
// d_qkv[M, 3C] <- {dq, dk, dv} (each [B,H,T,D] with arbitrary B/H/T strides), fused with the qkv bias gradient
// db[3C] += colsum(d_qkv): one pass over the data instead of three strided copies and a column reduction.
struct QkvSrc {
  const __nv_bfloat16* p[3];
  long long sB[3], sH[3], sT[3];
};

__global__ void __launch_bounds__(256) qkv_gather_colsum_kernel(QkvSrc src, __nv_bfloat16* __restrict__ out,
                                                                float* __restrict__ db, int M, int T, int C, int D,
                                                                int rows_per_block, int mc) {
  __shared__ float red[8][256];
  const int N = 3 * C;
  const int cg = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int col0 = blockIdx.x * 256 + cg * 8;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(M, r0 + rows_per_block);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (col0 < N) {
    const int sel = col0 / C, within = col0 - sel * C;
    const int h = within / D, d = within - h * D;
    const __nv_bfloat16* base = src.p[sel] + h * src.sH[sel] + d;
    const long long sB = src.sB[sel], sT = src.sT[sel];
    int r = r0 + rl;
    // two rows in flight per thread
    for (; r + 8 < r1; r += 16) {
      const int b0 = r / T, t0 = r - b0 * T, b1 = (r + 8) / T, t1 = (r + 8) - b1 * T;
      const uint4 u0 = *reinterpret_cast<const uint4*>(base + b0 * sB + t0 * sT);
      const uint4 u1 = *reinterpret_cast<const uint4*>(base + b1 * sB + t1 * sT);
      *reinterpret_cast<uint4*>(out + static_cast<size_t>(r) * N + col0) = u0;
      *reinterpret_cast<uint4*>(out + static_cast<size_t>(r + 8) * N + col0) = u1;
      const uint32_t w[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float2 f = unpack_bf16x2(w[j]);
        acc[2 * (j & 3)] += f.x; acc[2 * (j & 3) + 1] += f.y;
      }
    }
    for (; r < r1; r += 8) {
      const int b0 = r / T, t0 = r - b0 * T;
      const uint4 u0 = *reinterpret_cast<const uint4*>(base + b0 * sB + t0 * sT);
      *reinterpret_cast<uint4*>(out + static_cast<size_t>(r) * N + col0) = u0;
      const uint32_t w[4] = {u0.x, u0.y, u0.z, u0.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 f = unpack_bf16x2(w[j]);
        acc[2 * j] += f.x; acc[2 * j + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[rl][cg * 8 + j] = acc[j];
  __syncthreads();
  const int c = threadIdx.x;
  if (blockIdx.x * 256 + c < N) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][c];
    grad_add_f32(db + blockIdx.x * 256 + c, s, mc);
  }
}

// ------------------------------------------------------------------ grad norm (sum of squares)
__global__ void __launch_bounds__(512) sumsq_kernel(const float* __restrict__ g, size_t n, float* __restrict__ out) {
  __shared__ float sred[16];
  float s = 0.f;
  const size_t nvec = n / 4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float4 v = reinterpret_cast<const float4*>(g)[i];
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? sred[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) atomicAdd(out, t);
  }
}

// ------------------------------------------------------------------ AdamW over a flat buffer
// p,m,v fp32 master state; g fp32 grads (zeroed on the way out when zero_grad != 0);
// p16 bf16 compute copy refreshed in the same sweep. wd_mask[i / 256] selects weight decay.
// sumsq (device scalar, may be null) drives global-norm clipping without a host sync.
struct AdamArgs {
  float lr, beta1, beta2, eps, weight_decay, bc1, bc2, max_norm, grad_div;
  int zero_grad, sumsq_n, p16_mc;
};
__global__ void __launch_bounds__(256) adamw_kernel(float* __restrict__ p, float* __restrict__ g,
                                                    float* __restrict__ m, float* __restrict__ v,
                                                    __nv_bfloat16* __restrict__ p16,
                                                    const uint8_t* __restrict__ wd_mask,
                                                    const float* __restrict__ sumsq,
                                                    const float* __restrict__ dyn, size_t n, AdamArgs a) {
  // a.sumsq_n partial sums of squares (one per rank's shard in the owner-sharded mode; summed in rank order, so every
  // rank computes the identical clip factor); a.p16_mc: `p16` is an NVSwitch multicast address -- the refreshed bf16
  // parameters of this shard are stored into every rank's copy (sharded optimizer + all-gather in one sweep)
  // dyn (device, optional) = {lr, bias_correction1, bias_correction2}: lets a captured CUDA graph replay
  // with a per-step learning rate / step count without re-capturing.
  if (dyn != nullptr) { a.lr = dyn[0]; a.bc1 = dyn[1]; a.bc2 = dyn[2]; }
  float clip = 1.0f;
  if (sumsq != nullptr && a.max_norm > 0.f) {
    float total = 0.f;
    for (int i = 0; i < a.sumsq_n; ++i) total += sumsq[i];
    const float norm = sqrtf(total) / a.grad_div;
    if (norm > a.max_norm) clip = a.max_norm / (norm + 1e-6f);
  }
  const float gmul = clip / a.grad_div;
  const size_t nvec = n / 4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float4 pv = reinterpret_cast<float4*>(p)[i];
    float4 gv = reinterpret_cast<float4*>(g)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    const float wd = wd_mask[(i * 4) >> 8] ? a.weight_decay : 0.f;
    float* pp = reinterpret_cast<float*>(&pv);
    float* gg = reinterpret_cast<float*>(&gv);
    float* mm = reinterpret_cast<float*>(&mv);
    float* vq = reinterpret_cast<float*>(&vv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gr = gg[j] * gmul;
      mm[j] = a.beta1 * mm[j] + (1.f - a.beta1) * gr;
      vq[j] = a.beta2 * vq[j] + (1.f - a.beta2) * gr * gr;
      const float mh = mm[j] / a.bc1, vh = vq[j] / a.bc2;
      pp[j] = pp[j] - a.lr * (mh / (sqrtf(vh) + a.eps) + wd * pp[j]);
    }
    reinterpret_cast<float4*>(p)[i] = pv;
    reinterpret_cast<float4*>(m)[i] = mv;
    reinterpret_cast<float4*>(v)[i] = vv;
    if (a.zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    uint2 o;
    o.x = pack_bf16x2(pp[0], pp[1]);
    o.y = pack_bf16x2(pp[2], pp[3]);
    if (a.p16_mc) mc_store_v2_b32(reinterpret_cast<uint2*>(p16) + i, o.x, o.y);
    else reinterpret_cast<uint2*>(p16)[i] = o;
  }
}

// Owner-sharded mode: the locally accumulated 1-D gradients (biases, LayerNorm; built from many scalar atomics) go to
// their owners in one sweep -- dst is the LOCAL address of the segment in the symmetric gradient buffer, each 16-byte
// piece is added into the copy of the rank that owns it; src is cleared.
__global__ void __launch_bounds__(256) peer_push_kernel(float* __restrict__ dst, float* __restrict__ src, size_t n) {
  const size_t nvec = n / 4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float4 v = reinterpret_cast<float4*>(src)[i];
    red_add_v4_f32(peer_ptr(dst + i * 4), v.x, v.y, v.z, v.w);
    reinterpret_cast<float4*>(src)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// This rank's partial sum of squared gradients goes into slot `rank` of every rank's `parts` array (multicast store).
__global__ void norm_share_kernel(float* __restrict__ parts_mc, const float* __restrict__ mine, int rank) {
  if (threadIdx.x == 0 && blockIdx.x == 0) mc_store_f32(parts_mc + rank, *mine);
}

// Push a locally accumulated fp32 gradient segment into every peer's buffer through the switch and clear it:
// dst_mc[i] (+)= src[i]; src[i] = 0.  Used for the small 1-D parameters (biases, LayerNorm) whose gradients are
// built from many scalar atomics that would be wasteful to send over NVLink one by one.
__global__ void __launch_bounds__(256) mc_push_kernel(float* __restrict__ dst_mc, float* __restrict__ src, size_t n) {
  const size_t nvec = n / 4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float4 v = reinterpret_cast<float4*>(src)[i];
    mc_red_add_v4_f32(dst_mc + i * 4, v.x, v.y, v.z, v.w);
    reinterpret_cast<float4*>(src)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

__global__ void __launch_bounds__(256) cast_f32_bf16_kernel(const float* __restrict__ in,
                                                            __nv_bfloat16* __restrict__ out, size_t n) {
  const size_t nvec = n / 4;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float4 v = reinterpret_cast<const float4*>(in)[i];
    uint2 o;
    o.x = pack_bf16x2(v.x, v.y);
    o.y = pack_bf16x2(v.z, v.w);
    reinterpret_cast<uint2*>(out)[i] = o;
  }
}

// GELU forward/backward as standalone kernels (used when the GEMM backend is the library path).
__global__ void __launch_bounds__(256) gelu_fwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                       __nv_bfloat16* __restrict__ y, size_t n) {
  const size_t nvec = n / 8;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    uint4 u = reinterpret_cast<const uint4*>(x)[i];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 f = unpack_bf16x2(w[j]);
      ow[j] = pack_bf16x2(gelu_tanh(f.x), gelu_tanh(f.y));
    }
    reinterpret_cast<uint4*>(y)[i] = o;
  }
}
__global__ void __launch_bounds__(256) gelu_bwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                       const __nv_bfloat16* __restrict__ dy,
                                                       __nv_bfloat16* __restrict__ dx, size_t n) {
  const size_t nvec = n / 8;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    uint4 u = reinterpret_cast<const uint4*>(x)[i];
    uint4 d = reinterpret_cast<const uint4*>(dy)[i];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w}, dw[4] = {d.x, d.y, d.z, d.w};
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 f = unpack_bf16x2(w[j]), g = unpack_bf16x2(dw[j]);
      ow[j] = pack_bf16x2(g.x * gelu_tanh_grad(f.x), g.y * gelu_tanh_grad(f.y));
    }
    reinterpret_cast<uint4*>(dx)[i] = o;
  }
}

// SM count of the current device: grids are capped at a few CTAs per SM and loop over the rest
static int sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

static int grid_for(size_t work_items, int threads, int max_blocks) {
  size_t b = (work_items + threads - 1) / threads;
  if (b > static_cast<size_t>(max_blocks)) b = max_blocks;
  if (b < 1) b = 1;
  return static_cast<int>(b);
}

}  // namespace aitj

extern "C" {
using namespace aitj;
#define S(p) reinterpret_cast<cudaStream_t>(p)
#define BF(p) reinterpret_cast<__nv_bfloat16*>(p)
#define CBF(p) reinterpret_cast<const __nv_bfloat16*>(p)
#define LAUNCH_OK() (cudaPeekAtLastError() == cudaSuccess ? 0 : -30)

int aitj_layernorm_fwd(const void* x, const void* gamma, const void* beta, void* y, void* mean, void* rstd, int M,
                       int C, float eps, void* stream) {
  if (C % 256 || C > 2048) return -1;
  const int blocks = min((M + 7) / 8, sms() * 2);
#define LN_F(V) layernorm_fwd_kernel<V><<<blocks, 256, 0, S(stream)>>>(CBF(x), CBF(gamma), CBF(beta), BF(y), \
    reinterpret_cast<float*>(mean), reinterpret_cast<float*>(rstd), M, eps)
  switch (C / 256) {
    case 1: LN_F(1); break; case 2: LN_F(2); break; case 3: LN_F(3); break; case 4: LN_F(4); break;
    case 6: LN_F(6); break; case 8: LN_F(8); break; default: return -1;
  }
#undef LN_F
  return LAUNCH_OK();
}

int aitj_layernorm_bwd(const void* dy, const void* x, const void* gamma, const void* mean, const void* rstd,
                       const void* dres, void* dx, void* dgamma, void* dbeta, void* dxsum, int M, int C, int mc,
                       void* stream) {
  if (C % 256 || C > 1024) return -1;
  const int blocks = min((M + kLnBwdWarps - 1) / kLnBwdWarps, sms());
#define LN_B(V) layernorm_bwd_kernel<V><<<blocks, kLnBwdWarps * 32, 0, S(stream)>>>(CBF(dy), CBF(x), CBF(gamma), \
    reinterpret_cast<const float*>(mean), reinterpret_cast<const float*>(rstd), CBF(dres), BF(dx), \
    reinterpret_cast<float*>(dgamma), reinterpret_cast<float*>(dbeta), reinterpret_cast<float*>(dxsum), M, mc)
  switch (C / 256) {
    case 1: LN_B(1); break; case 2: LN_B(2); break; case 3: LN_B(3); break; case 4: LN_B(4); break;
    default: return -1;
  }
#undef LN_B
  return LAUNCH_OK();
}

int aitj_embedding_fwd(const void* tok, const void* wte, const void* wpe, void* out, int M, int T, int C,
                       void* stream) {
  if (C % 8) return -1;
  const size_t total = static_cast<size_t>(M) * (C / 8);
  embedding_fwd_kernel<<<grid_for(total, 256, sms() * 16), 256, 0, S(stream)>>>(
      reinterpret_cast<const int64_t*>(tok), CBF(wte), CBF(wpe), BF(out), M, T, C);
  return LAUNCH_OK();
}

int aitj_embedding_bwd(const void* tok, const void* dx, void* dwte, void* dwpe, int M, int T, int C, int mc,
                       void* stream) {
  if (C % 4) return -1;
  const size_t total = static_cast<size_t>(M) * (C / 4);
  embedding_bwd_kernel<<<grid_for(total, 256, sms() * 16), 256, 0, S(stream)>>>(
      reinterpret_cast<const int64_t*>(tok), CBF(dx), reinterpret_cast<float*>(dwte), reinterpret_cast<float*>(dwpe),
      M, T, C, mc);
  return LAUNCH_OK();
}

// embeddings with a third (token-type) table: out = wte[tok] + wpe[pos] + wtt[typ]
int aitj_embedding3_fwd(const void* tok, const void* typ, const void* wte, const void* wpe, const void* wtt, void* out,
                        int M, int T, int C, void* stream) {
  if (C % 8) return -1;
  const size_t total = static_cast<size_t>(M) * (C / 8);
  embedding_fwd_kernel<<<grid_for(total, 256, sms() * 16), 256, 0, S(stream)>>>(
      reinterpret_cast<const int64_t*>(tok), CBF(wte), CBF(wpe), BF(out), M, T, C,
      reinterpret_cast<const int64_t*>(typ), CBF(wtt));
  return LAUNCH_OK();
}

int aitj_embedding3_bwd(const void* tok, const void* typ, const void* dx, void* dwte, void* dwpe, void* dwtt, int M, int T,
                        int C, int mc, void* stream) {
  if (C % 4) return -1;
  const size_t total = static_cast<size_t>(M) * (C / 4);
  embedding_bwd_kernel<<<grid_for(total, 256, sms() * 16), 256, 0, S(stream)>>>(
      reinterpret_cast<const int64_t*>(tok), CBF(dx), reinterpret_cast<float*>(dwte), reinterpret_cast<float*>(dwpe),
      M, T, C, mc, reinterpret_cast<const int64_t*>(typ), reinterpret_cast<float*>(dwtt));
  return LAUNCH_OK();
}

int aitj_softmax_xent(void* logits, const void* target, void* loss, int M, int V, int Vp, float gscale,
                      void* stream) {
  if (Vp % 8 || V > Vp) return -1;
  // The row is staged in shared memory (100 KB at Vp = 50304, so two CTAs fit an SM's 228 KB): one HBM read and one
  // write per logit, and the second CTA's loads overlap the first one's exponentials.
  const int smem = Vp * 2;
  if (smem > 200 * 1024) return -2;
  static int configured = 0;
  if (configured < smem) {
    if (cudaFuncSetAttribute(softmax_xent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
      return -20;
    configured = smem;
  }
  softmax_xent_kernel<<<M, 512, smem, S(stream)>>>(BF(logits), reinterpret_cast<const int64_t*>(target),
                                                    reinterpret_cast<float*>(loss), V, Vp, gscale);
  return LAUNCH_OK();
}

// Finish the EPI_XENT GEMM's cross-entropy (see xent_finish_kernel): part float2 [M, nblk], tgt_logit fp32 [M], target
// int64 [M] -> loss fp32 [M]; acc fp64 [2] += (sum of losses, rows with a target).
int aitj_xent_finish(const void* part, const void* tgt_logit, const void* target, void* loss, void* acc, int M, int nblk,
                     void* stream) {
  if (M <= 0) return 0;
  if (nblk < 1) return -1;
  xent_finish_kernel<<<grid_for(M, kXentWarps, sms() * 8), kXentWarps * 32, 0, S(stream)>>>(
      reinterpret_cast<const float2*>(part), reinterpret_cast<const float*>(tgt_logit),
      reinterpret_cast<const int64_t*>(target), reinterpret_cast<float*>(loss), reinterpret_cast<double*>(acc), M, nblk);
  return LAUNCH_OK();
}

int aitj_colsum(const void* dy, void* db, int M, int N, int mc, void* stream) {
  if (N % 8) return -1;
  const int col_blocks = (N + 255) / 256;
  int rows_per_block = 512;
  while (rows_per_block > 32 && col_blocks * ((M + rows_per_block - 1) / rows_per_block) < sms() * 4) rows_per_block /= 2;
  dim3 grid(col_blocks, (M + rows_per_block - 1) / rows_per_block);
  colsum_kernel<<<grid, 256, 0, S(stream)>>>(CBF(dy), reinterpret_cast<float*>(db), M, N, rows_per_block, mc);
  return LAUNCH_OK();
}

int aitj_qkv_gather_colsum(const void* dq, const void* dk, const void* dv, const long long* strides, void* out,
                           void* db, int B, int T, int H, int D, int mc, void* stream) {
  // strides: 9 element strides {dq.sB, dq.sH, dq.sT, dk.., dv..}; the D stride must be 1
  if (D % 8) return -1;
  QkvSrc src;
  src.p[0] = CBF(dq); src.p[1] = CBF(dk); src.p[2] = CBF(dv);
  for (int i = 0; i < 3; ++i) { src.sB[i] = strides[3 * i]; src.sH[i] = strides[3 * i + 1]; src.sT[i] = strides[3 * i + 2]; }
  const int M = B * T, C = H * D, N = 3 * C;
  const int col_blocks = (N + 255) / 256;
  int rows_per_block = 512;
  while (rows_per_block > 32 && col_blocks * ((M + rows_per_block - 1) / rows_per_block) < sms() * 4) rows_per_block /= 2;
  dim3 grid(col_blocks, (M + rows_per_block - 1) / rows_per_block);
  qkv_gather_colsum_kernel<<<grid, 256, 0, S(stream)>>>(src, BF(out), reinterpret_cast<float*>(db), M, T, C, D,
                                                         rows_per_block, mc);
  return LAUNCH_OK();
}

int aitj_sumsq(const void* g, long long n, void* out, void* stream) {
  if (n % 4) return -1;
  sumsq_kernel<<<grid_for(static_cast<size_t>(n) / 4, 512, sms() * 4), 512, 0, S(stream)>>>(
      reinterpret_cast<const float*>(g), static_cast<size_t>(n), reinterpret_cast<float*>(out));
  return LAUNCH_OK();
}

static int g_adam_sumsq_n = 1, g_adam_p16_mc = 0;   // consumed by the next aitj_adamw call
int aitj_adamw_set_shard(int sumsq_n, int p16_mc) { g_adam_sumsq_n = sumsq_n; g_adam_p16_mc = p16_mc; return 0; }

int aitj_fused_set_peers(const void* base, const long long* delta, const long long* bound, int n) {
  if (n < 1 || n > 8) return -1;
  PeerTable t;
  memset(&t, 0, sizeof(t));
  t.base = reinterpret_cast<const float*>(base);
  for (int i = 0; i < n; ++i) t.delta[i] = delta[i];
  for (int i = 0; i <= n; ++i) t.bound[i] = bound[i];
  t.n = n;
  return cudaMemcpyToSymbol(c_peers, &t, sizeof(t)) == cudaSuccess ? 0 : -2;
}

int aitj_peer_push(void* dst_local, void* src, long long n, void* stream) {
  if (n % 4) return -1;
  peer_push_kernel<<<grid_for(static_cast<size_t>(n) / 4, 256, sms() * 2), 256, 0, S(stream)>>>(
      reinterpret_cast<float*>(dst_local), reinterpret_cast<float*>(src), static_cast<size_t>(n));
  return LAUNCH_OK();
}

int aitj_norm_share(void* parts_mc, const void* mine, int rank, void* stream) {
  norm_share_kernel<<<1, 32, 0, S(stream)>>>(reinterpret_cast<float*>(parts_mc), reinterpret_cast<const float*>(mine),
                                             rank);
  return LAUNCH_OK();
}

int aitj_adamw(void* p, void* g, void* m, void* v, void* p16, const void* wd_mask, const void* sumsq,
               const void* dyn, long long n, float lr, float beta1, float beta2, float eps, float weight_decay, int step, float max_norm,
               float grad_div, int zero_grad, void* stream) {
  AdamArgs a;
  a.sumsq_n = g_adam_sumsq_n; a.p16_mc = g_adam_p16_mc;
  g_adam_sumsq_n = 1; g_adam_p16_mc = 0;   // taken before the refusal: a refused sweep does not pass them on
  if (n % 256) return -1;
  a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.weight_decay = weight_decay;
  a.bc1 = 1.0f - powf(beta1, static_cast<float>(step));
  a.bc2 = 1.0f - powf(beta2, static_cast<float>(step));
  a.max_norm = max_norm; a.grad_div = grad_div; a.zero_grad = zero_grad;
  adamw_kernel<<<grid_for(static_cast<size_t>(n) / 4, 256, sms() * 8), 256, 0, S(stream)>>>(
      reinterpret_cast<float*>(p), reinterpret_cast<float*>(g), reinterpret_cast<float*>(m),
      reinterpret_cast<float*>(v), BF(p16), reinterpret_cast<const uint8_t*>(wd_mask),
      reinterpret_cast<const float*>(sumsq), reinterpret_cast<const float*>(dyn), static_cast<size_t>(n), a);
  return LAUNCH_OK();
}

int aitj_mc_push(void* dst_mc, void* src, long long n, void* stream) {
  if (n % 4) return -1;
  mc_push_kernel<<<grid_for(static_cast<size_t>(n) / 4, 256, sms() * 2), 256, 0, S(stream)>>>(
      reinterpret_cast<float*>(dst_mc), reinterpret_cast<float*>(src), static_cast<size_t>(n));
  return LAUNCH_OK();
}

int aitj_cast_f32_bf16(const void* in, void* out, long long n, void* stream) {
  if (n % 4) return -1;
  cast_f32_bf16_kernel<<<grid_for(static_cast<size_t>(n) / 4, 256, sms() * 8), 256, 0, S(stream)>>>(
      reinterpret_cast<const float*>(in), BF(out), static_cast<size_t>(n));
  return LAUNCH_OK();
}

int aitj_gelu_fwd(const void* x, void* y, long long n, void* stream) {
  if (n % 8) return -1;
  gelu_fwd_kernel<<<grid_for(static_cast<size_t>(n) / 8, 256, sms() * 8), 256, 0, S(stream)>>>(CBF(x), BF(y),
                                                                                             static_cast<size_t>(n));
  return LAUNCH_OK();
}
int aitj_gelu_bwd(const void* x, const void* dy, void* dx, long long n, void* stream) {
  if (n % 8) return -1;
  gelu_bwd_kernel<<<grid_for(static_cast<size_t>(n) / 8, 256, sms() * 8), 256, 0, S(stream)>>>(
      CBF(x), CBF(dy), BF(dx), static_cast<size_t>(n));
  return LAUNCH_OK();
}
}  // extern "C"

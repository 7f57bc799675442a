// LayerNorm forward and backward for rows of any width C that is a multiple of 8, up to 2048 (sm_90a): the widths of
// GPT-2 large (1280) and XL (1600), which the fused_ops.cu pair does not serve (it needs C % 256 == 0, and its backward
// keeps every lane's dgamma / dbeta / dxsum partials in registers, which spills from C = 1024 on).
//
// One warp per row; lane `l` owns the 8-column vectors j = i * 32 + l (i < V = ceil(C / 256)), so only the last i is
// partial.  Every input is read from HBM once and every output written once.  Row-independent per-column values --
// gamma, beta, and the backward's per-column partial sums -- live in shared memory as float4 pairs: the 8 columns of
// vector i * 32 + l are slots (2i) * 32 + l and (2i + 1) * 32 + l, so a warp's float4 accesses cover 512 contiguous
// bytes and never conflict on a bank.
#include "ptx.cuh"

namespace aitj {
namespace lnw {

constexpr int kMaxC = 2048;
constexpr int kFwdWarps = 8;   // 2 blocks per SM
constexpr int kBwdWarps = 8;   // 1 block per SM: its shared memory holds 3 partial rows per warp

__device__ __forceinline__ int slot(int i, int half, int lane) { return (2 * i + half) * 32 + lane; }
// first column of float4 slot s
__device__ __forceinline__ int slot_col(int s) { return ((s >> 6) * 32 + (s & 31)) * 8 + ((s >> 5) & 1) * 4; }

template <int V>
__device__ __forceinline__ void load_row(uint4 (&r)[V], const __nv_bfloat16* __restrict__ p, int nvec, int lane) {
#pragma unroll
  for (int i = 0; i < V; ++i)
    r[i] = (i * 32 + lane < nvec) ? *reinterpret_cast<const uint4*>(p + (i * 32 + lane) * 8) : make_uint4(0, 0, 0, 0);
}

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 t = unpack_bf16x2(w[j]);
    f[2 * j] = t.x; f[2 * j + 1] = t.y;
  }
}

// A bf16 vector of the C columns into float4 slots (zeros past C).
template <int V>
__device__ void stage_param(float4* dst, const __nv_bfloat16* __restrict__ src, int nvec) {
  for (int s = threadIdx.x; s < 2 * V * 32; s += blockDim.x) {
    const int c = slot_col(s);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < nvec * 8) {
      const uint2 u = *reinterpret_cast<const uint2*>(src + c);
      const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
      v = make_float4(a.x, a.y, b.x, b.y);
    }
    dst[s] = v;
  }
}

// ------------------------------------------------------------------ forward
// y = (x - mean) * rstd * gamma + beta; mean / rstd (fp32, per row) are kept for the backward.  Persistent warps with
// the next row's loads in flight while the current one is normalised, as in fused_ops.cu; x stays packed bf16 in
// registers and is unpacked on each of the three passes.
template <int V>
__global__ void __launch_bounds__(kFwdWarps * 32, 2) layernorm_wide_fwd_kernel(
    const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ gamma, const __nv_bfloat16* __restrict__ beta,
    __nv_bfloat16* __restrict__ y, float* __restrict__ mean_out, float* __restrict__ rstd_out, int M, int C, float eps) {
  __shared__ float4 sg[2 * V * 32], sb[2 * V * 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = C / 8;
  stage_param<V>(sg, gamma, nvec);
  stage_param<V>(sb, beta, nvec);
  __syncthreads();
  const float inv_c = 1.0f / C;
  const int stride = gridDim.x * kFwdWarps;
  int row = blockIdx.x * kFwdWarps + warp;
  uint4 nxt[V];
  if (row < M) load_row<V>(nxt, x + static_cast<size_t>(row) * C, nvec, lane);
  for (; row < M; row += stride) {
    uint4 cur[V];
#pragma unroll
    for (int i = 0; i < V; ++i) cur[i] = nxt[i];
    if (row + stride < M) load_row<V>(nxt, x + static_cast<size_t>(row + stride) * C, nvec, lane);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      float f[8];
      unpack8(cur[i], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += f[j];
    }
    const float mean = warp_sum(s) * inv_c;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      if (i * 32 + lane >= nvec) continue;
      float f[8];
      unpack8(cur[i], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = f[j] - mean; q += d * d; }
    }
    const float rstd = rsqrtf(warp_sum(q) * inv_c + eps);
    __nv_bfloat16* yr = y + static_cast<size_t>(row) * C;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      if (i * 32 + lane >= nvec) continue;
      float f[8];
      unpack8(cur[i], f);
      const float4 g0 = sg[slot(i, 0, lane)], g1 = sg[slot(i, 1, lane)];
      const float4 b0 = sb[slot(i, 0, lane)], b1 = sb[slot(i, 1, lane)];
      const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      uint4 o;
      uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        ow[j] = pack_bf16x2((f[2 * j] - mean) * rstd * g[2 * j] + b[2 * j],
                            (f[2 * j + 1] - mean) * rstd * g[2 * j + 1] + b[2 * j + 1]);
      *reinterpret_cast<uint4*>(yr + (i * 32 + lane) * 8) = o;
    }
    if (lane == 0) { mean_out[row] = mean; rstd_out[row] = rstd; }
  }
}

// ------------------------------------------------------------------ backward
// dx = rstd * (dy * gamma - mean(dy * gamma) - h * mean(dy * gamma * h)) (+ dres), h = (x - mean) * rstd, written as
// bf16.  dgamma += sum_rows dy * h, dbeta += sum_rows dy and, when given, dxsum += sum_rows dx (the bias gradient of the
// linear layer that fed this LayerNorm).  Each warp adds its rows' terms into a partial row of its own in shared
// memory (no per-lane register accumulators, so no spills at any width); at the end the block sums its warps' partials
// and adds them into the fp32 gradient buffer with one grad_add_f32 per column.
template <int V>
constexpr int bwd_smem_bytes() { return (1 + 3 * kBwdWarps) * 2 * V * 32 * static_cast<int>(sizeof(float4)); }

template <int V>
__global__ void __launch_bounds__(kBwdWarps * 32, 1) layernorm_wide_bwd_kernel(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ gamma,
    const float* __restrict__ mean_in, const float* __restrict__ rstd_in, const __nv_bfloat16* __restrict__ dres,
    __nv_bfloat16* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dxsum,
    int M, int C, int mc) {
  constexpr int S = 2 * V * 32;              // float4 slots of one row
  extern __shared__ float4 smem[];
  float4* sg = smem;                         // gamma
  float4* part = smem + S;                   // [warp][dgamma, dbeta, dxsum][S]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = C / 8;
  stage_param<V>(sg, gamma, nvec);
  for (int s = threadIdx.x; s < 3 * kBwdWarps * S; s += blockDim.x) part[s] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  float4* pg = part + warp * 3 * S;
  float4* pb = pg + S;
  float4* ps = pb + S;
  const bool has_res = dres != nullptr;
  const float inv_c = 1.0f / C;

  for (int row = blockIdx.x * kBwdWarps + warp; row < M; row += gridDim.x * kBwdWarps) {
    const size_t base = static_cast<size_t>(row) * C;
    uint4 xu[V], du[V], ru[V];
    load_row<V>(xu, x + base, nvec, lane);
    load_row<V>(du, dy + base, nvec, lane);
    if (has_res) load_row<V>(ru, dres + base, nvec, lane);
    const float mean = mean_in[row], rstd = rstd_in[row];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      if (i * 32 + lane >= nvec) continue;
      float xf[8], df[8];
      unpack8(xu[i], xf);
      unpack8(du[i], df);
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int k = slot(i, half, lane);
        const float4 g = sg[k];
        const float gg[4] = {g.x, g.y, g.z, g.w};
        float h[4], a[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          h[e] = (xf[half * 4 + e] - mean) * rstd;
          a[e] = df[half * 4 + e] * gg[e];
          s1 += a[e];
          s2 += a[e] * h[e];
        }
        float4 t = pg[k];
        t.x += df[half * 4] * h[0]; t.y += df[half * 4 + 1] * h[1];
        t.z += df[half * 4 + 2] * h[2]; t.w += df[half * 4 + 3] * h[3];
        pg[k] = t;
        t = pb[k];
        t.x += df[half * 4]; t.y += df[half * 4 + 1]; t.z += df[half * 4 + 2]; t.w += df[half * 4 + 3];
        pb[k] = t;
      }
    }
    s1 = warp_sum(s1) * inv_c;
    s2 = warp_sum(s2) * inv_c;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      if (i * 32 + lane >= nvec) continue;
      float xf[8], df[8], rf[8];
      unpack8(xu[i], xf);
      unpack8(du[i], df);
      if (has_res) unpack8(ru[i], rf);
      else
#pragma unroll
        for (int j = 0; j < 8; ++j) rf[j] = 0.f;
      float o[8];
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int k = slot(i, half, lane);
        const float4 g = sg[k];
        const float gg[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int j = half * 4 + e;
          const float h = (xf[j] - mean) * rstd;
          o[j] = rstd * (df[j] * gg[e] - s1 - h * s2) + rf[j];
        }
        float4 t = ps[k];
        t.x += o[half * 4]; t.y += o[half * 4 + 1]; t.z += o[half * 4 + 2]; t.w += o[half * 4 + 3];
        ps[k] = t;
      }
      uint4 u;
      u.x = pack_bf16x2(o[0], o[1]); u.y = pack_bf16x2(o[2], o[3]);
      u.z = pack_bf16x2(o[4], o[5]); u.w = pack_bf16x2(o[6], o[7]);
      *reinterpret_cast<uint4*>(dx + base + (i * 32 + lane) * 8) = u;
    }
  }
  __syncthreads();
  float* const dst[3] = {dgamma, dbeta, dxsum};
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    const int c = slot_col(s);
    if (c >= C) continue;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (dst[a] == nullptr) continue;
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int w = 0; w < kBwdWarps; ++w) {
        const float4 p = part[(w * 3 + a) * S + s];
        t.x += p.x; t.y += p.y; t.z += p.z; t.w += p.w;
      }
      grad_add_f32(dst[a] + c, t.x, mc);
      grad_add_f32(dst[a] + c + 1, t.y, mc);
      grad_add_f32(dst[a] + c + 2, t.z, mc);
      grad_add_f32(dst[a] + c + 3, t.w, mc);
    }
  }
}

static int sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

template <int V>
static int launch_bwd(const void* dy, const void* x, const void* gamma, const void* mean, const void* rstd,
                      const void* dres, void* dx, void* dgamma, void* dbeta, void* dxsum, int M, int C, int mc,
                      cudaStream_t st) {
  constexpr int smem = bwd_smem_bytes<V>();
  static bool configured = false;
  if (!configured) {
    if (cudaFuncSetAttribute(layernorm_wide_bwd_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) !=
        cudaSuccess)
      return -20;
    configured = true;
  }
  const int blocks = min((M + kBwdWarps - 1) / kBwdWarps, sms());
  layernorm_wide_bwd_kernel<V><<<blocks, kBwdWarps * 32, smem, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const __nv_bfloat16*>(x),
      reinterpret_cast<const __nv_bfloat16*>(gamma), reinterpret_cast<const float*>(mean),
      reinterpret_cast<const float*>(rstd), reinterpret_cast<const __nv_bfloat16*>(dres),
      reinterpret_cast<__nv_bfloat16*>(dx), reinterpret_cast<float*>(dgamma), reinterpret_cast<float*>(dbeta),
      reinterpret_cast<float*>(dxsum), M, C, mc);
  return 0;
}

}  // namespace lnw
}  // namespace aitj

extern "C" {
using namespace aitj::lnw;

// These entry points refuse nothing: F.layernorm_wide_fwd / F.layernorm_wide_bwd check every argument (C a multiple of
// 8 in [8, 2048], shapes, dtypes, 16-byte alignment) before calling them.  A call with no rows, or a width that is not
// positive or exceeds 2048, launches nothing.
int aitj_layernorm_wide_fwd(const void* x, const void* gamma, const void* beta, void* y, void* mean, void* rstd, int M,
                            int C, float eps, void* stream) {
  if (M <= 0 || C <= 0 || C > kMaxC) return 0;
  const int blocks = min((M + kFwdWarps - 1) / kFwdWarps, sms() * 2);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define LNW_F(V)                                                                                                   \
  layernorm_wide_fwd_kernel<V><<<blocks, kFwdWarps * 32, 0, st>>>(                                                 \
      reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(gamma),                    \
      reinterpret_cast<const __nv_bfloat16*>(beta), reinterpret_cast<__nv_bfloat16*>(y),                          \
      reinterpret_cast<float*>(mean), reinterpret_cast<float*>(rstd), M, C, eps)
  switch ((C + 255) / 256) {
    case 1: LNW_F(1); break; case 2: LNW_F(2); break; case 3: LNW_F(3); break; case 4: LNW_F(4); break;
    case 5: LNW_F(5); break; case 6: LNW_F(6); break; case 7: LNW_F(7); break; default: LNW_F(8); break;
  }
#undef LNW_F
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -30;
}

int aitj_layernorm_wide_bwd(const void* dy, const void* x, const void* gamma, const void* mean, const void* rstd,
                            const void* dres, void* dx, void* dgamma, void* dbeta, void* dxsum, int M, int C, int mc,
                            void* stream) {
  if (M <= 0 || C <= 0 || C > kMaxC) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = 0;
#define LNW_B(V) rc = launch_bwd<V>(dy, x, gamma, mean, rstd, dres, dx, dgamma, dbeta, dxsum, M, C, mc, st)
  switch ((C + 255) / 256) {
    case 1: LNW_B(1); break; case 2: LNW_B(2); break; case 3: LNW_B(3); break; case 4: LNW_B(4); break;
    case 5: LNW_B(5); break; case 6: LNW_B(6); break; case 7: LNW_B(7); break; default: LNW_B(8); break;
  }
#undef LNW_B
  if (rc) return rc;
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -30;
}

}  // extern "C"

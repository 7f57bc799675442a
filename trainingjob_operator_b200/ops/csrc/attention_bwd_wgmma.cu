// Flash attention backward for sm_90a (head dim 64, bf16) on wgmma, reading q / k / v straight out of the packed
// [B*T, 3*H*64] activation and writing dq | dk | dv straight into the packed gradient of the same layout.
//
// One CTA (one warpgroup) owns a block of 64 keys of one (batch, head) and walks the query blocks that see it, keeping
// dK and dV in registers.  Per query block of 64 (Q and dO double-buffered by TMA):
//   S^T  = K Q^T,  dP^T = V dO^T                      (both operands in shared memory)
//   P^T  = exp(S^T * scale - lse),  dS^T = P^T * (dP^T - delta)
//   dV  += P^T dO,  dK += dS^T Q                        (P^T / dS^T straight from the accumulator registers)
//   dQ   = dS K                                         (dS^T staged in shared memory, read as a transposed A operand)
// and dQ is added into an fp32 scratch with red.global.add (several key blocks contribute to one query row); a last
// pass converts it to bf16 into the packed gradient and clears the scratch.  delta = rowsum(dO * O) comes first.
//
// Document mask (kDoc; see attention_wgmma.cu): key k is seen by the queries q >= k with doc_start[q] <= k.  A key block
// walks the query blocks from its own up to the one holding the last query that sees its last key, found by a binary
// search over the (monotone) doc_start of the sequence, and P = 0 where k < doc_start[q].
#include "ptx.cuh"

namespace aitj {

constexpr int AB_B = 64;    // keys per CTA, queries per step
constexpr int AB_D = 64;
constexpr int kAbThreads = 128;

struct AttnBwdArgs {
  int B, T, H;
  int causal;
  float scale;
  float scale_log2;
  const float* lse;     // [B, H, T] natural log
  const float* delta;   // [B, H, T]
  float* dq_acc;        // [B*T, H*64]
  __nv_bfloat16* d_qkv; // [B*T, 3*H*64]
  const int* doc_start; // [B*T] (kDoc only)
};

__device__ __forceinline__ void red_add_v2_f32_ab(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

template <bool kDoc>
__global__ void __launch_bounds__(kAbThreads) attn_bwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv,
                                                              const __grid_constant__ CUtensorMap tmap_do,
                                                              const AttnBwdArgs a) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sk = smem;                 // 64 keys x 128 B
  uint8_t* sv = smem + 8192;
  uint8_t* sq = smem + 16384;         // [2] x 64 queries x 128 B
  uint8_t* sdo = smem + 32768;        // [2]
  uint8_t* sds = smem + 49152;        // dS^T: 64 keys x 64 queries bf16, 128B-swizzled
  uint64_t* kv_full = reinterpret_cast<uint64_t*>(smem + 57344);
  uint64_t* q_full = kv_full + 1;     // [2]

  const int T = a.T, H = a.H, C = H * AB_D;
  const int kvt = blockIdx.x;                     // low key blocks see the most queries under the causal mask
  const int bh = blockIdx.y;
  const int b = bh / H, h = bh - b * H;
  const int row0 = b * T;
  const int kv0 = kvt * AB_B;
  const int i0 = a.causal ? kvt : 0;
  int n_q = T / AB_B;
  const int tid = threadIdx.x;
  const int* ds_seq = kDoc ? a.doc_start + row0 : nullptr;
  if (kDoc) {
    // the queries past this block's last key that still see it form a prefix of (kv_last, T): those whose document
    // starts at or before kv_last.  First index past that prefix, by binary search; then clamp the block range into
    // [i0 + 1, T / 64] (a malformed doc_start cannot move a TMA coordinate out of this sequence)
    const int kv_last = kv0 + AB_B - 1;
    int lo = kv_last + 1, hi = T;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (ds_seq[mid] <= kv_last) lo = mid + 1;
      else hi = mid;
    }
    n_q = min(max((lo + AB_B - 1) / AB_B, i0 + 1), n_q);
  }

  if (tid == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_do);
    mbar_init(kv_full, 1);
    mbar_init(&q_full[0], 1);
    mbar_init(&q_full[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(kv_full, 16384);
    tma_load_2d(sk, &tmap_qkv, kv_full, (H + h) * AB_D, row0 + kv0);
    tma_load_2d(sv, &tmap_qkv, kv_full, (2 * H + h) * AB_D, row0 + kv0);
    mbar_arrive_expect_tx(&q_full[0], 16384);
    tma_load_2d(sq, &tmap_qkv, &q_full[0], h * AB_D, row0 + i0 * AB_B);
    tma_load_2d(sdo, &tmap_do, &q_full[0], h * AB_D, row0 + i0 * AB_B);
  }

  const int wl = tid >> 5;
  const int lane = tid & 31;
  const int t4 = lane & 3;
  const int r_loc = wl * 16 + (lane >> 2);        // this thread's accumulator rows: r_loc and r_loc + 8
  const uint32_t k_addr = smem_u32(sk), v_addr = smem_u32(sv), ds_addr = smem_u32(sds);
  const float* lse = a.lse + static_cast<size_t>(bh) * T;
  const float* delta = a.delta + static_cast<size_t>(bh) * T;
  float dk[32], dv[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dk[i] = 0.f; dv[i] = 0.f; }

  mbar_wait(kv_full, 0);
  for (int i = i0, it = 0; i < n_q; ++i, ++it) {
    const int buf = it & 1;
    if (tid == 0 && i + 1 < n_q) {
      // the other buffer was last read in the previous step, which every thread has left (barrier at its end)
      mbar_arrive_expect_tx(&q_full[buf ^ 1], 16384);
      tma_load_2d(sq + (buf ^ 1) * 8192, &tmap_qkv, &q_full[buf ^ 1], h * AB_D, row0 + (i + 1) * AB_B);
      tma_load_2d(sdo + (buf ^ 1) * 8192, &tmap_do, &q_full[buf ^ 1], h * AB_D, row0 + (i + 1) * AB_B);
    }
    mbar_wait(&q_full[buf], (it >> 1) & 1);
    const uint32_t q_addr = smem_u32(sq) + buf * 8192, do_addr = smem_u32(sdo) + buf * 8192;
    float st[32], dpt[32];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < AB_D / 16; ++ks)
      wgmma_m64n64_ss<0, 0>(st, make_wgmma_desc(k_addr + ks * 32, 16, 1024), make_wgmma_desc(q_addr + ks * 32, 16, 1024),
                            ks > 0 ? 1 : 0);
#pragma unroll
    for (int ks = 0; ks < AB_D / 16; ++ks)
      wgmma_m64n64_ss<0, 0>(dpt, make_wgmma_desc(v_addr + ks * 32, 16, 1024),
                            make_wgmma_desc(do_addr + ks * 32, 16, 1024), ks > 0 ? 1 : 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(st);
    fence_regs(dpt);

    const int qb = i * AB_B;
    const bool mask = a.causal && i == kvt;        // the diagonal block: key kv0 + r sees queries >= kv0 + r only
    // kDoc: some query of this block starts its document past this block's first key (the block's last query has the
    // largest document start)
    const bool dmask = kDoc && kv0 < ds_seq[qb + AB_B - 1];
    if (dmask) {     // (a separate loop: blocks without a document boundary run the causal kernel's loop unchanged)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int qc = qb + 8 * jj + 2 * t4;
        const float2 ls = *reinterpret_cast<const float2*>(lse + qc);
        const float2 dl = *reinterpret_cast<const float2*>(delta + qc);
        const int2 dsq = *reinterpret_cast<const int2*>(ds_seq + qc);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int idx = 4 * jj + 2 * hh + e;
            float p = fast_exp2(st[idx] * a.scale_log2 - (e ? ls.y : ls.x) * 1.4426950408889634f);
            if ((mask && 8 * jj + 2 * t4 + e < r_loc + 8 * hh) || kv0 + r_loc + 8 * hh < (e ? dsq.y : dsq.x)) p = 0.f;
            st[idx] = p;
            dpt[idx] = p * (dpt[idx] - (e ? dl.y : dl.x));
          }
      }
    } else {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int qc = qb + 8 * jj + 2 * t4;
        const float2 ls = *reinterpret_cast<const float2*>(lse + qc);
        const float2 dl = *reinterpret_cast<const float2*>(delta + qc);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int idx = 4 * jj + 2 * hh + e;
            float p = fast_exp2(st[idx] * a.scale_log2 - (e ? ls.y : ls.x) * 1.4426950408889634f);
            if (mask && 8 * jj + 2 * t4 + e < r_loc + 8 * hh) p = 0.f;
            st[idx] = p;
            dpt[idx] = p * (dpt[idx] - (e ? dl.y : dl.x));
          }
      }
    }
    uint32_t pa[4][4], dsa[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        pa[kk][r] = pack_bf16x2(st[8 * kk + 2 * r], st[8 * kk + 2 * r + 1]);
        dsa[kk][r] = pack_bf16x2(dpt[8 * kk + 2 * r], dpt[8 * kk + 2 * r + 1]);
      }
    // dS^T -> shared memory in the 128B-swizzle pattern (16-byte chunk c of row r at chunk c ^ (r & 7))
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int r = r_loc + 8 * hh;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(sds + r * 128 + ((jj ^ (r & 7)) << 4) + 4 * t4) = dsa[jj >> 1][(jj & 1) * 2 + hh];
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AB_B / 16; ++kk)
      wgmma_m64n64_rs<1>(dv, pa[kk], make_wgmma_desc(do_addr + kk * 2048, 8192, 1024), 1);
#pragma unroll
    for (int kk = 0; kk < AB_B / 16; ++kk)
      wgmma_m64n64_rs<1>(dk, dsa[kk], make_wgmma_desc(q_addr + kk * 2048, 8192, 1024), 1);
    wgmma_commit();
    fence_proxy_async_smem();          // the generic-proxy dS^T stores become visible to wgmma
    __syncthreads();
    float dq[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AB_B / 16; ++kk)
      wgmma_m64n64_ss<1, 1>(dq, make_wgmma_desc(ds_addr + kk * 2048, 8192, 1024),
                            make_wgmma_desc(k_addr + kk * 2048, 8192, 1024), kk > 0 ? 1 : 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(dq);
    fence_regs(dk);
    fence_regs(dv);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float* dst = a.dq_acc + static_cast<size_t>(row0 + qb + r_loc + 8 * hh) * C + h * AB_D + 2 * t4;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        red_add_v2_f32_ab(dst + 8 * jj, dq[4 * jj + 2 * hh] * a.scale, dq[4 * jj + 2 * hh + 1] * a.scale);
    }
    __syncthreads();                   // Q / dO of this step and dS^T are free for the next loads / stores
  }

#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    __nv_bfloat16* dst = a.d_qkv + static_cast<size_t>(row0 + kv0 + r_loc + 8 * hh) * 3 * C + 2 * t4;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      *reinterpret_cast<uint32_t*>(dst + (H + h) * AB_D + 8 * jj) =
          pack_bf16x2(dk[4 * jj + 2 * hh] * a.scale, dk[4 * jj + 2 * hh + 1] * a.scale);
      *reinterpret_cast<uint32_t*>(dst + (2 * H + h) * AB_D + 8 * jj) =
          pack_bf16x2(dv[4 * jj + 2 * hh], dv[4 * jj + 2 * hh + 1]);
    }
  }
}

// delta[b, h, t] = sum_d dO[b*T+t, h*64+d] * O[b*T+t, h*64+d]; one thread per (row, head): consecutive threads read
// consecutive 128-byte segments
__global__ void __launch_bounds__(256) attn_delta_kernel(const __nv_bfloat16* __restrict__ dO,
                                                         const __nv_bfloat16* __restrict__ O, float* __restrict__ delta,
                                                         int B, int T, int H) {
  const size_t n = static_cast<size_t>(B) * T * H;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < n;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t rowi = idx / H;
    const int h = static_cast<int>(idx - rowi * H);
    const uint4* a = reinterpret_cast<const uint4*>(dO + idx * AB_D);
    const uint4* b = reinterpret_cast<const uint4*>(O + idx * AB_D);
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const uint4 u = a[q], v = b[q];
      const uint32_t uw[4] = {u.x, u.y, u.z, u.w}, vw[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 x = unpack_bf16x2(uw[j]), y = unpack_bf16x2(vw[j]);
        s = fmaf(x.x, y.x, fmaf(x.y, y.y, s));
      }
    }
    const size_t bi = rowi / T;
    const int tt = static_cast<int>(rowi - bi * T);
    delta[(bi * H + h) * T + tt] = s;
  }
}

// d_qkv[:, 0:C] <- bf16(dq_acc); dq_acc <- 0 (ready for the next layer's backward)
__global__ void __launch_bounds__(256) attn_dq_finish_kernel(float* __restrict__ dq_acc, __nv_bfloat16* __restrict__ d_qkv,
                                                             size_t rows, int C) {
  const int vec_per_row = C / 8;
  const size_t total = rows * vec_per_row;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t r = idx / vec_per_row;
    const int c = static_cast<int>(idx - r * vec_per_row) * 8;
    float4* src = reinterpret_cast<float4*>(dq_acc + r * C + c);
    const float4 a = src[0], b = src[1];
    src[0] = make_float4(0.f, 0.f, 0.f, 0.f);
    src[1] = make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<uint4*>(d_qkv + r * 3 * C + c) =
        make_uint4(pack_bf16x2(a.x, a.y), pack_bf16x2(a.z, a.w), pack_bf16x2(b.x, b.y), pack_bf16x2(b.z, b.w));
  }
}

typedef CUresult (*EncodeTiledFnB)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int ab_encode_2d(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld_elems,
                        uint32_t box_inner, uint32_t box_outer) {
  static EncodeTiledFnB fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) return -10;
    fn = reinterpret_cast<EncodeTiledFnB>(p);
  }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld_elems * 2u};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 100;
}

}  // namespace aitj

extern "C" {

// qkv bf16 [B*T, 3*H*64]; out, d_out bf16 [B*T, H*64]; lse fp32 [B,H,T] (natural log, from aitj_attn_fwd);
// delta fp32 [B,H,T] scratch; dq_acc fp32 [B*T, H*64] scratch that MUST be zero on entry (it is zero again on exit);
// d_qkv bf16 [B*T, 3*H*64] receives dq | dk | dv.  T % 128 == 0.  scale <= 0 selects 1/sqrt(64).
// doc_start: null, or the int32 [B*T] document starts the forward was given (causal only).
int aitj_attn_bwd(const void* qkv, const void* out, const void* d_out, const void* lse, void* delta, void* dq_acc,
                  void* d_qkv, const void* doc_start, int B, int T, int H, int causal, float scale, void* stream_ptr) {
  using namespace aitj;
  if (B <= 0 || T <= 0 || H <= 0) return 0;
  if (T % 128) return -1;
  if (doc_start && !causal) return -5;
  if (reinterpret_cast<uintptr_t>(doc_start) & 7) return -4;   // read as int2 pairs
  const int C = H * AB_D;
  const uint64_t rows = static_cast<uint64_t>(B) * T;
  CUtensorMap tq, tdo;
  int rc = ab_encode_2d(&tq, qkv, 3ull * C, rows, 3ull * C, AB_D, AB_B);
  if (rc) return rc;
  rc = ab_encode_2d(&tdo, d_out, C, rows, C, AB_D, AB_B);
  if (rc) return rc - 1000;
  AttnBwdArgs a;
  a.B = B; a.T = T; a.H = H; a.causal = causal;
  if (scale <= 0.f) scale = 0.125f;
  a.scale = scale;
  a.scale_log2 = scale * 1.4426950408889634f;
  a.lse = reinterpret_cast<const float*>(lse);
  a.delta = reinterpret_cast<const float*>(delta);
  a.dq_acc = reinterpret_cast<float*>(dq_acc);
  a.d_qkv = reinterpret_cast<__nv_bfloat16*>(d_qkv);
  a.doc_start = reinterpret_cast<const int*>(doc_start);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_ptr);
  constexpr int kSmem = 57344 + 1024 + 64;
  static bool configured[2] = {false, false};
  const int v = doc_start ? 1 : 0;
  if (!configured[v]) {
    if (cudaFuncSetAttribute(v ? attn_bwd_kernel<true> : attn_bwd_kernel<false>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem) != cudaSuccess) return -20;
    configured[v] = true;
  }
  static int n_sms = 0;
  if (!n_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sms, cudaDevAttrMultiProcessorCount, dev);
  }
  const size_t n_stat = static_cast<size_t>(B) * T * H;
  int blocks = static_cast<int>((n_stat + 255) / 256);
  if (blocks > n_sms * 8) blocks = n_sms * 8;
  attn_delta_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(d_out),
                                            reinterpret_cast<const __nv_bfloat16*>(out), reinterpret_cast<float*>(delta), B, T, H);
  if (v)
    attn_bwd_kernel<true><<<dim3(T / AB_B, B * H), kAbThreads, kSmem, st>>>(tq, tdo, a);
  else
    attn_bwd_kernel<false><<<dim3(T / AB_B, B * H), kAbThreads, kSmem, st>>>(tq, tdo, a);
  const size_t nvec = rows * (C / 8);
  blocks = static_cast<int>((nvec + 255) / 256);
  if (blocks > n_sms * 8) blocks = n_sms * 8;
  attn_dq_finish_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<float*>(dq_acc), reinterpret_cast<__nv_bfloat16*>(d_qkv),
                                                rows, C);
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -30;
}

}  // extern "C"

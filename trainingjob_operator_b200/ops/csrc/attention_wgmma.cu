// Flash attention forward for sm_90a (head dim 64, bf16): S = Q K^T and O += P V on wgmma with the accumulators in
// registers, online softmax on the S fragments, operands moved by TMA straight out of the packed [B*T, 3*H*64] qkv
// activation -- no split / transpose / contiguous copies -- and the output written as [B*T, H*64], the layout the
// projection GEMM consumes.
//
// One CTA = one 128-row query tile of one (batch, head): two warpgroups of 64 query rows share the K / V blocks (64 keys
// each, double-buffered, the next block's TMA load in flight while the current one is used).  P never leaves the
// registers: the fp32 S fragment of a warpgroup has the row / column layout of a wgmma A operand, so P is packed to
// bf16 in place and multiplied with V (read transposed from shared memory: V is stored key-major).
//
// Document mask (kDoc, packed sequences): doc_start[b*T + t] is the sequence-local index of the first token of the
// document holding token t (non-decreasing along the sequence, 0 at t = 0); query q sees key k iff
// doc_start[q] <= k <= q.  A tile's key loop starts at the block of its first row's document start instead of block 0,
// so with short documents most key blocks are never loaded.
#include "ptx.cuh"

namespace aitj {

constexpr int ATT_BM = 128;   // query rows per CTA
constexpr int ATT_BN = 64;    // keys per block
constexpr int ATT_D = 64;
constexpr int kAttThreads = 256;

struct AttnArgs {
  int B, T, H;
  int causal;
  float scale_log2;   // softmax scale * log2(e)
  float* lse;         // [B, H, T] natural-log sum-exp of the scaled scores (what the backward needs)
  __nv_bfloat16* out; // [B*T, H*64]
  const int* doc_start; // [B*T] (kDoc only)
};

template <bool kDoc>
__global__ void __launch_bounds__(kAttThreads) attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv,
                                                               const AttnArgs a) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sq = smem;                    // 128 rows x 128 B
  uint8_t* sk = smem + 16384;            // [2] x 64 rows x 128 B
  uint8_t* sv = smem + 32768;            // [2] x 64 rows x 128 B
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + 49152);
  uint64_t* kv_full = q_full + 1;        // [2]

  const int T = a.T, H = a.H;
  const int qt = gridDim.x - 1 - blockIdx.x;      // the longest causal tiles first
  const int bh = blockIdx.y;
  const int b = bh / H, h = bh - b * H;
  const int row0 = b * T;                          // first row of this sequence in the packed activation
  const int q0 = qt * ATT_BM;
  const int n_kv = a.causal ? (q0 + ATT_BM) / ATT_BN : T / ATT_BN;
  const int tid = threadIdx.x;
  // first key block: the one holding the document start of the tile's first row (the smallest in the tile), clamped
  // into [0, q0] so that a malformed doc_start cannot move a TMA coordinate out of this sequence
  const int j0 = kDoc ? min(max(a.doc_start[row0 + q0], 0), q0) / ATT_BN : 0;

  if (tid == 0) {
    tma_prefetch_desc(&tmap_qkv);
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1);
    mbar_init(&kv_full[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(q_full, 16384);
    tma_load_2d(sq, &tmap_qkv, q_full, h * ATT_D, row0 + q0);
    tma_load_2d(sq + 8192, &tmap_qkv, q_full, h * ATT_D, row0 + q0 + 64);
    mbar_arrive_expect_tx(&kv_full[0], 16384);
    tma_load_2d(sk, &tmap_qkv, &kv_full[0], (H + h) * ATT_D, row0 + j0 * ATT_BN);
    tma_load_2d(sv, &tmap_qkv, &kv_full[0], (2 * H + h) * ATT_D, row0 + j0 * ATT_BN);
  }

  const int wg = tid >> 7;
  const int wl = (tid >> 5) & 3;
  const int lane = tid & 31;
  const int t4 = lane & 3;
  const int qrow = q0 + wg * 64 + wl * 16 + (lane >> 2);   // this thread's rows: qrow and qrow + 8 (sequence positions)
  // kDoc: the document starts of this thread's two rows, and the largest one of the warpgroup's 64 rows (its last row's):
  // key blocks that start at or past it need only the causal mask
  int ds[2] = {0, 0}, ds_hi = 0;
  if (kDoc) {
    ds[0] = min(max(a.doc_start[row0 + qrow], 0), qrow);
    ds[1] = min(max(a.doc_start[row0 + qrow + 8], 0), qrow + 8);
    ds_hi = a.doc_start[row0 + q0 + wg * 64 + 63];
  }
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const uint32_t q_addr = smem_u32(sq) + wg * 8192;

  mbar_wait(q_full, 0);
  for (int j = j0; j < n_kv; ++j) {
    const int it = j - j0;
    const int buf = it & 1;
    if (tid == 0 && j + 1 < n_kv) {
      // the other buffer was last read in iteration j-1, which every thread has left (barrier at its end)
      mbar_arrive_expect_tx(&kv_full[buf ^ 1], 16384);
      tma_load_2d(sk + (buf ^ 1) * 8192, &tmap_qkv, &kv_full[buf ^ 1], (H + h) * ATT_D, row0 + (j + 1) * ATT_BN);
      tma_load_2d(sv + (buf ^ 1) * 8192, &tmap_qkv, &kv_full[buf ^ 1], (2 * H + h) * ATT_D, row0 + (j + 1) * ATT_BN);
    }
    mbar_wait(&kv_full[buf], (it >> 1) & 1);
    const uint32_t k_addr = smem_u32(sk) + buf * 8192;
    const uint32_t v_addr = smem_u32(sv) + buf * 8192;
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < ATT_D / 16; ++ks)
      wgmma_m64n64_ss<0, 0>(s, make_wgmma_desc(q_addr + ks * 32, 16, 1024), make_wgmma_desc(k_addr + ks * 32, 16, 1024),
                            ks > 0 ? 1 : 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);

    const int kv0 = j * ATT_BN;
    const bool mask = a.causal && kv0 + ATT_BN - 1 > q0 + wg * 64;
    const bool dmask = kDoc && kv0 < ds_hi;
    float mx[2] = {-INFINITY, -INFINITY};
    if (dmask) {     // (a separate loop: blocks without a document boundary run the causal kernel's loop unchanged)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int idx = 4 * jj + 2 * hh + e;
            const int k = kv0 + 8 * jj + 2 * t4 + e;
            float v = s[idx] * a.scale_log2;
            if ((mask && k > qrow + 8 * hh) || k < ds[hh]) v = -INFINITY;
            s[idx] = v;
            mx[hh] = fmaxf(mx[hh], v);
          }
    } else {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int idx = 4 * jj + 2 * hh + e;
            float v = s[idx] * a.scale_log2;
            if (mask && kv0 + 8 * jj + 2 * t4 + e > qrow + 8 * hh) v = -INFINITY;
            s[idx] = v;
            mx[hh] = fmaxf(mx[hh], v);
          }
    }
    float alpha[2], m_sub[2], ls[2] = {0.f, 0.f};
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
      // without a document mask key 0 is visible to every query row and comes in block 0, so m is finite from then
      // on.  With one, a row whose document starts past this block has seen nothing but -inf yet: it keeps alpha = 1
      // and gets p = 0 (subtracting 0 instead of -inf), never exp2(-inf - -inf)
      const float m_new = fmaxf(m[hh], mx[hh]);
      if (kDoc && m_new == -INFINITY) {
        alpha[hh] = 1.f;
        m_sub[hh] = 0.f;
      } else {
        alpha[hh] = fast_exp2(m[hh] - m_new);
        m_sub[hh] = m_new;
      }
      m[hh] = m_new;
    }
#pragma unroll
    for (int idx = 0; idx < 32; ++idx) {
      const int hh = (idx >> 1) & 1;
      const float p = fast_exp2(s[idx] - m_sub[hh]);
      s[idx] = p;
      ls[hh] += p;
      o[idx] *= alpha[hh];
    }
    l[0] = l[0] * alpha[0] + ls[0];
    l[1] = l[1] * alpha[1] + ls[1];
    uint32_t pa[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) pa[kk][r] = pack_bf16x2(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk)
      wgmma_m64n64_rs<1>(o, pa[kk], make_wgmma_desc(v_addr + kk * 2048, 8192, 1024), 1);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    __syncthreads();
  }

  const int C = H * ATT_D;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float lt = l[hh];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const float inv = 1.f / lt;
    const int t = qrow + 8 * hh;
    __nv_bfloat16* dst = a.out + static_cast<size_t>(row0 + t) * C + h * ATT_D + 2 * t4;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
      *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
    if (t4 == 0) a.lse[static_cast<size_t>(bh) * T + t] = (m[hh] + __log2f(lt)) * 0.6931471805599453f;
  }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFnA)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int attn_encode_2d(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld,
                          uint32_t box_inner, uint32_t box_outer) {
  static EncodeTiledFnA fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) return -10;
    fn = reinterpret_cast<EncodeTiledFnA>(p);
  }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld * 2u};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 100;
}

}  // namespace aitj

extern "C" {

// qkv: bf16 [B*T, 3*H*64] (q | k | v, heads contiguous inside each third);  out: bf16 [B*T, H*64];
// lse: fp32 [B, H, T].  T must be a multiple of 128.  scale <= 0 selects 1/sqrt(64).
// doc_start: null, or int32 [B*T] document starts (see the top of this file; causal only).
int aitj_attn_fwd(const void* qkv, void* out, void* lse, const void* doc_start, int B, int T, int H, int causal,
                  float scale, void* stream_ptr) {
  using namespace aitj;
  if (B <= 0 || T <= 0 || H <= 0) return 0;
  if (T % ATT_BM) return -1;
  if (doc_start && !causal) return -5;
  if (reinterpret_cast<uintptr_t>(doc_start) & 7) return -4;   // read as int2 pairs
  if ((reinterpret_cast<uintptr_t>(qkv) & 15) || (reinterpret_cast<uintptr_t>(out) & 15)) return -4;
  const int C = H * ATT_D;
  CUtensorMap tq;
  int rc = attn_encode_2d(&tq, qkv, 3ull * C, static_cast<uint64_t>(B) * T, 3ull * C, ATT_D, 64);
  if (rc) return rc;
  AttnArgs a;
  a.B = B; a.T = T; a.H = H; a.causal = causal;
  if (scale <= 0.f) scale = 0.125f;
  a.scale_log2 = scale * 1.4426950408889634f;
  a.lse = reinterpret_cast<float*>(lse);
  a.out = reinterpret_cast<__nv_bfloat16*>(out);
  a.doc_start = reinterpret_cast<const int*>(doc_start);
  constexpr int kSmem = 49152 + 1024 + 64;
  static bool configured[2] = {false, false};
  const int v = doc_start ? 1 : 0;
  if (!configured[v]) {
    if (cudaFuncSetAttribute(v ? attn_fwd_kernel<true> : attn_fwd_kernel<false>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem) != cudaSuccess)
      return -20;
    configured[v] = true;
  }
  dim3 grid(T / ATT_BM, B * H);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_ptr);
  if (v)
    attn_fwd_kernel<true><<<grid, kAttThreads, kSmem, st>>>(tq, a);
  else
    attn_fwd_kernel<false><<<grid, kAttThreads, kSmem, st>>>(tq, a);
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -30;
}

}  // extern "C"

// Persistent, warp-specialised bf16 GEMM for sm_90a (H100): TMA -> 128B-swizzled shared-memory ring -> wgmma with the
// fp32 accumulators in registers -> epilogue straight from the registers with fused bias / GELU / dGELU / residual /
// pre-activation save, fp32 store or fp32 reduce-add (split-K, gradient accumulation) and optional column sums.
//
//   out[M,N] (+)= opA[M,K] * opB[N,K]^T
//     a_mn == 0 : A stored [M,K] row-major (K contiguous, "K-major")
//     a_mn == 1 : A stored [K,M] row-major (M contiguous, "MN-major")   -> used by wgrad
//     b_mn == 0 : B stored [N,K] row-major                               -> forward  (x @ W^T)
//     b_mn == 1 : B stored [K,N] row-major                               -> dgrad    (dy @ W), wgrad
//
// One CTA per SM computes 128 x kBN tiles (kBN = 128 or 256, BK = 64) in a persistent loop.  384 threads: warpgroup 0
// is the TMA producer (one thread), warpgroups 1 and 2 are consumers that each own 64 rows of the tile and issue
// wgmma.m64n{kBN}k16 with both operands read from shared memory.  While the consumers run the epilogue of one tile, the
// producer is already filling the ring with the next tile's operands.
//
// Clusters of kCM CTAs (kCM = 2 or 4, selected by block_n = 512 / 1024) work on vertically adjacent tiles that need the
// same B tile: each CTA loads 1/kCM of it and multicasts the slice to every CTA of the cluster, so each B byte is read
// from L2 once per cluster instead of once per CTA.  A stage is free again only when the consumers of every CTA of the
// cluster have released it (a peer's multicast writes into this CTA's ring).
#include "ptx.cuh"
#include <string.h>

namespace aitj {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int WG_K = 16;
constexpr int kGemmThreads = 384;   // warpgroup 0 TMA producer, warpgroups 1..2 consumers

enum : int {
  EPI_BIAS = 1,       // + bias[N]
  EPI_GELU = 2,       // gelu_tanh(.)
  EPI_RESIDUAL = 4,   // + residual[M,ldc]
  EPI_SAVE_PRE = 8,   // aux[M,ldc] <- value before GELU (bf16)
  EPI_DGELU = 16,     // * gelu'(aux[M,ldc])
  EPI_OUT_F32 = 32,   // out is fp32 (plain store)
  EPI_ACCUM = 64,     // out is fp32, red.global.add (split-K / grad accumulation)
  EPI_MC = 128,       // with EPI_ACCUM: `out` is an NVSwitch multicast address; reduce with multimem.red (GEMM + all-reduce in one kernel)
  EPI_PEER = 16384    // with EPI_ACCUM: `out` lies in the symmetric, owner-sharded gradient buffer; every element is added into the
                      // copy of the rank that owns it (red.global.add over NVLink peer memory): weight-gradient GEMM +
                      // reduce-scatter in one kernel.  With split-K the splits add into the local copy and
                      // peer_move_kernel sends the finished sums to their owners once
};

struct GemmArgs {
  int M, N, K;
  int ldc;
  void* out;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* residual;
  __nv_bfloat16* aux;
  int flags;
  int split_k;
  int tiles_m, tiles_n;
  int k_blocks, k_per_split;
  // optional (bf16 output): colsum[N] += column sums of the stored output, i.e. the bias gradient of the layer whose
  // input gradient this GEMM produces
  float* colsum;
};

struct WorkItem {
  int m_blk, n_blk, kb0, kb1;
};

// Grouped rasterisation: GROUP_M row blocks sweep the N tiles together, so consecutive work items share A and B in L2.
__device__ __forceinline__ WorkItem decode_work(const GemmArgs& a, int w) {
  const int num_tiles = a.tiles_m * a.tiles_n;
  const int split = w / num_tiles;
  const int t = w - split * num_tiles;
  constexpr int GROUP_M = 8;
  const int group_sz = GROUP_M * a.tiles_n;
  const int g = t / group_sz;
  const int first_m = g * GROUP_M;
  const int gm = min(a.tiles_m - first_m, GROUP_M);
  const int r = t - g * group_sz;
  WorkItem wi;
  wi.m_blk = first_m + (r % gm);
  wi.n_blk = r / gm;
  wi.kb0 = split * a.k_per_split;
  wi.kb1 = min(a.k_blocks, wi.kb0 + a.k_per_split);
  return wi;
}

__device__ __forceinline__ void red_add_v2_f32(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

// Epilogue of one consumer warpgroup: its 64 rows x kBN columns of accumulators in the wgmma fragment layout -- register
// 4j + 2h + e holds row (r_base + 8h), column (c_base + 8j + e).
template <int kBN>
__device__ __forceinline__ void epilogue(const GemmArgs& a, float (&acc)[kBN / 2], int r_base, int c_base) {
  const int flags = a.flags;
  const int lane = threadIdx.x & 31;
  if (flags & (EPI_OUT_F32 | EPI_ACCUM)) {
    float* obase = reinterpret_cast<float*>(a.out);
#pragma unroll
    for (int j = 0; j < kBN / 8; ++j) {
      const int col = c_base + 8 * j;
      if (col >= a.N) break;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r_base + 8 * h;
        if (row >= a.M) continue;
        float* p = obase + static_cast<size_t>(row) * a.ldc + col;
        const float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
        if (!(flags & EPI_ACCUM)) {
          *reinterpret_cast<float2*>(p) = make_float2(x0, x1);
        } else if (flags & EPI_MC) {
          mc_red_add_f32(p, x0);
          mc_red_add_f32(p + 1, x1);
        } else {
          red_add_v2_f32((flags & EPI_PEER) ? peer_ptr(p) : p, x0, x1);
        }
      }
    }
    return;
  }
  __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(a.out);
#pragma unroll
  for (int j = 0; j < kBN / 8; ++j) {
    const int col = c_base + 8 * j;
    if (col >= a.N) break;       // N % 8 == 0: a column pair is either wholly inside or wholly outside
    float2 bv = make_float2(0.f, 0.f);
    if (flags & EPI_BIAS) bv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(a.bias + col));
    float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r_base + 8 * h;
      if (row >= a.M) continue;
      const size_t off = static_cast<size_t>(row) * a.ldc + col;
      float x0 = acc[4 * j + 2 * h] + bv.x, x1 = acc[4 * j + 2 * h + 1] + bv.y;
      if (flags & EPI_SAVE_PRE) *reinterpret_cast<uint32_t*>(a.aux + off) = pack_bf16x2(x0, x1);
      if (flags & EPI_GELU) { x0 = gelu_tanh(x0); x1 = gelu_tanh(x1); }
      if (flags & EPI_DGELU) {
        const float2 pre = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(a.aux + off));
        x0 *= gelu_tanh_grad(pre.x);
        x1 *= gelu_tanh_grad(pre.y);
      }
      if (flags & EPI_RESIDUAL) {
        const float2 r = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(a.residual + off));
        x0 += r.x;
        x1 += r.y;
      }
      const uint32_t packed = pack_bf16x2(x0, x1);
      *reinterpret_cast<uint32_t*>(out + off) = packed;
      const float2 stored = unpack_bf16x2(packed);
      cs0 += stored.x;
      cs1 += stored.y;
    }
    if (a.colsum != nullptr) {
      // the eight lanes with the same (lane & 3) hold the same two columns of the warp's 16 rows
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        cs0 += __shfl_xor_sync(0xffffffffu, cs0, o);
        cs1 += __shfl_xor_sync(0xffffffffu, cs1, o);
      }
      if (lane < 4) {
        atomicAdd(a.colsum + col, cs0);
        atomicAdd(a.colsum + col + 1, cs1);
      }
    }
  }
}

template <int kBN>
__host__ __device__ constexpr int gemm_stages() { return kBN == 256 ? 4 : 6; }
template <int kBN>
__host__ __device__ constexpr int gemm_smem_bytes() { return gemm_stages<kBN>() * (BLOCK_M + kBN) * BLOCK_K * 2 + 1024 + 256; }

template <int kBN, bool kAMN, bool kBMN, int kCM>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const GemmArgs args) {
  constexpr int kStages = gemm_stages<kBN>();
  constexpr int kStageA = BLOCK_M * BLOCK_K * 2;
  constexpr int kStageB = kBN * BLOCK_K * 2;
  constexpr int kStageBytes = kStageA + kStageB;
  constexpr int kSliceN = kBN / kCM;               // rows of the B tile this CTA loads and multicasts
  static_assert(!kBMN || kSliceN % 64 == 0, "MN-major B slices are whole 64-column chunks");

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = kCM > 1 ? cluster_ctarank() : 0u;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);          // this CTA's producer: arrive(expect_tx) + the bytes of A and all B slices
      mbar_init(&empty_bar[i], 2 * kCM);   // both consumer warpgroups of every CTA of the cluster
    }
    fence_barrier_init();
  }
  if constexpr (kCM > 1) cluster_sync_all();   // no multicast may reach a peer before its barriers exist
  else __syncthreads();

  GemmArgs sched = args;
  sched.tiles_m = (args.tiles_m + kCM - 1) / kCM;     // a work item is kCM vertically adjacent tiles
  const int num_work = sched.tiles_m * args.tiles_n * args.split_k;
  const int cluster_id = blockIdx.x / kCM;
  const int num_clusters = gridDim.x / kCM;

  if (warp < 4) {
    // ------------------------------------------------------------ TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = cluster_id; w < num_work; w += num_clusters) {
        const WorkItem wi = decode_work(sched, w);
        const int m0 = (wi.m_blk * kCM + static_cast<int>(rank)) * BLOCK_M;
        const int n0 = wi.n_blk * kBN;
        for (int kb = wi.kb0; kb < wi.kb1; ++kb) {
          if constexpr (kCM > 1) mbar_wait_cluster(&empty_bar[stage], phase ^ 1u);
          else mbar_wait(&empty_bar[stage], phase ^ 1u);
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
          uint8_t* sa = smem + stage * kStageBytes;
          uint8_t* sb = sa + kStageA;
          if constexpr (!kAMN) {
            tma_load_2d(sa, &tmap_a, &full_bar[stage], kb * BLOCK_K, m0);
          } else {
#pragma unroll
            for (int j = 0; j < BLOCK_M / 64; ++j)
              tma_load_2d(sa + j * 8192, &tmap_a, &full_bar[stage], m0 + j * 64, kb * BLOCK_K);
          }
          constexpr uint16_t kMask = static_cast<uint16_t>((1u << kCM) - 1u);
          if constexpr (!kBMN) {
            const int r0 = static_cast<int>(rank) * kSliceN;
            if constexpr (kCM > 1) tma_load_2d_mcast(sb + r0 * 128, &tmap_b, &full_bar[stage], kb * BLOCK_K, n0 + r0, kMask);
            else tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * BLOCK_K, n0);
          } else {
#pragma unroll
            for (int j = 0; j < kSliceN / 64; ++j) {
              const int c = static_cast<int>(rank) * (kSliceN / 64) + j;
              if constexpr (kCM > 1) tma_load_2d_mcast(sb + c * 8192, &tmap_b, &full_bar[stage], n0 + c * 64, kb * BLOCK_K, kMask);
              else tma_load_2d(sb + c * 8192, &tmap_b, &full_bar[stage], n0 + c * 64, kb * BLOCK_K);
            }
          }
          if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumers (warpgroups 1, 2: 64 rows each)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    const int wg = (warp >> 2) - 1;
    const bool signaller = (threadIdx.x & 127) == 0;
    float acc[kBN / 2];
    int stage = 0;
    uint32_t phase = 0;
    auto release = [&](int s) {
      if (signaller) {
        if constexpr (kCM > 1) {
#pragma unroll
          for (int c = 0; c < kCM; ++c) mbar_arrive_remote(&empty_bar[s], static_cast<uint32_t>(c));
        } else {
          mbar_arrive(&empty_bar[s]);
        }
      }
    };
    for (int w = cluster_id; w < num_work; w += num_clusters) {
      const WorkItem wi = decode_work(sched, w);
      const int nk = wi.kb1 - wi.kb0;
      int prev = -1;
      for (int kb = 0; kb < nk; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(smem + stage * kStageBytes) + wg * 8192;
        const uint32_t b_addr = smem_u32(smem + stage * kStageBytes) + kStageA;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < BLOCK_K / WG_K; ++ks) {
          const uint64_t da = kAMN ? make_wgmma_desc(a_addr + ks * 2048, 8192, 1024)
                                   : make_wgmma_desc(a_addr + ks * WG_K * 2, 16, 1024);
          const uint64_t db = kBMN ? make_wgmma_desc(b_addr + ks * 2048, 8192, 1024)
                                   : make_wgmma_desc(b_addr + ks * WG_K * 2, 16, 1024);
          if constexpr (kBN == 256) wgmma_m64n256_ss<kAMN, kBMN>(acc, da, db, (kb > 0 || ks > 0) ? 1 : 0);
          else wgmma_m64n128_ss<kAMN, kBMN>(acc, da, db, (kb > 0 || ks > 0) ? 1 : 0);
        }
        wgmma_commit();
        wgmma_wait<1>();            // the previous stage's MMAs have retired: its buffers can be refilled
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0) release(prev);
      if (nk > 0) {
        const int wl = warp & 3;
        const int m_blk = wi.m_blk * kCM + static_cast<int>(rank);
        epilogue<kBN>(args, acc, m_blk * BLOCK_M + wg * 64 + wl * 16 + (lane >> 2), wi.n_blk * kBN + 2 * (lane & 3));
      }
    }
  }
  if constexpr (kCM > 1) {
    __syncwarp();
    cluster_sync_all();   // peers may still multicast into this CTA's ring / arrive on its barriers until all are done
  }
}

// EPI_PEER with split_k > 1: the splits accumulate into this rank's LOCAL copy of the gradient (plain red.add, as on one
// GPU); this pass then adds every element another rank owns into the owner's copy and clears the local one, so each
// gradient element crosses NVLink once instead of once per split.  Outside this window the local copy of a range this
// rank does not own is zero.  Ownership bounds are 256-element aligned, so a float4 never straddles two owners.
__global__ void __launch_bounds__(256) peer_move_kernel(float* __restrict__ out, int M, int N, int ldc) {
  const int vec_per_row = N >> 2;
  const size_t total = static_cast<size_t>(M) * vec_per_row;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t r = i / vec_per_row;
    const int c = static_cast<int>(i - r * vec_per_row) * 4;
    float* p = out + r * ldc + c;
    const long long delta = c_peers.delta[peer_owner(p)];
    if (delta == 0) continue;                     // this rank owns it: the sum is already where it belongs
    const float4 v = __ldcg(reinterpret_cast<const float4*>(p));
    red_add_v4_f32(reinterpret_cast<float*>(reinterpret_cast<char*>(p) + delta), v.x, v.y, v.z, v.w);
    __stcg(reinterpret_cast<float4*>(p), make_float4(0.f, 0.f, 0.f, 0.f));
  }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
      return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D bf16 tensor map (128B swizzle): `inner` contiguous elements per row, `outer` rows, row stride `ld` elements.
static int encode_2d(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld,
                     uint32_t box_inner, uint32_t box_outer) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return -10;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld * 2u};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 100;
}

static int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

template <int kBN, bool kAMN, bool kBMN, int kCM>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& args, int max_ctas,
                       cudaStream_t stream) {
  constexpr int kSmem = gemm_smem_bytes<kBN>();
  static int max_clusters = 0;
  auto kern = gemm_bf16_wgmma_kernel<kBN, kAMN, kBMN, kCM>;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = kCM; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = kSmem;
  cfg.stream = stream;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  if (!max_clusters) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem) != cudaSuccess) return -20;
    // how many clusters the GPU holds at once (a GPC whose SM count is not a multiple of kCM strands a few SMs)
    int n = num_sms() / kCM;
    if (kCM > 1) {
      cfg.gridDim = dim3(num_sms() / kCM * kCM);
      int q = 0;
      if (cudaOccupancyMaxActiveClusters(&q, kern, &cfg) == cudaSuccess && q > 0) n = q;
      else cudaGetLastError();
    }
    max_clusters = n;
  }
  const int num_work = ((args.tiles_m + kCM - 1) / kCM) * args.tiles_n * args.split_k;
  int clusters = max_clusters;
  if (num_work < clusters) clusters = num_work;
  if (max_ctas > 0 && clusters > max_ctas / kCM) clusters = max_ctas / kCM;
  if (clusters < 1) clusters = 1;
  cfg.gridDim = dim3(clusters * kCM);
  if (cudaLaunchKernelEx(&cfg, kern, ta, tb, args) != cudaSuccess) return -30;
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -30;
}

}  // namespace aitj

static float* g_gemm_colsum = nullptr;   // consumed by the next aitj_gemm_bf16 call

extern "C" {

// The next aitj_gemm_bf16 call (bf16 output) also accumulates the column sums of its output into buf[N] (fp32).
// One-shot: cleared by that call.
int aitj_gemm_set_colsum(void* buf) { g_gemm_colsum = reinterpret_cast<float*>(buf); return 0; }

// Returns 0 on success. See file header for operand conventions. lda/ldb/ldc in elements.
// block_n: 128 or 256 (0 = auto); 512 / 1024: 128x256 tiles in clusters of 2 / 4 CTAs sharing B by TMA multicast.
// split_k > 1 requires EPI_ACCUM. max_ctas: 0 = all SMs.
int aitj_gemm_bf16(const void* A, const void* B, void* out, int M, int N, int K, int lda, int ldb, int ldc,
                   int a_mn, int b_mn, const void* bias, const void* residual, void* aux, int flags, int split_k,
                   int block_n, int max_ctas, void* stream_ptr) {
  using namespace aitj;
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((N & 7) || (ldc & 7) || (lda & 7) || (ldb & 7)) return -1;
  if ((reinterpret_cast<uintptr_t>(out) & 15) || ((flags & EPI_SAVE_PRE) && (reinterpret_cast<uintptr_t>(aux) & 15))) return -4;
  if (split_k > 1 && !(flags & EPI_ACCUM)) return -2;
  if ((flags & (EPI_MC | EPI_PEER)) && !(flags & EPI_ACCUM)) return -5;
  const int cm = block_n == 1024 ? 4 : (block_n == 512 ? 2 : 1);
  if (cm > 1) block_n = 256;
  if (block_n == 0) block_n = (N > 128) ? 256 : 128;
  if (block_n != 128 && block_n != 256) return -3;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_ptr);

  GemmArgs args;
  args.M = M; args.N = N; args.K = K; args.ldc = ldc; args.out = out;
  args.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  args.residual = reinterpret_cast<const __nv_bfloat16*>(residual);
  args.aux = reinterpret_cast<__nv_bfloat16*>(aux);
  args.flags = flags;
  args.colsum = g_gemm_colsum;
  g_gemm_colsum = nullptr;
  if (args.colsum && (flags & (EPI_OUT_F32 | EPI_ACCUM))) return -6;   // column sums of a bf16 output only
  args.tiles_m = (M + BLOCK_M - 1) / BLOCK_M;
  args.tiles_n = (N + block_n - 1) / block_n;
  args.k_blocks = (K + BLOCK_K - 1) / BLOCK_K;
  if (split_k < 1) split_k = 1;
  if (split_k > args.k_blocks) split_k = args.k_blocks;
  args.k_per_split = (args.k_blocks + split_k - 1) / split_k;
  args.split_k = (args.k_blocks + args.k_per_split - 1) / args.k_per_split;

  CUtensorMap ta, tb;
  int rc;
  if (!a_mn) rc = encode_2d(&ta, A, K, M, lda, BLOCK_K, BLOCK_M);
  else       rc = encode_2d(&ta, A, M, K, lda, 64, BLOCK_K);
  if (rc) return rc;
  if (!b_mn) rc = encode_2d(&tb, B, K, N, ldb, BLOCK_K, block_n / cm);
  else       rc = encode_2d(&tb, B, N, K, ldb, 64, BLOCK_K);
  if (rc) return rc - 1000;
  const bool peer_move = (flags & EPI_PEER) && args.split_k > 1;
  if (peer_move) args.flags &= ~EPI_PEER;

#define AITJ_DISPATCH(BN, CM)                                                                         \
  if (!a_mn && !b_mn) rc = launch_gemm<BN, false, false, CM>(ta, tb, args, max_ctas, stream);        \
  else if (!a_mn && b_mn) rc = launch_gemm<BN, false, true, CM>(ta, tb, args, max_ctas, stream);     \
  else if (a_mn && !b_mn) rc = launch_gemm<BN, true, false, CM>(ta, tb, args, max_ctas, stream);     \
  else rc = launch_gemm<BN, true, true, CM>(ta, tb, args, max_ctas, stream);
  if (cm == 4) { AITJ_DISPATCH(256, 4) }
  else if (cm == 2) { AITJ_DISPATCH(256, 2) }
  else if (block_n == 256) { AITJ_DISPATCH(256, 1) }
  else { AITJ_DISPATCH(128, 1) }
#undef AITJ_DISPATCH
  if (rc || !peer_move) return rc;
  const size_t nvec = static_cast<size_t>(M) * (N / 4);
  int blocks = static_cast<int>((nvec + 255) / 256);
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  peer_move_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<float*>(out), M, N, ldc);
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -30;
}

// Ownership table of the symmetric gradient buffer for EPI_PEER (see ptx.cuh: PeerTable); one copy per translation unit.
int aitj_gemm_set_peers(const void* base, const long long* delta, const long long* bound, int n) {
  if (n < 1 || n > 8) return -1;
  aitj::PeerTable t;
  memset(&t, 0, sizeof(t));
  t.base = reinterpret_cast<const float*>(base);
  for (int i = 0; i < n; ++i) t.delta[i] = delta[i];
  for (int i = 0; i <= n; ++i) t.bound[i] = bound[i];
  t.n = n;
  return cudaMemcpyToSymbol(aitj::c_peers, &t, sizeof(t)) == cudaSuccess ? 0 : -2;
}

int aitj_num_sms() { return aitj::num_sms(); }

}  // extern "C"

// Persistent, warp-specialised bf16 GEMM for sm_90a (H100): TMA -> 128B-swizzled shared-memory ring -> wgmma with the
// fp32 accumulators in registers -> epilogue with fused bias / GELU / dGELU / residual / pre-activation save and
// optional column sums, whose bf16 outputs leave through shared memory by TMA store (inputs arrive by TMA load), or an
// fp32 store or fp32 reduce-add (split-K, gradient accumulation) straight from the registers.
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
//
// The epilogue variant is a template parameter (kEpi, EPI_* bits), so a kernel contains only the paths its variant
// uses.  An epilogue that tests every flag at run time unrolls to ~20k instructions per 256-wide kernel, and the
// consumer warps fetch that code again on every tile; with a plain-store epilogue the whole kernel is under 1k.  Only
// the (layout, epilogue) pairs in kGemmKernels are compiled; aitj_gemm_bf16 returns -7 for any other.
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
  EPI_COLSUM = 256,   // bf16 out only: colsum[N] += column sums of the stored output (set by aitj_gemm_set_colsum)
  EPI_XENT = 512,     // no [M, N] output: per-row cross-entropy partials of the logits (set by aitj_gemm_set_xent)
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
  int split_k;
  int tiles_m, tiles_n;
  int k_blocks, k_per_split;
  // EPI_COLSUM: colsum[N] += column sums of the stored output, i.e. the bias gradient of the layer whose input gradient
  // this GEMM produces
  float* colsum;
  // EPI_XENT: for row r and 128-column block b, xent_part[r * xent_ld + b] <- (max, sum of exp(x - max)) over the
  // block's columns below xent_vocab; xent_tgt[r] <- the logit of column xent_target[r].  Rows with a negative target
  // are skipped.
  const int64_t* xent_target;
  float2* xent_part;
  float* xent_tgt;
  int xent_vocab, xent_ld;
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

template <int kEpi>
__host__ __device__ constexpr bool bf16_out() { return (kEpi & (EPI_OUT_F32 | EPI_ACCUM)) == 0; }
// bf16 epilogues that read a second [M, ldc] input: the residual, or the saved pre-activation for GELU'
template <int kEpi>
__host__ __device__ constexpr bool epi_reads() { return (kEpi & (EPI_RESIDUAL | EPI_DGELU)) != 0; }

// fp32 epilogue of one consumer warpgroup: its 64 rows x kBN columns of accumulators in the wgmma fragment layout --
// register 4j + 2h + e holds row (r_base + 8h), column (c_base + 8j + e).
template <int kBN, int kEpi>
__device__ __forceinline__ void epilogue_f32(const GemmArgs& a, float (&acc)[kBN / 2], int r_base, int c_base) {
  constexpr int flags = kEpi;
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
      if constexpr (!(flags & EPI_ACCUM)) {
        *reinterpret_cast<float2*>(p) = make_float2(x0, x1);
      } else if constexpr ((flags & EPI_MC) != 0) {
        mc_red_add_f32(p, x0);
        mc_red_add_f32(p + 1, x1);
      } else {
        red_add_v2_f32((flags & EPI_PEER) ? peer_ptr(p) : p, x0, x1);
      }
    }
  }
}

// Cross-entropy epilogue of one consumer warpgroup (EPI_XENT): the logits never leave the registers.  Each thread holds
// two rows (r_base, r_base + 8) x kBN / 4 columns in the layout of epilogue_f32; the four lanes of a quad share a row,
// so a row's (max, sum of exp) over a 128-column block is the quad's combination of its lanes' 32 values.  Lane 0 of
// the quad stores the pair with one plain 8-byte store, and the lane holding the target column stores its logit: no
// atomics, and each (row, block) and each row's target logit is written by exactly one thread.
template <int kBN>
__device__ __forceinline__ void epilogue_xent(const GemmArgs& a, const float (&acc)[kBN / 2], int r_base, int c_base,
                                              int n0) {
  constexpr float kLog2e = 1.4426950408889634f;
  constexpr int kBlocks = kBN / 128;
  const bool leader = (threadIdx.x & 3) == 0;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = r_base + 8 * h;
    // a padding row (negative target) or a row past M stores nothing; its quad still joins the shuffles, which take
    // the whole warp
    const long long tgt = row < a.M ? a.xent_target[row] : -1;
    const bool live = tgt >= 0;
#pragma unroll
    for (int b = 0; b < kBlocks; ++b) {
      const int blk_col0 = n0 + 128 * b;
      if (blk_col0 >= a.N) break;
      float mx = -INFINITY;
#pragma unroll
      for (int j = 16 * b; j < 16 * b + 16; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (c_base + 8 * j + e < a.xent_vocab) mx = fmaxf(mx, acc[4 * j + 2 * h + e]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      // a block wholly past the vocabulary keeps (-inf, 0); the finish kernel skips such pairs
      const float moff = mx == -INFINITY ? 0.f : mx * kLog2e;
      float sum = 0.f;
#pragma unroll
      for (int j = 16 * b; j < 16 * b + 16; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (c_base + 8 * j + e < a.xent_vocab) sum += exp2f(fmaf(acc[4 * j + 2 * h + e], kLog2e, -moff));
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      if (live && leader) a.xent_part[static_cast<size_t>(row) * a.xent_ld + (blk_col0 >> 7)] = make_float2(mx, sum);
    }
    // the target column: register 4j + 2h + e of the lane whose quad offset covers it
    const long long off = tgt - c_base;
    if (live && off >= 0 && off < kBN && (off & 7) < 2) {
      const int jt = static_cast<int>(off >> 3), et = static_cast<int>(off & 1);
      float x = 0.f;
#pragma unroll
      for (int j = 0; j < kBN / 8; ++j)
        if (j == jt) x = et ? acc[4 * j + 2 * h + 1] : acc[4 * j + 2 * h];
      a.xent_tgt[row] = x;
    }
  }
}

// bf16 epilogues leave through shared memory.  Each consumer warpgroup owns two 8 KB slots; a slot holds one 64 x 64
// box of a bf16 tensor map with SWIZZLE_128B (row r at byte 128 r, its 16-byte chunk c at chunk c ^ (r % 8)), so the
// stmatrix / ldmatrix rows of one 8 x 8 matrix fall on eight different chunks and never share a bank.  The warpgroup
// stages its 64 x kBN share one box ("unit") at a time, alternating slots, and one thread stores each box with TMA:
// whole 128-byte lines leave in the background instead of 8-row x 16-byte scattered stores, and the tensor map's
// bounds clip the M and N tails.  The warpgroup never waits for a store's writes, only (before it reuses a slot) for
// the store to have read the slot.  RESIDUAL and DGELU inputs arrive by TMA in the slot their output leaves from.
constexpr int kSlotBytes = 64 * 64 * 2;
constexpr int kStagingBytes = 2 * 2 * kSlotBytes;   // 2 consumer warpgroups x 2 slots

struct Staging {
  uint8_t* slots;      // this warpgroup's two slots
  uint64_t* in_bar;    // [2]: a slot's input box has landed (RESIDUAL / DGELU)
  uint32_t unit;       // boxes staged so far; box u goes through slot u % 2
  uint32_t in_phase;   // parity of each in_bar
  int wg;
  bool issuer;         // thread 0 of the warpgroup issues its TMA loads and stores
};

// Shared address of the 16-byte row of fragment group p (columns 16p .. 16p + 15 of a box) that this lane gives to
// stmatrix / ldmatrix: lanes 8i .. 8i + 7 address the rows of matrix i = (8-column half i / 2, 8-row half i % 2).
__device__ __forceinline__ uint32_t box_addr(const uint8_t* slot, int p) {
  const int lane = threadIdx.x & 31;
  const int row = ((threadIdx.x >> 5) & 3) * 16 + (lane & 8) + (lane & 7);
  return smem_u32(slot) + row * 128 + (((2 * p + (lane >> 4)) ^ (lane & 7)) << 4);
}

// Load the input box at column c0, row m0 into slot s, the slot its output will leave from.
__device__ __forceinline__ void load_input_box(Staging& st, const CUtensorMap* in_map, uint32_t s, int c0, int m0) {
  mbar_arrive_expect_tx(&st.in_bar[s], kSlotBytes);
  tma_load_2d(st.slots + s * kSlotBytes, in_map, &st.in_bar[s], c0, m0);
}

// Stage box `cb` (columns n0 + 64 cb ..) of the warpgroup's share in the next slot and store it through `map`: the
// pre-activation if kPre, else the epilogue's output, computed exactly as a register epilogue would, in the same order.
// The box is written in four 16-column groups, one stmatrix each, so that only four packed registers are live beside
// the accumulators.
template <int kBN, int kEpi, bool kPre>
__device__ __forceinline__ void stage_box(const GemmArgs& a, const CUtensorMap* map, const CUtensorMap* in_map,
                                          float (&acc)[kBN / 2], Staging& st, int cb, int m0, int n0) {
  constexpr int flags = kEpi;
  constexpr bool kReads = epi_reads<kEpi>() && !kPre;
  const int lane = threadIdx.x & 31;
  const int row = m0 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);   // rows row and row + 8 of the fragments
  const uint32_t s = st.unit & 1u;
  uint8_t* slot = st.slots + s * kSlotBytes;
  if constexpr (kReads) {
    mbar_wait(&st.in_bar[s], (st.in_phase >> s) & 1u);
    st.in_phase ^= 1u << s;
  }
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    uint32_t v[4];   // matrix i of the group: pair (j = 8 cb + 2p + i / 2, h = i % 2) of the register layout
    if constexpr (kReads) ldmatrix_x4(box_addr(slot, p), v);
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int j = 8 * cb + 2 * p + q;
      const int col = n0 + 8 * j + 2 * (lane & 3);
      float2 bv = make_float2(0.f, 0.f);
      if constexpr ((flags & EPI_BIAS) != 0)
        if (col < a.N) bv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(a.bias + col));
      float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float x0 = acc[4 * j + 2 * h] + bv.x, x1 = acc[4 * j + 2 * h + 1] + bv.y;
        if constexpr (kPre) {
          v[2 * q + h] = pack_bf16x2(x0, x1);
          continue;
        }
        if constexpr ((flags & EPI_GELU) != 0) { x0 = gelu_tanh(x0); x1 = gelu_tanh(x1); }
        if constexpr ((flags & EPI_DGELU) != 0) {
          const float2 pre = unpack_bf16x2(v[2 * q + h]);
          x0 *= gelu_tanh_grad(pre.x);
          x1 *= gelu_tanh_grad(pre.y);
        }
        if constexpr ((flags & EPI_RESIDUAL) != 0) {
          const float2 r = unpack_bf16x2(v[2 * q + h]);
          x0 += r.x;
          x1 += r.y;
        }
        const uint32_t packed = pack_bf16x2(x0, x1);
        v[2 * q + h] = packed;
        if constexpr ((flags & EPI_COLSUM) != 0) {
          if (row + 8 * h < a.M) {
            const float2 stored = unpack_bf16x2(packed);
            cs0 += stored.x;
            cs1 += stored.y;
          }
        }
      }
      if constexpr (!kPre && (flags & EPI_COLSUM) != 0) {
        // the eight lanes with the same (lane & 3) hold the same two columns of the warp's 16 rows
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          cs0 += __shfl_xor_sync(0xffffffffu, cs0, o);
          cs1 += __shfl_xor_sync(0xffffffffu, cs1, o);
        }
        if (lane < 4 && col < a.N) {
          atomicAdd(a.colsum + col, cs0);
          atomicAdd(a.colsum + col + 1, cs1);
        }
      }
    }
    stmatrix_x4(box_addr(slot, p), v[0], v[1], v[2], v[3]);
  }
  fence_proxy_async_smem();
  // the previous box's store has read the other slot: once the barrier is passed, the next box may be written there
  if (st.issuer) tma_store_wait_read<0>();
  named_bar_sync(1 + st.wg, 128);
  if (st.issuer) {
    tma_store_2d(map, slot, n0 + 64 * cb, m0);
    tma_store_commit();
    // this slot receives the input of the box after next once the store has read it
    if (kReads && cb + 2 < kBN / 64 && n0 + 64 * (cb + 2) < a.N) {
      tma_store_wait_read<0>();
      load_input_box(st, in_map, s, n0 + 64 * (cb + 2), m0);
    }
  }
  ++st.unit;
}

// bf16 epilogue of one consumer warpgroup: rows m0 .. m0 + 63, columns n0 .. n0 + kBN - 1, accumulators in the
// register layout of epilogue_f32.
template <int kBN, int kEpi>
__device__ __forceinline__ void epilogue_bf16(const GemmArgs& a, const CUtensorMap* out_map, const CUtensorMap* aux_map,
                                              const CUtensorMap* in_map, float (&acc)[kBN / 2], Staging& st, int m0,
                                              int n0) {
#pragma unroll
  for (int cb = 0; cb < kBN / 64; ++cb) {
    if (n0 + 64 * cb >= a.N) break;
    if constexpr ((kEpi & EPI_SAVE_PRE) != 0) stage_box<kBN, kEpi, true>(a, aux_map, in_map, acc, st, cb, m0, n0);
    stage_box<kBN, kEpi, false>(a, out_map, in_map, acc, st, cb, m0, n0);
  }
}

template <int kBN>
__host__ __device__ constexpr int gemm_stages() { return kBN == 256 ? 4 : 6; }
template <int kBN, int kEpi>
__host__ __device__ constexpr int gemm_smem_bytes() {
  return gemm_stages<kBN>() * (BLOCK_M + kBN) * BLOCK_K * 2 + (bf16_out<kEpi>() ? kStagingBytes : 0) + 1024 + 256;
}

template <int kBN, bool kAMN, bool kBMN, int kCM, int kEpi>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_aux,
                       const __grid_constant__ CUtensorMap tmap_res, const GemmArgs args) {
  constexpr int kStages = gemm_stages<kBN>();
  constexpr int kStageA = BLOCK_M * BLOCK_K * 2;
  constexpr int kStageB = kBN * BLOCK_K * 2;
  constexpr int kStageBytes = kStageA + kStageB;
  constexpr int kSliceN = kBN / kCM;               // rows of the B tile this CTA loads and multicasts
  static_assert(!kBMN || kSliceN % 64 == 0, "MN-major B slices are whole 64-column chunks");
  static_assert(!(kEpi & EPI_RESIDUAL) || !(kEpi & (EPI_DGELU | EPI_SAVE_PRE)), "one second bf16 tensor per epilogue");
  static_assert(!(kEpi & EPI_DGELU) || !(kEpi & EPI_SAVE_PRE), "one second bf16 tensor per epilogue");
  static_assert(!(kEpi & EPI_XENT) || kEpi == (EPI_XENT | EPI_OUT_F32), "the cross-entropy epilogue combines with no other");
  constexpr int kStaging = bf16_out<kEpi>() ? kStagingBytes : 0;
  const CUtensorMap* in_map = (kEpi & EPI_RESIDUAL) ? &tmap_res : &tmap_aux;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* staging = smem + kStages * kStageBytes;   // 1024-aligned: every stage is a multiple of 1024 bytes
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + kStaging);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* in_bar = empty_bar + kStages;             // [2 warpgroups][2 slots]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = kCM > 1 ? cluster_ctarank() : 0u;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if constexpr (bf16_out<kEpi>()) tma_prefetch_desc(&tmap_out);
    if constexpr ((kEpi & EPI_SAVE_PRE) != 0) tma_prefetch_desc(&tmap_aux);
    if constexpr (epi_reads<kEpi>()) tma_prefetch_desc(in_map);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);          // this CTA's producer: arrive(expect_tx) + the bytes of A and all B slices
      mbar_init(&empty_bar[i], 2 * kCM);   // both consumer warpgroups of every CTA of the cluster
    }
    if constexpr (epi_reads<kEpi>())
      for (int i = 0; i < 4; ++i) mbar_init(&in_bar[i], 1);   // the warpgroup's issuer: arrive(expect_tx) + one box
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
    // lane c of the warpgroup's first warp frees the stage in CTA c of the cluster
    const bool signaller = (threadIdx.x & 127) < kCM;
    float acc[kBN / 2];
    int stage = 0;
    uint32_t phase = 0;
    Staging st{staging + wg * 2 * kSlotBytes, in_bar + 2 * wg, 0u, 0u, wg, (threadIdx.x & 127) == 0};
    auto release = [&](int s) {
      if (signaller) {
        if constexpr (kCM > 1) mbar_arrive_remote(&empty_bar[s], static_cast<uint32_t>(lane));
        else mbar_arrive(&empty_bar[s]);
      }
    };
    for (int w = cluster_id; w < num_work; w += num_clusters) {
      const WorkItem wi = decode_work(sched, w);
      const int nk = wi.kb1 - wi.kb0;
      const int m0 = (wi.m_blk * kCM + static_cast<int>(rank)) * BLOCK_M + wg * 64;   // this warpgroup's rows
      const int n0 = wi.n_blk * kBN;
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
        if constexpr (epi_reads<kEpi>()) {
          // the epilogue's first two input boxes load under the first k-block's MMAs, as soon as the previous tile's
          // last stores have read their slots
          if (kb == 0 && st.issuer && m0 < args.M) {
            tma_store_wait_read<0>();
#pragma unroll
            for (int cb = 0; cb < 2; ++cb)
              if (n0 + 64 * cb < args.N) load_input_box(st, in_map, (st.unit + cb) & 1u, n0 + 64 * cb, m0);
          }
        }
        wgmma_wait<1>();            // the previous stage's MMAs have retired: its buffers can be refilled
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0) release(prev);
      if (nk > 0) {
        if constexpr (bf16_out<kEpi>()) {
          if (m0 < args.M) epilogue_bf16<kBN, kEpi>(args, &tmap_out, &tmap_aux, in_map, acc, st, m0, n0);
        } else if constexpr ((kEpi & EPI_XENT) != 0) {
          epilogue_xent<kBN>(args, acc, m0 + (warp & 3) * 16 + (lane >> 2), n0 + 2 * (lane & 3), n0);
        } else {
          epilogue_f32<kBN, kEpi>(args, acc, m0 + (warp & 3) * 16 + (lane >> 2), n0 + 2 * (lane & 3));
        }
      }
    }
    // the shared memory of the last stores stays valid until they have read it
    if constexpr (bf16_out<kEpi>())
      if (st.issuer) tma_store_wait_read<0>();
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

// The operands' tensor maps and, for bf16 outputs, those of the epilogue's tensors (64 x 64 boxes); maps a variant does
// not use stay zero.
struct GemmMaps {
  CUtensorMap a, b, out, aux, res;
};

template <int kBN, bool kAMN, bool kBMN, int kCM, int kEpi>
static int launch_gemm(const GemmMaps& maps, const GemmArgs& args, int max_ctas, cudaStream_t stream) {
  constexpr int kSmem = gemm_smem_bytes<kBN, kEpi>();
  static int max_clusters = 0;
  auto kern = gemm_bf16_wgmma_kernel<kBN, kAMN, kBMN, kCM, kEpi>;
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
  if (cudaLaunchKernelEx(&cfg, kern, maps.a, maps.b, maps.out, maps.aux, maps.res, args) != cudaSuccess) return -30;
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -30;
}

typedef int (*LaunchFn)(const GemmMaps&, const GemmArgs&, int, cudaStream_t);

struct GemmKernel {
  bool a_mn, b_mn;
  int epi;            // EPI_* bits, EPI_COLSUM included
  int block_n, cm;    // tile width and CTAs per cluster
  LaunchFn launch;
};

// Every tile configuration of one (operand layout, epilogue) pair: 128- and 256-wide tiles on single CTAs, and 256-wide
// tiles in clusters of 2 and 4.
#define GEMM_TILES(AMN, BMN, EPI)                          \
  {AMN, BMN, EPI, 128, 1, launch_gemm<128, AMN, BMN, 1, EPI>},  \
  {AMN, BMN, EPI, 256, 1, launch_gemm<256, AMN, BMN, 1, EPI>},  \
  {AMN, BMN, EPI, 256, 2, launch_gemm<256, AMN, BMN, 2, EPI>},  \
  {AMN, BMN, EPI, 256, 4, launch_gemm<256, AMN, BMN, 4, EPI>}

// The kernels aitj_gemm_bf16 can launch: the epilogues GPT2Engine and BertEngine use (BERT shares GPT-2's GEMM
// front-ends) and the ones ops/selfcheck.py checks.
static const GemmKernel kGemmKernels[] = {
    // forward, x[M,K] @ W[N,K]^T: logits; qkv; fc (+ GELU, pre-activation saved); attn proj and fc2 (+ skip connection)
    GEMM_TILES(false, false, 0),
    GEMM_TILES(false, false, EPI_BIAS),
    GEMM_TILES(false, false, EPI_BIAS | EPI_GELU | EPI_SAVE_PRE),
    GEMM_TILES(false, false, EPI_BIAS | EPI_RESIDUAL),
    // evaluation: the logits GEMM with the cross-entropy epilogue (GPT2Engine.eval_forward); its only outputs are fp32
    // plain stores (the partials), so its kernel is keyed as an fp32 variant: no staging slots, no TMA store
    GEMM_TILES(false, false, EPI_XENT | EPI_OUT_F32),
    // epilogues of the other layouts, checked on this one (selfcheck)
    GEMM_TILES(false, false, EPI_DGELU),
    GEMM_TILES(false, false, EPI_DGELU | EPI_COLSUM),
    GEMM_TILES(false, false, EPI_OUT_F32),
    GEMM_TILES(false, false, EPI_ACCUM),
    // input gradient, dy[M,N] @ W[N,K]: fc2 (* GELU', + fc bias gradient); qkv with the skip connection's gradient (BERT)
    GEMM_TILES(false, true, 0),
    GEMM_TILES(false, true, EPI_DGELU),
    GEMM_TILES(false, true, EPI_DGELU | EPI_COLSUM),
    GEMM_TILES(false, true, EPI_RESIDUAL),
    // weight gradient, dW[N,K] += dy[M,N]^T x[M,K]: local, NVSwitch multicast, owner-sharded
    GEMM_TILES(true, true, 0),
    GEMM_TILES(true, true, EPI_ACCUM),
    GEMM_TILES(true, true, EPI_ACCUM | EPI_MC),
    GEMM_TILES(true, true, EPI_ACCUM | EPI_PEER),
    GEMM_TILES(true, false, 0),
};
#undef GEMM_TILES

}  // namespace aitj

static float* g_gemm_colsum = nullptr;   // consumed by the next aitj_gemm_bf16 call
static struct {
  const int64_t* target;
  float2* part;
  float* tgt;
  int vocab;
} g_gemm_xent = {nullptr, nullptr, nullptr, 0};   // consumed by the next aitj_gemm_bf16 call

extern "C" {

// The next aitj_gemm_bf16 call (bf16 output) also accumulates the column sums of its output into buf[N] (fp32).
// One-shot: cleared by that call.
int aitj_gemm_set_colsum(void* buf) { g_gemm_colsum = reinterpret_cast<float*>(buf); return 0; }

// The next aitj_gemm_bf16 call with flags == EPI_XENT writes no output: for every row r with target[r] >= 0 (int64) it
// stores part[r, b] = (max, sum of exp(x - max)) (float2 [M, ceil(N / 128)]) over the columns c < vocab of each
// 128-column block b of row r of the product, and tgt_logit[r] (fp32) = its column target[r].  One-shot: cleared by
// that call.  aitj_xent_finish (fused_ops.cu) turns the partials into per-row losses.
int aitj_gemm_set_xent(const void* target, void* part, void* tgt_logit, int vocab) {
  g_gemm_xent.target = reinterpret_cast<const int64_t*>(target);
  g_gemm_xent.part = reinterpret_cast<float2*>(part);
  g_gemm_xent.tgt = reinterpret_cast<float*>(tgt_logit);
  g_gemm_xent.vocab = vocab;
  return 0;
}

// Returns 0 on success. See file header for operand conventions. lda/ldb/ldc in elements.
// block_n: 128 or 256 (0 = auto); 512 / 1024: 128x256 tiles in clusters of 2 / 4 CTAs sharing B by TMA multicast.
// split_k > 1 requires EPI_ACCUM. max_ctas: 0 = all SMs.  -7: no kernel is compiled for this operand layout and
// epilogue (kGemmKernels).  EPI_XENT (after aitj_gemm_set_xent) takes no other bit and no split, and `out` may be null;
// -8: it was asked for without its buffers, with another bit or a split, or with vocab outside [1, N].
int aitj_gemm_bf16(const void* A, const void* B, void* out, int M, int N, int K, int lda, int ldb, int ldc,
                   int a_mn, int b_mn, const void* bias, const void* residual, void* aux, int flags, int split_k,
                   int block_n, int max_ctas, void* stream_ptr) {
  using namespace aitj;
  // both one-shot buffers are taken before any refusal, so that a refused call cannot hand them to the next GEMM
  const auto xent = g_gemm_xent;
  g_gemm_xent = {nullptr, nullptr, nullptr, 0};
  float* const colsum = g_gemm_colsum;
  g_gemm_colsum = nullptr;
  if (flags & EPI_XENT) {
    // the max and the sum of exponentials of a row cannot be formed from the partial products of a K split
    if (flags != EPI_XENT || split_k > 1 || !xent.target || !xent.part || !xent.tgt || xent.vocab < 1 ||
        xent.vocab > N || (reinterpret_cast<uintptr_t>(xent.part) & 7))
      return -8;
  } else if (xent.target) {
    return -8;                                   // cross-entropy buffers given to a GEMM without EPI_XENT
  }
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((N & 7) || (ldc & 7) || (lda & 7) || (ldb & 7)) return -1;
  // TMA needs 16-byte aligned tensors
  if ((reinterpret_cast<uintptr_t>(out) & 15) ||
      ((flags & (EPI_SAVE_PRE | EPI_DGELU)) && (reinterpret_cast<uintptr_t>(aux) & 15)) ||
      ((flags & EPI_RESIDUAL) && (reinterpret_cast<uintptr_t>(residual) & 15)))
    return -4;
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
  args.colsum = colsum;
  if (args.colsum && (flags & (EPI_OUT_F32 | EPI_ACCUM | EPI_XENT))) return -6;   // column sums of a bf16 output only
  args.xent_target = xent.target;
  args.xent_part = xent.part;
  args.xent_tgt = xent.tgt;
  args.xent_vocab = xent.vocab;
  args.xent_ld = (N + 127) / 128;
  args.tiles_m = (M + BLOCK_M - 1) / BLOCK_M;
  args.tiles_n = (N + block_n - 1) / block_n;
  args.k_blocks = (K + BLOCK_K - 1) / BLOCK_K;
  if (split_k < 1) split_k = 1;
  if (split_k > args.k_blocks) split_k = args.k_blocks;
  args.k_per_split = (args.k_blocks + split_k - 1) / split_k;
  args.split_k = (args.k_blocks + args.k_per_split - 1) / args.k_per_split;
  const bool peer_move = (flags & EPI_PEER) && args.split_k > 1;
  int epi = flags & ~EPI_COLSUM;
  if (args.colsum) epi |= EPI_COLSUM;
  if (flags & EPI_XENT) epi |= EPI_OUT_F32;
  if (peer_move) epi &= ~EPI_PEER;
  const GemmKernel* kernel = nullptr;
  for (const GemmKernel& k : kGemmKernels)
    if (k.a_mn == (a_mn != 0) && k.b_mn == (b_mn != 0) && k.epi == epi && k.block_n == block_n && k.cm == cm) kernel = &k;
  if (!kernel) return -7;

  GemmMaps maps;
  memset(&maps, 0, sizeof(maps));
  int rc;
  if (!a_mn) rc = encode_2d(&maps.a, A, K, M, lda, BLOCK_K, BLOCK_M);
  else       rc = encode_2d(&maps.a, A, M, K, lda, 64, BLOCK_K);
  if (rc) return rc;
  if (!b_mn) rc = encode_2d(&maps.b, B, K, N, ldb, BLOCK_K, block_n / cm);
  else       rc = encode_2d(&maps.b, B, N, K, ldb, 64, BLOCK_K);
  if (rc) return rc - 1000;
  if (!(flags & (EPI_OUT_F32 | EPI_ACCUM | EPI_XENT))) {
    rc = encode_2d(&maps.out, out, N, M, ldc, 64, 64);
    if (!rc && (flags & (EPI_SAVE_PRE | EPI_DGELU))) rc = encode_2d(&maps.aux, aux, N, M, ldc, 64, 64);
    if (!rc && (flags & EPI_RESIDUAL)) rc = encode_2d(&maps.res, residual, N, M, ldc, 64, 64);
    if (rc) return rc - 2000;
  }
  rc = kernel->launch(maps, args, max_ctas, stream);
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

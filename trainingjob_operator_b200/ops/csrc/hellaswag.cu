// HellaSwag scoring of completions packed as documents into training-shaped rows (sm_90a).
//
// runtime/hellaswag.py packs every completion (context + one ending) of an example into consecutive positions of a
// row, as a document of its own; the attention sees it through the document mask (attention_wgmma.cu's doc_start).
// Two kernels complete the forward:
//
// * embedding_doc_fwd: out[r] = wte[tok[r]] + wpe[(r mod T) - doc_start[r]], the embedding with positions counted from
//   each document's first token, so a completion is embedded as if it stood alone at position 0 of a row.
// * choice_score: one warp per example turns the per-token NLL of the completions' ending-predicting positions (what
//   aitj_xent_finish leaves in the loss vector) into each completion's mean NLL, picks the lowest (the first on a tie)
//   and adds (correct, examples) to an fp64 accumulator with one atomic each per block.
//
// The C entry points refuse nothing: ops/functional.py checks every argument before it calls them.
#include "ptx.cuh"

namespace aitj {
namespace hellaswag {

constexpr int kChoices = 4;
constexpr int kScoreWarps = 8;

__global__ void __launch_bounds__(256) embedding_doc_fwd_kernel(const int64_t* __restrict__ tok,
                                                                const __nv_bfloat16* __restrict__ wte,
                                                                const __nv_bfloat16* __restrict__ wpe,
                                                                const int* __restrict__ doc_start,
                                                                __nv_bfloat16* __restrict__ out, int M, int T, int C) {
  const int vec_per_row = C / 8;
  const size_t total = static_cast<size_t>(M) * vec_per_row;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(i / vec_per_row), c = static_cast<int>(i % vec_per_row) * 8;
    const int pos = m % T - doc_start[m];
    const uint4 a = *reinterpret_cast<const uint4*>(wte + tok[m] * C + c);
    const uint4 b = *reinterpret_cast<const uint4*>(wpe + static_cast<size_t>(pos) * C + c);
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 fa = unpack_bf16x2(aw[j]), fb = unpack_bf16x2(bw[j]);
      ow[j] = pack_bf16x2(fa.x + fb.x, fa.y + fb.y);
    }
    *reinterpret_cast<uint4*>(out + static_cast<size_t>(m) * C + c) = o;
  }
}

// spans int2 [E, 4]: (first row, rows) of each completion's ending-predicting positions in `loss`.  The sum of a
// completion runs in a fixed order (lane-strided fp64 partials, then a butterfly), so a completion's mean depends only on
// its own losses, not on where it was packed or how many ranks share the work.
__global__ void __launch_bounds__(kScoreWarps * 32) choice_score_kernel(const float* __restrict__ loss,
                                                                        const int2* __restrict__ spans,
                                                                        const int* __restrict__ labels, int E,
                                                                        float* __restrict__ mean,
                                                                        double* __restrict__ acc) {
  __shared__ int correct[kScoreWarps], seen[kScoreWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int e = blockIdx.x * kScoreWarps + warp;
  int ok = 0;
  if (e < E) {
    float best = 0.f;
    int pick = 0;
#pragma unroll
    for (int c = 0; c < kChoices; ++c) {
      const int2 sp = spans[e * kChoices + c];
      double s = 0.0;
      for (int i = lane; i < sp.y; i += 32) s += loss[sp.x + i];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float m = static_cast<float>(s / sp.y);
      if (c == 0 || m < best) { best = m; pick = c; }
      if (lane == 0) mean[e * kChoices + c] = m;
    }
    ok = pick == labels[e];
  }
  if (lane == 0) { correct[warp] = ok; seen[warp] = e < E; }
  __syncthreads();
  if (threadIdx.x < 2) {
    int t = 0;
#pragma unroll
    for (int w = 0; w < kScoreWarps; ++w) t += threadIdx.x == 0 ? correct[w] : seen[w];
    if (t != 0) atomicAdd(acc + threadIdx.x, static_cast<double>(t));
  }
}

}  // namespace hellaswag
}  // namespace aitj

extern "C" {
using namespace aitj::hellaswag;

// out[r] = wte[tok[r]] + wpe[(r mod T) - doc_start[r]] (bf16 [M, C], fp32 sum; tok int64, doc_start int32 [M]).
int aitj_embedding_doc_fwd(const void* tok, const void* wte, const void* wpe, const void* doc_start, void* out, int M,
                           int T, int C, void* stream) {
  if (M <= 0 || C <= 0) return 0;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const size_t total = static_cast<size_t>(M) * (C / 8);
  size_t blocks = (total + 255) / 256;
  if (blocks > static_cast<size_t>(sms) * 16) blocks = static_cast<size_t>(sms) * 16;
  embedding_doc_fwd_kernel<<<static_cast<int>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const int64_t*>(tok), reinterpret_cast<const __nv_bfloat16*>(wte),
      reinterpret_cast<const __nv_bfloat16*>(wpe), reinterpret_cast<const int*>(doc_start),
      reinterpret_cast<__nv_bfloat16*>(out), M, T, C);
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -30;
}

// mean fp32 [E, 4] <- the mean of loss[first, first + rows) of each completion (spans int32 [E, 4, 2]); acc fp64 [2] +=
// (examples whose lowest mean, the first on a tie, is labels[e], examples).
int aitj_choice_score(const void* loss, const void* spans, const void* labels, int E, void* mean, void* acc,
                      void* stream) {
  if (E <= 0) return 0;
  choice_score_kernel<<<(E + kScoreWarps - 1) / kScoreWarps, kScoreWarps * 32, 0,
                        reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float*>(loss), reinterpret_cast<const int2*>(spans), reinterpret_cast<const int*>(labels),
      E, reinterpret_cast<float*>(mean), reinterpret_cast<double*>(acc));
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -30;
}

}  // extern "C"

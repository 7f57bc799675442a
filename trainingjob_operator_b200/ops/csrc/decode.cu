// Autoregressive decoding of GPT-2 on a KV cache (sm_90a): one decode step of S sequences in lockstep.
//
// The S sequences share their position `pos`, which lives in device memory (int32): the host never passes it, so one
// captured decode step (embedding -> layers -> logits -> sampling -> pos + 1) is replayed for every token.
//
// * attention_decode: the new token's k and v go into the layer's cache at `pos`, and its q attends over cache positions
//   [0, pos].  Flash-decoding: the keys are split into 64-position chunks, one CTA per (chunk, head, sequence) streams
//   its chunk of K and V into shared memory with cp.async and leaves a partial (max, sum, acc); a second kernel merges
//   the partials of each (head, sequence).  The grid is sized for the cache length, so CTAs whose chunk starts past
//   `pos` exit at once and a replay stays correct as `pos` grows; at S = 1 the grid still has H x (pos / 64 + 1) CTAs.
// * embedding_decode: x[s] = wte[tok[s]] + wpe[pos].
// * sample_tokens: one CTA per sequence over its bf16 logits row (staged in shared memory): greedy argmax, or a draw
//   from softmax(logits / temperature) restricted to the top_k largest (radix select on the bf16 bits, -0 equal to +0),
//   keyed by a counter-based Philox of (seed, sequence, pos); prompt positions are forced.  The last CTA to finish moves
//   `pos` on.
//
// The C entry points refuse nothing: ops/functional.py checks every argument before it calls them.
#include "ptx.cuh"

namespace aitj {
namespace decode {

constexpr int kHeadDim = 64;
constexpr int kChunk = 64;                 // cache positions per attention CTA
constexpr int kAttnThreads = 128;
constexpr int kSampleThreads = 1024;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}

// ------------------------------------------------------------------ attention, one decode step
// qkv [S, 3C] (q | k | v, head-major inside each), cache [S, Tmax, 2, H, 64], part fp32 [S, H, nsplit, 64 + 2].
// K / V rows of the chunk sit in shared memory with their 16-byte pieces XOR-swizzled by the row, so that the
// per-key dot products (one warp per key, two dims per lane) and the per-dim accumulation read without conflicts.
__global__ void __launch_bounds__(kAttnThreads) attention_decode_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                                        __nv_bfloat16* __restrict__ cache,
                                                                        const int* __restrict__ pos_p,
                                                                        float* __restrict__ part, int H, int Tmax,
                                                                        int nsplit) {
  const int split = blockIdx.x, h = blockIdx.y, s = blockIdx.z;
  const int pos = *pos_p;
  const int t0 = split * kChunk;
  if (t0 > pos) return;                    // past the current position: nothing to attend (grid sized for Tmax)
  const int C = H * kHeadDim;
  const int n = min(kChunk, pos + 1 - t0); // keys of this chunk
  __shared__ __align__(16) __nv_bfloat16 ks[kChunk][kHeadDim];
  __shared__ __align__(16) __nv_bfloat16 vs[kChunk][kHeadDim];
  __shared__ float sc[kChunk];
  __shared__ float qf[kHeadDim];
  __shared__ float red[2][kHeadDim];
  const int tid = threadIdx.x;
  const __nv_bfloat16* row_new = qkv + static_cast<size_t>(s) * 3 * C;
  const size_t seq_base = static_cast<size_t>(s) * Tmax * 2 * C;
  // stage the chunk: 8 16-byte pieces per row of K and of V; the row at `pos` comes from this step's qkv
  for (int i = tid; i < 2 * kChunk * 8; i += kAttnThreads) {
    const int kv = i / (kChunk * 8), r = (i / 8) % kChunk, piece = i % 8;
    if (r >= n) continue;
    const int t = t0 + r;
    __nv_bfloat16* dst = (kv ? &vs[r][0] : &ks[r][0]) + ((piece ^ (r & 7)) * 8);
    const __nv_bfloat16* src = t == pos ? row_new + (1 + kv) * C + h * kHeadDim + piece * 8
                                        : cache + seq_base + (static_cast<size_t>(t) * 2 + kv) * C + h * kHeadDim + piece * 8;
    cp_async16(dst, src);
  }
  if (tid < kHeadDim) qf[tid] = __bfloat162float(row_new[h * kHeadDim + tid]) * (0.125f * 1.4426950408889634f);
  if (t0 + kChunk > pos) {
    // this CTA holds position `pos`: it writes the new k and v of head h into the cache
    if (tid < 16) {
      const int kv = tid / 8, piece = tid % 8;
      const uint4 v = *reinterpret_cast<const uint4*>(row_new + (1 + kv) * C + h * kHeadDim + piece * 8);
      *reinterpret_cast<uint4*>(cache + seq_base + (static_cast<size_t>(pos) * 2 + kv) * C + h * kHeadDim + piece * 8) = v;
    }
  }
  cp_async_wait_all();
  __syncthreads();
  // scores (log2 domain): warp w takes keys w, w + 4, ...; lane l the dims 2l, 2l + 1
  const int warp = tid >> 5, lane = tid & 31;
  for (int r = warp; r < n; r += kAttnThreads / 32) {
    const int d = 2 * lane;
    const __nv_bfloat162 k2 = *reinterpret_cast<const __nv_bfloat162*>(&ks[r][((d / 8) ^ (r & 7)) * 8 + d % 8]);
    const float2 kf = __bfloat1622float2(k2);
    const float dot = warp_sum(kf.x * qf[d] + kf.y * qf[d + 1]);
    if (lane == 0) sc[r] = dot;
  }
  __syncthreads();
  float m = -INFINITY;
  for (int r = 0; r < n; ++r) m = fmaxf(m, sc[r]);
  // acc[d] over the chunk's keys: thread tid takes dim tid % 64 of keys of parity tid / 64
  const int d = tid % kHeadDim, half = tid / kHeadDim;
  float acc = 0.f;
  for (int r = half; r < n; r += 2) {
    const float p = exp2f(sc[r] - m);
    acc += p * __bfloat162float(vs[r][((d / 8) ^ (r & 7)) * 8 + d % 8]);
  }
  red[half][d] = acc;
  __syncthreads();
  float* out = part + ((static_cast<size_t>(s) * H + h) * nsplit + split) * (kHeadDim + 2);
  if (half == 0) {
    out[d] = acc + red[1][d];
    if (d == 0) {
      float lsum = 0.f;
      for (int r = 0; r < n; ++r) lsum += exp2f(sc[r] - m);
      out[kHeadDim] = m;
      out[kHeadDim + 1] = lsum;
    }
  }
}

// out[s, h*64 + d] = merged partials of the chunks [0, pos / 64]
__global__ void __launch_bounds__(kHeadDim) attention_decode_merge_kernel(const float* __restrict__ part,
                                                                          const int* __restrict__ pos_p,
                                                                          __nv_bfloat16* __restrict__ out, int H,
                                                                          int nsplit) {
  const int h = blockIdx.x, s = blockIdx.y, d = threadIdx.x;
  const int used = *pos_p / kChunk + 1;
  const float* p = part + (static_cast<size_t>(s) * H + h) * nsplit * (kHeadDim + 2);
  float M = -INFINITY;
  for (int i = 0; i < used; ++i) M = fmaxf(M, p[i * (kHeadDim + 2) + kHeadDim]);
  float L = 0.f, acc = 0.f;
  for (int i = 0; i < used; ++i) {
    const float* q = p + i * (kHeadDim + 2);
    const float w = exp2f(q[kHeadDim] - M);
    L += w * q[kHeadDim + 1];
    acc += w * q[d];
  }
  out[static_cast<size_t>(s) * H * kHeadDim + h * kHeadDim + d] = __float2bfloat16(acc / L);
}

// ------------------------------------------------------------------ embedding at the shared position
__global__ void __launch_bounds__(256) embedding_decode_kernel(const int64_t* __restrict__ tok,
                                                               const __nv_bfloat16* __restrict__ wte,
                                                               const __nv_bfloat16* __restrict__ wpe,
                                                               const int* __restrict__ pos_p,
                                                               __nv_bfloat16* __restrict__ out, int C) {
  const int s = blockIdx.x;
  const int64_t t = tok[s];
  const int pos = *pos_p;
  for (int c = threadIdx.x * 8; c < C; c += blockDim.x * 8) {
    const uint4 a = *reinterpret_cast<const uint4*>(wte + t * C + c);
    const uint4 b = *reinterpret_cast<const uint4*>(wpe + static_cast<size_t>(pos) * C + c);
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 fa = unpack_bf16x2(aw[j]), fb = unpack_bf16x2(bw[j]);
      ow[j] = pack_bf16x2(fa.x + fb.x, fa.y + fb.y);
    }
    *reinterpret_cast<uint4*>(out + static_cast<size_t>(s) * C + c) = o;
  }
}

// ------------------------------------------------------------------ sampling
// Philox4x32-10 (Salmon et al., SC'11): counter (pos, sequence, 0, 0), key (seed low, seed high) -> the first word.
__device__ __forceinline__ uint32_t philox_first_word(uint64_t seed, uint32_t seq, uint32_t pos) {
  uint32_t c0 = pos, c1 = seq, c2 = 0, c3 = 0;
  uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c0;
}

// order-preserving 16-bit key of a bf16 value: a larger value has a larger key, and -0 has the key of +0, 0x8000 (they
// are equal, so a -0 ties with a +0 top_k-th logit and is kept); a negative of magnitude m > 0 has 0x8000 - m
__device__ __forceinline__ uint32_t bf16_key(uint16_t b) {
  return (b & 0x8000u) ? (0x10000u - b) : (b | 0x8000u);
}

struct SampleArgs {
  const __nv_bfloat16* logits;
  int ld, vocab;
  int64_t* tok;                 // [S]: the next step's input
  int64_t* out;                 // [S, ld_out]
  int ld_out;
  const int64_t* prompt;        // [S, ld_prompt]
  int ld_prompt, prompt_len;
  int* pos;                     // pos[0]: position; pos[1]: CTAs done with this step (zero between steps)
  float temperature;
  int top_k;
  uint64_t seed;
  int first_seq;                // sequence index of row 0 (the Philox counter takes first_seq + row)
};

__device__ __forceinline__ void argmax_merge(float& v, int& i, float v2, int i2) {
  if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
}

__global__ void __launch_bounds__(kSampleThreads) sample_tokens_kernel(SampleArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint16_t* row = reinterpret_cast<uint16_t*>(smem_raw);
  __shared__ uint32_t hist[256];
  __shared__ float wv[32];
  __shared__ int wi[32];
  __shared__ float wsum[32];
  __shared__ int sel_token, sel_thread;
  __shared__ uint32_t thr_key, k_rem, bin_hi;
  const int s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nwarps = kSampleThreads / 32;
  const int pos = a.pos[0];
  const int V = a.vocab;
  int token;
  if (pos + 1 < a.prompt_len) {
    token = static_cast<int>(a.prompt[static_cast<size_t>(s) * a.ld_prompt + pos + 1]);   // prompt forcing
  } else {
    const uint16_t* src = reinterpret_cast<const uint16_t*>(a.logits + static_cast<size_t>(s) * a.ld);
    // stage the row (columns < vocab) and find the argmax, lowest index on ties
    float bv = -INFINITY;
    int bi = 0x7FFFFFFF;
    for (int c = tid; c < V; c += kSampleThreads) {
      const uint16_t b = src[c];
      row[c] = b;
      argmax_merge(bv, bi, __uint_as_float(static_cast<uint32_t>(b) << 16), c);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      argmax_merge(bv, bi, __shfl_xor_sync(0xffffffffu, bv, o), __shfl_xor_sync(0xffffffffu, bi, o));
    if (lane == 0) { wv[warp] = bv; wi[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
      bv = lane < nwarps ? wv[lane] : -INFINITY;
      bi = lane < nwarps ? wi[lane] : 0x7FFFFFFF;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
        argmax_merge(bv, bi, __shfl_xor_sync(0xffffffffu, bv, o), __shfl_xor_sync(0xffffffffu, bi, o));
      if (lane == 0) { wv[0] = bv; wi[0] = bi; }
    }
    __syncthreads();
    const float zmax = wv[0];
    const int amax = wi[0];
    if (a.temperature == 0.f || a.top_k == 1) {
      token = amax;
    } else {
      // threshold key: the top_k-th largest logit (radix select, high byte then low byte); 0 keeps every column
      uint32_t thr = 0;
      if (a.top_k > 0 && a.top_k < V) {
        for (int pass = 0; pass < 2; ++pass) {
          for (int i = tid; i < 256; i += kSampleThreads) hist[i] = 0;
          __syncthreads();
          for (int c = tid; c < V; c += kSampleThreads) {
            const uint32_t k = bf16_key(row[c]);
            if (pass == 0) atomicAdd(&hist[k >> 8], 1u);
            else if ((k >> 8) == bin_hi) atomicAdd(&hist[k & 0xFFu], 1u);
          }
          __syncthreads();
          if (tid == 0) {
            const uint32_t want = pass == 0 ? static_cast<uint32_t>(a.top_k) : k_rem;
            uint32_t cum = 0;
            int b = 255;
            for (; b > 0 && cum + hist[b] < want; --b) cum += hist[b];
            if (pass == 0) { bin_hi = b; k_rem = want - cum; }
            else thr_key = (bin_hi << 8) | b;
          }
          __syncthreads();
        }
        thr = thr_key;
      }
      // p(c) = exp((z_c - zmax) / T) over the kept columns; each thread sums a contiguous run of columns, so the
      // prefix over threads orders the columns
      const float scale = 1.4426950408889634f / a.temperature;
      const int per = (V + kSampleThreads - 1) / kSampleThreads;
      const int c0 = min(V, tid * per), c1 = min(V, c0 + per);
      float part = 0.f;
      for (int c = c0; c < c1; ++c)
        if (bf16_key(row[c]) >= thr) part += exp2f((__uint_as_float(static_cast<uint32_t>(row[c]) << 16) - zmax) * scale);
      // inclusive scan over the threads
      float incl = part;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      if (lane == 31) wsum[warp] = incl;
      if (tid == 0) sel_thread = -1;
      __syncthreads();
      if (warp == 0) {
        float w = lane < nwarps ? wsum[lane] : 0.f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const float y = __shfl_up_sync(0xffffffffu, w, o);
          if (lane >= o) w += y;
        }
        if (lane < nwarps) wsum[lane] = w;
      }
      __syncthreads();
      if (warp > 0) incl += wsum[warp - 1];
      const float excl = incl - part;
      const float total = wsum[nwarps - 1];
      const uint32_t r = philox_first_word(a.seed, static_cast<uint32_t>(a.first_seq + s), static_cast<uint32_t>(pos));
      float target = static_cast<float>(r >> 8) * (1.0f / 16777216.0f) * total;    // [0, total)
      if (!(target < total)) target = nextafterf(total, 0.f);
      // The run holding the target belongs to the last thread with nonzero mass whose exclusive prefix does not pass
      // it.  The threads' [excl, incl) do not tile [0, total): the tree-ordered sums round differently, so neighbours
      // can overlap or leave a gap of an ulp, and even taking excl from the predecessor's incl would not do, since the
      // scan is not monotone (a thread with no mass can end below the one before it).  This rule gives every target
      // exactly one owner whenever the row has mass: the first thread with mass has excl 0.
      const unsigned starts = __ballot_sync(0xffffffffu, part > 0.f && excl <= target);
      if (lane == 0 && starts) atomicMax(&sel_thread, warp * 32 + 31 - __clz(starts));
      __syncthreads();
      if (tid == sel_thread) {
        // a target past the run's rounded sum takes its last column of nonzero probability
        float accp = excl;
        int pick = -1, last = -1;
        for (int c = c0; c < c1; ++c) {
          if (bf16_key(row[c]) < thr) continue;
          const float p = exp2f((__uint_as_float(static_cast<uint32_t>(row[c]) << 16) - zmax) * scale);
          if (p > 0.f) last = c;
          accp += p;
          if (target < accp) { pick = c; break; }
        }
        sel_token = pick >= 0 ? pick : last;
      }
      __syncthreads();
      token = sel_thread >= 0 ? sel_token : amax;
    }
  }
  if (tid == 0) {
    a.tok[s] = token;
    if (pos + 1 < a.ld_out) a.out[static_cast<size_t>(s) * a.ld_out + pos + 1] = token;
    // every CTA has read pos[0] before it counts itself done: the last one moves the shared position on
    __threadfence();
    const int done = atomicAdd(&a.pos[1], 1);
    if (done == static_cast<int>(gridDim.x) - 1) {
      a.pos[1] = 0;
      a.pos[0] = pos + 1;
      __threadfence();
    }
  }
}

}  // namespace decode
}  // namespace aitj

extern "C" {
using namespace aitj::decode;

// One decode step of one layer for S sequences at the position *pos (device int32): see attention_decode_kernel.
// part: fp32 scratch of S * H * ceil(Tmax / 64) * 66 elements.
int aitj_attention_decode(const void* qkv, void* cache, const void* pos, void* out, void* part, int S, int H, int Tmax,
                          void* stream) {
  if (S <= 0 || H <= 0 || Tmax <= 0) return 0;
  const int nsplit = (Tmax + kChunk - 1) / kChunk;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  attention_decode_kernel<<<dim3(nsplit, H, S), kAttnThreads, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(qkv), reinterpret_cast<__nv_bfloat16*>(cache),
      reinterpret_cast<const int*>(pos), reinterpret_cast<float*>(part), H, Tmax, nsplit);
  attention_decode_merge_kernel<<<dim3(H, S), kHeadDim, 0, st>>>(
      reinterpret_cast<const float*>(part), reinterpret_cast<const int*>(pos), reinterpret_cast<__nv_bfloat16*>(out), H,
      nsplit);
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -30;
}

// x[s] = wte[tok[s]] + wpe[*pos] (bf16 [S, C], fp32 sum).
int aitj_embedding_decode(const void* tok, const void* wte, const void* wpe, const void* pos, void* out, int S, int C,
                          void* stream) {
  if (S <= 0 || C <= 0) return 0;
  embedding_decode_kernel<<<S, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const int64_t*>(tok), reinterpret_cast<const __nv_bfloat16*>(wte),
      reinterpret_cast<const __nv_bfloat16*>(wpe), reinterpret_cast<const int*>(pos),
      reinterpret_cast<__nv_bfloat16*>(out), C);
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -30;
}

// The next token of each of S sequences from their logits rows (bf16 [S, ld], columns < vocab): tok[s] and
// out[s, *pos + 1] <- the prompt's token while *pos + 1 < prompt_len, else the argmax (temperature 0 or top_k 1) or a
// draw from softmax(logits / temperature) over the top_k largest (0 = all; ties with the top_k-th are kept), keyed by
// Philox(seed, first_seq + s, *pos).  Then *pos += 1; pos[1] counts finished CTAs and is zero again on exit.
int aitj_sample_tokens(const void* logits, int ld, int vocab, void* tok, void* out, int ld_out, const void* prompt,
                       int ld_prompt, int prompt_len, void* pos, float temperature, int top_k, long long seed,
                       int first_seq, int S, void* stream) {
  if (S <= 0) return 0;
  const int smem = ((vocab * 2 + 15) / 16) * 16;
  static int configured = 0;
  if (configured < smem) {
    if (cudaFuncSetAttribute(sample_tokens_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
      return -20;
    configured = smem;
  }
  SampleArgs a;
  a.logits = reinterpret_cast<const __nv_bfloat16*>(logits);
  a.ld = ld; a.vocab = vocab;
  a.tok = reinterpret_cast<int64_t*>(tok);
  a.out = reinterpret_cast<int64_t*>(out);
  a.ld_out = ld_out;
  a.prompt = reinterpret_cast<const int64_t*>(prompt);
  a.ld_prompt = ld_prompt; a.prompt_len = prompt_len;
  a.pos = reinterpret_cast<int*>(pos);
  a.temperature = temperature; a.top_k = top_k;
  a.seed = static_cast<uint64_t>(seed);
  a.first_seq = first_seq;
  sample_tokens_kernel<<<S, kSampleThreads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -30;
}

}  // extern "C"

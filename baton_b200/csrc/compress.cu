// Top-k sparsification with error feedback (parallel/compress.py): the exact, deterministic selection of the k
// largest-magnitude entries of a client update, and its compaction into the sparse wire format of the fused collective.
//
//   u = fl32(fl32(theta - global) + e)      (e: the client's residual; without error feedback u = theta - global)
//   key(x) = bits(x) & 0x7FFFFFFF, NaN -> 0x7FC00000 (above +inf); order: key descending, then index ascending
//
// Selection is a radix select on the 31-bit keys with integer counts, so its result depends on nothing but u:
//   hist0   u is computed and written to the u buffer (in place over e with error feedback); histogram of key >> 20
//   pick    one CTA finds the bucket that holds the k-th key: prefix bits and the count still needed inside it
//   hist1   histogram of bits 19..9 over the keys whose bits 30..20 match, pick
//   hist2   histogram of bits 8..0 over the keys whose bits 30..9 match, pick -> threshold key tau and the tie quota
//           q = k - #(key > tau): the first q elements with key == tau (by index) are kept
//   count   one warp per 1024-element granule counts key > tau and key == tau
//   scan    one CTA: ties before each granule, the ties it keeps, and the exclusive scan of the kept counts (rowptr)
//   write   one warp per granule emits its entries in index order: 16-bit offset in the granule and cast(u) in the wire
//           dtype at rowptr[g] + rank; with error feedback, e = 0 on the kept entries (e already holds u elsewhere)
// The logical-client fold replaces `write` with `fold`: acc (+)= n_k * topk(u), e updated, the replica reset.  The
// nonzero compaction (after fold_finish) runs count / scan / write with "theta != global" as the selection.
// Atomics only add integers into histograms, and every output position comes from a scan, so two launches give the same
// bits and the grid size (the SM count) changes nothing.
#include "pdl.cuh"
#include "ptx.cuh"
#include "launch.h"

namespace b200 {

constexpr int TK_THREADS = 256;
constexpr int TK_GRANULE = 1024;
constexpr uint32_t TK_NAN_KEY = 0x7FC00000u;
// work layout (int32 words): three histograms, the selection state, per-granule counts / tie quotas, row pointers
constexpr int TK_H0 = 0, TK_H1 = 2048, TK_H2 = 4096, TK_STATE = 4608, TK_GRAN = 4624;
// state: [0] key prefix (tau after the last pick), [1] count still needed inside the prefix's bucket (q at the end)

__device__ __forceinline__ uint32_t tk_key(float x) {
  const uint32_t m = __float_as_uint(x) & 0x7FFFFFFFu;
  return m > 0x7F800000u ? TK_NAN_KEY : m;
}

// level 0: u = (theta - global) [+ e] into u, histogram of key >> 20
__global__ void __launch_bounds__(TK_THREADS)
topk_hist0_kernel(const float* __restrict__ theta, const float* __restrict__ global_w, float* u, int ef, long long n,
                  int* __restrict__ work) {
  __shared__ uint32_t h[2048];
  for (int i = threadIdx.x; i < 2048; i += TK_THREADS) h[i] = 0;
  __syncthreads();
  const long long nv = n >> 2;
  for (long long i = blockIdx.x * static_cast<long long>(TK_THREADS) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * TK_THREADS) {
    const float4 t = __ldcs(reinterpret_cast<const float4*>(theta) + i);
    const float4 g = __ldcs(reinterpret_cast<const float4*>(global_w) + i);
    float4 v = make_float4(__fsub_rn(t.x, g.x), __fsub_rn(t.y, g.y), __fsub_rn(t.z, g.z), __fsub_rn(t.w, g.w));
    if (ef) {
      const float4 e = reinterpret_cast<const float4*>(u)[i];
      v = make_float4(__fadd_rn(v.x, e.x), __fadd_rn(v.y, e.y), __fadd_rn(v.z, e.z), __fadd_rn(v.w, e.w));
    }
    reinterpret_cast<float4*>(u)[i] = v;
    atomicAdd(&h[tk_key(v.x) >> 20], 1u);
    atomicAdd(&h[tk_key(v.y) >> 20], 1u);
    atomicAdd(&h[tk_key(v.z) >> 20], 1u);
    atomicAdd(&h[tk_key(v.w) >> 20], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2048; i += TK_THREADS)
    if (h[i]) atomicAdd(reinterpret_cast<unsigned*>(work + TK_H0) + i, h[i]);
}

// levels 1 and 2: histogram of the next bits over the keys that match the prefix chosen so far
template <int LEVEL>
__global__ void __launch_bounds__(TK_THREADS) topk_hist_kernel(const float* __restrict__ u, long long n, int* work) {
  constexpr int HSHIFT = LEVEL == 1 ? 20 : 9;        // bits above the histogrammed ones must match the prefix
  constexpr int BSHIFT = LEVEL == 1 ? 9 : 0;
  constexpr uint32_t BMASK = LEVEL == 1 ? 2047u : 511u;
  __shared__ uint32_t h[2048];
  for (int i = threadIdx.x; i < 2048; i += TK_THREADS) h[i] = 0;
  __syncthreads();
  const uint32_t want = static_cast<uint32_t>(work[TK_STATE]) >> HSHIFT;
  const long long nv = n >> 2;
  for (long long i = blockIdx.x * static_cast<long long>(TK_THREADS) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * TK_THREADS) {
    const float4 v = __ldcs(reinterpret_cast<const float4*>(u) + i);
    const uint32_t k[4] = {tk_key(v.x), tk_key(v.y), tk_key(v.z), tk_key(v.w)};
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if ((k[j] >> HSHIFT) == want) atomicAdd(&h[(k[j] >> BSHIFT) & BMASK], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2048; i += TK_THREADS)
    if (h[i]) atomicAdd(reinterpret_cast<unsigned*>(work + (LEVEL == 1 ? TK_H1 : TK_H2)) + i, h[i]);
}

// one warp: the bucket (from the top) in which the running count reaches the count still needed; 64 buckets per lane
template <int LEVEL>
__global__ void topk_pick_kernel(int* work, long long k) {
  constexpr int NB = LEVEL == 2 ? 512 : 2048;
  constexpr int PER = NB / 32;
  constexpr int SHIFT = LEVEL == 0 ? 20 : LEVEL == 1 ? 9 : 0;
  const unsigned* h = reinterpret_cast<const unsigned*>(work + (LEVEL == 0 ? TK_H0 : LEVEL == 1 ? TK_H1 : TK_H2));
  const int lane = threadIdx.x;
  const unsigned long long need = LEVEL == 0 ? static_cast<unsigned long long>(k) : static_cast<unsigned>(work[TK_STATE + 1]);
  // lane l holds buckets NB-1-l*PER down to NB-(l+1)*PER: lane 0 the highest
  unsigned long long mine = 0;
  for (int j = 0; j < PER; ++j) mine += h[NB - 1 - lane * PER - j];
  unsigned long long incl = mine;      // inclusive prefix over the lanes (from the top)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  const unsigned long long excl = incl - mine;
  if (excl < need && need <= incl) {   // exactly one lane
    unsigned long long above = excl;
    int b = NB - 1 - lane * PER;
    for (int j = 0; j < PER; ++j, --b) {
      const unsigned c = h[b];
      if (above + c >= need) break;
      above += c;
    }
    const uint32_t prefix = (LEVEL == 0 ? 0u : static_cast<uint32_t>(work[TK_STATE])) | (static_cast<uint32_t>(b) << SHIFT);
    work[TK_STATE] = static_cast<int>(prefix);
    work[TK_STATE + 1] = static_cast<int>(need - above);
  }
}

// the selection of one 32-element chunk of a granule: lane's element is kept when its key is above tau, or equal to it
// and among the granule's first `quota` ties (ties_seen counts the ties of the earlier chunks)
__device__ __forceinline__ bool tk_selected(uint32_t key, uint32_t tau, int quota, int& ties_seen, uint32_t lt_mask) {
  const bool eq = key == tau;
  const uint32_t eq_mask = __ballot_sync(0xffffffffu, eq);
  const bool sel = key > tau || (eq && ties_seen + __popc(eq_mask & lt_mask) < quota);
  ties_seen += __popc(eq_mask);
  return sel;
}

// MODE 0 (top-k): counts of key > tau and key == tau per granule; MODE 1 (nonzero): count of theta != global
template <int MODE>
__global__ void __launch_bounds__(TK_THREADS)
topk_count_kernel(const float* __restrict__ u, const float* __restrict__ theta, const float* __restrict__ global_w,
                  long long n_gran, int* __restrict__ work) {
  const int lane = threadIdx.x & 31;
  const uint32_t tau = static_cast<uint32_t>(work[TK_STATE]);
  int* cnt_gt = work + TK_GRAN;
  int* cnt_eq = cnt_gt + n_gran;
  for (long long g = (blockIdx.x * static_cast<long long>(TK_THREADS) + threadIdx.x) >> 5; g < n_gran;
       g += (static_cast<long long>(gridDim.x) * TK_THREADS) >> 5) {
    int gt = 0, eq = 0;
    const long long base = g * TK_GRANULE;
#pragma unroll 8
    for (int c = 0; c < TK_GRANULE / 32; ++c) {
      const long long i = base + c * 32 + lane;
      if constexpr (MODE == 0) {
        const uint32_t key = tk_key(__ldcs(u + i));
        gt += key > tau;
        eq += key == tau;
      } else {
        gt += __ldcs(theta + i) != __ldcs(global_w + i);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      gt += __shfl_xor_sync(0xffffffffu, gt, o);
      eq += __shfl_xor_sync(0xffffffffu, eq, o);
    }
    if (lane == 0) {
      cnt_gt[g] = gt;
      cnt_eq[g] = eq;
    }
  }
}

// block-wide exclusive scan of one value per thread (1024 threads); returns the exclusive prefix, total the sum
__device__ __forceinline__ long long tk_block_scan(long long v, long long* sh, long long& total) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const long long y = threadIdx.x >= static_cast<unsigned>(o) ? sh[threadIdx.x - o] : 0;
    __syncthreads();
    sh[threadIdx.x] += y;
    __syncthreads();
  }
  const long long incl = sh[threadIdx.x];
  total = sh[1023];
  __syncthreads();
  return incl - v;
}

// one CTA of 1024 threads, each over a contiguous run of granules: the ties kept per granule (the first q by index) and
// rowptr = the exclusive scan of the kept counts, clamped at cap
__global__ void __launch_bounds__(1024) topk_scan_kernel(int* work, long long n_gran, uint32_t* rowptr, long long cap,
                                                         int mode) {
  __shared__ long long sh[1024];
  int* cnt_gt = work + TK_GRAN;
  int* cnt_eq = cnt_gt + n_gran;
  int* quota = cnt_eq + n_gran;
  const long long q = mode == 0 ? static_cast<long long>(work[TK_STATE + 1]) : 0;
  const long long per = (n_gran + 1023) / 1024;
  const long long g0 = threadIdx.x * per, g1 = g0 + per < n_gran ? g0 + per : n_gran;
  long long s = 0, total;
  for (long long g = g0; g < g1; ++g) s += cnt_eq[g];
  long long ties = tk_block_scan(s, sh, total);
  long long kept = 0;
  for (long long g = g0; g < g1; ++g) {
    const long long e = cnt_eq[g];
    long long qg = q - ties;
    qg = qg < 0 ? 0 : (qg > e ? e : qg);
    quota[g] = static_cast<int>(qg);
    ties += e;
    kept += cnt_gt[g] + qg;
  }
  long long pos = tk_block_scan(kept, sh, total);
  for (long long g = g0; g < g1; ++g) {
    rowptr[g] = static_cast<uint32_t>(pos < cap ? pos : cap);
    pos += cnt_gt[g] + quota[g];
  }
  if (threadIdx.x == 1023) rowptr[n_gran] = static_cast<uint32_t>(total < cap ? total : cap);
}

__device__ __forceinline__ void tk_store_value(void* val, long long pos, float x, int wire_kind) {
  if (wire_kind == 0) reinterpret_cast<float*>(val)[pos] = x;
  else reinterpret_cast<__nv_bfloat16*>(val)[pos] = __float2bfloat16_rn(x);
}

// MODE 0: the kept entries of u (e = 0 there when ef); MODE 1: the entries where theta != global, value theta - global
template <int MODE>
__global__ void __launch_bounds__(TK_THREADS)
topk_write_kernel(float* __restrict__ u, const float* __restrict__ theta, const float* __restrict__ global_w, int ef,
                  long long n_gran, const int* __restrict__ work, const uint32_t* __restrict__ rowptr,
                  uint16_t* __restrict__ off, void* __restrict__ val, int wire_kind, long long cap) {
  const int lane = threadIdx.x & 31;
  const uint32_t lt = (1u << lane) - 1u;
  const uint32_t tau = static_cast<uint32_t>(work[TK_STATE]);
  const int* quota = work + TK_GRAN + 2 * n_gran;
  for (long long g = (blockIdx.x * static_cast<long long>(TK_THREADS) + threadIdx.x) >> 5; g < n_gran;
       g += (static_cast<long long>(gridDim.x) * TK_THREADS) >> 5) {
    const long long base = g * TK_GRANULE;
    long long pos = rowptr[g];
    const int qg = MODE == 0 ? quota[g] : 0;
    int ties = 0;
#pragma unroll 4
    for (int c = 0; c < TK_GRANULE / 32; ++c) {
      const long long i = base + c * 32 + lane;
      float x;
      bool sel;
      if constexpr (MODE == 0) {
        x = u[i];
        sel = tk_selected(tk_key(x), tau, qg, ties, lt);
      } else {
        const float t = __ldcs(theta + i), gw = __ldcs(global_w + i);
        x = __fsub_rn(t, gw);
        sel = t != gw;
      }
      const uint32_t sm = __ballot_sync(0xffffffffu, sel);
      const long long p = pos + __popc(sm & lt);
      if (sel && p < cap) {
        off[p] = static_cast<uint16_t>(c * 32 + lane);
        tk_store_value(val, p, x, wire_kind);
      }
      if (MODE == 0 && ef && sel) u[i] = 0.f;
      pos += __popc(sm);
    }
  }
}

// logical-client fold: acc (+)= nk * topk(u) (acc = 0 first), e = 0 on the kept entries (ef), replica reset (reset)
__global__ void __launch_bounds__(TK_THREADS)
topk_fold_kernel(float* __restrict__ u, int ef, long long n_gran, const int* __restrict__ work, float* __restrict__ acc,
                 float nk, int first, float* __restrict__ theta, const float* __restrict__ global_w,
                 __nv_bfloat16* __restrict__ wb, float* __restrict__ mom, long long n_mom, int reset) {
  const int lane = threadIdx.x & 31;
  const uint32_t lt = (1u << lane) - 1u;
  const uint32_t tau = static_cast<uint32_t>(work[TK_STATE]);
  const int* quota = work + TK_GRAN + 2 * n_gran;
  for (long long g = (blockIdx.x * static_cast<long long>(TK_THREADS) + threadIdx.x) >> 5; g < n_gran;
       g += (static_cast<long long>(gridDim.x) * TK_THREADS) >> 5) {
    const long long base = g * TK_GRANULE;
    const int qg = quota[g];
    int ties = 0;
#pragma unroll 4
    for (int c = 0; c < TK_GRANULE / 32; ++c) {
      const long long i = base + c * 32 + lane;
      const float x = u[i];
      const bool sel = tk_selected(tk_key(x), tau, qg, ties, lt);
      float a = first ? 0.f : acc[i];
      if (sel) a = fmaf(nk, x, a);
      acc[i] = a;
      if (ef && sel) u[i] = 0.f;
      if (reset) {
        const float gw = global_w[i];
        theta[i] = gw;
        if (wb != nullptr) wb[i] = __float2bfloat16_rn(gw);
        if (mom != nullptr && i < n_mom) mom[i] = 0.f;
      }
    }
  }
}

static int tk_grid(long long work_items, int per_block) {
  long long g = (work_items + per_block - 1) / per_block;
  const long long cap = 4ll * device_sm_count();
  if (g > cap) g = cap;
  return static_cast<int>(g < 1 ? 1 : g);
}

// passes hist0 .. scan of a top-k selection (rowptr: where the scan writes the row pointers)
static int topk_select_passes(const float* theta, const float* global_w, float* u, int ef, long long n, long long k,
                              int* work, uint32_t* rowptr, long long cap, cudaStream_t s) {
  const long long n_gran = n / TK_GRANULE;
  cudaError_t e = cudaMemsetAsync(work, 0, TK_GRAN * sizeof(int), s);
  if (e != cudaSuccess) return static_cast<int>(e);
  const int ge = tk_grid(n / 4, TK_THREADS), gg = tk_grid(n_gran, TK_THREADS / 32);
  topk_hist0_kernel<<<ge, TK_THREADS, 0, s>>>(theta, global_w, u, ef, n, work);
  topk_pick_kernel<0><<<1, 32, 0, s>>>(work, k);
  topk_hist_kernel<1><<<ge, TK_THREADS, 0, s>>>(u, n, work);
  topk_pick_kernel<1><<<1, 32, 0, s>>>(work, k);
  topk_hist_kernel<2><<<ge, TK_THREADS, 0, s>>>(u, n, work);
  topk_pick_kernel<2><<<1, 32, 0, s>>>(work, k);
  topk_count_kernel<0><<<gg, TK_THREADS, 0, s>>>(u, nullptr, nullptr, n_gran, work);
  topk_scan_kernel<<<1, 1024, 0, s>>>(work, n_gran, rowptr, cap, 0);
  return static_cast<int>(cudaGetLastError());
}

static bool tk_shape_ok(const float* theta, const float* global_w, const float* u, long long n, long long k) {
  return n > 0 && n % TK_GRANULE == 0 && k >= 1 && k <= n && n / TK_GRANULE < (1ll << 30) &&
         ((reinterpret_cast<uintptr_t>(theta) | reinterpret_cast<uintptr_t>(global_w) | reinterpret_cast<uintptr_t>(u)) &
          15) == 0;
}

}  // namespace b200

extern "C" int b200_topk_pack(const float* theta, const float* global_w, float* u, int ef, long long n, long long k,
                              int* work, uint32_t* rowptr, uint16_t* off, void* val, int wire_kind, long long cap,
                              cudaStream_t stream) {
  using namespace b200;
  if (!tk_shape_ok(theta, global_w, u, n, k) || (wire_kind != 0 && wire_kind != 1) || cap < k) return -2;
  int rc = topk_select_passes(theta, global_w, u, ef, n, k, work, rowptr, cap, stream);
  if (rc) return rc;
  topk_write_kernel<0><<<tk_grid(n / TK_GRANULE, TK_THREADS / 32), TK_THREADS, 0, stream>>>(
      u, nullptr, nullptr, ef, n / TK_GRANULE, work, rowptr, off, val, wire_kind, cap);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int b200_topk_fold(float* theta, const float* global_w, float* u, int ef, long long n, long long k, int* work,
                              float* acc, float nk, int first, void* w_bf16, float* mom, long long n_mom, int reset,
                              cudaStream_t stream) {
  using namespace b200;
  if (!tk_shape_ok(theta, global_w, u, n, k) || acc == nullptr) return -2;
  const long long n_gran = n / TK_GRANULE;
  uint32_t* rowptr = reinterpret_cast<uint32_t*>(work + TK_GRAN + 3 * n_gran);
  int rc = topk_select_passes(theta, global_w, u, ef, n, k, work, rowptr, n, stream);
  if (rc) return rc;
  topk_fold_kernel<<<tk_grid(n_gran, TK_THREADS / 32), TK_THREADS, 0, stream>>>(
      u, ef, n_gran, work, acc, nk, first, theta, global_w, reinterpret_cast<__nv_bfloat16*>(w_bf16), mom, n_mom, reset);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int b200_nonzero_pack(const float* theta, const float* global_w, long long n, int* work, uint32_t* rowptr,
                                 uint16_t* off, void* val, int wire_kind, long long cap, cudaStream_t stream) {
  using namespace b200;
  if (!tk_shape_ok(theta, global_w, theta, n, 1) || (wire_kind != 0 && wire_kind != 1) || cap < 1) return -2;
  const long long n_gran = n / TK_GRANULE;
  const int gg = tk_grid(n_gran, TK_THREADS / 32);
  topk_count_kernel<1><<<gg, TK_THREADS, 0, stream>>>(nullptr, theta, global_w, n_gran, work);
  topk_scan_kernel<<<1, 1024, 0, stream>>>(work, n_gran, rowptr, cap, 1);
  topk_write_kernel<1><<<gg, TK_THREADS, 0, stream>>>(nullptr, theta, global_w, 0, n_gran, work, rowptr, off, val,
                                                       wire_kind, cap);
  return static_cast<int>(cudaGetLastError());
}

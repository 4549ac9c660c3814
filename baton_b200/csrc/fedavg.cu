// Fused FedAvg collective over NVLink / NVSwitch -- ONE persistent kernel per round that does
//
//   (wire formats: fp32, bf16, or block-scaled fp8 = e4m3 + one UE8M0 scale per 32 elements)
//   phase 0  pack      wire_r[t]  = cast( s_r * (theta_r[t] - global[t]) )   (delta mode)
//                                   cast( s_r * theta_r[t] )                 (weights mode)
//   barrier  per-CTA 64-bit flags in peer-mapped pads, st.release.sys / ld.acquire.sys; the flag
//            word carries this client's sample count n_r, so the n_k exchange that FedAvg needs
//            (weights w_k = n_k / N, reference manager.py:119-126) costs no extra message
//   phase 1  reduce    owner(t) pulls tile t from every participant with 16 B peer loads over
//            + bcast   NVLink (or ONE multimem.ld_reduce: the switch adds the replicas), sums in
//                      fp32 in fixed rank order, casts, and pushes the result into tile t of every
//                      live replica's wire buffer (peer stores, or ONE multimem.st replicated by
//                      the switch).  In place: owner(t) is the only reader and writer of tile t.
//   barrier
//   phase 2  apply     global += result ; theta = global ; bf16 shadow = bf16(theta) ; momentum = 0
//                      (the reference's load_state_dict, worker.py:98, with no extra pass), then
//                      publish a per-tile arrival flag so the next forward's first GEMM
//                      (gemm_wgmma, flag-gated TMA producer) can start on its weight tiles while
//                      the rest of the arena is still in flight.
//   barrier  (closing: wire / pads may be reused by the next round)
//
// This replaces the reference's upload (worker.py:108-118), CPU reduce (manager.py:119-126),
// broadcast (manager.py:77-86) and load_state_dict (worker.py:98).  No NCCL call on this path.
// The per-epoch loss history is reduced the same way (manager.py:127-130) by CTA 0.
//
// Tile t (tile_elems elements) is owned by the (t mod A)-th live rank and handled by CTA
// ((t div A) mod G) on EVERY rank in every phase, so a per-CTA cross-GPU barrier is enough:
// CTA b only ever consumes data produced by CTA b of some rank.
//
// Participation: n_k == 0 -> rank k is not read (P2P) / packs zeros (NVLS);
// alive_mask bit k == 0 -> rank k is neither read, written nor waited for (dead process), so a
// dead peer cannot hang the collective the way a blocking NCCL call would; a bounded spin turns a
// peer that dies mid-collective into an error status instead of a hang.
#define B200_TU_TAG 7
#include "pdl.cuh"
#include <type_traits>

#include "ptx.cuh"
#include "launch.h"
#include "mx.cuh"
#include "dp.cuh"
#include "secagg.cuh"

namespace b200 {

constexpr int FEDAVG_THREADS = 512;
constexpr int FLAG_GRANULE = 1024;   // elements covered by one arrival flag (bcast_gemm consumers)

__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Per-CTA barrier across the live ranks.  pads[k] is rank k's pad (peer-mapped); slot layout
// pad[cta * B200_MAX_RANKS + src_rank], word = (epoch << 32) | payload.  Epochs only grow, so no
// reset races.  payload_out[k] (shared memory) receives rank k's payload.
__device__ __forceinline__ bool cta_barrier_all_ranks(const FedAvgArgs& a, uint32_t epoch, uint32_t payload,
                                                      uint32_t* payload_out) {
  __syncthreads();
  const int t = threadIdx.x;
  bool ok = true;
  if (t < a.world && ((a.alive_mask >> t) & 1u)) {
    fence_sys();
    const unsigned long long word = (static_cast<unsigned long long>(epoch) << 32) | payload;
    st_release_sys_u64(a.pads[t] + (static_cast<size_t>(blockIdx.x) * B200_MAX_RANKS + a.rank), word);
    const unsigned long long* mine = a.pads[a.rank] + (static_cast<size_t>(blockIdx.x) * B200_MAX_RANKS + t);
    unsigned long long spins = 0, v;
    const unsigned long long limit = a.timeout_log2 > 0 ? (1ull << a.timeout_log2) : ~0ull;
    while (static_cast<int32_t>(static_cast<uint32_t>((v = ld_acquire_sys_u64(mine)) >> 32) - epoch) < 0) {
      if (++spins > limit) {
        ok = false;
        if (a.status != nullptr) atomicExch(a.status, 1 + t);
        break;
      }
    }
    if (payload_out != nullptr) payload_out[t] = static_cast<uint32_t>(v);
  }
  const int all_ok = __syncthreads_and(ok ? 1 : 0);
  return all_ok != 0;
}

__device__ __forceinline__ uint2 ld_volatile_v2(const void* p) {
  uint2 r;
  asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void st_na_v2(void* p, const uint2& v) {
  asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}
__device__ __forceinline__ uint32_t ld_volatile_u8(const void* p) {
  uint32_t r;
  asm volatile("ld.volatile.global.u8 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void st_volatile_u8(void* p, uint32_t v) {
  asm volatile("st.volatile.global.u8 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Wire formats.  WIRE 0: fp32 (4 per 16 B), 1: bf16 (8 per 16 B), 2: MXFP8 -- e4m3 payload (8 per 8 B
// thread vector) plus one UE8M0 scale byte per 32 consecutive elements, stored behind the payload.
template <int WIRE>
struct Wire;
template <>
struct Wire<1> {
  static constexpr int VEC = 8, VBYTES = 16;
  static constexpr bool SCALED = false;
  __device__ static void unpack(const uint4& u, float (&f)[8], float) {
    float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
  }
  __device__ static uint4 pack(const float (&f)[8], float) {
    uint4 u;
    u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
    u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
    return u;
  }
  __device__ static uint4 ld(const void* p) { return ld_volatile_v4(p); }
  __device__ static void st(void* p, const uint4& v) { *reinterpret_cast<uint4*>(p) = v; }
  __device__ static void st_na(void* p, const uint4& v) { st_na_v4(p, v); }
  __device__ static uint4 mc_reduce(const void* p) { return multimem_ld_reduce_bf16x8(p); }
};
template <>
struct Wire<0> {
  static constexpr int VEC = 4, VBYTES = 16;
  static constexpr bool SCALED = false;
  __device__ static void unpack(const uint4& u, float (&f)[4], float) {
    f[0] = __uint_as_float(u.x); f[1] = __uint_as_float(u.y);
    f[2] = __uint_as_float(u.z); f[3] = __uint_as_float(u.w);
  }
  __device__ static uint4 pack(const float (&f)[4], float) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
  }
  __device__ static uint4 ld(const void* p) { return ld_volatile_v4(p); }
  __device__ static void st(void* p, const uint4& v) { *reinterpret_cast<uint4*>(p) = v; }
  __device__ static void st_na(void* p, const uint4& v) { st_na_v4(p, v); }
  __device__ static uint4 mc_reduce(const void* p) {
    float4 r = multimem_ld_reduce_f32x4(p);
    return make_uint4(__float_as_uint(r.x), __float_as_uint(r.y), __float_as_uint(r.z), __float_as_uint(r.w));
  }
};
template <>
struct Wire<2> {
  static constexpr int VEC = 8, VBYTES = 8;
  static constexpr bool SCALED = true;
  __device__ static void unpack(const uint4& u, float (&f)[8], float scale) {
    const float2 a = from_e4m3x2(static_cast<uint16_t>(u.x & 0xFFFFu)), b = from_e4m3x2(static_cast<uint16_t>(u.x >> 16));
    const float2 c = from_e4m3x2(static_cast<uint16_t>(u.y & 0xFFFFu)), d = from_e4m3x2(static_cast<uint16_t>(u.y >> 16));
    f[0] = a.x * scale; f[1] = a.y * scale; f[2] = b.x * scale; f[3] = b.y * scale;
    f[4] = c.x * scale; f[5] = c.y * scale; f[6] = d.x * scale; f[7] = d.y * scale;
  }
  __device__ static uint4 pack(const float (&f)[8], float inv) {
    uint4 u;
    u.x = to_e4m3x2(f[0] * inv, f[1] * inv) | (static_cast<uint32_t>(to_e4m3x2(f[2] * inv, f[3] * inv)) << 16);
    u.y = to_e4m3x2(f[4] * inv, f[5] * inv) | (static_cast<uint32_t>(to_e4m3x2(f[6] * inv, f[7] * inv)) << 16);
    u.z = 0; u.w = 0;
    return u;
  }
  __device__ static uint4 ld(const void* p) { const uint2 v = ld_volatile_v2(p); return make_uint4(v.x, v.y, 0, 0); }
  __device__ static void st(void* p, const uint4& v) { *reinterpret_cast<uint2*>(p) = make_uint2(v.x, v.y); }
  __device__ static void st_na(void* p, const uint4& v) { st_na_v2(p, make_uint2(v.x, v.y)); }
  __device__ static uint4 mc_reduce(const void*) { return make_uint4(0, 0, 0, 0); }   // the switch cannot apply block scales
};
// WIRE 3: the int32 ring of a secure-aggregation round, 4 per 16 B.  Its pack (encode + masks) and reduce (wrapping
// integer adds) are secagg_pack / secagg_reduce; the apply phase reads fp32(int32) and scales it by 2^-f.
template <>
struct Wire<3> {
  static constexpr int VEC = 4, VBYTES = 16;
  static constexpr bool SCALED = false;
  __device__ static void unpack(const uint4& u, float (&f)[4], float) {
    f[0] = __int2float_rn(static_cast<int>(u.x)); f[1] = __int2float_rn(static_cast<int>(u.y));
    f[2] = __int2float_rn(static_cast<int>(u.z)); f[3] = __int2float_rn(static_cast<int>(u.w));
  }
  __device__ static uint4 ld(const void* p) { return ld_volatile_v4(p); }
  __device__ static void st_na(void* p, const uint4& v) { st_na_v4(p, v); }
  // the generic reduce loop names these, but a secure round never runs it
  __device__ static uint4 pack(const float (&)[4], float) { return make_uint4(0, 0, 0, 0); }
  __device__ static uint4 mc_reduce(const void*) { return make_uint4(0, 0, 0, 0); }   // ptxas has no .v4.u32 ld_reduce
};

// shared exponent of the 32-element block owned by a quad of adjacent lanes (8 elements each);
// every lane of the warp must call this
template <int VEC>
__device__ __forceinline__ int quad_block_exponent(const float (&f)[VEC]) {
  float amax = 0.f;
#pragma unroll
  for (int j = 0; j < VEC; ++j) amax = fmaxf(amax, fabsf(f[j]));
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
  amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
  return mx_exponent(amax);
}

// Optional in-kernel phase timestamps (multi-GPU kernels with spin barriers cannot be replayed under ncu):
// thread 0 of the first and of the last CTA record %globaltimer at every phase boundary.
// Compiled in only with -DB200_FEDAVG_PHASE_TIMING (BATON_BUILD_PHASE_TIMING=1 python -m baton_b200.build_ext), so
// the default build keeps the exact instruction stream that was validated on hardware.
__device__ __forceinline__ void phase_stamp(const FedAvgArgs& a, int slot) {
#ifdef B200_FEDAVG_PHASE_TIMING
  if (a.phase_ns != nullptr && threadIdx.x == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1)) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    a.phase_ns[(blockIdx.x == 0 ? 0 : 8) + slot] = t;
  }
#else
  (void)a; (void)slot;
#endif
}

// ---------------------------------------------------------------- SCAFFOLD: the control-variate segment
// Segment 1 of a SCAFFOLD round is a second wire of n elements at byte offset `off` of every rank's wire half (fp8:
// its scale bytes behind its n payload bytes).  Its tiles are mapped to owners and CTAs exactly like segment 0's
// (owner = (t mod A)-th live rank, CTA = (t div A) mod G), so the per-CTA barriers of the round cover it too.  The three
// phases below are kept apart from fedavg_round's own loops so the plain and DP kernels keep their instruction streams.

// phase 0: wire = cast(src) over the tiles this CTA packs
template <int WIRE>
__device__ __forceinline__ void seg_pack(uint8_t* wire, const float* __restrict__ src, long long n, int T, int A, int G) {
  using W = Wire<WIRE>;
  constexpr int VEC = W::VEC;
  constexpr size_t esz = W::VBYTES / VEC;
  const long long n_tiles = (n + T - 1) / T;
  const int lane_elems = static_cast<int>(threadIdx.x & 31) * VEC;
  for (long long q = blockIdx.x; q * A < n_tiles; q += G) {
    for (int r = 0; r < A; ++r) {
      const long long t = q * A + r;
      if (t >= n_tiles) break;
      const long long base = t * T;
      const int len = static_cast<int>((n - base) < T ? (n - base) : T);
      for (int i = threadIdx.x * VEC; i - lane_elems < len; i += FEDAVG_THREADS * VEC) {   // warp-uniform bound
        const bool valid = i < len;
        float f[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) f[j] = 0.f;
        if (valid) {
#pragma unroll
          for (int j = 0; j < VEC; j += 4) {
            const float4 v = __ldcs(reinterpret_cast<const float4*>(src + base + i + j));
            f[j] = v.x; f[j + 1] = v.y; f[j + 2] = v.z; f[j + 3] = v.w;
          }
        }
        float inv = 1.f;
        if constexpr (W::SCALED) {
          const int e = quad_block_exponent<VEC>(f);
          inv = exp2_int(-e);
          if (valid && (threadIdx.x & 3) == 0) wire[n + ((base + i) >> 5)] = static_cast<uint8_t>(e + 127);
        }
        if (valid) W::st(wire + (base + i) * esz, W::pack(f, inv));
      }
    }
  }
}

// phase 1: the owner of a tile sums weight * wire_k over the participants (part[k] != 0, fixed rank order) and stores
// the cast result into that tile of every live rank's segment
template <int WIRE>
__device__ __forceinline__ void seg_reduce(uint8_t* const* s_wire, const float* part, size_t off, float weight,
                                           long long n, int T, int A, int G, int my_pos) {
  using W = Wire<WIRE>;
  constexpr int VEC = W::VEC;
  constexpr int KG = 4;                          // peers whose loads are issued together
  constexpr size_t esz = W::VBYTES / VEC;
  const long long n_tiles = (n + T - 1) / T;
  const int lane_elems = static_cast<int>(threadIdx.x & 31) * VEC;
  for (long long t = my_pos + static_cast<long long>(blockIdx.x) * A; t < n_tiles; t += static_cast<long long>(G) * A) {
    const long long base = t * T;
    const int len = static_cast<int>((n - base) < T ? (n - base) : T);
    for (int i = threadIdx.x * VEC; i - lane_elems < len; i += FEDAVG_THREADS * VEC) {
      const bool valid = i < len;
      const size_t eo = off + (base + i) * esz, so = off + n + ((base + i) >> 5);
      float acc[VEC];
#pragma unroll
      for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
#pragma unroll 1
      for (int k0 = 0; k0 < A; k0 += KG) {
        uint4 v[KG];
        uint32_t sc[KG];
        if (valid) {
#pragma unroll
          for (int k = 0; k < KG; ++k)
            if (k0 + k < A && part[k0 + k] != 0.f) {
              v[k] = W::ld(s_wire[k0 + k] + eo);
              if constexpr (W::SCALED) sc[k] = ld_volatile_u8(s_wire[k0 + k] + so);
            }
#pragma unroll
          for (int k = 0; k < KG; ++k)
            if (k0 + k < A && part[k0 + k] != 0.f) {
              float f[VEC];
              float scale = 1.f;
              if constexpr (W::SCALED) scale = exp2_int(static_cast<int>(sc[k]) - 127);
              W::unpack(v[k], f, scale);
#pragma unroll
              for (int j = 0; j < VEC; ++j) acc[j] = fmaf(weight, f[j], acc[j]);
            }
        }
      }
      float inv = 1.f;
      int e = 0;
      if constexpr (W::SCALED) {
        e = quad_block_exponent<VEC>(acc);
        inv = exp2_int(-e);
      }
      if (valid) {
        const uint4 out = W::pack(acc, inv);
        for (int k = 0; k < A; ++k) {
          W::st_na(s_wire[k] + eo, out);
          if constexpr (W::SCALED)
            if ((threadIdx.x & 3) == 0) st_volatile_u8(s_wire[k] + so, static_cast<uint32_t>(e + 127));
        }
      }
    }
  }
}

// phase 2: dst += the reduced segment, over the tiles this CTA applies (the ones it packed)
template <int WIRE>
__device__ __forceinline__ void seg_apply_add(const uint8_t* wire, float* __restrict__ dst, long long n, int T, int A,
                                              int G) {
  using W = Wire<WIRE>;
  constexpr int VEC = W::VEC;
  constexpr size_t esz = W::VBYTES / VEC;
  const long long n_tiles = (n + T - 1) / T;
  for (long long q = blockIdx.x; q * A < n_tiles; q += G) {
    for (int r = 0; r < A; ++r) {
      const long long t = q * A + r;
      if (t >= n_tiles) break;
      const long long base = t * T;
      const int len = static_cast<int>((n - base) < T ? (n - base) : T);
      for (int i = threadIdx.x * VEC; i < len; i += FEDAVG_THREADS * VEC) {
        const uint4 wv = W::ld(wire + (base + i) * esz);
        float scale = 1.f;
        if constexpr (W::SCALED) scale = exp2_int(static_cast<int>(ld_volatile_u8(wire + n + ((base + i) >> 5))) - 127);
        float f[VEC];
        W::unpack(wv, f, scale);
#pragma unroll
        for (int j = 0; j < VEC; j += 4) {
          float4 c = *reinterpret_cast<const float4*>(dst + base + i + j);
          c.x += f[j]; c.y += f[j + 1]; c.z += f[j + 2]; c.w += f[j + 3];
          *reinterpret_cast<float4*>(dst + base + i + j) = c;
        }
      }
    }
  }
}

// ---------------------------------------------------------------- robust rounds: coordinate-wise median / trimmed mean
// Phase 1 of a robust round replaces the weighted sum with a selection across the P participating client segments.  The
// owner of a tile walks it in chunks of CH = ROBUST_STAGE / NP elements (NP = P rounded up to 8, 16 or 32):
//   load    all threads pull the chunk of every segment with 16-byte (fp8: 8-byte) loads, 32 / VEC per thread issued
//           before the first use, decode to fp32 and store order-preserving uint32 keys into shared memory [NP][CH];
//   select  thread c takes column c into registers (padding rows: key 0xFFFFFFFF, above every value), sorts it with a
//           bitonic network (NP = 32: two runs of 16 and a bitonic merge through shared memory), writes it back and
//           puts the selected value into row 0 of its own column;
//   store   the threads cast row 0 to the wire format (fp8: the quad's block exponent) and store it into seg 0 of every
//           live replica, where the plain apply phase finds it.
// The result of an element depends only on the multiset of its P values, never on the tile size, the CTA count, the
// owner or the order of the segments.  IEEE-rounded intrinsics keep --use_fast_math from reassociating or approximating.
constexpr int ROBUST_STAGE = 16384;   // uint32 keys staged per chunk (64 KB of dynamic shared memory)
constexpr int ROBUST_SMEM = ROBUST_STAGE * 4 + B200_MAX_ROBUST_CLIENTS * 8 + 16;

// total order on floats as uint32 keys: -inf < ... < -0 < +0 < ... < +inf < NaN (every NaN canonicalised to 0x7FC00000)
__device__ __forceinline__ uint32_t robust_key(float x) {
  uint32_t u = __float_as_uint(x);
  if ((u & 0x7FFFFFFFu) > 0x7F800000u) u = 0x7FC00000u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float robust_unkey(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

template <int NP>
__device__ __forceinline__ void bitonic_sort(uint32_t (&k)[NP]) {
#pragma unroll
  for (int size = 2; size <= NP; size <<= 1)
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1)
#pragma unroll
      for (int i = 0; i < NP; ++i) {
        const int j = i ^ stride;
        if (j > i) {
          const uint32_t lo = min(k[i], k[j]), hi = max(k[i], k[j]);
          const bool up = (i & size) == 0;
          k[i] = up ? lo : hi;
          k[j] = up ? hi : lo;
        }
      }
}

// ascending bitonic merge: sorts a bitonic sequence of N keys
template <int N>
__device__ __forceinline__ void bitonic_merge(uint32_t (&k)[N]) {
#pragma unroll
  for (int stride = N >> 1; stride > 0; stride >>= 1)
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const int j = i ^ stride;
      if (j > i) {
        const uint32_t lo = min(k[i], k[j]), hi = max(k[i], k[j]);
        k[i] = lo;
        k[j] = hi;
      }
    }
}

// median: x[P/2] for odd P, 0.5 * (x[(P-1)/2] + x[P/2]) for even P; trimmed mean: (x[b] + ... + x[P-b-1]) / (P - 2b),
// added in ascending order from 0; P == 0: 0 (the round changes nothing).  x = the sorted column col of the stage.
__device__ __forceinline__ float robust_select(const uint32_t* col, int stride, int P, int kind, int b) {
  if (P == 0) return 0.f;
  if (kind == 0) {
    const int i0 = (P - 1) >> 1, i1 = P >> 1;
    const float x1 = robust_unkey(col[i1 * stride]);
    return i0 == i1 ? x1 : __fmul_rn(0.5f, __fadd_rn(robust_unkey(col[i0 * stride]), x1));
  }
  float acc = 0.f;
  for (int j = b; j < P - b; ++j) acc = __fadd_rn(acc, robust_unkey(col[j * stride]));
  return __fdiv_rn(acc, static_cast<float>(P - 2 * b));
}

// load: elements [e0, e0 + clen) of the P segments src[0 .. P) into the stage [NP][CH] as order-preserving keys, RG
// wire vectors per thread issued before the first decode (shared by the selection and Krum's distance pass)
template <int WIRE, int NP>
__device__ __forceinline__ void robust_stage(const uint8_t* const* src, uint32_t* stage, int P, long long n, long long e0,
                                             int clen) {
  using W = Wire<WIRE>;
  constexpr int VEC = W::VEC;
  constexpr size_t esz = W::VBYTES / VEC;
  constexpr int CH = ROBUST_STAGE / NP;          // elements per chunk
  constexpr int VPR = CH / VEC;                  // wire vectors per segment row of a chunk
  constexpr int R = NP * VPR / FEDAVG_THREADS;   // loads per thread per chunk
  constexpr int RG = 4;                          // ... in groups of RG in flight
  static_assert(R * FEDAVG_THREADS == NP * VPR && R % RG == 0, "the stage must split evenly over the threads");
#pragma unroll 1
  for (int r0 = 0; r0 < R; r0 += RG) {
    uint4 v[RG];
    uint32_t sc[RG];
#pragma unroll
    for (int r = 0; r < RG; ++r) {
      const int w = threadIdx.x + (r0 + r) * FEDAVG_THREADS, p = w / VPR, q = (w % VPR) * VEC;
      if (p < P && q < clen) {
        v[r] = W::ld(src[p] + (e0 + q) * esz);
        if constexpr (W::SCALED) sc[r] = ld_volatile_u8(src[p] + n + ((e0 + q) >> 5));
      }
    }
#pragma unroll
    for (int r = 0; r < RG; ++r) {
      const int w = threadIdx.x + (r0 + r) * FEDAVG_THREADS, p = w / VPR, q = (w % VPR) * VEC;
      if (p < P && q < clen) {
        float f[VEC];
        float scale = 1.f;
        if constexpr (W::SCALED) scale = exp2_int(static_cast<int>(sc[r]) - 127);
        W::unpack(v[r], f, scale);
#pragma unroll
        for (int j = 0; j < VEC; j += 4)
          *reinterpret_cast<uint4*>(stage + p * CH + q + j) =
              make_uint4(robust_key(f[j]), robust_key(f[j + 1]), robust_key(f[j + 2]), robust_key(f[j + 3]));
      }
    }
  }
}

template <int WIRE, int NP>
__device__ __forceinline__ void robust_tiles(const FedAvgRobustArgs& a, uint8_t* const* s_wire, const uint8_t* const* src,
                                             uint32_t* stage, int P, int A, int my_pos) {
  using W = Wire<WIRE>;
  constexpr int VEC = W::VEC;
  constexpr size_t esz = W::VBYTES / VEC;
  constexpr int CH = ROBUST_STAGE / NP;          // elements per chunk
  const int G = gridDim.x;
  const long long n = a.n;
  const int T = a.tile_elems;
  const long long n_tiles = (n + T - 1) / T;
  const int b = a.trim_b[P];
  const int lane_elems = static_cast<int>(threadIdx.x & 31) * VEC;
  for (long long t = my_pos + static_cast<long long>(blockIdx.x) * A; t < n_tiles; t += static_cast<long long>(G) * A) {
    const long long base = t * T;
    const int len = static_cast<int>((n - base) < T ? (n - base) : T);
    for (int c0 = 0; c0 < len; c0 += CH) {
      const int clen = len - c0 < CH ? len - c0 : CH;
      const long long e0 = base + c0;
      robust_stage<WIRE, NP>(src, stage, P, n, e0, clen);
      __syncthreads();
      // ---- select: one column per thread
#pragma unroll 1
      for (int c = threadIdx.x; c < clen; c += FEDAVG_THREADS) {
        // sorted back into the column (only this thread reads it), then selected from there.  32 rows do not fit in
        // registers as one network: they are sorted as two runs of 16, a half-cleaner (row i against row 31 - i) puts
        // the 16 smallest keys into rows 0..15 and the 16 largest into rows 16..31, each half bitonic, and a 16-wide
        // bitonic merge sorts each half
        constexpr int NR = NP < 16 ? NP : 16;
        uint32_t* col = stage + c;
#pragma unroll
        for (int h = 0; h < NP; h += NR) {
          uint32_t k[NR];
#pragma unroll
          for (int j = 0; j < NR; ++j) k[j] = h + j < P ? col[(h + j) * CH] : 0xFFFFFFFFu;
          bitonic_sort<NR>(k);
#pragma unroll
          for (int j = 0; j < NR; ++j)
            if (NP > 16 || j < P) col[(h + j) * CH] = k[j];
        }
        if constexpr (NP > 16) {
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const uint32_t x = col[i * CH], y = col[(31 - i) * CH];
            col[i * CH] = min(x, y);
            col[(31 - i) * CH] = max(x, y);
          }
#pragma unroll
          for (int h = 0; h < 32; h += 16) {
            uint32_t k[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) k[j] = col[(h + j) * CH];
            bitonic_merge<16>(k);
#pragma unroll
            for (int j = 0; j < 16; ++j) col[(h + j) * CH] = k[j];
          }
        }
        stage[c] = __float_as_uint(robust_select(col, CH, P, a.kind, b));
      }
      __syncthreads();
      // ---- cast + store into seg 0 of every live replica (warp-uniform bound: the fp8 quads shuffle)
      for (int i = threadIdx.x * VEC; i - lane_elems < clen; i += FEDAVG_THREADS * VEC) {
        const bool valid = i < clen;
        float f[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) f[j] = valid ? __uint_as_float(stage[i + j]) : 0.f;
        float inv = 1.f;
        int e = 0;
        if constexpr (W::SCALED) {
          e = quad_block_exponent<VEC>(f);
          inv = exp2_int(-e);
        }
        if (valid) {
          const size_t off = (e0 + i) * esz;
          const uint4 out = W::pack(f, inv);
#pragma unroll 1
          for (int k = 0; k < A; ++k) {
            W::st_na(s_wire[k] + off, out);
            if constexpr (W::SCALED)
              if ((threadIdx.x & 3) == 0) st_volatile_u8(s_wire[k] + n + ((e0 + i) >> 5), static_cast<uint32_t>(e + 127));
          }
        }
      }
      __syncthreads();   // the next chunk reuses the stage
    }
  }
}

// phase 1 of a robust round: gather the P client segments of the live ranks (counts from their pages), then select
// the P client segments of the live ranks in segment order (rank position, then the rank's segment order) into src
__device__ __forceinline__ int robust_gather(const FedAvgRobustArgs& a, uint8_t* const* s_wire, const int* s_rank, int A,
                                             const uint8_t** src, int* s_P) {
  if (threadIdx.x == 0) {
    int P = 0;
    for (int k = 0; k < A; ++k) {
      const uint32_t m = *reinterpret_cast<const volatile uint32_t*>(a.seg_page[s_rank[k]]);
      for (uint32_t j = 0; j < m && P < B200_MAX_ROBUST_CLIENTS; ++j)   // the host keeps P <= 32
        src[P++] = s_wire[k] + static_cast<size_t>(j) * static_cast<size_t>(a.seg_stride);
    }
    *s_P = P;
  }
  __syncthreads();
  return *s_P;
}

template <int WIRE>
__device__ __forceinline__ void robust_reduce(const FedAvgRobustArgs& a, uint8_t* const* s_wire, const int* s_rank, int A,
                                              int my_pos) {
  extern __shared__ __align__(16) uint8_t robust_smem[];
  uint32_t* stage = reinterpret_cast<uint32_t*>(robust_smem);
  const uint8_t** src = reinterpret_cast<const uint8_t**>(robust_smem + ROBUST_STAGE * 4);
  int* s_P = reinterpret_cast<int*>(robust_smem + ROBUST_STAGE * 4 + B200_MAX_ROBUST_CLIENTS * 8);
  const int P = robust_gather(a, s_wire, s_rank, A, src, s_P);
  if (P <= 8) robust_tiles<WIRE, 8>(a, s_wire, src, stage, P, A, my_pos);
  else if (P <= 16) robust_tiles<WIRE, 16>(a, s_wire, src, stage, P, A, my_pos);
  else robust_tiles<WIRE, 32>(a, s_wire, src, stage, P, A, my_pos);
}

// ---------------------------------------------------------------- Multi-Krum rounds (see launch.h / parallel/robust.py)
// Phase 1 of a Krum round, between barrier 1 (epoch + 1) and barrier 2 (epoch + 3):
//   distances  the owner of a tile stages the P segments chunk by chunk (robust_stage) and adds the upper-triangle
//              pair sums (x_i - x_j)^2 from shared memory: 4 x 4 register blocks of rows, 4 columns per lane, 16 fp32
//              sums per lane reduced over the warp by a transpose-reduce (16 shuffles), the 128-column slices of a
//              chunk added in slice order in fp32, and the chunk's sum added to one fp64 accumulator per pair;
//   rank       every CTA writes its P(P-1)/2 fp64 partials into its slot of a local work buffer; the last CTA to
//              arrive (a device counter the launcher zeroes) adds the slots in CTA order into this rank's distance page;
//              the other CTAs wait for it with a bounded spin (not a grid sync: a CTA whose cross-GPU barrier timed
//              out has returned, and an unbounded grid-wide wait would hang the rest of the grid);
//   exchange   a per-CTA cross-rank barrier at epoch + 2: once CTA b passes it, CTA b of every live rank has passed
//              the rank step, so every page is complete.  Every CTA adds the A pages in rank order: every CTA of every
//              rank holds the same D bits and computes the same scores and kept set;
//   kept mean  robust_tiles over the m kept segments with the trimmed mean and b = 0 (the host sets kind and trim_b).
// P <= 2 skips the distances and the exchange on every rank alike (P is known identically after barrier 1): all
// scores tie and the first m segments are kept.
constexpr int KRUM_PAIRS = B200_KRUM_PAIRS;
constexpr int KRUM_ITEMS = 144;                 // (block pair, 128-column slice) items per chunk at NP = 32 (the most)
constexpr int KRUM_PART_OFF = ROBUST_SMEM;      // float [KRUM_ITEMS][16]: per-item pair sums of a chunk
constexpr int KRUM_D_OFF = KRUM_PART_OFF + KRUM_ITEMS * 16 * 4;              // double [32][32]
constexpr int KRUM_SCORE_OFF = KRUM_D_OFF + B200_MAX_ROBUST_CLIENTS * B200_MAX_ROBUST_CLIENTS * 8;   // double [32]
constexpr int KRUM_KEPT_OFF = KRUM_SCORE_OFF + B200_MAX_ROBUST_CLIENTS * 8;  // int [32] + the "last CTA" word
constexpr int KRUM_SMEM = KRUM_KEPT_OFF + (B200_MAX_ROBUST_CLIENTS + 4) * 4;

__device__ __forceinline__ uint32_t ld_acquire_gpu_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// pair p of the upper triangle of P rows (row-major: (0,1), (0,2), ..., (1,2), ...)
__device__ __forceinline__ void krum_pair(int p, int P, int& i, int& j) {
  i = 0;
  while (p >= P - 1 - i) {
    p -= P - 1 - i;
    ++i;
  }
  j = i + 1 + p;
}

// one step of the warp transpose-reduce of 16 values: lanes with bit 2H set keep values H .. 2H-1, the others 0 .. H-1,
// each added to its partner's copy
template <int H>
__device__ __forceinline__ void krum_reduce_step(float (&v)[16], int lane) {
  const bool upper = (lane & (2 * H)) != 0;
#pragma unroll
  for (int q = 0; q < H; ++q) {
    const float send = upper ? v[q] : v[q + H];
    const float keep = upper ? v[q + H] : v[q];
    v[q] = __fadd_rn(keep, __shfl_xor_sync(0xffffffffu, send, 2 * H));
  }
}

// this CTA's fp64 sums of (x_i - x_j)^2 over its tiles, for the pair (pi, pj) of this thread (pi < 0: none)
template <int WIRE, int NP>
__device__ __forceinline__ double krum_distances(const FedAvgKrumArgs& a, const uint8_t* const* src, uint32_t* stage,
                                                 float* part, int P, int A, int my_pos, int pi, int pj) {
  constexpr int CH = ROBUST_STAGE / NP;
  constexpr int NB = NP / 4;                      // 4-row blocks
  constexpr int NBLK = NB * (NB + 1) / 2;         // block pairs bi <= bj
  constexpr int SLICES = CH / 128;                // 128-column slices: 4 columns per lane
  constexpr int ITEMS = NBLK * SLICES;
  static_assert(ITEMS % (FEDAVG_THREADS / 32) == 0 && ITEMS <= KRUM_ITEMS, "items must split evenly over the warps");
  const int G = gridDim.x;
  const long long n = a.n;
  const int T = a.tile_elems;
  const long long n_tiles = (n + T - 1) / T;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int my_item = -1, my_idx = 0;
  if (pi >= 0) {
    const int bi = pi >> 2, bj = pj >> 2;
    my_item = (bi * NB - bi * (bi - 1) / 2 + bj - bi) * SLICES;
    my_idx = (pi & 3) * 4 + (pj & 3);
  }
  double acc = 0.0;
  for (long long t = my_pos + static_cast<long long>(blockIdx.x) * A; t < n_tiles; t += static_cast<long long>(G) * A) {
    const long long base = t * T;
    const int len = static_cast<int>((n - base) < T ? (n - base) : T);
    for (int c0 = 0; c0 < len; c0 += CH) {
      const int clen = len - c0 < CH ? len - c0 : CH;
      robust_stage<WIRE, NP>(src, stage, P, n, base + c0, clen);
      __syncthreads();
#pragma unroll 1
      for (int it = warp; it < ITEMS; it += FEDAVG_THREADS / 32) {
        int bi = 0, r = it / SLICES;
        while (r >= NB - bi) {
          r -= NB - bi;
          ++bi;
        }
        const int bj = bi + r, c1 = (it % SLICES) * 128 + lane;
        float v[16];
#pragma unroll
        for (int q = 0; q < 16; ++q) v[q] = 0.f;
#pragma unroll 1
        for (int u = 0; u < 4; ++u) {
          const int c = c1 + 32 * u;
          if (c < clen) {
            float xi[4], xj[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              xi[q] = robust_unkey(stage[(4 * bi + q) * CH + c]);
              xj[q] = robust_unkey(stage[(4 * bj + q) * CH + c]);
            }
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
              for (int w = 0; w < 4; ++w) {
                const float d = __fsub_rn(xi[q], xj[w]);
                v[q * 4 + w] = __fmaf_rn(d, d, v[q * 4 + w]);
              }
          }
        }
        // transpose-reduce: after the step over lane bit o, a lane keeps the half of its values selected by that bit;
        // lane l ends with the warp sum of value ((l >> 1) & 15) (the last step adds the two lanes that share it)
        krum_reduce_step<8>(v, lane);
        krum_reduce_step<4>(v, lane);
        krum_reduce_step<2>(v, lane);
        krum_reduce_step<1>(v, lane);
        v[0] = __fadd_rn(v[0], __shfl_xor_sync(0xffffffffu, v[0], 1));
        if ((lane & 1) == 0) part[it * 16 + (lane >> 1)] = v[0];
      }
      __syncthreads();
      if (my_item >= 0) {
        float sum = 0.f;
#pragma unroll 1
        for (int sl = 0; sl < SLICES; ++sl) sum = __fadd_rn(sum, part[(my_item + sl) * 16 + my_idx]);
        acc += static_cast<double>(sum);
      }
      // the next chunk's stage load may start: the stage was last read before the barrier above, and part is rewritten
      // only after the barrier that follows that load
    }
  }
  return acc;
}

// CTA partials -> this rank's distance page (last CTA to arrive, CTA order); false on timeout (status written)
__device__ __forceinline__ bool krum_rank_reduce(const FedAvgKrumArgs& a, double acc, int npairs, int* s_last) {
  const int G = gridDim.x;
  if (static_cast<int>(threadIdx.x) < npairs) a.work[static_cast<size_t>(blockIdx.x) * KRUM_PAIRS + threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    *s_last = atomicAdd(a.sync, 1u) == static_cast<unsigned>(G - 1);
  }
  __syncthreads();
  bool ok = true;
  if (*s_last) {
    __threadfence();
    if (static_cast<int>(threadIdx.x) < npairs) {
      double d = 0.0;
      for (int b = 0; b < G; ++b)
        d += *reinterpret_cast<const volatile double*>(a.work + static_cast<size_t>(b) * KRUM_PAIRS + threadIdx.x);
      a.dist_page[a.rank][threadIdx.x] = d;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence_system();
      atomicExch(a.sync + 1, 1u);
    }
  } else if (threadIdx.x == 0) {
    unsigned long long spins = 0;
    const unsigned long long limit = a.timeout_log2 > 0 ? (1ull << a.timeout_log2) : ~0ull;
    while (ld_acquire_gpu_u32(a.sync + 1) == 0u) {
      if (++spins > limit) {
        ok = false;
        if (a.status != nullptr) atomicExch(a.status, 1 + a.rank);
        break;
      }
    }
  }
  return __syncthreads_and(ok ? 1 : 0) != 0;
}

template <int WIRE>
__device__ __forceinline__ bool krum_reduce(const FedAvgKrumArgs& a, uint8_t* const* s_wire, const int* s_rank, int A,
                                            int my_pos) {
  extern __shared__ __align__(16) uint8_t robust_smem[];
  uint32_t* stage = reinterpret_cast<uint32_t*>(robust_smem);
  const uint8_t** src = reinterpret_cast<const uint8_t**>(robust_smem + ROBUST_STAGE * 4);
  int* s_P = reinterpret_cast<int*>(robust_smem + ROBUST_STAGE * 4 + B200_MAX_ROBUST_CLIENTS * 8);
  float* part = reinterpret_cast<float*>(robust_smem + KRUM_PART_OFF);
  double* Dm = reinterpret_cast<double*>(robust_smem + KRUM_D_OFF);
  double* score = reinterpret_cast<double*>(robust_smem + KRUM_SCORE_OFF);
  int* kept = reinterpret_cast<int*>(robust_smem + KRUM_KEPT_OFF);
  const int P = robust_gather(a, s_wire, s_rank, A, src, s_P);
  constexpr int MC = B200_MAX_ROBUST_CLIENTS;
  for (int i = threadIdx.x; i < MC * MC; i += FEDAVG_THREADS) Dm[i] = 0.0;
  if (P > 2) {
    const int npairs = P * (P - 1) / 2;
    int pi = -1, pj = -1;
    if (static_cast<int>(threadIdx.x) < npairs) krum_pair(threadIdx.x, P, pi, pj);
    double acc;
    if (P <= 8) acc = krum_distances<WIRE, 8>(a, src, stage, part, P, A, my_pos, pi, pj);
    else if (P <= 16) acc = krum_distances<WIRE, 16>(a, src, stage, part, P, A, my_pos, pi, pj);
    else acc = krum_distances<WIRE, 32>(a, src, stage, part, P, A, my_pos, pi, pj);
    if (!krum_rank_reduce(a, acc, npairs, kept + MC)) return false;
    if (!cta_barrier_all_ranks(a, a.epoch + 2, 0u, nullptr)) return false;
    if (pi >= 0) {
      double d = 0.0;
      for (int k = 0; k < A; ++k) d += *reinterpret_cast<const volatile double*>(a.dist_page[s_rank[k]] + threadIdx.x);
      if ((__double_as_longlong(d) & 0x7FF0000000000000ll) == 0x7FF0000000000000ll) d = __longlong_as_double(0x7FF0000000000000ll);
      Dm[pi * MC + pj] = d;
      Dm[pj * MC + pi] = d;
    }
  }
  __syncthreads();
  // score_i: the k smallest D[i][j], j != i, added in ascending order in fp64
  const int kk = a.krum_k[P], m = a.krum_m[P];
  if (static_cast<int>(threadIdx.x) < P) {
    const int i = threadIdx.x;
    uint32_t taken = 1u << i;
    double acc = 0.0;
    for (int t = 0; t < kk; ++t) {
      int bj = -1;
      double best = 0.0;
      for (int j = 0; j < P; ++j)
        if (!((taken >> j) & 1u) && (bj < 0 || Dm[i * MC + j] < best)) {
          bj = j;
          best = Dm[i * MC + j];
        }
      taken |= 1u << bj;
      acc += best;
    }
    score[i] = acc;
  }
  __syncthreads();
  if (static_cast<int>(threadIdx.x) < P) {
    const int i = threadIdx.x;
    int r = 0;
    for (int j = 0; j < P; ++j) r += (score[j] < score[i] || (score[j] == score[i] && j < i)) ? 1 : 0;
    kept[i] = r < m ? 1 : 0;
  }
  __syncthreads();
  if (blockIdx.x == 0 && a.report != nullptr) {
    for (int i = threadIdx.x; i < MC * MC; i += FEDAVG_THREADS) a.report[1 + i] = Dm[i];
    if (static_cast<int>(threadIdx.x) < MC) {
      a.report[1 + MC * MC + threadIdx.x] = static_cast<int>(threadIdx.x) < P ? score[threadIdx.x] : 0.0;
      a.report[1 + MC * MC + MC + threadIdx.x] = static_cast<int>(threadIdx.x) < P ? kept[threadIdx.x] : 0;
    }
    if (threadIdx.x == 0) a.report[0] = P;
  }
  if (threadIdx.x == 0) {     // the kept segments, in segment order
    int w = 0;
    for (int i = 0; i < P; ++i)
      if (kept[i]) src[w++] = src[i];
  }
  __syncthreads();
  if (m <= 8) robust_tiles<WIRE, 8>(a, s_wire, src, stage, m, A, my_pos);
  else if (m <= 16) robust_tiles<WIRE, 16>(a, s_wire, src, stage, m, A, my_pos);
  else robust_tiles<WIRE, 32>(a, s_wire, src, stage, m, A, my_pos);
  return true;
}

// ---------------------------------------------------------------- top-k rounds (see launch.h / parallel/compress.py)
// Phase 1 of a top-k round: the owner of a tile walks it in chunks of TOPK_CHUNK_G granules (1024 elements each).
//   stage   the chunk's TOPK_CHUNK_G + 1 row pointers of every live participant, one remote load per (rank, word), into
//           shared memory, and the fp32 accumulator tile of the chunk is zeroed;
//   add     warp w owns granule w of the chunk: for every live participant in rank order it adds w_k * value at the
//           entries' offsets, four entries per lane in flight.  Offsets inside one rank's granule are distinct, so the
//           lanes never collide; the __syncwarp between ranks orders the adds of one element by rank, and the sum of
//           every element is fmaf(w_k, x, acc) from 0 over the ranks that sent it, as the dense reduce computes it
//           (a rank that did not send an element would add w_k * 0, which changes nothing);
//   store   the tile is cast to the wire format and stored into seg 0 of every live replica, where the apply finds it.
constexpr int TOPK_CHUNK_G = FEDAVG_THREADS / 32;                  // one granule per warp
constexpr int TOPK_SMEM = TOPK_CHUNK_G * FLAG_GRANULE * 4 + B200_MAX_RANKS * (TOPK_CHUNK_G + 1) * 4;

__device__ __forceinline__ uint32_t ld_volatile_u32(const void* p) {
  uint32_t r;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ uint32_t ld_volatile_u16(const void* p) {
  uint16_t r;
  asm volatile("ld.volatile.global.u16 %0, [%1];" : "=h"(r) : "l"(p) : "memory");
  return r;
}

template <int WIRE>
__device__ __forceinline__ void topk_reduce(const FedAvgTopkArgs& a, uint8_t* const* s_wire, const float* s_w, int A,
                                            int my_pos) {
  static_assert(WIRE == 0 || WIRE == 1, "top-k rounds carry fp32 or bf16 values");
  using W = Wire<WIRE>;
  constexpr int VEC = W::VEC;
  constexpr size_t esz = W::VBYTES / VEC;
  constexpr int U = 4;                               // entries per lane in flight
  extern __shared__ __align__(16) uint8_t topk_smem[];
  float* acc = reinterpret_cast<float*>(topk_smem);
  uint32_t* rp = reinterpret_cast<uint32_t*>(topk_smem + TOPK_CHUNK_G * FLAG_GRANULE * 4);   // [rank pos][CHUNK_G + 1]
  const int G = gridDim.x;
  const long long n = a.n;
  const int T = a.tile_elems;
  const long long n_tiles = (n + T - 1) / T;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long long t = my_pos + static_cast<long long>(blockIdx.x) * A; t < n_tiles; t += static_cast<long long>(G) * A) {
    const long long base = t * T;
    const int ng = static_cast<int>(((n - base) < T ? (n - base) : T) / FLAG_GRANULE);
    for (int c0 = 0; c0 < ng; c0 += TOPK_CHUNK_G) {
      const int cg = ng - c0 < TOPK_CHUNK_G ? ng - c0 : TOPK_CHUNK_G;
      const long long g0 = base / FLAG_GRANULE + c0;
      for (int i = threadIdx.x; i < A * (TOPK_CHUNK_G + 1); i += FEDAVG_THREADS) {
        const int k = i / (TOPK_CHUNK_G + 1), j = i % (TOPK_CHUNK_G + 1);
        if (j <= cg && s_w[k] != 0.f) rp[i] = ld_volatile_u32(s_wire[k] + a.rowptr_off + (g0 + j) * 4);
      }
      for (int i = threadIdx.x * 4; i < cg * FLAG_GRANULE; i += FEDAVG_THREADS * 4)
        *reinterpret_cast<float4*>(acc + i) = make_float4(0.f, 0.f, 0.f, 0.f);
      __syncthreads();
      if (warp < cg) {
        float* ag = acc + warp * FLAG_GRANULE;
#pragma unroll 1
        for (int k = 0; k < A; ++k) {
          const float w = s_w[k];
          if (w == 0.f) continue;
          const uint8_t* src = s_wire[k];
          const uint32_t e1 = rp[k * (TOPK_CHUNK_G + 1) + warp + 1];
#pragma unroll 1
          for (uint32_t e = rp[k * (TOPK_CHUNK_G + 1) + warp] + lane; e < e1; e += 32 * U) {
            uint32_t o[U], v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
              const uint32_t j = e + 32 * u;
              if (j < e1) {
                o[u] = ld_volatile_u16(src + a.off_off + static_cast<size_t>(j) * 2);
                v[u] = WIRE == 0 ? ld_volatile_u32(src + a.val_off + static_cast<size_t>(j) * 4)
                                 : ld_volatile_u16(src + a.val_off + static_cast<size_t>(j) * 2);
              }
            }
#pragma unroll
            for (int u = 0; u < U; ++u)
              if (e + 32 * u < e1) {
                const float x = WIRE == 0 ? __uint_as_float(v[u]) : __uint_as_float(v[u] << 16);
                ag[o[u]] = fmaf(w, x, ag[o[u]]);
              }
          }
          __syncwarp();
        }
      }
      __syncthreads();
      for (int i = threadIdx.x * VEC; i < cg * FLAG_GRANULE; i += FEDAVG_THREADS * VEC) {
        float f[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) f[j] = acc[i + j];
        const uint4 out = W::pack(f, 1.f);
        const size_t off = (base + static_cast<long long>(c0) * FLAG_GRANULE + i) * esz;
#pragma unroll 1
        for (int k = 0; k < A; ++k) W::st_na(s_wire[k] + off, out);
      }
      __syncthreads();   // the next chunk reuses the tile and the row pointers
    }
  }
}

// ---------------------------------------------------------------- secure aggregation (see launch.h / parallel/secagg.py)
// phase 0 of a secure round, after the count barrier: this participant's masked upload over the tiles this CTA packs,
// one 16-element ChaCha20 block per thread and trip (tile_elems % 16 == 0, so a block never straddles a tile).  keys[p] /
// add[p]: the n_peers other participants' pair keys and signs (+ for a higher rank); w: this rank's weight.
__device__ __forceinline__ void secagg_pack(const FedAvgSecAggArgs& a, uint8_t* my_wire, const uint32_t (*keys)[8],
                                            const int* add, int n_peers, float w, int A, int G) {
  const long long n = a.n;
  const int T = a.tile_elems;
  const long long n_tiles = (n + T - 1) / T;
  int sat = 0;
  for (long long q = blockIdx.x; q * A < n_tiles; q += G) {
    for (int r = 0; r < A; ++r) {
      const long long t = q * A + r;
      if (t >= n_tiles) break;
      const long long base = t * T;
      const int len = static_cast<int>((n - base) < T ? (n - base) : T);
      for (int i = threadIdx.x * 16; i < len; i += FEDAVG_THREADS * 16) {
        const int valid = len - i < 16 ? len - i : 16;     // a multiple of 4 (n % 8 == 0)
        float x[16];
#pragma unroll
        for (int j = 0; j < 16; j += 4) {
          float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
          if (j < valid) {
            const float4 th = __ldcs(reinterpret_cast<const float4*>(a.theta + base + i + j));
            const float4 g = __ldcs(reinterpret_cast<const float4*>(a.global_w + base + i + j));
            d = make_float4(__fsub_rn(th.x, g.x), __fsub_rn(th.y, g.y), __fsub_rn(th.z, g.z), __fsub_rn(th.w, g.w));
          }
          x[j] = d.x; x[j + 1] = d.y; x[j + 2] = d.z; x[j + 3] = d.w;
        }
        uint32_t u[16];
        sat += secagg_encode_block(x, valid, w, a.range, a.two_f, n_peers, [&](int p) { return keys[p]; },
                                   [&](int p) { return add[p] != 0; }, static_cast<uint32_t>((base + i) >> 4), a.epoch,
                                   0u, 0u, u);
#pragma unroll
        for (int j = 0; j < 16; j += 4)
          if (j < valid) *reinterpret_cast<uint4*>(my_wire + (base + i + j) * 4) = make_uint4(u[j], u[j + 1], u[j + 2], u[j + 3]);
      }
    }
  }
  if (sat != 0 && a.saturated != nullptr) atomicAdd(a.saturated, static_cast<unsigned long long>(sat));
}

// phase 1 of a secure round: the owner of a tile adds the participants' (part[k] > 0) uploads as uint32 with
// wrap-around, in rank order, eight peer loads in flight, and stores the sum into that tile of every live replica
__device__ __forceinline__ void secagg_reduce(const FedAvgSecAggArgs& a, uint8_t* const* s_wire, const float* part, int A,
                                              int my_pos) {
  constexpr int KG = 8;
  const int G = gridDim.x;
  const long long n = a.n;
  const int T = a.tile_elems;
  const long long n_tiles = (n + T - 1) / T;
  for (long long t = my_pos + static_cast<long long>(blockIdx.x) * A; t < n_tiles; t += static_cast<long long>(G) * A) {
    const long long base = t * T;
    const int len = static_cast<int>((n - base) < T ? (n - base) : T);
    for (int i = threadIdx.x * 4; i < len; i += FEDAVG_THREADS * 4) {
      const size_t off = (base + i) * 4;
      uint4 acc = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 1
      for (int k0 = 0; k0 < A; k0 += KG) {
        uint4 v[KG];
#pragma unroll
        for (int k = 0; k < KG; ++k)
          if (k0 + k < A && part[k0 + k] > 0.f) v[k] = ld_volatile_v4(s_wire[k0 + k] + off);
#pragma unroll
        for (int k = 0; k < KG; ++k)
          if (k0 + k < A && part[k0 + k] > 0.f) {
            acc.x += v[k].x; acc.y += v[k].y; acc.z += v[k].z; acc.w += v[k].w;
          }
      }
#pragma unroll 1
      for (int k = 0; k < A; ++k) st_na_v4(s_wire[k] + off, acc);
    }
  }
}

// ---------------------------------------------------------------- server optimizer (see launch.h / parallel/server_opt.py)
// one element: the state update, then the model update, each operation rounded separately (no FMA contraction)
__device__ __forceinline__ float sopt_step(float x, float d, float& m, float& v, int kind, const float* c) {
  if (kind == 0) {
    m = __fadd_rn(__fmul_rn(c[0], m), d);
    return __fadd_rn(x, __fmul_rn(c[4], m));
  }
  m = __fadd_rn(__fmul_rn(c[0], m), __fmul_rn(c[1], d));
  const float dd = __fmul_rn(d, d);
  if (kind == 1) {
    v = __fadd_rn(v, dd);
  } else if (kind == 2) {
    const float s = __fsub_rn(v, dd);
    v = __fsub_rn(v, __fmul_rn(__fmul_rn(c[3], dd), s > 0.f ? 1.f : (s < 0.f ? -1.f : 0.f)));
  } else {
    v = __fadd_rn(__fmul_rn(c[2], v), __fmul_rn(c[3], dd));
  }
  return __fadd_rn(x, __fdiv_rn(__fmul_rn(c[4], m), __fadd_rn(__fsqrt_rn(v), c[5])));
}

// the apply phase of one tile in a server-optimizer round: ONE wire vector per trip (the plain loop's two, plus m and v,
// would not fit under the 96-register cap).  Parameter vectors (n_param % 8 == 0: a vector never straddles it) take
// the step, or keep the global model when the round had no weight (step == false); buffers take global += d as in the
// plain loop.  Then theta, the bf16 shadow and the momentum reset, as there.
// Personalized rounds (LocalArgs): the shift from logical element e to its physical arena element, which skips the
// local range [lo, lo + len); 0 in every other round, so their address arithmetic is unchanged.  e and e + VEC - 1 are
// on the same side of lo (a multiple of 1024), so one shift serves a whole wire vector.
template <bool LOCAL, typename Args>
__device__ __forceinline__ long long local_shift(const Args& a, long long e) {
  if constexpr (LOCAL) return e >= a.lo ? a.len : 0ll;
  else return 0ll;
}

template <int WIRE, bool LOCAL, typename Args>
__device__ __forceinline__ void sopt_apply_tile(const Args& a, const uint8_t* my_wire, long long base, int len,
                                                float apply_scale, bool step) {
  using W = Wire<WIRE>;
  constexpr int VEC = W::VEC;
  constexpr size_t esz = W::VBYTES / VEC;
  const size_t sc_off = static_cast<size_t>(a.n);
  for (int i = threadIdx.x * VEC; i < len; i += FEDAVG_THREADS * VEC) {
    const long long le = base + i;                    // logical: the wire
    const uint4 wv = W::ld(my_wire + le * esz);
    float scale = 1.f;
    if constexpr (W::SCALED) scale = exp2_int(static_cast<int>(ld_volatile_u8(my_wire + sc_off + (le >> 5))) - 127);
    float f[VEC];
    W::unpack(wv, f, scale);
    const long long e = le + local_shift<LOCAL>(a, le);   // physical: the replica and the server state
    const bool opt = e < a.n_param;
#pragma unroll
    for (int j = 0; j < VEC; j += 4) {
      const float4 g = *reinterpret_cast<const float4*>(a.global_w + e + j);
      float4 nw = g;
      if (opt) {
        if (step) {
          float4 m4 = *reinterpret_cast<const float4*>(a.m + e + j);
          float4 v4 = make_float4(0.f, 0.f, 0.f, 0.f);
          if (a.kind != 0) v4 = *reinterpret_cast<const float4*>(a.v + e + j);
          nw.x = sopt_step(g.x, __fmul_rn(f[j], apply_scale), m4.x, v4.x, a.kind, a.coef);
          nw.y = sopt_step(g.y, __fmul_rn(f[j + 1], apply_scale), m4.y, v4.y, a.kind, a.coef);
          nw.z = sopt_step(g.z, __fmul_rn(f[j + 2], apply_scale), m4.z, v4.z, a.kind, a.coef);
          nw.w = sopt_step(g.w, __fmul_rn(f[j + 3], apply_scale), m4.w, v4.w, a.kind, a.coef);
          *reinterpret_cast<float4*>(a.m + e + j) = m4;
          if (a.kind != 0) *reinterpret_cast<float4*>(a.v + e + j) = v4;
        }
      } else {
        nw = make_float4(f[j] * apply_scale + g.x, f[j + 1] * apply_scale + g.y, f[j + 2] * apply_scale + g.z,
                         f[j + 3] * apply_scale + g.w);
      }
      *reinterpret_cast<float4*>(a.global_w + e + j) = nw;
      *reinterpret_cast<float4*>(a.theta + e + j) = nw;
      if (a.momentum != nullptr && e + j < a.n_momentum)
        *reinterpret_cast<float4*>(a.momentum + e + j) = make_float4(0.f, 0.f, 0.f, 0.f);
      if (a.theta_bf16 != nullptr) {
        const uint2 o = make_uint2(pack_bf16x2(nw.x, nw.y), pack_bf16x2(nw.z, nw.w));
        *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(a.theta_bf16) + (e + j) * 2) = o;
      }
    }
  }
}

// The kind of aggregation a round runs.  Every kind is one args struct of launch.h, and RoundOf maps the struct to its
// kind (and whether the apply phase runs the server optimizer): fedavg_round_kernel<WIRE, Args> is the round's kernel.
enum class Agg { mean, dp, scaffold, robust, krum, topk, secagg };
template <class Args> struct RoundOf;
template <Agg K> struct RoundKind {
  static constexpr Agg kind = K;
  static constexpr bool sopt = false, local = false;
};
template <> struct RoundOf<FedAvgArgs> : RoundKind<Agg::mean> {};
template <> struct RoundOf<FedAvgDPArgs> : RoundKind<Agg::dp> {};
template <> struct RoundOf<FedAvgScaffoldArgs> : RoundKind<Agg::scaffold> {};
template <> struct RoundOf<FedAvgRobustArgs> : RoundKind<Agg::robust> {};
template <> struct RoundOf<FedAvgKrumArgs> : RoundKind<Agg::krum> {};
template <> struct RoundOf<FedAvgTopkArgs> : RoundKind<Agg::topk> {};
template <> struct RoundOf<FedAvgSecAggArgs> : RoundKind<Agg::secagg> {};
template <class Base> struct RoundOf<ServerOptArgs<Base>> {
  static constexpr Agg kind = RoundOf<Base>::kind;
  static constexpr bool sopt = true, local = false;
};
template <class Base> struct RoundOf<LocalArgs<Base>> {
  static constexpr Agg kind = RoundOf<Base>::kind;
  static constexpr bool sopt = RoundOf<Base>::sopt, local = true;
};

// K == Agg::mean: the weighted mean w_k = n_k / N.
// Agg::dp: DP-FedAvg (see launch.h / DESIGN.md): w_k = n_k s_k / N with s_k from rank k's clip page, and the owner of a
// tile adds sigma C / N * z[i] to its fp32 sum before the cast.  The loss and the integer side arena keep the weights
// n_k / N.
// Agg::scaffold: a SCAFFOLD round -- segment 1 (the control variates, see seg_pack) rides between the same barriers;
// every participant weighs 1 / N there.
// Agg::robust: a robust round (robust_reduce above); every rank publishes its segment count before barrier 1.
// Agg::krum: a Multi-Krum round (krum_reduce above), a robust round whose exchange barrier takes epoch + 2 and barrier 2
// epoch + 3.
// Agg::topk: a top-k round (topk_reduce above): no pack phase, the uploads are sparse lists written before the launch.
// Agg::secagg: a secure-aggregation round (WIRE 3, see launch.h): the count barrier (epoch + 1) comes before the pack
// (secagg_pack above), barrier 1 takes epoch + 2, the reduce is secagg_reduce, barrier 2 takes epoch + 3.
// SOPT (with any kind): a server-optimizer round -- the apply phase runs sopt_apply_tile.
// LOCAL (with the mean): a personalized round -- n is the logical element count, and the pack and apply phases address
// the replica at the physical element local_shift gives (see LocalArgs in launch.h).
// The whole round; Args is the kind's args struct (ServerOptArgs<that> when SOPT, LocalArgs<...> when LOCAL), see RoundOf.
template <int WIRE, Agg K, bool SOPT, bool LOCAL, typename Args>
__device__ __forceinline__ void fedavg_round(const Args& a) {
  constexpr bool DP = K == Agg::dp, SCAF = K == Agg::scaffold, KRUM = K == Agg::krum, TOPK = K == Agg::topk;
  constexpr bool ROBUST = K == Agg::robust || KRUM;
  constexpr bool SECAGG = K == Agg::secagg;
  using W = Wire<WIRE>;
  constexpr int VEC = W::VEC;
  constexpr bool SCALED = W::SCALED;
  const int G = gridDim.x;
  __shared__ uint8_t* s_wire[B200_MAX_RANKS];   // indexed by position among the live ranks
  __shared__ long long* s_int[B200_MAX_RANKS];
  __shared__ float* s_loss[B200_MAX_RANKS];
  __shared__ int s_rank[B200_MAX_RANKS];
  __shared__ float s_w[B200_MAX_RANKS];
  __shared__ uint32_t s_payload[B200_MAX_RANKS];  // indexed by rank
  __shared__ float s_inv_total;
  __shared__ float s_part[DP || SECAGG ? B200_MAX_RANKS : 1];   // DP: participation weights n_k / N (loss, integer
                                                                 // arena); secure rounds: the counts n_k
  __shared__ uint32_t s_key[SECAGG ? B200_MAX_RANKS : 1][8];     // secure rounds: the other participants' pair keys
  __shared__ int s_add[SECAGG ? B200_MAX_RANKS : 1];             // ... and signs (1: a higher rank, added)
  __shared__ int s_npeer;
  int A = 0, my_pos = -1;
  for (int k = 0; k < a.world; ++k)
    if ((a.alive_mask >> k) & 1u) {
      if (k == a.rank) my_pos = A;
      if (threadIdx.x == 0) {
        s_wire[A] = reinterpret_cast<uint8_t*>(a.wire[k]);
        s_int[A] = a.int_wire[k];
        s_loss[A] = a.loss_wire[k];
        s_rank[A] = k;
      }
      ++A;
    }
  if (my_pos < 0 || A == 0) return;
  const long long n = a.n;
  const int T = a.tile_elems;
  const long long n_tiles = (n + T - 1) / T;
  const float my_n = a.n_samples[a.rank];
  constexpr size_t esz = W::VBYTES / VEC;         // payload bytes per element
  const size_t sc_off = static_cast<size_t>(n);   // SCALED: scale bytes live behind the n payload bytes
  const int lane_elems = static_cast<int>(threadIdx.x & 31) * VEC;
  uint8_t* my_wire = reinterpret_cast<uint8_t*>(a.wire[a.rank]);
  const float* __restrict__ theta_r = a.theta;
  const float* __restrict__ global_r = a.global_w;

  // ---------------------------------------------------------------- phase 0: pack (+ prescale) + cast
  // P2P mode applies w_k on the reader side (the upload keeps full wire precision); NVLS mode needs
  // the scaled value on the wire because the switch can only add: scale by n_k now, by 1/N in phase 2.
  // Loop bounds are warp-uniform (first lane's element) so the block-scale shuffles are legal.
  const float pack_scale = a.use_nvls ? my_n * a.nvls_prescale : 1.0f;
  phase_stamp(a, 0);                                   // start
  if constexpr (SECAGG) {
    // the count barrier: every rank learns the counts, hence the participants and the weights, before anyone packs
    if (!cta_barrier_all_ranks(a, a.epoch + 1, __float_as_uint(my_n), s_payload)) return;
    if (threadIdx.x == 0) {          // IEEE-rounded operations: the weights are bit-equal to the host reference's
      float total = 0.f;
      for (int k = 0; k < A; ++k) {
        const float nk = a.counts_from_flags ? __uint_as_float(s_payload[s_rank[k]]) : a.n_samples[s_rank[k]];
        s_part[k] = nk;
        total = __fadd_rn(total, nk);
      }
      const float inv = total > 0.f ? __fdiv_rn(1.f, total) : 0.f;
      int np = 0;
      for (int k = 0; k < A; ++k) {
        s_w[k] = __fmul_rn(s_part[k], inv);
        if (k != my_pos && s_part[k] > 0.f) {
          s_add[np] = s_rank[k] > a.rank ? 1 : 0;
          for (int j = 0; j < 8; ++j) s_key[np][j] = a.keys[s_rank[k]][j];
          ++np;
        }
      }
      s_npeer = np;
      s_inv_total = inv;
    }
    __syncthreads();
    if (s_part[my_pos] > 0.f) secagg_pack(a, my_wire, s_key, s_add, s_npeer, s_w[my_pos], A, G);
  } else if (!TOPK && (my_n != 0.f || a.use_nvls) && !a.prepacked) {
    for (long long q = blockIdx.x; q * A < n_tiles; q += G) {
      for (int r = 0; r < A; ++r) {
        const long long t = q * A + r;
        if (t >= n_tiles) break;
        const long long base = t * T;
        const int len = static_cast<int>((n - base) < T ? (n - base) : T);
        constexpr int STEP = FEDAVG_THREADS * VEC;
        for (int i0 = threadIdx.x * VEC; i0 - lane_elems < len; i0 += 2 * STEP) {
          // two independent wire vectors per trip, every load issued before the first store
          float4 th[2][VEC / 4], gg[2][VEC / 4];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int i = i0 + u * STEP;
            if (i < len) {
              const long long sh = local_shift<LOCAL>(a, base + i);
#pragma unroll
              for (int j = 0; j < VEC; j += 4) {
                th[u][j >> 2] = __ldcs(reinterpret_cast<const float4*>(theta_r + base + i + j + sh));
                if (a.delta) gg[u][j >> 2] = __ldcs(reinterpret_cast<const float4*>(global_r + base + i + j + sh));
              }
            }
          }
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int i = i0 + u * STEP;
            const bool valid = i < len;
            float f[VEC];
#pragma unroll
            for (int j = 0; j < VEC; ++j) f[j] = 0.f;
            if (valid) {
#pragma unroll
              for (int j = 0; j < VEC; j += 4) {
                float4 t4 = th[u][j >> 2];
                if (a.delta) {
                  const float4 g = gg[u][j >> 2];
                  t4.x -= g.x; t4.y -= g.y; t4.z -= g.z; t4.w -= g.w;
                }
                f[j] = t4.x * pack_scale; f[j + 1] = t4.y * pack_scale;
                f[j + 2] = t4.z * pack_scale; f[j + 3] = t4.w * pack_scale;
              }
            }
            float inv = 1.f;
            if constexpr (SCALED) {
              if (i0 + u * STEP - lane_elems < len) {          // warp-uniform
                const int e = quad_block_exponent<VEC>(f);
                inv = exp2_int(-e);
                if (valid && (threadIdx.x & 3) == 0) my_wire[sc_off + ((base + i) >> 5)] = static_cast<uint8_t>(e + 127);
              }
            }
            if (valid) W::st(my_wire + (base + i) * esz, W::pack(f, inv));
          }
        }
      }
    }
  }
  if constexpr (SCAF) {
    if (my_n != 0.f) seg_pack<WIRE>(my_wire + a.seg1_off, a.dc, a.n_c, T, A, G);
  }
  if (blockIdx.x == 0) {
    // integer side arena (num_batches_tracked ...) and the local per-epoch losses
    for (int i = threadIdx.x; i < a.n_int; i += FEDAVG_THREADS) a.int_wire[a.rank][i] = a.int_local[i];
    for (int i = threadIdx.x; i < a.n_loss; i += FEDAVG_THREADS) a.loss_wire[a.rank][i] = a.loss_local[i];
  }
  if constexpr (ROBUST) {
    // every CTA publishes the count (same value): CTA b's barrier then covers it for CTA b of every peer
    if (threadIdx.x == 0) *reinterpret_cast<volatile uint32_t*>(a.seg_page[a.rank]) = a.my_segs;
  }
  phase_stamp(a, 1);                                   // pack done
  if (!cta_barrier_all_ranks(a, a.epoch + (SECAGG ? 2 : 1), __float_as_uint(my_n), s_payload)) return;
  phase_stamp(a, 2);                                   // barrier 1 passed

  // weights w_k = n_k / N from the counts that rode on the barrier flags (or the host's plan)
  if (!SECAGG && threadIdx.x == 0) {
    float total = 0.f;
    for (int k = 0; k < A; ++k) {
      const float nk = a.counts_from_flags ? __uint_as_float(s_payload[s_rank[k]]) : a.n_samples[s_rank[k]];
      s_w[k] = nk;
      total += nk;
    }
    const float inv = total > 0.f ? 1.f / total : 0.f;
    if constexpr (DP) {
      for (int k = 0; k < A; ++k) {
        s_part[k] = s_w[k] * inv;
        // a non-participant's page may hold an older round's factor: only read it for n_k != 0
        s_w[k] = s_w[k] != 0.f ? s_w[k] * *reinterpret_cast<const volatile float*>(a.clip_page[s_rank[k]]) : 0.f;
      }
    }
    for (int k = 0; k < A; ++k) s_w[k] *= inv;
    s_inv_total = inv;
  }
  __syncthreads();

  // ---------------------------------------------------------------- phase 1: reduce + broadcast
  // A remote 16-byte load costs a full NVLink round trip (microseconds); with few ranks a thread that handles ONE wire
  // vector per trip has only A loads in flight and cannot keep the link busy.  Each trip therefore handles U vectors, U chosen so that
  // about eight remote loads per thread are in flight whatever the number of ranks.
  auto reduce_tiles = [&](auto u_tag) {
    constexpr int U = decltype(u_tag)::value;
    constexpr int KG = 8 / U;          // ranks per load group: U * KG = 8 wire vectors in flight per thread
    for (long long t = my_pos + static_cast<long long>(blockIdx.x) * A; t < n_tiles; t += static_cast<long long>(G) * A) {
      const long long base = t * T;
      const int len = static_cast<int>((n - base) < T ? (n - base) : T);
      constexpr int STEP = FEDAVG_THREADS * VEC;
      for (int i0 = threadIdx.x * VEC; i0 - lane_elems < len; i0 += U * STEP) {
        if (!SCALED && a.use_nvls) {
          uint4 out[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int i = i0 + u * STEP;
            if (i < len)      // the switch adds the replicas
              out[u] = W::mc_reduce(reinterpret_cast<const uint8_t*>(a.wire_mc) + (base + i) * esz);
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int i = i0 + u * STEP;
            if (i < len)      // the switch replicates the store
              multimem_st_v4(reinterpret_cast<uint8_t*>(a.wire_mc) + (base + i) * esz, out[u]);
          }
          continue;
        }
        // peers in groups of 8 (one NVSwitch box): issue the group's loads first (memory-level parallelism), then
        // accumulate in fixed rank order so the result is bitwise reproducible
        float acc[U][VEC];
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
          for (int j = 0; j < VEC; ++j) acc[u][j] = 0.f;
#pragma unroll 1
        for (int k0 = 0; k0 < A; k0 += KG) {
          uint4 v[U][KG];
          uint32_t sc[U][KG];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int i = i0 + u * STEP;
            if (i < len) {
              const size_t off = (base + i) * esz;
#pragma unroll
              for (int k = 0; k < KG; ++k)
                if (k0 + k < A && s_w[k0 + k] != 0.f) {
                  v[u][k] = W::ld(s_wire[k0 + k] + off);
                  if constexpr (SCALED) sc[u][k] = ld_volatile_u8(s_wire[k0 + k] + sc_off + ((base + i) >> 5));
                }
            }
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int i = i0 + u * STEP;
            if (i < len) {
#pragma unroll
              for (int k = 0; k < KG; ++k) {
                if (k0 + k < A) {
                  const float w = s_w[k0 + k];
                  if (w != 0.f) {
                    float f[VEC];
                    float scale = 1.f;
                    if constexpr (SCALED) scale = exp2_int(static_cast<int>(sc[u][k]) - 127);
                    W::unpack(v[u][k], f, scale);
#pragma unroll
                    for (int j = 0; j < VEC; ++j) acc[u][j] = fmaf(w, f[j], acc[u][j]);
                  }
                }
              }
            }
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int i = i0 + u * STEP;
          const bool valid = i < len;
          if constexpr (DP) {
            if (valid) {
              const float ns = a.noise_std * s_inv_total;
#pragma unroll
              for (int j = 0; j < VEC; j += 4) {
                const float4 z = dp_normal4(a.seed, a.round, static_cast<unsigned long long>(base + i + j) >> 2);
                acc[u][j] = fmaf(ns, z.x, acc[u][j]); acc[u][j + 1] = fmaf(ns, z.y, acc[u][j + 1]);
                acc[u][j + 2] = fmaf(ns, z.z, acc[u][j + 2]); acc[u][j + 3] = fmaf(ns, z.w, acc[u][j + 3]);
              }
            }
          }
          float inv = 1.f;
          int e = 0;
          if constexpr (SCALED) {
            if (i - lane_elems < len) {                  // warp-uniform: every lane of the warp takes part in the shuffles
              e = quad_block_exponent<VEC>(acc[u]);
              inv = exp2_int(-e);
            }
          }
          if (valid) {
            const size_t off = (base + i) * esz;
            const uint4 out = W::pack(acc[u], inv);
#pragma unroll
            for (int k = 0; k < B200_MAX_RANKS; ++k)
              if (k < A) {
                W::st_na(s_wire[k] + off, out);
                if constexpr (SCALED)
                  if ((threadIdx.x & 3) == 0)
                    st_volatile_u8(s_wire[k] + sc_off + ((base + i) >> 5), static_cast<uint32_t>(e + 127));
              }
          }
        }
      }
    }
  };
  if constexpr (KRUM) {
    if (!krum_reduce<WIRE>(a, s_wire, s_rank, A, my_pos)) return;
  } else if constexpr (TOPK) {
    topk_reduce<WIRE>(a, s_wire, s_w, A, my_pos);
  } else if constexpr (SECAGG) {
    secagg_reduce(a, s_wire, s_part, A, my_pos);
  } else if constexpr (ROBUST) {
    robust_reduce<WIRE>(a, s_wire, s_rank, A, my_pos);
  } else if constexpr (SCAF) {
    // one wire vector per trip: the same sums in the same rank order as the wider trips, in fewer registers
    reduce_tiles(std::integral_constant<int, 1>{});
  } else if constexpr (SOPT) {
    // at most two vectors per trip (one with DP's noise): with more, the server-optimizer kernels spill (the same sums
    // in the same order)
    if (!DP && A <= 4) reduce_tiles(std::integral_constant<int, 2>{});
    else reduce_tiles(std::integral_constant<int, 1>{});
  } else {
    if (A <= 2) reduce_tiles(std::integral_constant<int, 4>{});
    else if (A <= 4) reduce_tiles(std::integral_constant<int, 2>{});
    else reduce_tiles(std::integral_constant<int, 1>{});
  }
  if constexpr (SCAF) seg_reduce<WIRE>(s_wire, s_w, static_cast<size_t>(a.seg1_off), a.inv_clients, a.n_c, T, A, G, my_pos);
  // weighted per-epoch loss (manager.py:127-130); every rank computes the same tiny vector
  if (blockIdx.x == 0 && a.loss_out != nullptr) {
    for (int e = threadIdx.x; e < a.n_loss; e += FEDAVG_THREADS) {
      float acc = 0.f;
      for (int k = 0; k < A; ++k)
        if constexpr (DP) {
          if (s_part[k] != 0.f) acc = fmaf(s_part[k], *reinterpret_cast<volatile float*>(s_loss[k] + e), acc);
        } else if (s_w[k] != 0.f) {
          acc = fmaf(s_w[k], *reinterpret_cast<volatile float*>(s_loss[k] + e), acc);
        }
      a.loss_out[e] = acc;
    }
  }
  phase_stamp(a, 3);                                   // reduce + broadcast done
  if (!cta_barrier_all_ranks(a, a.epoch + (KRUM || SECAGG ? 3 : 2), 0u, nullptr)) return;
  phase_stamp(a, 4);                                   // barrier 2 passed

  // ---------------------------------------------------------------- phase 2: running-mean apply
  // CTA b applies exactly the tiles CTA b of the owners produced: (t / A) % G == b
  float apply_scale = a.use_nvls ? s_inv_total / a.nvls_prescale : 1.0f;
  if constexpr (SECAGG) apply_scale = a.inv_two_f;
  for (long long q = blockIdx.x; q * A < n_tiles; q += G) {
    for (int r = 0; r < A; ++r) {
      const long long t = q * A + r;
      if (t >= n_tiles) break;
      const long long base = t * T;
      const int len = static_cast<int>((n - base) < T ? (n - base) : T);
      constexpr int STEP = FEDAVG_THREADS * VEC;
      if constexpr (SOPT) sopt_apply_tile<WIRE, LOCAL>(a, my_wire, base, len, apply_scale, s_inv_total != 0.f);
      else for (int i0 = threadIdx.x * VEC; i0 < len; i0 += 2 * STEP) {
        uint4 wv[2];
        uint32_t sc[2];
        float4 gg[2][VEC / 4];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int i = i0 + u * STEP;
          if (i < len) {
            wv[u] = W::ld(my_wire + (base + i) * esz);
            if constexpr (SCALED) sc[u] = ld_volatile_u8(my_wire + sc_off + ((base + i) >> 5));
            if (a.delta) {
              const long long sh = local_shift<LOCAL>(a, base + i);
#pragma unroll
              for (int j = 0; j < VEC; j += 4)
                gg[u][j >> 2] = *reinterpret_cast<const float4*>(a.global_w + base + i + j + sh);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int i = i0 + u * STEP;
          if (i < len) {
            float f[VEC];
            float scale = 1.f;
            if constexpr (SCALED) scale = exp2_int(static_cast<int>(sc[u]) - 127);
            W::unpack(wv[u], f, scale);
            const long long sh = local_shift<LOCAL>(a, base + i);
#pragma unroll
            for (int j = 0; j < VEC; j += 4) {
              float4 nw = make_float4(f[j] * apply_scale, f[j + 1] * apply_scale, f[j + 2] * apply_scale,
                                      f[j + 3] * apply_scale);
              if (a.delta) {
                const float4 g = gg[u][j >> 2];
                nw.x += g.x; nw.y += g.y; nw.z += g.z; nw.w += g.w;
              }
              if (a.global_w != nullptr) *reinterpret_cast<float4*>(a.global_w + base + i + j + sh) = nw;
              *reinterpret_cast<float4*>(a.theta + base + i + j + sh) = nw;
              if (a.momentum != nullptr && base + i + j + sh < a.n_momentum)
                *reinterpret_cast<float4*>(a.momentum + base + i + j + sh) = make_float4(0.f, 0.f, 0.f, 0.f);
              if (a.theta_bf16 != nullptr) {
                const uint2 o = make_uint2(pack_bf16x2(nw.x, nw.y), pack_bf16x2(nw.z, nw.w));
                *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(a.theta_bf16) + (base + i + j + sh) * 2) = o;
              }
            }
          }
        }
      }
      if (a.tile_flags != nullptr) {
        // arrival flags have a FIXED granularity of FLAG_GRANULE elements (work tiles are multiples of it), so a consumer
        // captured in a CUDA graph indexes them without knowing this round's tile size: flag[e / 1024] >= round means
        // theta / global / bf16 shadow of elements [1024 f, 1024 f + 1024) carry the new global model
        __syncthreads();  // every thread's stores of this tile are done
        const int ng = (len + FLAG_GRANULE - 1) / FLAG_GRANULE;
        for (int g = threadIdx.x; g < ng; g += FEDAVG_THREADS) {
          __threadfence();
          st_release_sys(a.tile_flags + base / FLAG_GRANULE + g, a.flag_value);
        }
      }
    }
  }
  if constexpr (SCAF) seg_apply_add<WIRE>(my_wire + a.seg1_off, a.c, a.n_c, T, A, G);
  // integer side arena: max over participants (BatchNorm step counters only ever grow)
  if (a.n_int > 0 && blockIdx.x == 0) {
    for (int i = threadIdx.x; i < a.n_int; i += FEDAVG_THREADS) {
      long long m = a.int_local[i];
      for (int k = 0; k < A; ++k)
        if ((DP ? s_part[k] : s_w[k]) != 0.f) {
          const long long v = *reinterpret_cast<volatile long long*>(s_int[k] + i);
          m = v > m ? v : m;
        }
      a.int_local[i] = m;
    }
  }
  // No closing barrier: the wire buffer and the int / loss pages are DOUBLE-BUFFERED by round parity (the host passes
  // the addresses of this round's half).  A rank that races ahead packs round r+1 into the other half while a slow
  // peer still applies round r from this one; the half is reused in round r+2, and nobody can be there before every
  // rank has passed barrier 2 of round r+1, i.e. has left round r altogether.  The pads hold monotone epochs
  // (a faster rank's next-round arrival also satisfies this round's wait), so they need no parity.
  phase_stamp(a, 5);                                   // apply done
  phase_stamp(a, 6);
}

// One 512-thread CTA per SM, capped at 96 registers per thread (48 K of the SM's 64 K): the rest of the register file
// stays available to small kernels of the NEXT round (batch gather, im2col, the flag-gated weight staging of
// bcast_gemm) that are launched on the compute stream while this kernel is still running on its side stream -- and
// a flag-gated consumer that became resident first can never keep this (cooperatively launched) grid from fitting.
// Robust, Krum and top-k rounds also take dynamic shared memory (ROBUST_SMEM, KRUM_SMEM, TOPK_SMEM: see round_smem).
template <int WIRE, typename Args>
__global__ void __maxnreg__(96) fedavg_round_kernel(const __grid_constant__ Args a) {
  fedavg_round<WIRE, RoundOf<Args>::kind, RoundOf<Args>::sopt, RoundOf<Args>::local>(a);
}

// one logical client's upload into its wire segment: the phase-0 pack of fedavg_round (delta mode, scale 1) over the
// whole arena, plus fold_client_kernel's replica reset.  Loop bounds are warp-uniform so the fp8 quads can shuffle.
template <int WIRE>
__global__ void __launch_bounds__(256)
pack_client_kernel(uint8_t* __restrict__ seg, float* __restrict__ theta, const float* __restrict__ global_w,
                   __nv_bfloat16* __restrict__ wb, float* __restrict__ mom, long long n_mom, long long n, int reset) {
  using W = Wire<WIRE>;
  constexpr int VEC = W::VEC;
  constexpr size_t esz = W::VBYTES / VEC;
  const long long nvec = n / VEC;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const int lane = threadIdx.x & 31;
  for (long long v0 = static_cast<long long>(blockIdx.x) * blockDim.x + (threadIdx.x & ~31); v0 < nvec; v0 += stride) {
    const long long v = v0 + lane;
    const bool valid = v < nvec;
    float f[VEC];
    float4 g[VEC / 4];
#pragma unroll
    for (int j = 0; j < VEC; ++j) f[j] = 0.f;
    if (valid) {
#pragma unroll
      for (int j = 0; j < VEC; j += 4) {
        const float4 t = *reinterpret_cast<const float4*>(theta + v * VEC + j);
        g[j >> 2] = *reinterpret_cast<const float4*>(global_w + v * VEC + j);
        f[j] = t.x - g[j >> 2].x; f[j + 1] = t.y - g[j >> 2].y;
        f[j + 2] = t.z - g[j >> 2].z; f[j + 3] = t.w - g[j >> 2].w;
      }
    }
    float inv = 1.f;
    if constexpr (W::SCALED) {
      const int e = quad_block_exponent<VEC>(f);
      inv = exp2_int(-e);
      if (valid && (lane & 3) == 0) seg[n + ((v * VEC) >> 5)] = static_cast<uint8_t>(e + 127);
    }
    if (valid) {
      W::st(seg + v * VEC * esz, W::pack(f, inv));
      if (reset) {
#pragma unroll
        for (int j = 0; j < VEC; j += 4) {
          const long long i = v * VEC + j;
          *reinterpret_cast<float4*>(theta + i) = g[j >> 2];
          if (wb != nullptr)
            *reinterpret_cast<uint2*>(wb + i) = make_uint2(pack_bf16x2(g[j >> 2].x, g[j >> 2].y),
                                                           pack_bf16x2(g[j >> 2].z, g[j >> 2].w));
          if (mom != nullptr && i < n_mom) *reinterpret_cast<float4*>(mom + i) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    }
  }
}

// ---------------------------------------------------------------- DP clip factor and clipped logical-client fold
// ||theta - global||^2 over [0, n): a FIXED grid of B200_DP_NORM_BLOCKS CTAs (independent of the SM count), fp64
// throughout (differences and squares too, so no finite update overflows to a non-finite norm), one slot of `work` per
// CTA, and the last CTA to finish sums the slots in index order -- two launches on the same data give the same bits.  work[B200_DP_NORM_BLOCKS] is the arrival counter (reset by the last CTA).
constexpr int DP_NORM_THREADS = 256;
__global__ void __launch_bounds__(DP_NORM_THREADS)
dp_clip_factor_kernel(const float* __restrict__ theta, const float* __restrict__ global_w, long long n, float clip,
                      unsigned long long* __restrict__ work, float* s_out, float* norm_out, float* s_copy, int* nonfinite) {
  __shared__ double red[DP_NORM_THREADS / 32];
  __shared__ bool last;
  const long long nv = n >> 2;
  double d = 0.0;
  for (long long i = blockIdx.x * static_cast<long long>(DP_NORM_THREADS) + threadIdx.x; i < nv;
       i += static_cast<long long>(B200_DP_NORM_BLOCKS) * DP_NORM_THREADS) {
    const float4 t = __ldcs(reinterpret_cast<const float4*>(theta) + i);
    const float4 g = __ldcs(reinterpret_cast<const float4*>(global_w) + i);
    const double dx = static_cast<double>(t.x) - g.x, dy = static_cast<double>(t.y) - g.y;
    const double dz = static_cast<double>(t.z) - g.z, dw = static_cast<double>(t.w) - g.w;
    d = fma(dx, dx, d); d = fma(dy, dy, d); d = fma(dz, dz, d); d = fma(dw, dw, d);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = d;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
    for (int w = 0; w < DP_NORM_THREADS / 32; ++w) b += red[w];
    reinterpret_cast<double*>(work)[blockIdx.x] = b;
    __threadfence();
    last = atomicAdd(work + B200_DP_NORM_BLOCKS, 1ull) == B200_DP_NORM_BLOCKS - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  double sq = 0.0;
  for (int b = 0; b < B200_DP_NORM_BLOCKS; ++b) sq += reinterpret_cast<const volatile double*>(work)[b];
  work[B200_DP_NORM_BLOCKS] = 0ull;
  const double norm = sqrt(sq);
  float s;
  if (!isfinite(norm)) {
    s = 0.f;
    if (nonfinite != nullptr) atomicAdd(nonfinite, 1);
  } else {
    s = norm > static_cast<double>(clip) ? static_cast<float>(static_cast<double>(clip) / norm) : 1.f;
  }
  s_out[0] = s;
  if (s_copy != nullptr) s_copy[0] = s;
  norm_out[0] = static_cast<float>(norm);
}

// acc (+)= s * (theta - global) with s = *s_dev (written by dp_clip_factor_kernel just before), and the replica reset of
// fold_client_kernel (elementwise.cu), which this mirrors; kept separate so that kernel's instruction stream is unchanged.
// Unlike it, this one is launched without programmatic dependent launch: it follows the norm kernel, a plain launch.
// s == 0 (non-finite update): the client adds nothing, and its NaNs never reach acc.
__global__ void __launch_bounds__(DP_NORM_THREADS)
fold_client_scaled_kernel(float* __restrict__ acc, float* __restrict__ theta, const float* __restrict__ global_w,
                          __nv_bfloat16* __restrict__ wb, float* __restrict__ mom, long long n_mom, long long n,
                          const float* __restrict__ s_dev, int first, int reset) {
  const float s = *s_dev;
  const long long nv = n >> 2;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 g = reinterpret_cast<const float4*>(global_w)[i];
    const float4 t = reinterpret_cast<const float4*>(theta)[i];
    float4 a = first ? make_float4(0.f, 0.f, 0.f, 0.f) : reinterpret_cast<const float4*>(acc)[i];
    if (s != 0.f) {
      a.x = fmaf(s, t.x - g.x, a.x); a.y = fmaf(s, t.y - g.y, a.y);
      a.z = fmaf(s, t.z - g.z, a.z); a.w = fmaf(s, t.w - g.w, a.w);
    }
    reinterpret_cast<float4*>(acc)[i] = a;
    if (reset) {
      reinterpret_cast<float4*>(theta)[i] = g;
      if (wb != nullptr) reinterpret_cast<uint2*>(wb)[i] = make_uint2(pack_bf16x2(g.x, g.y), pack_bf16x2(g.z, g.w));
      if (mom != nullptr && (i << 2) < n_mom) reinterpret_cast<float4*>(mom)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// the standalone encode + mask (b200_secagg_encode): one 16-element block per thread and trip, the peers' keys in
// shared memory; the same secagg_encode_block as the collective's pack
constexpr int SECAGG_THREADS = 256;
__global__ void __launch_bounds__(SECAGG_THREADS)
secagg_encode_kernel(const float* __restrict__ theta, const float* __restrict__ global_w, long long n, float w, float R,
                     float two_f, const __grid_constant__ B200SecAggPeers peers, uint32_t n0, uint32_t n1, uint32_t n2,
                     uint32_t counter0, uint32_t* __restrict__ out, unsigned long long* saturated) {
  __shared__ uint32_t s_key[B200_MAX_RANKS][8];
  __shared__ int s_add[B200_MAX_RANKS];
  for (int i = threadIdx.x; i < peers.n * 8; i += SECAGG_THREADS) s_key[i >> 3][i & 7] = peers.key[i >> 3][i & 7];
  if (static_cast<int>(threadIdx.x) < peers.n) s_add[threadIdx.x] = peers.sign[threadIdx.x] > 0;
  __syncthreads();
  const long long nb = (n + 15) >> 4;
  int sat = 0;
  for (long long b = blockIdx.x * static_cast<long long>(SECAGG_THREADS) + threadIdx.x; b < nb;
       b += static_cast<long long>(gridDim.x) * SECAGG_THREADS) {
    const long long e0 = b << 4;
    const int valid = n - e0 < 16 ? static_cast<int>(n - e0) : 16;
    float x[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      x[j] = 0.f;
      if (j < valid) x[j] = global_w != nullptr ? __fsub_rn(theta[e0 + j], global_w[e0 + j]) : theta[e0 + j];
    }
    uint32_t u[16];
    sat += secagg_encode_block(x, valid, w, R, two_f, peers.n, [&](int p) { return s_key[p]; },
                               [&](int p) { return s_add[p] != 0; }, counter0 + static_cast<uint32_t>(b), n0, n1, n2, u);
#pragma unroll
    for (int j = 0; j < 16; ++j)
      if (j < valid) out[e0 + j] = u[j];
  }
  if (sat != 0 && saturated != nullptr) atomicAdd(saturated, static_cast<unsigned long long>(sat));
}

}  // namespace b200

// The kernel spins on cross-GPU flags per CTA, so every CTA of the grid must be resident at the same time or the ranks
// deadlock each other.  It is therefore launched COOPERATIVELY: the runtime refuses a grid that cannot be co-resident
// (cudaErrorCooperativeLaunchTooLarge) and schedules all CTAs together, also next to work on other streams -- instead
// of the plain <<<>>> of round 1, which was only safe on an otherwise idle GPU.  The grid is clamped to what
// cudaOccupancyMaxActiveBlocksPerMultiprocessor allows on this device, cached per kernel (each kind takes its own
// dynamic shared memory).
template <int WIRE, class Args>
static int launch_round_kernel(const Args* args, int n_ctas, cudaStream_t stream) {
  using namespace b200;
  constexpr Agg K = RoundOf<Args>::kind;
  constexpr int smem = K == Agg::krum ? KRUM_SMEM : K == Agg::robust ? ROBUST_SMEM : K == Agg::topk ? TOPK_SMEM : 0;
  const void* kernel = reinterpret_cast<const void*>(fedavg_round_kernel<WIRE, Args>);
  static int max_ctas = -1;
  if (max_ctas < 0) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (smem != 0) {
      cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      if (e != cudaSuccess) return static_cast<int>(e);
    }
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, FEDAVG_THREADS, smem);
    max_ctas = sms * per_sm;
    if (max_ctas < 1) max_ctas = 1;
  }
  if (n_ctas > max_ctas) n_ctas = max_ctas;
  if constexpr (K == Agg::krum) {
    // the rank step's arrival counter and done flag start at zero every launch (also after a timed-out one)
    cudaError_t e = cudaMemsetAsync(args->sync, 0, 2 * sizeof(unsigned int), stream);
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  void* kargs[] = {const_cast<Args*>(args)};
  cudaError_t e = cudaLaunchCooperativeKernel(kernel, dim3(n_ctas), dim3(FEDAVG_THREADS), kargs, smem, stream);
  if (e != cudaSuccess) return static_cast<int>(e);
  return static_cast<int>(cudaGetLastError());
}

static bool robust_args_ok(const FedAvgRobustArgs* args) {
  // a selection is not a sum: robust rounds run on peer loads, never on the switch
  if (args->use_nvls || !args->delta || args->tile_flags != nullptr || args->my_segs > B200_MAX_ROBUST_CLIENTS ||
      args->seg_stride % 256 != 0 || (args->kind != 0 && args->kind != 1) || args->world > B200_MAX_RANKS)
    return false;
  for (int k = 0; k < args->world; ++k)
    if (((args->alive_mask >> k) & 1u) && args->seg_page[k] == nullptr) return false;
  return true;
}

static bool krum_args_ok(const FedAvgKrumArgs* args) {
  // the kept mean is the trimmed mean with b = 0: the host passes kind 1 and a zero trim table
  if (args->use_nvls || !args->delta || args->tile_flags != nullptr || args->my_segs > B200_MAX_ROBUST_CLIENTS ||
      args->seg_stride % 256 != 0 || args->kind != 1 || args->world > B200_MAX_RANKS || args->work == nullptr ||
      args->sync == nullptr)
    return false;
  for (int p = 0; p <= B200_MAX_ROBUST_CLIENTS; ++p)
    if (args->trim_b[p] != 0 || args->krum_m[p] > p || (p > 0 && args->krum_m[p] < 1) || args->krum_k[p] >= (p > 0 ? p : 1))
      return false;
  for (int k = 0; k < args->world; ++k)
    if (((args->alive_mask >> k) & 1u) && (args->seg_page[k] == nullptr || args->dist_page[k] == nullptr)) return false;
  return true;
}

static bool dp_args_ok(const FedAvgDPArgs* args) {
  // the switch adds the raw wire values, but the clip factors are applied on the reader side: DP runs on peer loads
  if (args->use_nvls || !args->delta || args->world > B200_MAX_RANKS) return false;
  for (int k = 0; k < args->world; ++k)
    if (((args->alive_mask >> k) & 1u) && args->clip_page[k] == nullptr) return false;
  return true;
}

static bool scaffold_args_ok(const FedAvgScaffoldArgs* args) {
  // 1 / N weighs every participant's raw wire value on the reader side: SCAFFOLD runs on peer loads
  return !(args->use_nvls || !args->delta || args->dc == nullptr || args->c == nullptr || args->n_c <= 0 ||
           args->n_c % 8 != 0 || args->seg1_off % 16 != 0);
}

// a sum of sparse lists needs the peer loads (the switch adds dense vectors), the delta, the lists written before the
// launch, whole granules per tile and aligned list offsets; fp8's block scales have no meaning on a list
static bool topk_args_ok(const FedAvgTopkArgs* args) {
  using b200::FLAG_GRANULE;
  return !(args->use_nvls || !args->delta || !args->prepacked || args->tile_flags != nullptr ||
           args->world > B200_MAX_RANKS || args->n % FLAG_GRANULE != 0 || args->tile_elems <= 0 ||
           args->tile_elems % FLAG_GRANULE != 0 || args->rowptr_off % 4 != 0 || args->off_off % 2 != 0 ||
           args->val_off % 4 != 0 || (args->wire_kind != 0 && args->wire_kind != 1));
}

// a ring sum needs peer loads (on sm_90a the switch adds u32 only in scalar form), the delta, the fp32-sized wire, the
// kernel's own pack after the count barrier, 16-element blocks inside a tile, a block counter that cannot wrap, and
// f, 2^f, 2^-f consistent with R
static bool secagg_args_ok(const FedAvgSecAggArgs* args) {
  return !(args->use_nvls || !args->delta || args->prepacked || args->tile_flags != nullptr || args->wire_kind != 0 ||
           args->global_w == nullptr || args->tile_elems <= 0 || args->tile_elems % 16 != 0 ||
           args->n >= B200_SECAGG_MAX_ELEMS || !(args->range >= 0x1p-20f && args->range <= 0x1p20f) ||
           args->frac_bits < 10 || args->frac_bits > 50 || args->two_f != ldexpf(1.f, args->frac_bits) ||
           args->inv_two_f != ldexpf(1.f, -args->frac_bits) || args->world > B200_MAX_RANKS);
}

// the server step needs the pseudo-gradient (delta mode), the global copy and the state over [0, n_param)
// (n_phys: the physical arena elements, args->n except in a personalized round)
template <class Base>
static bool sopt_args_ok(const ServerOptArgs<Base>* args, long long n_phys) {
  return args->delta && args->global_w != nullptr && args->m != nullptr && args->kind >= 0 && args->kind <= 3 &&
         (args->kind == 0 || args->v != nullptr) && args->n_param >= 0 && args->n_param % 8 == 0 &&
         args->n_param <= n_phys;
}

// a personalized round: whole 1024-element granules on both edges of the local range (no wire vector or fp8 block
// crosses one), the range inside the physical arena, the plain mean and no arrival flags (they index physical granules)
template <class Args>
static bool local_args_ok(const Args* args) {
  using b200::FLAG_GRANULE;
  return b200::RoundOf<Args>::kind == b200::Agg::mean && args->tile_flags == nullptr && args->lo >= 0 &&
         args->len > 0 && args->lo % FLAG_GRANULE == 0 && args->len % FLAG_GRANULE == 0 && args->lo <= args->n;
}

template <class Args>
int b200_fedavg_round(const Args* args, int n_ctas, cudaStream_t stream) {
  using namespace b200;
  constexpr Agg K = RoundOf<Args>::kind;
  if (args->world > B200_MAX_RANKS || args->n % 8 != 0 || args->tile_elems % 8 != 0) return -2;
  if (args->tile_flags != nullptr && args->tile_elems % FLAG_GRANULE != 0) return -2;
  // block-scaled fp8 wire: 32-element blocks must not straddle tiles, and the switch cannot rescale
  if (args->wire_kind == 2 && (args->tile_elems % 32 != 0 || args->use_nvls)) return -2;
  long long n_phys = args->n;
  if constexpr (RoundOf<Args>::local) {
    if (!local_args_ok(args)) return -2;
    n_phys += args->len;
  }
  if constexpr (RoundOf<Args>::sopt) {
    if (!sopt_args_ok(args, n_phys)) return -2;
  }
  if constexpr (K == Agg::dp) {
    if (!dp_args_ok(args)) return -2;
  } else if constexpr (K == Agg::scaffold) {
    if (!scaffold_args_ok(args)) return -2;
  } else if constexpr (K == Agg::robust) {
    if (!robust_args_ok(args)) return -2;
  } else if constexpr (K == Agg::krum) {
    if (!krum_args_ok(args)) return -2;
    if (n_ctas > B200_KRUM_MAX_CTAS) n_ctas = B200_KRUM_MAX_CTAS;
  } else if constexpr (K == Agg::topk) {
    if (!topk_args_ok(args)) return -2;
  } else if constexpr (K == Agg::secagg) {
    if (!secagg_args_ok(args)) return -2;
  }
  if (n_ctas < 1) n_ctas = 1;
  if constexpr (K == Agg::secagg) {   // the int32 ring
    return launch_round_kernel<3>(args, n_ctas, stream);
  } else {
    if constexpr (K != Agg::topk) {   // top-k rounds carry fp32 or bf16 values only
      if (args->wire_kind == 2) return launch_round_kernel<2>(args, n_ctas, stream);
    }
    if (args->wire_kind == 1) return launch_round_kernel<1>(args, n_ctas, stream);
    return launch_round_kernel<0>(args, n_ctas, stream);
  }
}

template int b200_fedavg_round(const FedAvgArgs*, int, cudaStream_t);
template int b200_fedavg_round(const FedAvgDPArgs*, int, cudaStream_t);
template int b200_fedavg_round(const FedAvgScaffoldArgs*, int, cudaStream_t);
template int b200_fedavg_round(const FedAvgRobustArgs*, int, cudaStream_t);
template int b200_fedavg_round(const FedAvgKrumArgs*, int, cudaStream_t);
template int b200_fedavg_round(const FedAvgTopkArgs*, int, cudaStream_t);
template int b200_fedavg_round(const ServerOptArgs<FedAvgArgs>*, int, cudaStream_t);
template int b200_fedavg_round(const ServerOptArgs<FedAvgDPArgs>*, int, cudaStream_t);
template int b200_fedavg_round(const ServerOptArgs<FedAvgScaffoldArgs>*, int, cudaStream_t);
template int b200_fedavg_round(const ServerOptArgs<FedAvgRobustArgs>*, int, cudaStream_t);
template int b200_fedavg_round(const ServerOptArgs<FedAvgKrumArgs>*, int, cudaStream_t);
template int b200_fedavg_round(const ServerOptArgs<FedAvgTopkArgs>*, int, cudaStream_t);
template int b200_fedavg_round(const FedAvgSecAggArgs*, int, cudaStream_t);
template int b200_fedavg_round(const ServerOptArgs<FedAvgSecAggArgs>*, int, cudaStream_t);
template int b200_fedavg_round(const LocalArgs<FedAvgArgs>*, int, cudaStream_t);
template int b200_fedavg_round(const LocalArgs<ServerOptArgs<FedAvgArgs>>*, int, cudaStream_t);

extern "C" int b200_pack_client(void* seg, float* theta, const float* global_w, void* w_bf16, float* mom, long long n_mom,
                                long long n, int wire_kind, int reset, cudaStream_t stream) {
  using namespace b200;
  if (n <= 0) return 0;
  if (n % 8 != 0 || wire_kind < 0 || wire_kind > 2) return -2;
  if ((reinterpret_cast<uintptr_t>(theta) | reinterpret_cast<uintptr_t>(global_w) | reinterpret_cast<uintptr_t>(seg)) & 15)
    return -2;
  const int vec = wire_kind == 0 ? 4 : 8;
  long long g = (n / vec + 255) / 256;
  const long long cap = 8ll * device_sm_count();
  if (g > cap) g = cap;
  auto* wb = reinterpret_cast<__nv_bfloat16*>(w_bf16);
  auto* s = static_cast<uint8_t*>(seg);
  if (wire_kind == 2)
    pack_client_kernel<2><<<static_cast<unsigned>(g), 256, 0, stream>>>(s, theta, global_w, wb, mom, n_mom, n, reset);
  else if (wire_kind == 1)
    pack_client_kernel<1><<<static_cast<unsigned>(g), 256, 0, stream>>>(s, theta, global_w, wb, mom, n_mom, n, reset);
  else
    pack_client_kernel<0><<<static_cast<unsigned>(g), 256, 0, stream>>>(s, theta, global_w, wb, mom, n_mom, n, reset);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int b200_dp_clip_factor(const float* theta, const float* global_w, long long n, float clip, void* work,
                                   float* s_out, float* norm_out, float* s_copy, int* nonfinite, cudaStream_t stream) {
  using namespace b200;
  if (n % 4 != 0 || !(clip >= 0.f) || work == nullptr || s_out == nullptr || norm_out == nullptr) return -2;
  if ((reinterpret_cast<uintptr_t>(theta) | reinterpret_cast<uintptr_t>(global_w)) & 15) return -2;
  dp_clip_factor_kernel<<<B200_DP_NORM_BLOCKS, DP_NORM_THREADS, 0, stream>>>(
      theta, global_w, n, clip, static_cast<unsigned long long*>(work), s_out, norm_out, s_copy, nonfinite);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int b200_fold_client_scaled(float* acc, float* theta, const float* global_w, void* w_bf16, float* mom,
                                       long long n_mom, long long n, const float* s, int first, int reset,
                                       cudaStream_t stream) {
  using namespace b200;
  if (n <= 0) return 0;
  if (n & 3) return -2;
  long long g = (n / 4 + DP_NORM_THREADS - 1) / DP_NORM_THREADS;
  const long long cap = 8ll * device_sm_count();
  if (g > cap) g = cap;
  fold_client_scaled_kernel<<<static_cast<unsigned>(g), DP_NORM_THREADS, 0, stream>>>(
      acc, theta, global_w, reinterpret_cast<__nv_bfloat16*>(w_bf16), mom, n_mom, n, s, first, reset);
  return static_cast<int>(cudaGetLastError());
}

extern "C" int b200_secagg_encode(const float* theta, const float* global_w, long long n, float w, float range,
                                  int frac_bits, const B200SecAggPeers* peers, const uint32_t* nonce, uint32_t counter0,
                                  uint32_t* out, unsigned long long* saturated, cudaStream_t stream) {
  using namespace b200;
  if (n <= 0) return 0;
  if (peers == nullptr || nonce == nullptr || peers->n < 0 || peers->n >= B200_MAX_RANKS || frac_bits < 10 ||
      frac_bits > 50 || !(range >= 0x1p-20f && range <= 0x1p20f) ||
      static_cast<unsigned long long>(counter0) + static_cast<unsigned long long>((n + 15) >> 4) > (1ull << 32))
    return -2;
  long long g = ((n + 15) / 16 + SECAGG_THREADS - 1) / SECAGG_THREADS;
  const long long cap = 8ll * device_sm_count();
  if (g > cap) g = cap;
  secagg_encode_kernel<<<static_cast<unsigned>(g), SECAGG_THREADS, 0, stream>>>(
      theta, global_w, n, w, range, ldexpf(1.f, frac_bits), *peers, nonce[0], nonce[1], nonce[2], counter0, out, saturated);
  return static_cast<int>(cudaGetLastError());
}

B200_TRACE_REGISTER(fedavg)

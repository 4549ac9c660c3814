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

// DP: DP-FedAvg (see launch.h / DESIGN.md): w_k = n_k s_k / N with s_k from rank k's clip page, and the owner of a tile
// adds sigma C / N * z[i] to its fp32 sum before the cast.  The loss and the integer side arena keep the weights n_k / N.
// SCAF: a SCAFFOLD round -- segment 1 (the control variates, see seg_pack) rides between the same barriers; every
// participant weighs 1 / N there.
// The whole round; Args is FedAvgDPArgs when DP, FedAvgScaffoldArgs when SCAF.
template <int WIRE, bool DP, bool SCAF = false, typename Args>
__device__ __forceinline__ void fedavg_round(const Args& a) {
  static_assert(!(DP && SCAF), "DP-FedAvg and SCAFFOLD are exclusive");
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
  __shared__ float s_part[DP ? B200_MAX_RANKS : 1];   // DP: participation weights n_k / N (loss, integer arena)
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
  if ((my_n != 0.f || a.use_nvls) && !a.prepacked) {
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
#pragma unroll
              for (int j = 0; j < VEC; j += 4) {
                th[u][j >> 2] = __ldcs(reinterpret_cast<const float4*>(theta_r + base + i + j));
                if (a.delta) gg[u][j >> 2] = __ldcs(reinterpret_cast<const float4*>(global_r + base + i + j));
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
  phase_stamp(a, 1);                                   // pack done
  if (!cta_barrier_all_ranks(a, a.epoch + 1, __float_as_uint(my_n), s_payload)) return;
  phase_stamp(a, 2);                                   // barrier 1 passed

  // weights w_k = n_k / N from the counts that rode on the barrier flags (or the host's plan)
  if (threadIdx.x == 0) {
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
  if constexpr (SCAF) {
    // one wire vector per trip: the same sums in the same rank order as the wider trips, in fewer registers
    reduce_tiles(std::integral_constant<int, 1>{});
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
  if (!cta_barrier_all_ranks(a, a.epoch + 2, 0u, nullptr)) return;
  phase_stamp(a, 4);                                   // barrier 2 passed

  // ---------------------------------------------------------------- phase 2: running-mean apply
  // CTA b applies exactly the tiles CTA b of the owners produced: (t / A) % G == b
  const float apply_scale = a.use_nvls ? s_inv_total / a.nvls_prescale : 1.0f;
  for (long long q = blockIdx.x; q * A < n_tiles; q += G) {
    for (int r = 0; r < A; ++r) {
      const long long t = q * A + r;
      if (t >= n_tiles) break;
      const long long base = t * T;
      const int len = static_cast<int>((n - base) < T ? (n - base) : T);
      constexpr int STEP = FEDAVG_THREADS * VEC;
      for (int i0 = threadIdx.x * VEC; i0 < len; i0 += 2 * STEP) {
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
#pragma unroll
              for (int j = 0; j < VEC; j += 4) gg[u][j >> 2] = *reinterpret_cast<const float4*>(a.global_w + base + i + j);
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
#pragma unroll
            for (int j = 0; j < VEC; j += 4) {
              float4 nw = make_float4(f[j] * apply_scale, f[j + 1] * apply_scale, f[j + 2] * apply_scale,
                                      f[j + 3] * apply_scale);
              if (a.delta) {
                const float4 g = gg[u][j >> 2];
                nw.x += g.x; nw.y += g.y; nw.z += g.z; nw.w += g.w;
              }
              if (a.global_w != nullptr) *reinterpret_cast<float4*>(a.global_w + base + i + j) = nw;
              *reinterpret_cast<float4*>(a.theta + base + i + j) = nw;
              if (a.momentum != nullptr && base + i + j < a.n_momentum)
                *reinterpret_cast<float4*>(a.momentum + base + i + j) = make_float4(0.f, 0.f, 0.f, 0.f);
              if (a.theta_bf16 != nullptr) {
                const uint2 o = make_uint2(pack_bf16x2(nw.x, nw.y), pack_bf16x2(nw.z, nw.w));
                *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(a.theta_bf16) + (base + i + j) * 2) = o;
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
template <int WIRE>
__global__ void __maxnreg__(96) fedavg_allreduce_kernel(const __grid_constant__ FedAvgArgs a) {
  fedavg_round<WIRE, false>(a);
}
template <int WIRE>
__global__ void __maxnreg__(96) fedavg_allreduce_dp_kernel(const __grid_constant__ FedAvgDPArgs a) {
  fedavg_round<WIRE, true>(a);
}
template <int WIRE>
__global__ void __maxnreg__(96) fedavg_allreduce_scaffold_kernel(const __grid_constant__ FedAvgScaffoldArgs a) {
  fedavg_round<WIRE, false, true>(a);
}

// stand-alone cross-GPU barrier on the pads (one CTA): fences host-side phases
__global__ void flag_barrier_kernel(FedAvgArgs a, int slot) {
  const int t = threadIdx.x;
  if (t < a.world && ((a.alive_mask >> t) & 1u)) {
    fence_sys();
    st_release_sys_u64(a.pads[t] + (static_cast<size_t>(slot) * B200_MAX_RANKS + a.rank),
                       static_cast<unsigned long long>(a.epoch) << 32);
    const unsigned long long* mine = a.pads[a.rank] + (static_cast<size_t>(slot) * B200_MAX_RANKS + t);
    while (static_cast<int32_t>(static_cast<uint32_t>(ld_acquire_sys_u64(mine) >> 32) - a.epoch) < 0) {
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

}  // namespace b200

// The kernel spins on cross-GPU flags per CTA, so every CTA of the grid must be resident at the same time or the ranks
// deadlock each other.  It is therefore launched COOPERATIVELY: the runtime refuses a grid that cannot be co-resident
// (cudaErrorCooperativeLaunchTooLarge) and schedules all CTAs together, also next to work on other streams -- instead
// of the plain <<<>>> of round 1, which was only safe on an otherwise idle GPU.  The grid is clamped to what
// cudaOccupancyMaxActiveBlocksPerMultiprocessor allows on this device.
template <int WIRE, bool DP, bool SCAF, typename Args>
static int launch_fedavg(const Args* args, int n_ctas, cudaStream_t stream) {
  using namespace b200;
  static int max_ctas = -1;
  const void* kernel = SCAF ? reinterpret_cast<const void*>(fedavg_allreduce_scaffold_kernel<WIRE>)
                       : DP ? reinterpret_cast<const void*>(fedavg_allreduce_dp_kernel<WIRE>)
                            : reinterpret_cast<const void*>(fedavg_allreduce_kernel<WIRE>);
  if (max_ctas < 0) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, FEDAVG_THREADS, 0);
    max_ctas = sms * per_sm;
    if (max_ctas < 1) max_ctas = 1;
  }
  if (n_ctas > max_ctas) n_ctas = max_ctas;
  void* kargs[] = {const_cast<Args*>(args)};
  cudaError_t e = cudaLaunchCooperativeKernel(kernel, dim3(n_ctas), dim3(FEDAVG_THREADS), kargs, 0, stream);
  if (e != cudaSuccess) return static_cast<int>(e);
  return static_cast<int>(cudaGetLastError());
}

template <bool DP, bool SCAF, typename Args>
static int fedavg_dispatch(const Args* args, int n_ctas, cudaStream_t stream) {
  using namespace b200;
  if (args->world > B200_MAX_RANKS || args->n % 8 != 0 || args->tile_elems % 8 != 0) return -2;
  if (args->tile_flags != nullptr && args->tile_elems % FLAG_GRANULE != 0) return -2;
  if (n_ctas < 1) n_ctas = 1;
  if (args->wire_kind == 2) {
    // block-scaled fp8 wire: 32-element blocks must not straddle tiles, and the switch cannot rescale
    if (args->tile_elems % 32 != 0 || args->use_nvls) return -2;
    return launch_fedavg<2, DP, SCAF>(args, n_ctas, stream);
  }
  if (args->wire_kind == 1) return launch_fedavg<1, DP, SCAF>(args, n_ctas, stream);
  return launch_fedavg<0, DP, SCAF>(args, n_ctas, stream);
}

extern "C" int b200_fedavg_allreduce(const FedAvgArgs* args, int n_ctas, cudaStream_t stream) {
  return fedavg_dispatch<false, false>(args, n_ctas, stream);
}

extern "C" int b200_fedavg_allreduce_dp(const FedAvgDPArgs* args, int n_ctas, cudaStream_t stream) {
  // the switch adds the raw wire values, but the clip factors are applied on the reader side: DP runs on peer loads
  if (args->use_nvls || !args->delta || args->world > B200_MAX_RANKS) return -2;
  for (int k = 0; k < args->world; ++k)
    if (((args->alive_mask >> k) & 1u) && args->clip_page[k] == nullptr) return -2;
  return fedavg_dispatch<true, false>(args, n_ctas, stream);
}

extern "C" int b200_fedavg_allreduce_scaffold(const FedAvgScaffoldArgs* args, int n_ctas, cudaStream_t stream) {
  // 1 / N weighs every participant's raw wire value on the reader side: SCAFFOLD runs on peer loads
  if (args->use_nvls || !args->delta || args->dc == nullptr || args->c == nullptr || args->n_c <= 0 ||
      args->n_c % 8 != 0 || args->seg1_off % 16 != 0)
    return -2;
  return fedavg_dispatch<false, true>(args, n_ctas, stream);
}

extern "C" int b200_flag_barrier(unsigned long long* const* pads, int rank, int world, uint32_t alive_mask,
                                 uint32_t epoch, int slot, cudaStream_t stream) {
  using namespace b200;
  if (world > B200_MAX_RANKS) return -2;
  FedAvgArgs a = {};
  for (int k = 0; k < world; ++k) a.pads[k] = pads[k];
  a.rank = rank; a.world = world; a.alive_mask = alive_mask; a.epoch = epoch;
  flag_barrier_kernel<<<1, 32, 0, stream>>>(a, slot);
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

B200_TRACE_REGISTER(fedavg)

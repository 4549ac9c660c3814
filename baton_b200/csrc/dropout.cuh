// Dropout masks of BERT training (baton_b200/data/dropout.py states the contract): element i of a dropout site keeps
// its value iff word i & 3 of
//     philox4x32_10(counter = (i >> 2, 0x80000000 | site << 22 | t, stream_lo, stream_hi), key)
// is >= thresh, where t = epoch * steps + step is the local step of the run.  The per-epoch words {epoch, stream_lo,
// stream_hi} are read from device memory (a captured epoch graph replays them for every round, client and epoch); site,
// step, steps, thresh and the scale are launch arguments.  A kept value is multiplied by scale = fp32(1 / (1 - p)).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dp.cuh"
#include "launch.h"

namespace b200 {

struct DropArgs {
  const int* words;        // device {epoch, stream_lo, stream_hi}
  uint32_t key_lo, key_hi;
  uint32_t site, step, steps;
  uint32_t thresh;         // floor(p * 2^32)
  float scale;             // fp32(1 / (1 - p))
};

inline DropArgs drop_args(const B200Dropout* d) {
  return DropArgs{d->words, static_cast<uint32_t>(d->key), static_cast<uint32_t>(d->key >> 32), d->site, d->step,
                  d->steps, d->thresh, d->scale};
}

// the counter words of one launch; read after griddep_wait()
struct DropCtr {
  uint32_t w1, s_lo, s_hi;
  uint2 key;
  uint32_t thresh;
};

__device__ __forceinline__ DropCtr drop_ctr(const DropArgs& a) {
  DropCtr c;
  const uint32_t epoch = static_cast<uint32_t>(__ldg(a.words));
  c.s_lo = static_cast<uint32_t>(__ldg(a.words + 1));
  c.s_hi = static_cast<uint32_t>(__ldg(a.words + 2));
  c.w1 = 0x80000000u | (a.site << 22) | (epoch * a.steps + a.step);
  c.key = make_uint2(a.key_lo, a.key_hi);
  c.thresh = a.thresh;
  return c;
}

// keep bits of elements 4q .. 4q + 3 (bit j: element 4q + j is kept)
__device__ __forceinline__ uint32_t drop_keep4(const DropCtr& c, uint32_t q) {
  const uint4 x = philox4x32_10(make_uint4(q, c.w1, c.s_lo, c.s_hi), c.key);
  return static_cast<uint32_t>(x.x >= c.thresh) | (static_cast<uint32_t>(x.y >= c.thresh) << 1) |
         (static_cast<uint32_t>(x.z >= c.thresh) << 2) | (static_cast<uint32_t>(x.w >= c.thresh) << 3);
}

// keep bits of the 8 elements i0 .. i0 + 7, i0 % 8 == 0
__device__ __forceinline__ uint32_t drop_keep8(const DropCtr& c, unsigned long long i0) {
  const uint32_t q = static_cast<uint32_t>(i0 >> 2);
  return drop_keep4(c, q) | (drop_keep4(c, q + 1) << 4);
}

// keep bit of one element
__device__ __forceinline__ bool drop_keep1(const DropCtr& c, unsigned long long i) {
  return (drop_keep4(c, static_cast<uint32_t>(i >> 2)) >> (i & 3)) & 1u;
}

// v * scale when bit j of the keep bits is set, else 0
__device__ __forceinline__ float kept(uint32_t bits, int j, float v, float scale) {
  return ((bits >> j) & 1u) ? v * scale : 0.f;
}

}  // namespace b200

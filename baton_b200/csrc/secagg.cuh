// Secure aggregation (parallel/secagg.py): the ChaCha20 block function (RFC 8439) and the fixed-point encode + pairwise
// mask of one 16-element block.  The fused collective's pack phase (Agg::secagg, fedavg.cu) and the standalone
// b200_secagg_encode call these same functions, so both produce the bits of the numpy reference.
#pragma once
#include <stdint.h>

namespace b200 {

__device__ __forceinline__ uint32_t chacha_rotl(uint32_t x, int n) { return __funnelshift_l(x, x, n); }

#define B200_CHACHA_QR(a, b, c, d)                   \
  a += b; d = chacha_rotl(d ^ a, 16);                \
  c += d; b = chacha_rotl(b ^ c, 12);                \
  a += b; d = chacha_rotl(d ^ a, 8);                 \
  c += d; b = chacha_rotl(b ^ c, 7);

// u[0..16) += sign * ChaCha20(key, counter, nonce) (mod 2^32): the 16 output words of one block.  key: 8 words
// (little-endian key bytes), read here so they need not stay in registers across the rounds.
__device__ __forceinline__ void chacha20_mask_add(uint32_t (&u)[16], const uint32_t* key, uint32_t counter,
                                                  uint32_t n0, uint32_t n1, uint32_t n2, bool add) {
  uint32_t x0 = 0x61707865u, x1 = 0x3320646Eu, x2 = 0x79622D32u, x3 = 0x6B206574u;
  uint32_t x4 = key[0], x5 = key[1], x6 = key[2], x7 = key[3], x8 = key[4], x9 = key[5], x10 = key[6], x11 = key[7];
  uint32_t x12 = counter, x13 = n0, x14 = n1, x15 = n2;
#pragma unroll 1
  for (int r = 0; r < 10; ++r) {
    B200_CHACHA_QR(x0, x4, x8, x12) B200_CHACHA_QR(x1, x5, x9, x13)
    B200_CHACHA_QR(x2, x6, x10, x14) B200_CHACHA_QR(x3, x7, x11, x15)
    B200_CHACHA_QR(x0, x5, x10, x15) B200_CHACHA_QR(x1, x6, x11, x12)
    B200_CHACHA_QR(x2, x7, x8, x13) B200_CHACHA_QR(x3, x4, x9, x14)
  }
  const uint32_t s[16] = {x0 + 0x61707865u, x1 + 0x3320646Eu, x2 + 0x79622D32u, x3 + 0x6B206574u,
                          x4 + key[0], x5 + key[1], x6 + key[2], x7 + key[3],
                          x8 + key[4], x9 + key[5], x10 + key[6], x11 + key[7],
                          x12 + counter, x13 + n0, x14 + n1, x15 + n2};
#pragma unroll
  for (int i = 0; i < 16; ++i) u[i] = add ? u[i] + s[i] : u[i] - s[i];
}
#undef B200_CHACHA_QR

// q = int32(rint_even(fp32(w * clamp(x, -R, R)) * 2^f)), NaN -> 0 (two_f = 2^f, exact); returns 1 when x was clamped or
// not finite.  IEEE-rounded intrinsics: --use_fast_math must not flush or contract.
__device__ __forceinline__ int secagg_encode1(float x, float w, float R, float two_f, uint32_t& q) {
  const bool sat = !(fabsf(x) <= R);
  const float y = x != x ? 0.f : fminf(fmaxf(x, -R), R);
  q = static_cast<uint32_t>(__float2int_rn(__fmul_rn(__fmul_rn(w, y), two_f)));
  return sat ? 1 : 0;
}

// The masked upload of elements [e0, e0 + 16) (e0 % 16 == 0): u = encode(x) + sum over the peers of sign_p * S_p,
// block counter counter0 + e0 / 16.  peer_key(p) gives peer p's 8 key words, peer_add(p) its sign; x[i] with i >= valid
// is not encoded (the keystream words still are, and the caller does not store them).  Returns the saturated count.
template <class KeyOf, class AddOf>
__device__ __forceinline__ int secagg_encode_block(const float (&x)[16], int valid, float w, float R, float two_f,
                                                   int n_peers, KeyOf peer_key, AddOf peer_add, uint32_t counter,
                                                   uint32_t n0, uint32_t n1, uint32_t n2, uint32_t (&u)[16]) {
  int sat = 0;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    u[i] = 0u;
    if (i < valid) sat += secagg_encode1(x[i], w, R, two_f, u[i]);
  }
#pragma unroll 1
  for (int p = 0; p < n_peers; ++p) chacha20_mask_add(u, peer_key(p), counter, n0, n1, n2, peer_add(p));
  return sat;
}

}  // namespace b200

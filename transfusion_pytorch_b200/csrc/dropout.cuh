// Counter-based dropout masks (DESIGN.md §5).  The keep bit of an element is a pure function of WHAT is dropped, never of where a
// thread holds it, so the forward and the backward (and any future tiling) regenerate the same mask:
//
//   keep(key, site, layer, head, i, j):  Philox4x32-10 (Random123) with key (key0, key1) and counter (j >> 3, i, head, 2 * layer + site);
//   the four output words are eight 16-bit uniforms, element j & 7 takes half-word j & 7 (low half first); keep iff u16 >= thr,
//   thr = round(p * 65536).  Kept values are scaled by 1 / (1 - p) in fp32; p = 1 gives thr = 65536 and scale 0 (all dropped, no inf).
//
//   site 1 (FFN, after GEGLU): i = packed token row, j = inner column, head = 0.
//   site 0 (attention probabilities): i, j = packed query / key rows, head = the head.  No attention kernel applies it yet; the site word
//   keeps the two sites' masks independent, so adding it changes no FFN mask.
//
// oracle/dropout_mask.py restates exactly this definition for the tests.
#pragma once
#include <stdint.h>

namespace tfx {

enum : int { DROP_SITE_ATTN = 0, DROP_SITE_FFN = 1 };

// dropout parameters of one launch: the key lives on the device (a captured graph sees a new key on every replay)
struct DropParams {
  const uint32_t* key;     // device, 2 x u32
  uint32_t thr;            // keep iff u16 >= thr
  float scale;             // 1 / (1 - p), 0 for p = 1
  int layer;
};

__host__ inline DropParams make_drop_params(const void* key, float p, int layer) {
  DropParams d;
  d.key = static_cast<const uint32_t*>(key);
  const double t = (double)p * 65536.0 + 0.5;
  d.thr = p >= 1.f ? 65536u : (uint32_t)t;
  d.scale = p >= 1.f ? 0.f : (float)(1.0 / (1.0 - (double)p));
  d.layer = layer;
  return d;
}

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c;
}

// keep bits (bit e = column 8 g + e) of the 8-column group g = j >> 3 of row i
__device__ __forceinline__ uint32_t drop_keep8(const DropParams& d, uint32_t k0, uint32_t k1, int site, int head, uint32_t i, uint32_t g) {
  const uint4 w = philox4x32_10(make_uint4(g, i, (uint32_t)head, (uint32_t)(2 * d.layer + site)), k0, k1);
  const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
  uint32_t bits = 0;
#pragma unroll
  for (int e = 0; e < 8; ++e) bits |= (((ws[e >> 1] >> (16 * (e & 1))) & 0xFFFFu) >= d.thr ? 1u : 0u) << e;
  return bits;
}

}  // namespace tfx

// dropout.cuh — counter-based dropout masks of the training forward and backward (DESIGN.md §4.1, "Dropout").
//
// A keep / drop decision is a pure function of the 64-bit seed of the training forward and of the LOGICAL element it
// applies to, never of a tile, a packing or a launch shape, so the forward kernels and every backward kernel regenerate
// the same mask and no mask is stored.  Generator: Philox4x32-10 (Salmon et al., SC'11; the Random123 constants), key
// (seed & 0xffffffff, seed >> 32), counter (c0, c1, c2, c3):
//   hidden sites (site 0 embeddings, 2 attention output, 3 FFN output) of token t = b L + i, column n:
//       c0 = n >> 3, c1 = t, c2 = 0, c3 = stream(site, layer); the element's 16 bits: word (n >> 1) & 3, half n & 1
//   attention probabilities (site 1) of sequence b, head h, query i, key j:
//       c0 = 4 (j >> 5) + ((j >> 1) & 3), c1 = i, c2 = b heads + h, c3 = stream(1, layer); word (j >> 3) & 3, half j & 1
//       (one call covers the keys 32 (j >> 5) + 8 m + 2 ((j >> 1) & 3) + {0, 1}, m = 0..3: exactly the keys one lane holds
//       in a row of an m16n8 / m64nN accumulator fragment, so a lane never generates bits it does not use)
//   stream(site, layer) = 4 layer + site.
// half 0 is the low 16 bits of the word.  The element is kept when its 16 bits u satisfy u >= thr, thr = min(round(p 2^16),
// 65535), so the effective rate is thr / 2^16 (within 2^-17 of p); kept values are scaled by 1 / (1 - thr / 2^16).
#pragma once
#include <stdint.h>

namespace drop {

enum : uint32_t { kSiteEmbed = 0, kSiteAttn = 1, kSiteAttnOut = 2, kSiteFfnOut = 3 };

__host__ __device__ constexpr uint32_t stream(uint32_t site, int layer) { return 4u * static_cast<uint32_t>(layer) + site; }

// one dropout site of one launch: the Philox key, the threshold and scale, the counter word c3 (and, for the GEMM
// epilogue, the token stride of its rows: 1, or L when row r is the CLS row of sequence r; or, for a packed row plan, the
// token b L + i of every row, -1 for a row of no sequence)
struct Cfg {
  uint32_t k0, k1;
  uint32_t thr;
  uint32_t stream;
  float scale;
  int tok_stride;
  const int32_t* row_tok;   // null: row r is token r * tok_stride
};

__host__ __device__ __forceinline__ uint32_t row_token(const Cfg& c, int r) {
  return c.row_tok ? static_cast<uint32_t>(c.row_tok[r]) : static_cast<uint32_t>(r) * static_cast<uint32_t>(c.tok_stride);
}

__device__ __forceinline__ uint4 philox(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0;
    c1 = lo1;
    c2 = n2;
    c3 = lo0;
  }
  return make_uint4(c0, c1, c2, c3);
}

__device__ __forceinline__ uint32_t word(const uint4& w, int i) { return i == 0 ? w.x : i == 1 ? w.y : i == 2 ? w.z : w.w; }

// keep decision of the 16-bit half `half` of a generator word
__device__ __forceinline__ bool keep(uint32_t w, int half, uint32_t thr) { return ((w >> (16 * half)) & 0xFFFFu) >= thr; }

// Attention probabilities of keys whose index inside their sequence starts at a multiple of 8 but not of 32 (packed row
// plans: a sequence's keys start at any multiple of 16 of a tile): the 32 keys k0 + 8 m + 2 q4 + {0, 1} (m = 0..3) of a
// lane lie in the dense calls a = k0 >> 5 and a + 1; word m of the result is the word those keys use, with r = (k0 >> 3) & 3
// words taken from call a and the rest from call a + 1.
__device__ __forceinline__ uint4 splice(const uint4& wa, const uint4& wb, int r) {
  return r == 0 ? wa : r == 1 ? make_uint4(wa.y, wa.z, wa.w, wb.x) : r == 2 ? make_uint4(wa.z, wa.w, wb.x, wb.y)
                                                                             : make_uint4(wa.w, wb.x, wb.y, wb.z);
}

// the four words of the hidden-site call covering columns 8 g .. 8 g + 7 of token t
__device__ __forceinline__ uint4 hidden_bits(const Cfg& c, uint32_t t, uint32_t g) { return philox(c.k0, c.k1, g, t, 0u, c.stream); }

}  // namespace drop

// attention.cuh — fused multi-head self-attention for the encoder (K3 of SURVEY.md §2.3).
//
//   ctx = softmax(Q K^T / sqrt(64) + (1 - mask) * -10000) V         per (sequence, head)
//
// replaces HF RobertaSelfAttention / BertSelfAttention (transformers==2.3.0, eager) as reached from
// model/models.py:150-151,188-189,237-238.  The additive -10000 mask is reproduced literally
// (bias added in fp32 before the softmax), so an all-padding sequence gives the same finite
// "softmax of the raw scores" the reference gives, not NaN.
//
// Two kernels, both over work items (128-token query tile, head) and persistent (one CTA per SM):
//   attention_single_kernel   one 128-key block per item (L <= 128 dense or packed, row plans of sequences of up to 128
//                             tokens): warp-specialised, two MMA warpgroups with S, P and O in registers (below)
//   attention_multi_kernel    several key blocks per item (L = 256 / 512, packed sequences longer than 128): a TMA
//                             producer warp streams Q / K / V up to kStages key blocks ahead of one warpgroup that runs,
//                             per 128-key block of the same sequence:
//   S = Q K^T          wgmma m64n128k16 x (2 x 4)   (Q, K: TMA boxes of the [tokens, 3H] QKV buffer), written to a
//                      shared fp32 score tile
//   softmax            one warpgroup, thread = query row reading its row of the score tile, two passes per block with
//                      online rescaling; P written as 16-bit (FMT) into shared memory in the K-major SWIZZLE_128B layout
//   O_blk = P V        wgmma m64n64k16 x (2 x 8)    (V is the MN-major B operand), written over the score tile
//   o = o*alpha + O_blk in registers; after the last block ctx = o / l  (16-bit)
// Sequence lengths: a multiple of 128, or a divisor of 128 (then a tile holds 128/L sequences and
// cross-sequence scores are excluded).  head_dim is fixed at 64 (BERT/RoBERTa-base).
// Packed variable-length token matrices (kPacked with a row plan): every row r attends to the keys [row_lo[r], row_hi[r])
// of its own sequence.  Single-block plans: no sequence straddles a 128-row tile.  Otherwise an item's keys are the
// contiguous packed rows [kv0, kv0 + 128 nkv) covering every row's own range (tile_kv); the blocks of it outside a row's
// range are exact no-ops for that row, and the first block inside it takes the two-pass treatment the dense kernel gives
// block 0.
#pragma once
#include "act16.cuh"
#include "dropout.cuh"
#include "tc05.cuh"

namespace attn {

using namespace tc05;

constexpr int kTile = 128;   // query rows / keys per block
constexpr int kDh = 64;      // head dim

__device__ __forceinline__ float ex2_ftz(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

struct Params {
  int n_tokens;        // B * L
  int L;               // sequence length
  int heads;
  int hidden;          // heads * 64
  const float* kbias;  // [n_tokens] additive key bias * log2(e): 0 or -10000*log2e
  float scale_log2;    // log2(e) / sqrt(64)
  // Variable-length packing (kPacked kernels only; null = uniform L): token row r belongs to a sequence that occupies the
  // packed rows [row_lo[r], row_hi[r]) — whole sequences share tiles, nothing is padded inside a sequence (kbias is all
  // zero), rows that belong to no sequence attend to themselves only.
  const int32_t* row_lo;
  const int32_t* row_hi;
  // attention_multi_kernel<kPacked = true>: per 128-row tile, (first key row, number of 128-key blocks) of its work items
  const int2* tile_kv;
  // kDrop kernels: dropout of the probabilities, site 1 (dropout.cuh).  The dropped entries of the 16-bit P are zero, the
  // row sum l keeps every p, and ctx = O * (drop.scale / l).  With a row plan the counters are those of the dense batch:
  // row_tok[r] = b seq_L + i is the token of row r (-1: no sequence), its keys are counted from row_lo[r]; the plan's
  // sequences start at multiples of 8 rows (varlen_align 16).
  drop::Cfg drop;
  const int32_t* row_tok;
  int seq_L;
};

struct Smem {
  static constexpr int kStages = 3;                            // (K, V) stages
  static constexpr int kTileBytes = kTile * kDh * 2;           // 16 KB: one 128 x 64 16-bit operand tile
  static constexpr int kQ = 0;
  static constexpr int kKV = kQ + kTileBytes;                  // stage s: K at +0, V at +16 KB
  static constexpr int kP = kKV + kStages * 2 * kTileBytes;    // 128 x 128 16-bit (two 64-key halves)
  static constexpr int kSPitch = kTile + 4;                    // fp32 words per row of the score / output tile
  static constexpr int kS = kP + kTile * kTile * 2;            // S (128 x 128 fp32), then O_blk (128 x 64) over it
  static constexpr int kBias = kS + kTile * kSPitch * 4;       // 128 floats + 4 ballots
  static constexpr int kBiasStride = kTile * 4 + 16;
  static constexpr int kBar = kBias + kBiasStride;
  // q_full q_empty kv_full[S] kv_empty[S]
  static constexpr int kNumBars = 2 + 2 * kStages;
  static constexpr int kTotal = kBar + kNumBars * 8;
  static constexpr int kDynamic = kTotal + 1024;
  static_assert(kDynamic <= 232448, "attention smem exceeds 227 KB");
};

// a running maximum above this is the score of an unmasked key: masked keys sit near -10000 log2(e) = -14427
constexpr float kRealMax = -7000.0f;

constexpr int kThreads = 256;   // attention_multi_kernel: warp 0 TMA, 1-3 idle, 4-7 the softmax / MMA warpgroup

// Persistent, one CTA per SM.  The CTA walks its work items w = blockIdx.x + n * gridDim.x; the TMA producer runs
// up to kStages key/value blocks ahead (the HBM latency of a 48 KB Q/K/V fetch is longer than one item's
// arithmetic); producer and warpgroup derive the block order from the same loop nest.
// kPacked: a variable-length row plan (p.row_lo, p.tile_kv) of sequences longer than 128 tokens.
// FMT: 16-bit format of Q / K / V, of the probabilities P and of the output (act16.cuh).
template <bool kPacked, uint32_t FMT, bool kDrop = false>
__global__ void __launch_bounds__(kThreads, 1)
attention_multi_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmCTX, const Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Smem::kBar);
  uint64_t* q_full = bars + 0;
  uint64_t* q_empty = bars + 1;
  uint64_t* kv_full = bars + 2;                      // [kStages]
  uint64_t* kv_empty = bars + 2 + Smem::kStages;     // [kStages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = (p.n_tokens + kTile - 1) / kTile;
  const int total_work = n_tiles * p.heads;
  const int nkv_dense = (p.L >= kTile) ? p.L / kTile : 1;
  // keys of the items of a tile: first key row, number of 128-key blocks
  auto kv_of = [&](int tile, int& kv0, int& nkv) {
    if constexpr (kPacked) {
      const int2 t = __ldg(p.tile_kv + tile);
      kv0 = t.x;
      nkv = t.y;
    } else {
      kv0 = (p.L >= kTile) ? (tile * kTile / p.L) * p.L : tile * kTile;
      nkv = nkv_dense;
    }
  };

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmQKV);
    tma_prefetch_desc(&tmCTX);
    mbar_init(q_full, 1);
    mbar_init(q_empty, 4);          // the four warps of the warpgroup, after the last S of an item
    for (int s = 0; s < Smem::kStages; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 4);   // the four warps of the warpgroup, after the block's P V
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ================================ TMA producer ================================
    if (lane == 0) {
      Ring<Smem::kStages> kv;
      uint32_t qc = 0;
      for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
        const int tile = w / p.heads, h = w - tile * p.heads;
        const int tok0 = tile * kTile;
        int kv_tok0, nkv;
        kv_of(tile, kv_tok0, nkv);
        for (int j = 0; j < nkv; ++j) {
          if (j == 0) {
            mbar_wait(q_empty, (qc & 1) ^ 1, 10);
            ++qc;
            mbar_arrive_expect_tx(q_full, Smem::kTileBytes);
            tma_load_2d(smem + Smem::kQ, &tmQKV, q_full, h * kDh, tok0, kEvictFirst);
          }
          mbar_wait(&kv_empty[kv.stage], kv.phase ^ 1, 11);
          mbar_arrive_expect_tx(&kv_full[kv.stage], 2 * Smem::kTileBytes);
          uint8_t* st = smem + Smem::kKV + kv.stage * 2 * Smem::kTileBytes;
          tma_load_2d(st, &tmQKV, &kv_full[kv.stage], p.hidden + h * kDh, kv_tok0 + j * kTile, kEvictNormal);
          tma_load_2d(st + Smem::kTileBytes, &tmQKV, &kv_full[kv.stage], 2 * p.hidden + h * kDh, kv_tok0 + j * kTile,
                      kEvictNormal);
          kv.advance();
        }
      }
    }
  } else if (warp >= 4) {
    // =============================== softmax / output ==============================
    const int quad = warp & 3;                 // 32-row quarter of the tile this warp owns
    const int row = quad * 32 + lane;          // query row inside the tile
    uint8_t* sP = smem + Smem::kP;
    float* sS = reinterpret_cast<float*>(smem + Smem::kS);
    const uint32_t srow = smem_u32(sS) / 4u + static_cast<uint32_t>(row * Smem::kSPitch);   // this row, word address
    float* sbias = reinterpret_cast<float*>(smem + Smem::kBias);
    unsigned* smask = reinterpret_cast<unsigned*>(sbias + kTile);  // per-warp ballots of masked keys
    const int bar_id = 1;
    const uint32_t sq = smem_u32(smem + Smem::kQ);
    const uint32_t sp = smem_u32(sP);
    Ring<Smem::kStages> kv;
    uint32_t qc = 0;
    // additive key bias of block (w2, j2) for key `row` of that block (fetched one block ahead of its use)
    auto load_bias = [&](int w2, int j2) -> float {
      if (w2 >= total_work) return 0.f;
      int k0, nk;
      kv_of(w2 / p.heads, k0, nk);
      const int kt = k0 + j2 * kTile + row;
      return (kt < p.n_tokens) ? __ldg(p.kbias + kt) : -INFINITY;
    };
    // P (and the output tile) rows in shared memory: 128-byte spans, 16-byte chunk index ^= (row & 7)  (SWIZZLE_128B)
    auto store_chunks = [&](uint8_t* rowp, int chunk0, const uint32_t* pk) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int ch = (chunk0 + q) ^ (row & 7);
        *reinterpret_cast<uint4*>(rowp + ch * 16) = make_uint4(pk[q * 4], pk[q * 4 + 1], pk[q * 4 + 2], pk[q * 4 + 3]);
      }
    };
    float bv = load_bias(blockIdx.x, 0);
    for (int w = blockIdx.x; w < total_work; w += gridDim.x) {
      const int tile = w / p.heads, h = w - tile * p.heads;
      const int tok0 = tile * kTile;
      int kv0, nkv;
      kv_of(tile, kv0, nkv);
      const bool varlen = kPacked && p.row_lo != nullptr;
      int seq_lo = (p.L >= kTile) ? 0 : (row / p.L) * p.L;   // keys of this row's own sequence, relative to kv0
      int seq_hi = (p.L >= kTile) ? kTile : seq_lo + p.L;
      if (varlen) {
        seq_lo = __ldg(p.row_lo + tok0 + row) - kv0;
        seq_hi = __ldg(p.row_hi + tok0 + row) - kv0;
      }
      // end of the whole 32-key chunks of the own sequence (counted from its first key): the keys the dense kernel,
      // with the sequence at key 0, handles in unmasked chunks
      const int seq_full = seq_lo + ((seq_hi - seq_lo) & ~31);
      // kDrop (dense, L >= 256): this row is query qi of sequence tok / L; its keys are the item's kv0 .. kv0 + L - 1.
      // kDrop with a row plan: query and sequence from row_tok, keys counted from the row's own first key.
      uint32_t d_qi = kDrop ? static_cast<uint32_t>((tok0 + row) % p.L) : 0u;
      uint32_t d_c2 = kDrop ? static_cast<uint32_t>(((tok0 + row) / p.L) * p.heads + h) : 0u;
      if (kDrop && kPacked) {
        const int tk = max(__ldg(p.row_tok + tok0 + row), 0);
        d_qi = static_cast<uint32_t>(tk % p.seq_L);
        d_c2 = static_cast<uint32_t>((tk / p.seq_L) * p.heads + h);
      }
      float m_run = -INFINITY, l_run = 0.f;
      float o[kDh];
#pragma unroll
      for (int i = 0; i < kDh; ++i) o[i] = 0.f;
      for (int j = 0; j < nkv; ++j) {
        // key bias of this block -> smem (the previous block's readers are past their last use: they all passed
        // the barrier after the P V of that block)
        sbias[row] = bv;
        {
          const unsigned mk = __ballot_sync(0xffffffffu, bv < 0.f);
          if (lane == 0) smask[quad] = mk;
        }
        if (row == 0) bulk_wait_read_all();   // the previous item's output tile has left sP
        named_bar_sync(bar_id, kTile);
        bv = (j + 1 < nkv) ? load_bias(w, j + 1) : load_bias(w + gridDim.x, 0);
        // Per 32-key chunk, warp-uniform:  0 = every p is exactly 0 (keys of another packed sequence, or all keys
        // masked while the row has an unmasked key somewhere: exp2(-10000 log2e + s - m) flushes to zero, as
        // exp(-10000 + s - m) does in the reference's fp32 softmax),  1 = no key masked (no bias term),  2 = general.
        const unsigned mk[4] = {smask[0], smask[1], smask[2], smask[3]};
        // (variable-length tiles: a row whose sequence covers the whole block takes the same arithmetic as a full-length
        // sequence of the dense kernel, so that the two paths agree bit for bit)
        const int bl = seq_lo - j * kTile, bh = seq_hi - j * kTile;   // own keys, relative to this block
        const int bf = seq_full - j * kTile;
        const bool plain = kPacked ? (varlen && bl <= 0 && bh >= kTile) : ((mk[0] | mk[1] | mk[2] | mk[3]) == 0u);
        int st[4];
        if (varlen) {   // per row: chunk outside / inside / straddling the boundary of the row's own sequence
          // (several key blocks: "inside" also needs the chunk's keys to lie in whole 32-key chunks of the sequence, as
          // the unmasked chunks of the dense kernel do; the others take the dense kernel's partial-chunk arithmetic)
#pragma unroll
          for (int c = 0; c < 4; ++c)
            st[c] = (bh <= c * 32 || bl >= c * 32 + 32) ? 0 : (bl <= c * 32 && bf >= c * 32 + 32) ? 1 : 2;
        } else {
          bool own[4], any_unmasked = false;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            own[c] = !kPacked || (p.L >= 32 ? (c * 32 >= seq_lo && c * 32 < seq_hi) : c == quad);
            any_unmasked |= own[c] && mk[c] != 0xffffffffu;
          }
          const bool skip_ok = (kPacked && p.L < 32) ? false : (any_unmasked || m_run > kRealMax);
#pragma unroll
          for (int c = 0; c < 4; ++c)
            st[c] = !own[c] ? 0 : (mk[c] == 0xffffffffu && skip_ok) ? 0 : (mk[c] == 0u && !(kPacked && p.L < 32)) ? 1 : 2;
        }
        // S = Q K^T -> the score tile
        if (j == 0) mbar_wait(q_full, qc & 1, 12);
        mbar_wait(&kv_full[kv.stage], kv.phase, 13);
        const uint32_t sk = smem_u32(smem + Smem::kKV + kv.stage * 2 * Smem::kTileBytes);
        {
          float s0[kTile / 2], s1[kTile / 2];
#pragma unroll
          for (int i = 0; i < kTile / 2; ++i) s0[i] = s1[i] = 0.f;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kDh / 16; ++k) {
            const uint64_t bdesc = make_desc_k_sw128(sk + k * 32);
            wgmma_n128<FMT, 0>(s0, make_desc_k_sw128(sq + k * 32), bdesc, 1u);
            wgmma_n128<FMT, 0>(s1, make_desc_k_sw128(sq + 64 * 128 + k * 32), bdesc, 1u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_regs(s0);
          wgmma_fence_regs(s1);
          acc_store_frag(sS, Smem::kSPitch, 0, 0, s0);
          acc_store_frag(sS, Smem::kSPitch, 64, 0, s1);
        }
        if (j == nkv - 1) {   // the item's last read of Q
          __syncwarp();
          if (lane == 0) mbar_arrive(q_empty);
          ++qc;
        }
        named_bar_sync(bar_id, kTile);   // every row of S is in the tile
        float rsum, alpha = 1.f, m_new;
        const int stb = st[0] | (st[1] << 2) | (st[2] << 4) | (st[3] << 6);
        const bool all_skip = stb == 0;   // a fully masked block of a row that has real keys: contributes nothing
        // p = exp2(t - m_ref) for the whole block: row sum, 16-bit P into swizzled smem; returns max(t - m_ref)
        auto exp_pass = [&](float m_ref, float& rs_out) -> float {
          float rs_ = 0.f, mu = -INFINITY;
          const float nm = -m_ref;
#pragma unroll 1
          for (int c = 0; c < kTile; c += 32) {
            const int sc_ = (stb >> (c >> 4)) & 3;
            uint32_t pk[16];
            if (sc_ == 0) {
#pragma unroll
              for (int i = 0; i < 16; ++i) pk[i] = 0u;
            } else {
              uint32_t v[32];
              acc_ld_x32(srow + c, v);
              uint4 dw[4];   // kDrop: the four calls of this 32-key chunk (dw[q] covers the key pairs q, q + 4, q + 8, q + 12)
              if constexpr (kDrop && kPacked) {   // key index of column c in the row's sequence: any multiple of 8
                const int koff = j * kTile + c - seq_lo;
                const int a = koff >> 5, r8 = (koff >> 3) & 3;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                  const uint4 wa = drop::philox(p.drop.k0, p.drop.k1, 4u * static_cast<uint32_t>(a) + q, d_qi, d_c2, p.drop.stream);
                  dw[q] = r8 == 0 ? wa : drop::splice(wa, drop::philox(p.drop.k0, p.drop.k1, 4u * static_cast<uint32_t>(a + 1) + q,
                                                                       d_qi, d_c2, p.drop.stream), r8);
                }
              } else if constexpr (kDrop) {
#pragma unroll
                for (int q = 0; q < 4; ++q)
                  dw[q] = drop::philox(p.drop.k0, p.drop.k1, 4u * static_cast<uint32_t>((j * kTile + c) >> 5) + q, d_qi, d_c2,
                                       p.drop.stream);
              }
              // zero the dropped entries of the 16-bit P (after the row sum, which keeps them)
              auto dropped = [&](int k, uint32_t& pp) {
                if constexpr (kDrop) {
                  const uint32_t wq = drop::word(dw[(k >> 1) & 3], (k >> 3) & 3);
                  const uint32_t lo = drop::keep(wq, 0, p.drop.thr) ? 0x0000FFFFu : 0u;
                  const uint32_t hi = drop::keep(wq, 1, p.drop.thr) ? 0xFFFF0000u : 0u;
                  pp &= lo | hi;
                }
              };
              if (sc_ == 1) {
#pragma unroll
                for (int i = 0; i < 32; i += 2) {
                  const float u0 = fmaf(__uint_as_float(v[i]), p.scale_log2, nm);
                  const float u1 = fmaf(__uint_as_float(v[i + 1]), p.scale_log2, nm);
                  mu = fmaxf(mu, fmaxf(u0, u1));
                  const float p0 = ex2_ftz(u0), p1 = ex2_ftz(u1);
                  rs_ += p0 + p1;
                  pk[i >> 1] = act16::Act<FMT>::pack2(p0, p1);
                  dropped(i, pk[i >> 1]);
                }
              } else {
#pragma unroll
                for (int i = 0; i < 32; i += 2) {
                  float u0 = fmaf(__uint_as_float(v[i]), p.scale_log2, sbias[c + i]) + nm;
                  float u1 = fmaf(__uint_as_float(v[i + 1]), p.scale_log2, sbias[c + i + 1]) + nm;
                  if constexpr (kPacked) {   // other sequences' keys: nothing; keys of whole chunks: unmasked arithmetic
                    const int k0 = c + i, k1 = c + i + 1;
                    u0 = (k0 < bl || k0 >= bh) ? -INFINITY : (k0 < bf) ? fmaf(__uint_as_float(v[i]), p.scale_log2, nm) : u0;
                    u1 = (k1 < bl || k1 >= bh) ? -INFINITY : (k1 < bf) ? fmaf(__uint_as_float(v[i + 1]), p.scale_log2, nm) : u1;
                  }
                  mu = fmaxf(mu, fmaxf(u0, u1));
                  const float p0 = ex2_ftz(u0), p1 = ex2_ftz(u1);
                  rs_ += p0 + p1;
                  pk[i >> 1] = act16::Act<FMT>::pack2(p0, p1);
                  dropped(i, pk[i >> 1]);
                }
              }
            }
            store_chunks(sP + (c >> 6) * (kTile * 128) + row * 128, (c & 63) >> 3, pk);
          }
          rs_out = rs_;
          return mu;
        };
        // Blocks after the first: ONE trip over the scores, relative to the running maximum (the block's own maximum is
        // tracked on the way).  exp2(t - m_run) stays <= 2^8 unless a score exceeds every earlier one by more than 8
        // (log2 units) — then, and only then, the warp redoes the block relative to the true maximum.  The softmax is
        // the same function either way (numerator and denominator carry the same factor 2^(m_true - m_ref)).
        const bool optimistic = __all_sync(0xffffffffu, j > 0 && m_run > kRealMax);
        // (packed tiles: all_skip may differ between the rows of a warp, so the vote is taken by every lane; a skipped
        // row has over = -inf, and a redo leaves it as it was: m_new = m_run, alpha = 1, P = 0)
        if (optimistic) {
          m_new = m_run;
          alpha = 1.f;
          rsum = 0.f;
          float over = -INFINITY;
          if (!all_skip) {
            over = exp_pass(m_run, rsum);
          } else {
            float dummy;
            exp_pass(m_run, dummy);   // (writes the zero P tile; no score reads: every chunk state is 0)
          }
          if (__any_sync(0xffffffffu, over > 8.0f)) {
            m_new = fmaxf(m_run, m_run + over);
            alpha = exp2f(m_run - m_new);
            exp_pass(m_new, rsum);
          }
        } else {
          // first block of an item (or no real key seen yet): pass 1 = row max (of the raw scores when `plain`:
          // scale > 0 commutes with max), pass 2 = exp relative to it
          float m_blk = -INFINITY;
          if (!all_skip) {
#pragma unroll 1
            for (int c = 0; c < kTile; c += 32) {
              const int sc_ = (stb >> (c >> 4)) & 3;
              if (sc_ == 0) continue;
              uint32_t v[32];
              acc_ld_x32(srow + c, v);
              if (plain) {
#pragma unroll
                for (int i = 0; i < 32; ++i) m_blk = fmaxf(m_blk, __uint_as_float(v[i]));
              } else if (sc_ == 1) {
#pragma unroll
                for (int i = 0; i < 32; ++i) m_blk = fmaxf(m_blk, __uint_as_float(v[i]) * p.scale_log2);
              } else {
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                  float t = fmaf(__uint_as_float(v[i]), p.scale_log2, sbias[c + i]);
                  if (kPacked && (c + i < bl || c + i >= bh)) t = -INFINITY;
                  m_blk = fmaxf(m_blk, t);
                }
              }
            }
          }
          if (plain) m_blk *= p.scale_log2;
          m_new = fmaxf(m_run, m_blk);
          alpha = (m_run == -INFINITY) ? 0.f : exp2f(m_run - m_new);
          exp_pass(m_new, rsum);
        }
        fence_proxy_async_smem();
        named_bar_sync(bar_id, kTile);   // P complete; every read of S is done
        // O_blk = P V -> the same tile
        {
          const uint32_t sv = sk + Smem::kTileBytes;
          float o0[kDh / 2], o1[kDh / 2];
#pragma unroll
          for (int i = 0; i < kDh / 2; ++i) o0[i] = o1[i] = 0.f;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kTile / 16; ++k) {
            // A = P: keys [16k, 16k+16) live in 64-key half (k/4), 32 bytes per K step inside the span
            const uint32_t pa = sp + (k >> 2) * (kTile * 128) + (k & 3) * 32;
            // B = V (MN-major): 16 keys = two 8-row groups of 1024 bytes
            const uint64_t bdesc = make_desc_mn_sw128(sv + k * 2048, kTile * 128, 1024);
            wgmma_n64<FMT, 1>(o0, make_desc_k_sw128(pa), bdesc, 1u);
            wgmma_n64<FMT, 1>(o1, make_desc_k_sw128(pa + 64 * 128), bdesc, 1u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_regs(o0);
          wgmma_fence_regs(o1);
          __syncwarp();
          if (lane == 0) mbar_arrive(&kv_empty[kv.stage]);
          kv.advance();
          acc_store_frag(sS, Smem::kSPitch, 0, 0, o0);
          acc_store_frag(sS, Smem::kSPitch, 64, 0, o1);
        }
        named_bar_sync(bar_id, kTile);   // every row of O_blk is in the tile
        if (!all_skip) {   // (a skipped block has P = 0: its O_blk is exactly 0 and alpha is exactly 1)
#pragma unroll
          for (int c = 0; c < kDh; c += 32) {
            uint32_t v[32];
            acc_ld_x32(srow + c, v);
#pragma unroll
            for (int i = 0; i < 32; ++i) o[c + i] = fmaf(o[c + i], alpha, __uint_as_float(v[i]));
          }
          l_run = fmaf(l_run, alpha, rsum);
          m_run = m_new;
        }
      }
      // ctx tile = o / l in 16 bits: staged in this group's P buffer (the PV MMA has finished reading it), one TMA store
      {
        const float inv = kDrop ? p.drop.scale / l_run : 1.0f / l_run;
#pragma unroll
        for (int c = 0; c < kDh; c += 32) {
          uint32_t pk[16];
#pragma unroll
          for (int i = 0; i < 32; i += 2) {
            pk[i >> 1] = act16::Act<FMT>::pack2(o[c + i] * inv, o[c + i + 1] * inv);
          }
          store_chunks(sP + row * 128, c >> 3, pk);
        }
        fence_proxy_async_smem();
        named_bar_sync(bar_id, kTile);
        if (row == 0) {
          tma_store_2d(&tmCTX, sP, h * kDh, tok0);   // rows past n_tokens are clipped by the tensor map
          bulk_commit_group();
        }
      }
    }
    if (row == 0) bulk_wait_read_all();
  }

}

// =====================================================================================================================
// Single key block: L <= 128 dense or packed (a tile holds 128 / L sequences), or a row plan whose sequences never
// straddle a tile.  One work item = (128-row tile, head), the tile's own 128 rows as keys.
//
// Warp-specialised, persistent, one CTA of 384 threads per SM:
//   warpgroup 0   producer: warp g (g = 0, 1) streams (Q, K, V) of consumer g's items into g's two-stage ring
//   warpgroups 1, 2   consumers: consumer g walks its own items w = 2 blockIdx.x + g + n 2 gridDim.x, whole items each,
//                 so that one consumer's softmax (MUFU / FMA) overlaps the other's wgmmas and loads
// Per item a consumer runs, with S, P and O in registers (no fp32 tile in shared memory):
//   S = Q K^T      wgmma m64n128k16 x (2 x 4), SS form (the same instructions and k order as the multi-block kernel)
//   softmax        per row; thread t holds rows 16 (t/32) + (t%32)/4 + {0, 8, 64, 72} x keys 8 j + 2 (t%4) + {0, 1}
//   O = P V        wgmma m64n64k16 x (2 x 8), RS form: the 16-bit S fragment, packed in pairs, is the A fragment
//   ctx = O / l    16-bit, staged in the consumer's output tile, one TMA store
// Bit-identical to the row-per-thread softmax this kernel replaced: a lane's 32 keys of a row are exactly the keys
// (k >> 1) & 3 == t % 4 of that row's partial sum rs[(k >> 1) & 3] (pairs in rising order), and two xor shuffles (1,
// then 2) form (rs0 + rs1) + (rs2 + rs3); maxima are exact in any order; P, and the key order of P V, are unchanged.
struct SmemSingle {
  static constexpr int kStages = 2;                                   // (Q, K, V) stages per consumer
  static constexpr int kTileBytes = kTile * kDh * 2;                  // 16 KB
  static constexpr int kStageBytes = 3 * kTileBytes;                  // Q at +0, K at +16 KB, V at +32 KB
  static constexpr int kQKV = 0;                                      // [consumer][stage]
  static constexpr int kOut = kQKV + 2 * kStages * kStageBytes;       // [consumer] 128 x 64 16-bit output tile
  static constexpr int kBias = kOut + 2 * kTileBytes;                 // [consumer] 128 floats + 4 ballots
  static constexpr int kBiasStride = kTile * 4 + 16;
  static constexpr int kBar = kBias + 2 * kBiasStride;                // [consumer] full[kStages] empty[kStages]
  static constexpr int kNumBars = 2 * 2 * kStages;
  static constexpr int kTotal = kBar + kNumBars * 8;
  static constexpr int kDynamic = kTotal + 1024;
  static_assert(kDynamic <= 232448, "single-block attention smem exceeds 227 KB");
};

constexpr int kSingleThreads = 384;

// Per-row state of the single-block softmax.  st: 2 bits per 32-key chunk (0 = every p is exactly 0, 1 = no key
// masked, 2 = general); plain: max of the raw scores, scaled afterwards; [bl, bh): the row's own keys (kPacked).
struct RowSt {
  int st, bl, bh;
  bool plain;
};

// kDrop: a row's dropout counter words: query index qi in its sequence, c2 = sequence * heads + head, and lo, the tile
// column of the sequence's key 0 (dense: a multiple of L; a row plan: a multiple of 8)
struct DropRow {
  uint32_t qi, c2;
  int lo;
};

// the dropout call of 32-key chunk cc (tile columns 32 cc ..) of a row, as the lane with q4 uses it: word m covers the
// columns 32 cc + 8 m + 2 q4 + {0, 1}.  A sequence shorter than 32 keys (L = 8, 16) lies in one call whose words are
// rotated by the sequence's offset inside its 32-key chunk; the columns of other sequences get words that are not theirs,
// where p is exactly 0.
__device__ __forceinline__ uint4 drop_bits(const drop::Cfg& dc, const DropRow& r, int L, int cc, int q4) {
  if (L < 32) {
    const uint4 w = drop::philox(dc.k0, dc.k1, static_cast<uint32_t>(q4), r.qi, r.c2, dc.stream);
    const int rot = (r.lo >> 3) & 3;
    return rot == 0 ? w : rot == 1 ? make_uint4(w.w, w.x, w.y, w.z) : rot == 2 ? make_uint4(w.z, w.w, w.x, w.y)
                                                                                : make_uint4(w.y, w.z, w.w, w.x);
  }
  const int k0 = 32 * cc - r.lo;   // key index of column 32 cc in the row's sequence
  const uint4 wa = drop::philox(dc.k0, dc.k1, 4u * static_cast<uint32_t>(k0 >> 5) + q4, r.qi, r.c2, dc.stream);
  if ((k0 & 31) == 0) return wa;
  return drop::splice(wa, drop::philox(dc.k0, dc.k1, 4u * static_cast<uint32_t>((k0 >> 5) + 1) + q4, r.qi, r.c2, dc.stream),
                      (k0 >> 3) & 3);
}

// Softmax of the two rows (r, r + 8) held by accumulator `d` (m64n128 fragment): P packed in pairs into `pk` (the A
// fragments of the 8 k steps of P V), row sums (reduced over the quad) into rsum.
template <bool kPacked, uint32_t FMT, bool kDrop = false>
__device__ __forceinline__ void softmax_pair(float (&d)[64], const RowSt& ra, const RowSt& rb, const float* sbias, int q4,
                                             float scale_log2, uint32_t (&pk)[32], float& la, float& lb,
                                             const Params* dp = nullptr, const DropRow* da = nullptr,
                                             const DropRow* db = nullptr) {
  const RowSt rs[2] = {ra, rb};
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int c = j >> 2;
    const float2 b2 = *reinterpret_cast<const float2*>(sbias + 8 * j + 2 * q4);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const RowSt& r = rs[e >> 1];
      const int col = 8 * j + 2 * q4 + (e & 1);
      const int s = (r.st >> (2 * c)) & 3;
      const float v = d[4 * j + e];
      float t = fmaf(v, scale_log2, (e & 1) ? b2.y : b2.x);
      if (kPacked && (col < r.bl || col >= r.bh)) t = -INFINITY;
      t = r.plain ? v : (s == 1) ? v * scale_log2 : t;
      d[4 * j + e] = t;
      if (s != 0) mx[e >> 1] = fmaxf(mx[e >> 1], t);
    }
  }
  float sc[2], nm[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float m = mx[i];
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    if (rs[i].plain) m *= scale_log2;
    sc[i] = rs[i].plain ? scale_log2 : 1.0f;
    nm[i] = -m;
  }
  float acc[2] = {0.f, 0.f};
  uint4 dw[2];   // kDrop: the dropout call of the current 32-key chunk, rows r and r + 8
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int c = j >> 2;
    if constexpr (kDrop) {
      if ((j & 3) == 0) {
        dw[0] = drop_bits(dp->drop, *da, dp->L, c, q4);
        dw[1] = drop_bits(dp->drop, *db, dp->L, c, q4);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {   // h: row r (d[4j], d[4j + 1]) or r + 8 (d[4j + 2], d[4j + 3])
      const bool zero = ((rs[h].st >> (2 * c)) & 3) == 0;
      const float p0 = zero ? 0.f : ex2_ftz(fmaf(d[4 * j + 2 * h], sc[h], nm[h]));
      const float p1 = zero ? 0.f : ex2_ftz(fmaf(d[4 * j + 2 * h + 1], sc[h], nm[h]));
      acc[h] += p0 + p1;
      pk[2 * j + h] = act16::Act<FMT>::pack2(p0, p1);
      if constexpr (kDrop) {   // the dropped entries of P become 0; the row sum keeps them
        const uint32_t wq = drop::word(dw[h], j & 3);
        pk[2 * j + h] &= (drop::keep(wq, 0, dp->drop.thr) ? 0x0000FFFFu : 0u) | (drop::keep(wq, 1, dp->drop.thr) ? 0xFFFF0000u : 0u);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {   // (rs0 + rs1) + (rs2 + rs3) on every lane of the quad
    acc[i] = acc[i] + __shfl_xor_sync(0xffffffffu, acc[i], 1);
    acc[i] = acc[i] + __shfl_xor_sync(0xffffffffu, acc[i], 2);
  }
  la = acc[0];
  lb = acc[1];
}

template <bool kPacked, uint32_t FMT, bool kDrop = false>
__global__ void __launch_bounds__(kSingleThreads, 1)
attention_single_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmCTX, const Params p) {
  using S = SmemSingle;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S::kBar);   // consumer g: full at 2 kStages g, empty after it

  // (broadcast from lane 0: ptxas then knows the warpgroup index, and every branch and loop bound derived from it, to
  // be warp-uniform, and keeps the wgmmas of the consumer path pipelined)
  const int wg = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 7), 0);
  const int n_tiles = (p.n_tokens + kTile - 1) / kTile;
  const int total_work = n_tiles * p.heads;
  const int stride = 2 * gridDim.x;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQKV);
    tma_prefetch_desc(&tmCTX);
    for (int g = 0; g < 2; ++g) {
      for (int s = 0; s < S::kStages; ++s) {
        mbar_init(bars + 2 * S::kStages * g + s, 1);
        mbar_init(bars + 2 * S::kStages * g + S::kStages + s, 4);   // the four warps of consumer g, after P V
      }
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ================================ TMA producers ================================
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp < 2 && lane == 0) {
      uint64_t* full = bars + 2 * S::kStages * warp;
      uint64_t* empty = full + S::kStages;
      uint8_t* ring = smem + S::kQKV + warp * S::kStages * S::kStageBytes;
      Ring<S::kStages> rq;
      for (int w = 2 * blockIdx.x + warp; w < total_work; w += stride) {
        const int tile = w / p.heads, h = w - tile * p.heads;
        const int tok0 = tile * kTile;
        mbar_wait(&empty[rq.stage], rq.phase ^ 1, 20);
        mbar_arrive_expect_tx(&full[rq.stage], S::kStageBytes);
        uint8_t* st = ring + rq.stage * S::kStageBytes;   // every byte is read once: evict first
        tma_load_2d(st, &tmQKV, &full[rq.stage], h * kDh, tok0, kEvictFirst);
        tma_load_2d(st + S::kTileBytes, &tmQKV, &full[rq.stage], p.hidden + h * kDh, tok0, kEvictFirst);
        tma_load_2d(st + 2 * S::kTileBytes, &tmQKV, &full[rq.stage], 2 * p.hidden + h * kDh, tok0, kEvictFirst);
        rq.advance();
      }
    }
    return;
  }

  // ================================== consumers ==================================
  const int g = wg - 1;
  const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31, q4 = lane & 3;
  const int r0 = 16 * warp + (lane >> 2);   // rows r0, r0 + 8 (accumulator 0) and r0 + 64, r0 + 72 (accumulator 1)
  uint64_t* full = bars + 2 * S::kStages * g;
  uint64_t* empty = full + S::kStages;
  const uint32_t ring = smem_u32(smem + S::kQKV + g * S::kStages * S::kStageBytes);
  uint8_t* sout = smem + S::kOut + g * S::kTileBytes;
  float* sbias = reinterpret_cast<float*>(smem + S::kBias + g * S::kBiasStride);
  unsigned* smask = reinterpret_cast<unsigned*>(sbias + kTile);   // per-warp ballots of masked keys
  const int bar_id = 1 + g;
  const bool varlen = kPacked && p.row_lo != nullptr;
  Ring<S::kStages> rq;
  // additive key bias of item w2 for key t of its tile (fetched one item ahead of its use)
  auto load_bias = [&](int w2) -> float {
    if (w2 >= total_work) return 0.f;
    const int kt = (w2 / p.heads) * kTile + t;
    return (kt < p.n_tokens) ? __ldg(p.kbias + kt) : -INFINITY;
  };
  float bv = load_bias(2 * blockIdx.x + g);
  for (int w = 2 * blockIdx.x + g; w < total_work; w += stride) {
    const int tile = w / p.heads, h = w - tile * p.heads;
    const int tok0 = tile * kTile;
    sbias[t] = bv;
    {
      const unsigned mk = __ballot_sync(0xffffffffu, bv < 0.f);
      if (lane == 0) smask[warp] = mk;
    }
    if (t == 0) bulk_wait_read_all();   // the previous item's output tile has left sout
    named_bar_sync(bar_id, kTile);
    bv = load_bias(w + stride);
    const unsigned mk[4] = {smask[0], smask[1], smask[2], smask[3]};
    // Per row and 32-key chunk: 0 = every p is exactly 0 (keys of another packed sequence, or all keys masked while the
    // row has an unmasked key somewhere: exp2(-10000 log2e + s - m) flushes to zero, as exp(-10000 + s - m) does in the
    // reference's fp32 softmax), 1 = no key masked (no bias term), 2 = general.
    RowSt rs[4];
    DropRow dr[4];   // kDrop (dense): query index, sequence / head word and own-key offset of each row
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = r0 + (i & 1) * 8 + (i >> 1) * 64;
      if constexpr (kDrop) {
        if (varlen) {
          const int tk = max(__ldg(p.row_tok + tok0 + row), 0);
          dr[i].qi = static_cast<uint32_t>(tk % p.seq_L);
          dr[i].c2 = static_cast<uint32_t>((tk / p.seq_L) * p.heads + h);
          dr[i].lo = __ldg(p.row_lo + tok0 + row) - tok0;
        } else {
          dr[i].qi = static_cast<uint32_t>((tok0 + row) % p.L);
          dr[i].c2 = static_cast<uint32_t>(((tok0 + row) / p.L) * p.heads + h);
          dr[i].lo = (p.L >= kTile) ? 0 : (row / p.L) * p.L;
        }
      }
      int lo = (p.L >= kTile) ? 0 : (row / p.L) * p.L;   // keys of this row's own sequence
      int hi = (p.L >= kTile) ? kTile : lo + p.L;
      if (varlen) {
        lo = __ldg(p.row_lo + tok0 + row) - tok0;
        hi = __ldg(p.row_hi + tok0 + row) - tok0;
      }
      int st = 0;
      if (varlen) {   // chunk outside / inside / straddling the boundary of the row's own sequence
#pragma unroll
        for (int c = 0; c < 4; ++c)
          st |= ((hi <= c * 32 || lo >= c * 32 + 32) ? 0 : (lo <= c * 32 && hi >= c * 32 + 32) ? 1 : 2) << (2 * c);
      } else {
        bool own[4], any_unmasked = false;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          own[c] = !kPacked || (p.L >= 32 ? (c * 32 >= lo && c * 32 < hi) : c == (row >> 5));
          any_unmasked |= own[c] && mk[c] != 0xffffffffu;
        }
        const bool skip_ok = (kPacked && p.L < 32) ? false : any_unmasked;
#pragma unroll
        for (int c = 0; c < 4; ++c)
          st |= (!own[c] ? 0 : (mk[c] == 0xffffffffu && skip_ok) ? 0 : (mk[c] == 0u && !(kPacked && p.L < 32)) ? 1 : 2)
                << (2 * c);
      }
      rs[i].st = st;
      rs[i].bl = lo;
      rs[i].bh = hi;
      rs[i].plain = kPacked ? (varlen && lo <= 0 && hi >= kTile) : ((mk[0] | mk[1] | mk[2] | mk[3]) == 0u);
    }

    mbar_wait(&full[rq.stage], rq.phase, 21);
    const uint32_t sq = ring + rq.stage * S::kStageBytes, sk = sq + S::kTileBytes, sv = sq + 2 * S::kTileBytes;
    // One 64-row half at a time: S = Q K^T, its softmax, O = P V (keys in the order of the multi-block kernel: 8 steps
    // of 16), then ctx = O / l in 16 bits into the output tile (SWIZZLE_128B: 16-byte chunk index ^= row & 7).  The P V
    // of half 0 is issued before the S of half 1, and wgmmas issue in program order, so the S of half 1 cannot be
    // hoisted above the softmax of half 0: one half of S, P and O is live at a time, and nothing spills.  (The other
    // consumer warpgroup covers the waits.)
    auto half = [&](int m0, const RowSt& ra, const RowSt& rb, const DropRow& da, const DropRow& db) {
      uint32_t pk[32];
      float l[2];
      {
        float s[kTile / 2];
#pragma unroll
        for (int i = 0; i < kTile / 2; ++i) s[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kDh / 16; ++k)
          wgmma_n128<FMT, 0>(s, make_desc_k_sw128(sq + m0 * 128 + k * 32), make_desc_k_sw128(sk + k * 32), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(s);
        softmax_pair<kPacked, FMT, kDrop>(s, ra, rb, sbias, q4, p.scale_log2, pk, l[0], l[1], &p, &da, &db);
      }
      float o[kDh / 2];
#pragma unroll
      for (int i = 0; i < kDh / 2; ++i) o[i] = 0.f;
      wgmma_fence_regs(pk);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kTile / 16; ++k) {
        const uint32_t a[4] = {pk[4 * k], pk[4 * k + 1], pk[4 * k + 2], pk[4 * k + 3]};
        wgmma_n64_rs<FMT>(o, a, make_desc_mn_sw128(sv + k * 2048, kTile * 128, 1024));   // 16 keys: two 8-row groups
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {   // rows m0 + r0 + 8 hh: o[4 j + 2 hh + 0..1], keys 8 j + 2 (t % 4) + 0..1
        const int row = m0 + r0 + 8 * hh;
        const float inv = kDrop ? p.drop.scale / l[hh] : 1.0f / l[hh];
        uint8_t* rowp = sout + row * 128 + q4 * 4;
#pragma unroll
        for (int j = 0; j < kDh / 8; ++j) {
          const int e = 4 * j + 2 * hh;
          *reinterpret_cast<uint32_t*>(rowp + ((j ^ (row & 7)) << 4)) = act16::Act<FMT>::pack2(o[e] * inv, o[e + 1] * inv);
        }
      }
    };
    half(0, rs[0], rs[1], dr[0], dr[1]);
    half(64, rs[2], rs[3], dr[2], dr[3]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[rq.stage]);   // this warp's last read of the stage
    rq.advance();
    fence_proxy_async_smem();
    named_bar_sync(bar_id, kTile);
    if (t == 0) {
      tma_store_2d(&tmCTX, sout, h * kDh, tok0);   // rows past n_tokens are clipped by the tensor map
      bulk_commit_group();
    }
  }
  if (t == 0) bulk_wait_read_all();
}

}  // namespace attn

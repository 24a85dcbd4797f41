/* ance_b200.h — C ABI of libance_b200.so: the H100-native replacement for the native arithmetic on
 * microsoft/ANCE's ANN-refresh path (drivers/run_ann_data_gen.py + model/models.py).
 *
 * The reference has no FFI of its own: the native work on this path is done by un-vendored
 * libraries called directly from Python.  Each entry point below names the reference call site it
 * replaces.  Plain C, opaque handles, int status (0 = ok), ance_last_error() for the message, no
 * exceptions and no torch types across the boundary.  All *_dev pointers are CUDA device pointers
 * on the device that was current when the handle was created; `stream` is a cudaStream_t passed as
 * void*.  Handles are not thread-safe; distinct handles may be used concurrently.
 *
 * There is NO CPU fallback: every compute entry point fails with ANCE_ERR_CUDA when no sm_90
 * device is present.
 */
#ifndef ANCE_B200_H_
#define ANCE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
  ANCE_OK = 0,
  ANCE_ERR_INVALID = 1,     /* bad argument */
  ANCE_ERR_CUDA = 2,        /* CUDA runtime / driver error, or no sm_90 device */
  ANCE_ERR_NOMEM = 3,
  ANCE_ERR_UNSUPPORTED = 4  /* shape outside what the kernels were built for */
};

/* 16-bit operand format of the tensor-core passes (wgmma runs both at the same rate). */
enum { ANCE_FMT_FP16 = 0, ANCE_FMT_BF16 = 1 };

const char* ance_version(void);
const char* ance_last_error(void);
/* number of kernels this library has launched in the calling process (bench.py's gpu_launches) */
int64_t ance_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Flat inner-product index  — replaces faiss.IndexFlatIP(dim) / .add / .search
 *   reference: drivers/run_ann_data_gen.py:269-276,303 ; drivers/run_ann_data_gen_dpr.py:238-252
 * Semantics (faiss IndexFlatIP): for each query the k rows with the largest fp32 inner product,
 * sorted by score descending; labels are row numbers in insertion order (+ row_offset), int64;
 * when fewer than k rows exist the tail is label -1 / score -FLT_MAX.  Ties are broken by the
 * smaller row number (faiss leaves tie order unspecified; ours is deterministic).
 * Scores are the exact fp32-input dot product accumulated in fp64 and rounded once to fp32.
 * ance_index_search fails with ANCE_ERR_UNSUPPORTED when an index row or a query is non-finite after rounding to the
 * 16-bit operand format (inf / NaN input, or |x| > 65504 with ANCE_FMT_FP16) instead of returning unverifiable results.
 * ------------------------------------------------------------------------------------------------ */
typedef struct ance_index* ance_index_t;

typedef struct {
  int64_t nq;             /* queries in the last search */
  int64_t n_tier2;        /* queries the first coarse pass could not certify -> second pass from their own thresholds */
  int64_t n_uncertified;  /* queries no coarse pass could certify -> exact brute-force fallback */
  int64_t n_candidates;   /* candidates rescored in fp32/fp64 */
  int32_t kprime;         /* candidates kept per (query, split) by the coarse pass */
  int32_t n_splits;       /* row-range splits of the corpus per query tile */
  float max_eps;          /* largest per-query coarse-score error bound used by the certificate */
} ance_search_stats;

int ance_index_create(int dim, int64_t capacity_rows, int operand_fmt, ance_index_t* out);
/* Same, over CALLER-OWNED fp32 row storage rows_dev [capacity_rows, dim] (16-byte aligned, must outlive the index; never
 * freed by it).  A producer that writes rows i .. i+n straight into rows_dev + i*dim and then calls
 * ance_index_add(idx, rows_dev + i*dim, n) adds them WITHOUT a copy: this is how the refresher keeps one fp32 copy of the
 * corpus instead of the reference's three (per-batch arrays -> concatenation -> faiss storage,
 * drivers/run_ann_data_gen.py:160-193,271). */
int ance_index_create_over(int dim, int64_t capacity_rows, int operand_fmt, float* rows_dev, ance_index_t* out);
/* HOST index: the fp32 rows live in page-locked host memory, the device keeps only the coarse pass's 16-bit operands and
 * 4 bytes per row (2 bytes per row element + 4 per row instead of 6 per element: 21,015,324 x 768 rows take 32.3 GB of
 * device memory instead of 97 GB).  rows_host == NULL: the library allocates capacity_rows x dim fp32 with cudaHostAlloc
 * and frees it in ance_index_destroy.  Otherwise rows_host is caller-owned page-locked memory mapped into the device
 * (e.g. a torch pinned tensor; 16-byte aligned, else ANCE_ERR_INVALID) that must outlive the index.
 * Results are the same exact top-k as a device index's.  What changes:
 *   - ance_index_prepare streams the rows H2D through a device staging buffer of at most 512 MB (two passes over
 *     4 * n * dim bytes when centring);
 *   - rescoring (tiers 1 and 2) first bounds every candidate's score from its 16-bit row and residual norm in HBM and
 *     reads over PCIe only the fp32 rows of candidates that can still reach the top k (ance_index_last_fetched);
 *   - the brute force (tier 3, ance_index_search_exact) copies the rows H2D slab by slab (at most 512 MB of staging)
 *     once per batch of <= 1024 queries (fewer for k > 512, as on a device index): one PCIe pass over the corpus per
 *     batch (21M x 768 rows: 64.6 GB), acceptable for a fallback. */
int ance_index_create_host(int dim, int64_t capacity_rows, int operand_fmt, float* rows_host, ance_index_t* out);
int ance_index_destroy(ance_index_t idx);
int ance_index_reset(ance_index_t idx);                       /* ntotal = 0, storage kept */
int64_t ance_index_ntotal(ance_index_t idx);
/* IndexFlatIP.add: append n rows (fp32, row-major [n, dim], device memory).  On a host index rows_dev may also be host
 * memory: device rows are copied D2H in stream order, other host rows by a plain (synchronous) copy, and the storage
 * slice rows_host + ntotal * dim itself is added without a copy. */
int ance_index_add(ance_index_t idx, const float* rows_dev, int64_t n, void* stream);
/* Build the 16-bit operands of the coarse pass from ALL rows added so far: the rows are centred on their column mean
 * (<q, p> = <q, p - mu> + <q, mu>: the ranking does not change, the certificate's error bound shrinks to the centred rows'
 * norms) and rounded to operand_fmt.  ance_index_search does this itself when rows were added since the last time
 * (8.84M rows: ~10 ms); call it explicitly to keep that cost out of the first search. */
int ance_index_prepare(ance_index_t idx, void* stream);
/* IndexFlatIP.search: Q [nq, dim] fp32 -> D [nq, k] fp32, I [nq, k] int64 (all device memory), 0 < k <= 2048
 * (ANCE_ERR_INVALID above).  k <= 512: reservoirs of 1024 / 2048 entries, k' <= 992.  512 < k <= 2048 (top-1000
 * evaluation, large --topk_training): reservoirs of 8192 entries, k' in [1024, 4096], queries processed in blocks of at
 * most 16,384 so that the workspace does not grow with nq; at k = 1000 and k = 2048 alike it peaks at about 2.2 GB on a
 * 132-SM H100 (reservoirs 1.11 GB, candidate ids <= 0.54 GB, brute-force keys <= 0.54 GB, query copies 0.05 GB), on top
 * of the index's own 6 bytes per row element (host index: 2 bytes per row element + 4 per row). */
int ance_index_search(ance_index_t idx, const float* q_dev, int64_t nq, int k, float* D_dev, int64_t* I_dev,
                      int64_t row_offset, void* stream);
/* Same contract (0 < k <= 2048), computed entirely by the exact fp32->fp64 brute-force kernel (validation path). */
int ance_index_search_exact(ance_index_t idx, const float* q_dev, int64_t nq, int k, float* D_dev,
                            int64_t* I_dev, int64_t row_offset, void* stream);
/* Statistics of the last search (ance_index_search has already synchronised its stream). */
int ance_index_last_stats(ance_index_t idx, ance_search_stats* out);
/* Memory the handle holds: *device_bytes = its own device allocations (rows it allocated, 16-bit operands, per-row norms,
 * search workspace grown so far), *host_bytes = its own pinned allocation (0 for caller-owned or device rows).  Unlike
 * cudaMemGetInfo this does not count other processes sharing the device. */
int ance_index_memory(ance_index_t idx, int64_t* device_bytes, int64_t* host_bytes);
/* Rows the last ance_index_search's rescoring (tiers 1 and 2) read from host memory; 0 for a device index. */
int64_t ance_index_last_fetched(ance_index_t idx);
/* Host address of a host index's fp32 rows [capacity_rows, dim] (the library's allocation or rows_host); NULL for a device
 * index.  Valid until ance_index_destroy. */
float* ance_index_host_rows(ance_index_t idx);
/* Tunables: "kprime" (multiple of 32 in [0, 4096]; 0 = auto: about 1.44 k for fp16 operands, 2 k + 32 for bf16, at least
 * 1024 when k > 512; a value below k, or above 992 when k <= 512, sends the search to the brute force), "n_splits"
 * (0 = auto), "cta_group" (1|2),
 * "max_ctas" (0 = all SMs), "tier2" (0|1), "exact_fallback" (0|1: measurement only — results of uncertified queries are
 * then NOT guaranteed), "pace_window" (tiles a sweeping CTA pair may run ahead of the slowest one; 0 = no soft
 * barrier), "operand_fmt" (ANCE_FMT_*: the rows already added are re-rounded from the fp32 copy at the next prepare / search),
 * "center" (0|1, default 1: centre the rows before rounding). */
int ance_index_set_param(ance_index_t idx, const char* name, double value);

/* Host k-way merge of per-shard results — replaces utils/util.py:87-146 barrier_array_merge +
 * the rank-0-only search (the reference's own precedent: utils/eval_mrr.py:175-183).
 * D[s], I[s]: [nq, k] sorted descending per shard (labels already global).  Output [nq, k]. */
int ance_merge_topk_host(const float* const* D, const int64_t* const* I, int n_shards, int64_t nq, int k,
                         float* D_out, int64_t* I_out, int n_threads);

/* ann_training_data_N writer (host only) — replaces the per-query formatting loop of drivers/run_ann_data_gen.py:318-329.
 * Line i = "qid \t pos \t n1,n2,...\n" of query order[i]; neg [n, neg_stride] holds counts[q] valid ids per row. */
int ance_write_training_data_host(const char* path, const int64_t* qids, const int64_t* pos, const int64_t* neg,
                                  const int64_t* counts, const int64_t* order, int64_t n, int neg_stride,
                                  int64_t* lines_written);

/* ------------------------------------------------------------------------------------------------
 * Dual-encoder forward — replaces the HF RobertaModel/BertModel forward + embeddingHead + norm
 *   reference: model/models.py:149-157 (RobertaDot_NLL_LN.query_emb/body_emb),
 *              model/models.py:165-199 (MultiChunk body_emb, caller reshapes [B,2048]->[4B,512]),
 *              model/models.py:223-259 (BiEncoder / HFBertEncoder, CLS of last layer, no head)
 * ------------------------------------------------------------------------------------------------ */
typedef struct ance_encoder* ance_encoder_t;

enum { ANCE_ARCH_ROBERTA = 0, ANCE_ARCH_BERT = 1 };

typedef struct {
  int arch;        /* ANCE_ARCH_ROBERTA: position ids = cumsum(ids != pad) * (ids != pad) + pad_id
                      ANCE_ARCH_BERT   : position ids = 0..L-1 */
  int n_layer, hidden, heads, ffn, vocab, max_pos, type_vocab, pad_id;
  float ln_eps;
  int has_head;    /* 1: out = LayerNorm(Linear(CLS)) (models.py:152-153); 0: out = CLS (models.py:237-239) */
  int operand_fmt; /* ANCE_FMT_FP16 (recommended) or ANCE_FMT_BF16: 16-bit storage format of weights and activations.
                      Both run the tensor cores at the same rate with fp32 accumulation; fp16 keeps 11 significant bits
                      instead of 8, i.e. 8x closer to the reference's fp32 forward.  A checkpoint whose activations
                      leave the fp16 range (|x| > 65504) produces non-finite embeddings, which ance_encoder_check
                      reports as ANCE_ERR_UNSUPPORTED: use ANCE_FMT_BF16 for such a model. */
} ance_encoder_config;

/* All weight pointers are HOST fp32 arrays in the checkpoint's own layout (Linear weight = [out, in]);
 * the library converts and uploads them once (Linear weights -> operand_fmt; embedding tables, biases and LayerNorm
 * parameters stay fp32). */
typedef struct {
  const float *q_w, *q_b, *k_w, *k_b, *v_w, *v_b;   /* attention.self.{query,key,value} */
  const float *ao_w, *ao_b, *ln1_g, *ln1_b;         /* attention.output.{dense,LayerNorm} */
  const float *ff1_w, *ff1_b;                       /* intermediate.dense */
  const float *ff2_w, *ff2_b, *ln2_g, *ln2_b;       /* output.{dense,LayerNorm} */
} ance_layer_weights;

typedef struct {
  const float *word_emb, *pos_emb, *type_emb, *emb_ln_g, *emb_ln_b;
  const ance_layer_weights* layers;                 /* [n_layer] */
  const float *head_w, *head_b, *head_ln_g, *head_ln_b; /* embeddingHead [hidden, hidden] + [hidden], norm [hidden] (has_head only) */
} ance_encoder_weights;

int ance_encoder_create(const ance_encoder_config* cfg, const ance_encoder_weights* w, int max_tokens,
                        ance_encoder_t* out);
int ance_encoder_destroy(ance_encoder_t enc);
/* ids_dev [B, L] int32.  Attention mask: lens_dev [B] int32 (mask = 1^len 0^(L-len), the
 * data/msmarco_data.py:275-303 form) or mask_dev [B, L] uint8 (data/DPR_data.py:283 form); exactly one
 * non-null.  Masked keys get the additive -10000 of HF 2.3.0, so an all-pad sequence yields the
 * finite "uniform attention" vector the reference yields.  out_dev [B, hidden] fp32. */
int ance_encoder_forward(ance_encoder_t enc, const int32_t* ids_dev, const int32_t* lens_dev,
                         const uint8_t* mask_dev, int B, int L, float* out_dev, void* stream);
/* Variable-length form of the same forward for L <= 128 (the MS MARCO passage / query caches): sequence b has lens[b]
 * real tokens followed by padding (data/msmarco_data.py:275-303), and only the real tokens are computed.  Whole sequences
 * are packed into 128-row attention tiles (a tile holds sequences of ANY lengths, none straddles a tile, every sequence
 * attends to its own tokens only), the linear layers and LayerNorms run on the packed token matrix, the CLS rows are
 * gathered for the last layer and the head.  lens_dev and lens_host hold the same B lengths, each in [1, L] (the tile
 * packing is planned on the host); B is unlimited (the call splits by the handle's max_tokens).  With the default
 * "varlen_align" = 1 the embeddings equal those of ance_encoder_forward up to fp32 summation order inside the softmax / P*V
 * of a tile (a sequence's terms are grouped by its offset in the tile; tests: |diff| <= 1e-2, both within the gate of the
 * fp32 reference); with "varlen_align" = 16 every sequence starts at a multiple of the tensor core's K step and the result
 * is bit-identical to ance_encoder_forward and independent of the batch composition, at ~12 % fewer real tokens per tile. */
int ance_encoder_forward_varlen(ance_encoder_t enc, const int32_t* ids_dev, const int32_t* lens_dev,
                                const int32_t* lens_host, int B, int L, float* out_dev, void* stream);
/* The same padding-free forward for any 0 < L <= 512 (within max_position_embeddings; the handle needs max_tokens >= L
 * rounded up to 128).  lens_dev / lens_host as above, each length in [1, L] (else ANCE_ERR_INVALID).  L <= 128 is
 * ance_encoder_forward_varlen.  For L > 128 sequences may span several tiles; the attention of a tile reads the keys of
 * every sequence it holds and skips, per row, the blocks outside the row's own sequence.  "varlen_align" = 16 (exact): a
 * sequence longer than 128 tokens starts on a tile boundary and fills ceil(len / 128) tiles (its rows padded to a multiple
 * of 32 with its own padding tokens), shorter ones start at a multiple of 16 rows of a tile; every embedding is
 * bit-identical to ance_encoder_forward at the same L, whatever else is in the batch.  "varlen_align" = 1 (densest): every
 * sequence starts where the previous one ends; the embeddings equal the dense forward's up to fp32 summation order. */
int ance_encoder_forward_packed(ance_encoder_t enc, const int32_t* ids_dev, const int32_t* lens_dev,
                                const int32_t* lens_host, int B, int L, float* out_dev, void* stream);
/* Tunables: "prune_last_layer" (default 1): in the last layer only token 0 of every sequence is read
 * downstream, so out-projection / FFN / LayerNorm run on those rows only (result-identical; bench.py reports
 * the executed FLOPs beside the algorithmic ones).  "ln_rows_per_warp" (1, 2, 4, or 3 = two rows held packed; default 2, process-wide): rows a warp
 * of the LayerNorm kernel normalises side by side (bit-identical results; default 2).  "varlen_align" (1 | 16):
 * see ance_encoder_forward_varlen and ance_encoder_forward_packed.  "train_max_len" (128, 256, 384 or 512; default 128,
 * per handle): the longest sequence ance_encoder_train_workspace, ance_encoder_forward_train and ance_dbg_train_layout
 * accept; above 128 they take the multiples of 128 up to it (the attention backward of L > 128 is a key-blocked kernel). */
int ance_encoder_set_param(ance_encoder_t enc, const char* name, double value);
/* Input / output validation, deferred so that forward stays asynchronous: synchronises `stream` and returns
 * ANCE_ERR_INVALID if any forward since the last check saw a token id outside [0, vocab_size) or a position
 * beyond max_position_embeddings (such lookups are clamped on the device; the reference's nn.Embedding raises
 * an index error, model/models.py:150-155 -> transformers modeling_roberta.py embeddings), ANCE_ERR_UNSUPPORTED if
 * any forward produced a non-finite embedding (fp16 range exceeded, or NaN weights).  The drivers call it once per
 * encode pass. */
int ance_encoder_check(ance_encoder_t enc, void* stream);
/* Debug / parity: copy the hidden states after layer `layer` (0 = embeddings) of the last forward
 * into out_dev [B*L, hidden] fp32 (with prune_last_layer the last layer holds its B CLS rows first). */
int ance_encoder_debug_hidden(ance_encoder_t enc, int layer, float* out_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training: gradients of the dense forward for sequences of up to 128 tokens, or up to 512 on a handle whose
 * "train_max_len" allows it (the trainer side of model/models.py:58-84, NLL.forward -> loss.backward()).
 * ------------------------------------------------------------------------------------------------ */
/* Gradient buffers: the layout of ance_encoder_weights / ance_layer_weights with DEVICE fp32 pointers (16-byte aligned),
 * every one required (the head's only with has_head).  ance_encoder_backward OVERWRITES them. */
typedef struct {
  float *q_w, *q_b, *k_w, *k_b, *v_w, *v_b;
  float *ao_w, *ao_b, *ln1_g, *ln1_b;
  float *ff1_w, *ff1_b;
  float *ff2_w, *ff2_b, *ln2_g, *ln2_b;
} ance_layer_grads;

typedef struct {
  float *word_emb, *pos_emb, *type_emb, *emb_ln_g, *emb_ln_b;
  const ance_layer_grads* layers;                    /* [n_layer], host array of device pointers */
  float *head_w, *head_b, *head_ln_g, *head_ln_b;
} ance_encoder_grads;

/* Bytes of device workspace one ance_encoder_forward_train of a [B, L] batch keeps for its backward (about
 * 16 hidden + 4 ffn bytes per token and layer: 24.6 KB at hidden 768, ffn 3072).  ANCE_ERR_UNSUPPORTED for L > 128 unless
 * L is a multiple of 128 up to the handle's "train_max_len" (ANCE_ERR_UNSUPPORTED above it). */
int ance_encoder_train_workspace(ance_encoder_t enc, int B, int L, size_t* bytes);
/* ance_encoder_forward with every activation the backward needs saved in ws_dev (256-byte aligned, the size above; one
 * workspace per forward whose backward is still to come; each forward_train is followed by at most one backward).  out_dev is bit-identical to ance_encoder_forward's.
 * L must be 8, 16, 32, 64 or 128, or a multiple of 128 up to "train_max_len" (ANCE_ERR_UNSUPPORTED above it), and
 * B * L <= max_tokens. */
int ance_encoder_forward_train(ance_encoder_t enc, const int32_t* ids_dev, const int32_t* lens_dev, const uint8_t* mask_dev,
                               int B, int L, void* ws_dev, float* out_dev, void* stream);
/* ance_encoder_forward_train in training mode: inverted dropout (keep with probability 1 - p, kept values scaled by
 * 1 / (1 - p)) at the four sites of a BERT / RoBERTa layer stack in training mode: the embedding LayerNorm's output, the
 * attention probabilities (p_attn), and the attention-output and FFN-output projections before their residual adds
 * (p_hidden); not the head.  Masks are regenerated from `seed` by a counter-based generator (Philox4x32-10) as functions of
 * the logical element (site, layer, token, column; layer, sequence, head, query, key), so the backward needs no stored mask:
 * ance_encoder_backward applies the masks this call used.  16 bits per decision: the effective rate is round(p 2^16) / 2^16.
 * Each rate must be finite and in [0, 1) (else ANCE_ERR_INVALID); a rate of 0 turns its sites off, and both 0 is
 * ance_encoder_forward_train exactly. */
int ance_encoder_forward_train_dropout(ance_encoder_t enc, const int32_t* ids_dev, const int32_t* lens_dev,
                                       const uint8_t* mask_dev, int B, int L, void* ws_dev, float* out_dev, float p_hidden,
                                       float p_attn, uint64_t seed, void* stream);
/* Packed variable-length training: the training forward of a [B, L] batch whose sequence b is the non-empty prefix of
 * lens_host[b] tokens, computing the real tokens only.  The batch is planned as ance_encoder_forward_packed plans it, at the
 * handle's "varlen_align", as ONE plan: ANCE_ERR_UNSUPPORTED when it needs more than max_tokens rows.  Lengths must lie in
 * [1, L]; L is any length up to 128, or up to the handle's "train_max_len" (ANCE_ERR_UNSUPPORTED above it).
 * ance_encoder_train_workspace_packed: the workspace bytes of that plan (its rows' activations, plus the plan and the CLS
 * rows of the pruned last layer, so that several packed forwards may precede their backwards).
 * ance_encoder_forward_train_packed: dropout as ance_encoder_forward_train_dropout (rates of 0: none), with the masks of the
 * dense [B, L] batch (token b L + i), so that with varlen_align 16 out_dev is bit-identical to the dense training forward's
 * at the same seed.  p_attn > 0 needs varlen_align 16 (ANCE_ERR_UNSUPPORTED otherwise).  ids_dev [B, L] int32 (the
 * padded batch), lens_host the lengths on the host (the plan and the kernels use them: the workspace keeps their copy),
 * lens_dev the same lengths on the device.  ance_encoder_backward then runs the
 * backward of this plan. */
int ance_encoder_train_workspace_packed(ance_encoder_t enc, const int32_t* lens_host, int B, int L, size_t* bytes);
int ance_encoder_forward_train_packed(ance_encoder_t enc, const int32_t* ids_dev, const int32_t* lens_dev,
                                      const int32_t* lens_host, int B, int L, void* ws_dev, float* out_dev, float p_hidden,
                                      float p_attn, uint64_t seed, void* stream);
/* Gradients of sum(d_out o out) with respect to every weight, for the forward that filled ws_dev (the weights must not
 * have changed since; dense or packed, as that forward was).  d_out_dev [B, hidden] fp32, 16-byte aligned.  The handle forgets ws_dev once this call is made:
 * a second backward from the same workspace is ANCE_ERR_INVALID.  Backward GEMM operands are bf16 whatever operand_fmt is, with fp32
 * accumulation; residual-stream and weight gradients are fp32.  Weight rows that the reference declares as padding_idx get
 * no gradient (word row pad_id; position row pad_id for RoBERTa).  The word / position gradients are scatter-added with
 * fp32 atomics: their summation order, and so their last bits, vary from run to run; everything else is deterministic. */
int ance_encoder_backward(ance_encoder_t enc, const float* d_out_dev, void* ws_dev, const ance_encoder_grads* g,
                          void* stream);
/* In-place weight refresh (after an optimizer step): w_dev holds DEVICE fp32 pointers in the layout of ance_encoder_create's
 * weights; they are converted into the handle's existing buffers in stream order, without a host round trip or a new
 * allocation.  The result is the handle ance_encoder_create would build from the same values. */
int ance_encoder_update_weights(ance_encoder_t enc, const ance_encoder_weights* w_dev, void* stream);
/* Debug / tests: the residual-stream gradients of the last ance_encoder_backward.  slot = -1 enables capture for backwards
 * of up to min(max_tokens, 4096) tokens (allocates (n_layer + 1) x that x hidden fp32; off by default).  With capture on,
 * slot n_layer holds d x_final [B, hidden] (the gradient into the last layer's CLS outputs, after the head; d_out itself
 * without a head) and slot l < n_layer holds d X_in(l) [B * L, hidden], the gradient into layer l's input (slot 0: into the
 * embedding LayerNorm's output).  slot >= 0 copies a whole slot, [min(max_tokens, 4096), hidden] fp32, into out_dev; it
 * is ANCE_ERR_INVALID when the last backward was not captured (none since capture was enabled, or one of more tokens than
 * the limit), so a read never returns an earlier backward's gradients. */
int ance_encoder_debug_grads(ance_encoder_t enc, int slot, float* out_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * LAMB optimizer step  — replaces utils/lamb.py's Lamb.step (one eager pass per parameter tensor)
 *   reference: utils/lamb.py:24-100, built at drivers/run_ann.py:81, utils/dpr_utils.py:90, drivers/run_warmup.py:77
 * One step over n contiguous fp32 device tensors: parameters p_dev[t], gradients g_dev[t], moment states m_dev[t] and
 * v_dev[t] (all four numel[t] elements, written in place except g), hyperparameters hyper[5 t .. 5 t + 4] = lr, beta1,
 * beta2, eps, weight_decay of the tensor's group.  With u = m / (sqrt(v) + eps) + weight_decay p (after the moment update,
 * p before this step's), w = min(||p||, 10), a = ||u||, r = w / a (1 when w or a is 0):
 *   m <- beta1 m + (1 - beta1) g,  v <- beta2 v + (1 - beta2) g^2,  p <- p - lr (adam ? 1 : r) u
 * and norms_dev[3 t .. 3 t + 2] = (w, a, r), r before the adam override.  No bias correction.  Three kernels on `stream`
 * whatever n (one when every numel is 0), no host synchronisation, no float atomics: the same inputs give the same bits.
 * The host arrays are consumed before the call returns.  Pointers need only 4-byte alignment (views at any offset);
 * numel may be 0 (then the pointers may be null).  At most 512 tensors and 16 distinct hyperparameter tuples per call
 * (the table travels as kernel parameters), else ANCE_ERR_UNSUPPORTED; split larger steps into several calls.  Bad
 * arguments are rejected before anything is enqueued. */
int ance_lamb_step(int n, float* const* p_dev, const float* const* g_dev, float* const* m_dev, float* const* v_dev,
                   const int64_t* numel, const double* hyper, int adam, float* norms_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * AdamW optimizer step  — replaces transformers 2.3.0's AdamW.step (one eager pass per parameter tensor)
 *   reference: built at utils/dpr_utils.py:88 (run_ann_dpr.py's default --optimizer adamW), drivers/run_ann.py:86,
 *   drivers/run_warmup.py:80
 * One step over n contiguous fp32 device tensors p_dev[t], g_dev[t], m_dev[t], v_dev[t] as for ance_lamb_step, with
 * hyper[5 t .. 5 t + 4] = step_size, beta1, beta2, eps, decay of the tensor: step_size = lr sqrt(1 - beta2^step) /
 * (1 - beta1^step) with the bias correction (lr without), computed by the caller from the tensor's own step count, and
 * decay = lr weight_decay.  Per element:
 *   m <- beta1 m + (1 - beta1) g,  v <- beta2 v + (1 - beta2) g^2,  p <- p - step_size m / (sqrt(v) + eps),
 *   then, only when decay > 0, p <- p - decay p (on the updated p)
 * with the roundings of the eager fp32 step (see csrc/optim.cu).  One kernel on `stream` whatever n (none when every
 * numel is 0), 28 bytes of traffic per element, no host synchronisation, no atomics: the same inputs give the same bits.
 * The host arrays are consumed before the call returns.  Pointers need only 4-byte alignment (views at any offset);
 * numel may be 0 (then the pointers may be null).  At most 512 tensors and 16 distinct (beta1, beta2, eps) per call
 * (the table travels as kernel parameters; step_size and decay may differ for every tensor), else
 * ANCE_ERR_UNSUPPORTED; split larger steps into several calls.  Bad arguments are rejected before anything is
 * enqueued. */
int ance_adamw_step(int n, float* const* p_dev, const float* const* g_dev, float* const* m_dev, float* const* v_dev,
                    const int64_t* numel, const double* hyper, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Device-time profile by kernel class (bench.py's roofline numbers): CUDA events recorded around every
 * launch on the launch stream.  Classes: 0 encoder GEMM, 1 attention, 2 LayerNorm/embedding/gather,
 * 3 operand quantisation, 4 coarse search GEMM, 5 exact rescore, 6 exact brute force, 7-10 encoder
 * GEMMs by role (QKV, attention out-proj, FFN up, FFN down; class 0 then holds the head GEMM only), 11 optimizer step.
 * ance_profile_read synchronises the device, returns milliseconds and launch counts per class
 * (arrays of length n <= 12) and optionally resets the accumulators.
 * ------------------------------------------------------------------------------------------------ */
int ance_profile_enable(int on);
int ance_profile_read(double* ms_by_class, int64_t* launches_by_class, int n, int reset);

/* ------------------------------------------------------------------------------------------------
 * Bring-up / test hooks (not part of the drop-in surface)
 * ------------------------------------------------------------------------------------------------ */
/* Host-only: the tile plan ance_encoder_forward_varlen makes for the first chunk of lens_host[0..B) on a handle created with
 * `max_tokens`: row0_out[i] = packed row of sequence i's first token (i < *n_placed), lo/hi_out [*n_tiles * 128] = own-sequence
 * key range of every packed row (may be null). */
int ance_dbg_pack_varlen(const int32_t* lens_host, int B, int max_tokens, int align, int32_t* row0_out, uint8_t* lo_out,
                         uint8_t* hi_out, int* n_placed, int* n_tiles);
/* Host-only: the plan ance_encoder_forward_packed makes for the first chunk of lens_host[0..B) at length L: row0_out[i] as
 * above, lo/hi_out [*n_tiles * 128] = own-sequence key range of every packed row in absolute packed rows (a row of no
 * sequence: [r, r + 1)), tile_kv_out [*n_tiles * 2] = (first key row, number of 128-key blocks) of each tile's attention
 * items.  The three arrays may be null. */
int ance_dbg_pack_packed(const int32_t* lens_host, int B, int L, int max_tokens, int align, int32_t* row0_out,
                         int32_t* lo_out, int32_t* hi_out, int32_t* tile_kv_out, int* n_placed, int* n_tiles);
/* Host-only: the rows of that plan as ance_encoder_forward_train_packed keeps them: row0_out[i] as above and
 * row_tok_out [*n_tiles * 128] = the dense token b L + i that each packed row computes (sequence b = token / L), -1 for a
 * row of no sequence. */
int ance_dbg_pack_rows(const int32_t* lens_host, int B, int L, int max_tokens, int align, int32_t* row0_out,
                       int32_t* row_tok_out, int* n_placed, int* n_tiles);
/* D[M,N] = act(A[M,K] * B[N,K]^T + bias) + R ; A,B 16-bit device arrays in `fmt`; R and the 16-bit output D are bf16
 * whatever `fmt` is; outputs optional; act 0 none, 1 GELU (erfc form), 2 GELU (logistic form).
 * variant (N tile BN, CTA cluster CG, operand stages): 0 = BN 128 CG 1 4 stages, 1 = BN 128 CG 1 3 stages,
 * 2 = BN 128 CG 2 4 stages, 3 = BN 64 CG 2 6 stages, 4 = BN 64 CG 1 6 stages */
int ance_dbg_gemm(const void* A_dev, const void* B_dev, int M, int N, int K, int fmt, int variant,
                  const float* bias_dev, const void* residual_bf16_dev, int act, void* C_bf16_dev,
                  float* C_f32_dev, void* stream);
/* The encoder's own GEMM launch (the instantiation every linear layer of the forward runs):
 * C[M,N] = act(A[M,K] W[N,K]^T + bias) + R with A rows at pitch lda, R rows at pitch ldr (ignored without R), C16 / C32
 * at pitch N.  A, W, R and C16 are 16-bit in `fmt`, bias and C32 fp32; bias, R and either output may be null.  act: 0 none,
 * 1 GELU (erfc form), 2 GELU (logistic form, the forward's default); the ANCE_B200_GELU environment variable is not read.
 * Every buffer 16-byte aligned, N, K, lda, ldr multiples of 8. */
int ance_dbg_linear(int fmt, const void* A_dev, int64_t lda, int M, const void* W_dev, int N, int K, const float* bias_dev,
                    const void* R_dev, int64_t ldr, int act, void* C16_dev, float* C32_dev, void* stream);
/* The encoder's own attention launch (same kernel selection and parameters as the forward): qkv [n_tokens, 3 * 64 heads]
 * 16-bit (Q | K | V, head-major inside each), kbias [n_tokens] fp32 additive key bias in log2 units (0 or
 * -10000 log2 e), ctx [n_tokens, 64 heads] 16-bit.  Dense (row_lo null): n_tokens / L sequences of L tokens.  Packed: the
 * device row plan of ance_dbg_pack_packed (row_lo / row_hi [n_tokens], absolute rows; tile_kv [n_tokens / 128 * 2], only
 * and always for L > 128), n_tokens a multiple of 128. */
int ance_dbg_attention(int fmt, const void* qkv_dev, int n_tokens, int L, int heads, const float* kbias_dev,
                       const int32_t* row_lo_dev, const int32_t* row_hi_dev, const int32_t* tile_kv_dev, void* ctx_dev,
                       void* stream);
/* The encoder's own LayerNorm launch: rows of `in` (16-bit in `fmt`, or fp32 when in_f32) at pitch in_ld -> out16 (16-bit)
 * and / or out32 (fp32) at pitch H, H in {256, 512, 768, 1024}.  rows_per_warp (1..4) stands in for the process-wide
 * "ln_rows_per_warp" tunable for this call only. */
int ance_dbg_layer_norm(int fmt, const void* in_dev, int in_f32, int64_t in_ld, int rows, int H, const float* gamma_dev,
                        const float* beta_dev, float eps, void* out16_dev, float* out32_dev, int rows_per_warp,
                        void* stream);
/* The backward's attention kernel: qkv [B * L, 3 * 64 heads] 16-bit in `fmt` and kbias [B * L] as for ance_dbg_attention
 * (dense, L <= 128), dout [B * L, 64 heads] bf16 (cls_only: [B, 64 heads], the gradient of token 0 of each sequence only)
 * -> dqkv [B * L, 3 * 64 heads] fp32. */
int ance_dbg_attention_backward(int fmt, const void* qkv_dev, const float* kbias_dev, const void* dout_bf16_dev,
                                int cls_only, int B, int L, int heads, float* dqkv_dev, void* stream);
/* The backward's attention kernels for L in {256, 384, 512} (the launch ance_encoder_backward makes there): the arguments
 * of ance_dbg_attention_backward, qkv, dout and dqkv 16-byte aligned.  Key-blocked on the tensor cores: a query-block
 * kernel writes dQ and per-row softmax statistics (scratch allocated per call), a key-block kernel then dK and dV. */
int ance_dbg_attention_backward_long(int fmt, const void* qkv_dev, const float* kbias_dev, const void* dout_bf16_dev,
                                     int cls_only, int B, int L, int heads, float* dqkv_dev, void* stream);
/* The backward's LayerNorm kernel: input rows as for ance_dbg_layer_norm, dy / dx fp32 [rows, H]; dgamma, dbeta and dsum
 * (column sum of dx) [H] may each be null. */
int ance_dbg_layer_norm_backward(int fmt, const void* in_dev, int in_f32, int64_t in_ld, int rows, int H,
                                 const float* gamma_dev, float eps, const float* dy_dev, float* dx_dev, float* dgamma_dev,
                                 float* dbeta_dev, float* dsum_dev, void* stream);
/* The backward's GELU kernel: g[i] *= gelu'(u[i]) for n elements, u 16-bit in `fmt`, g fp32. */
int ance_dbg_gelu_backward(int fmt, const void* u_dev, float* g_dev, int64_t n, void* stream);
/* The backward's embedding kernels: E [B * L, H] fp32 = (word[id] + pos[p]) + type[0], the LayerNorm input the backward
 * recomputes (positions by the arch's rule, roberta = 1 for RoBERTa's), then dword [vocab, H] and dpos [max_pos, H] are
 * zeroed and the rows of dE [B * L, H] scatter-added into them (no gradient for the padding_idx rows).  L <= 512. */
int ance_dbg_embedding_backward(const int32_t* ids_dev, int B, int L, int H, int roberta, int pad_id, int vocab, int max_pos,
                                const float* word_dev, const float* pos_dev, const float* type_dev, const float* dE_dev,
                                float* E_dev, float* dword_dev, float* dpos_dev, void* stream);
/* The backward's transpose: dst [C, dst_ld] bf16 = src [R, C]^T (src rows at pitch src_ld; src_kind 0 fp16, 1 bf16, 2 fp32),
 * columns R .. dst_ld - 1 of dst set to zero. */
int ance_dbg_transpose_bf16(int src_kind, const void* src_dev, int64_t src_ld, int R, int C, void* dst_dev, int64_t dst_ld,
                            void* stream);
/* The dropout generator's raw output: n Philox4x32-10 calls under the key (seed & 0xffffffff, seed >> 32); call i has
 * the counter (lo32(first_counter + i), hi32(first_counter + i), lo32(stream_word), hi32(stream_word)) and writes its four
 * words to out_dev[4 i .. 4 i + 3] (device, 16-byte aligned). */
int ance_dbg_dropout_bits(uint64_t seed, uint64_t stream_word, uint64_t first_counter, int64_t n, uint32_t* out_dev, void* stream);
/* The backward's attention kernels with dropout (what ance_encoder_backward launches after
 * ance_encoder_forward_train_dropout): the arguments of ance_dbg_attention_backward (L <= 128) or
 * ance_dbg_attention_backward_long (L in {256, 384, 512}), plus the probability rate p_attn (finite, in (0, 1)), the seed
 * and the layer whose site-1 mask to apply. */
int ance_dbg_attention_backward_dropout(int fmt, const void* qkv_dev, const float* kbias_dev, const void* dout_bf16_dev,
                                        int cls_only, int B, int L, int heads, float p_attn, uint64_t seed, int layer,
                                        float* dqkv_dev, void* stream);
/* The packed training backward's attention launch (ance_encoder_backward of a packed plan): sequence b occupies rows
 * seq_row0_dev[b] .. + seq_len_dev[b] of qkv [n_rows, 3 * 64 heads] (and of dout [n_rows, 64 heads] bf16, or dout [B, 64
 * heads] with cls_only), each at its own length <= L (<= 128: attn_bwd_kernel; up to 512: the key-blocked kernels).
 * dqkv_dev [n_rows, 3 * 64 heads] fp32 is zeroed first, as the backward does, so rows of no sequence come back 0.
 * p_attn > 0 applies the site-1 dropout of `layer` with `seed` (counters: sequence b, query and key in the sequence). */
int ance_dbg_attention_backward_packed(int fmt, const void* qkv_dev, const float* kbias_dev, const void* dout_bf16_dev,
                                       int cls_only, int B, int L, int heads, const int32_t* seq_row0_dev,
                                       const int32_t* seq_len_dev, int n_rows, float p_attn, uint64_t seed, int layer,
                                       float* dqkv_dev, void* stream);
/* Host-only: the byte offsets of the workspace ance_encoder_forward_train fills for a [B, L] batch (L <= 128, or a multiple
 * of 128 up to the handle's "train_max_len"), out[15] =
 * ids, kbias, layers, per_layer, x_in, qkv, ctx, t1, x1, u, ff, t2, x_final, head_in, total.  ids [B * L] int32 and kbias
 * [B * L] fp32 (log2 units) sit at their offsets; layer l's slots at layers + l * per_layer + (x_in .. t2); x_final
 * [B, hidden] 16-bit (the last layer's CLS outputs) and head_in [B, hidden] fp32 (the head LayerNorm's input) at theirs.
 * Every slot has room for B * L rows and is 16-bit in operand_fmt: x_in, ctx, t1, x1, t2 [., hidden], qkv [., 3 hidden],
 * u, ff [., ffn].  In the pruned last layer T1, X1, U, FF and T2 are compact: row b is sequence b's CLS row (B rows used);
 * CTX keeps its B * L rows (the CLS rows are read at pitch L * hidden); X_in and QKV are full. */
int ance_dbg_train_layout(ance_encoder_t enc, int B, int L, size_t* out);
/* Host-only: the workspace ance_encoder_forward_train_packed fills for the prefix lengths lens_host[B] of a [B, L] batch,
 * planned exactly as that call plans it (the handle's current "varlen_align"; the same refusals).  *n_tiles = the plan's
 * tiles, M = n_tiles * 128 packed rows; out[24] = the 15 fields of ance_dbg_train_layout for M rows (ids stays the dense
 * [B * L]; kbias and every per-layer slot hold M rows, the pruned last layer's compact slots B), then seq_row0 [B],
 * seq_len [B], row_lo, row_hi, row_tok [M] int32 (row_tok: the dense token b L + i of each row, -1 for a row of no
 * sequence), tile_kv [n_tiles] int2, cls_ctx, cls_x [B, hidden] 16-bit (the last layer's CTX and X_in rows at seq_row0)
 * and the total size. */
int ance_dbg_train_layout_packed(ance_encoder_t enc, const int32_t* lens_host, int B, int L, size_t* out, int* n_tiles);
/* Read-only copy of what a flat-IP index holds for the exactness certificate, into dst (host or device memory; the
 * stream is synchronised).  n_bytes must be the item's exact size, else ANCE_ERR_INVALID, as is an item the index does
 * not hold (no search since rows were added or the format changed; ndelta of a device index).  Items:
 *   rows (after the last prepare / search): MU fp32 [dim] (the centre; meaningful when CENTRED), CENTRED int32,
 *     P16 [n, dim] 16-bit operand rows, PSTATS [2] fp32 bits (max ||p^||, max ||p - mu - p^||), NDELTA fp32 [n] (host
 *     index: per-row ||p - mu - p^||, rounded up);
 *   the last ance_index_search's queries (its last block of <= 16,384 when k > 512): Q16 [nq, dim], QN_HAT, QN_DELTA fp32
 *     [nq]; the tier-1 uncertified list FLAGGED int32 [cnt] in slot order, FLAGGED_CNT int32, FLAGGED_THR fp32 [cnt]
 *     (tier 2's starting threshold of each slot);
 *   the last coarse pass (tier 1, or tier 2 when it ran; slot = query * n_splits + split, a tier-2 query is
 *     FLAGGED[query]): CAND_ID int32 [slots, out_cap], CAND_CNT int32 [slots], CAND_THR fp32 [slots] (every row of the
 *     split that is not a candidate has coarse score <= it), PASS int32 [6] = nq, n_splits, out_cap, k', rows per split
 *     (split s covers rows [s * it, (s + 1) * it)), tier. */
enum {
  ANCE_STATE_MU = 0, ANCE_STATE_CENTRED = 1, ANCE_STATE_P16 = 2, ANCE_STATE_PSTATS = 3, ANCE_STATE_NDELTA = 4,
  ANCE_STATE_Q16 = 5, ANCE_STATE_QN_HAT = 6, ANCE_STATE_QN_DELTA = 7, ANCE_STATE_CAND_ID = 8, ANCE_STATE_CAND_CNT = 9,
  ANCE_STATE_CAND_THR = 10, ANCE_STATE_PASS = 11, ANCE_STATE_FLAGGED = 12, ANCE_STATE_FLAGGED_CNT = 13,
  ANCE_STATE_FLAGGED_THR = 14
};
int ance_dbg_index_state(ance_index_t idx, int what, void* dst, int64_t n_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ANCE_B200_H_ */

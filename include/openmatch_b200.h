/* openmatch_b200 — C ABI of the H100-native dense-retrieval hot path (libopenmatch_b200.so).
 *
 * The reference (thunlp/OpenMatch, 100 % Python) has no FFI layer; the seams where its hot path crosses
 * into third-party compute are three Python call sites, and each entry point below replaces one of them
 * (paths relative to the reference tree):
 *
 *   encoder  : DRModel.encode -> model(**items)          src/openmatch/modeling/dense_retrieval_model.py:133-155
 *              + mean_pooling                             src/openmatch/utils.py:233-235
 *              + LinearHead.forward                       src/openmatch/modeling/linear.py:22-23
 *   index    : faiss.IndexFlatIP(dim) / .add / .search / .reset / .ntotal
 *                                                         src/openmatch/retriever/dense_retriever.py:38-41,105,133-137,180
 *              IndexShards merge behind index_cpu_to_gpu_multiple(shard=True)   ...:43-58
 *   loss     : torch.matmul + cross_entropy (+ autograd)  src/openmatch/loss.py:7-15,
 *                                                         src/openmatch/modeling/dense_retrieval_model.py:113-125
 *
 * Conventions: plain C symbols; every function returns 0 on success and a negative OM_E* code on
 * failure, om_last_error() then holds a thread-local message.  The caller owns all tensor memory and
 * passes raw pointers (host or device as stated) plus a CUDA stream handle (cudaStream_t cast to void*,
 * NULL = legacy default stream); the library owns only its opaque handles.  One process drives one GPU;
 * a handle is not thread-safe, distinct handles are.  There is no CPU fallback: every compute entry
 * point fails with OM_ENODEVICE when no sm_90 device is present.
 *
 * Streams.  `stream` may be any stream, including a non-blocking one that does not wait for the legacy
 * stream; the library issues the work of a call on that stream only.  The calls without a stream order
 * themselves: om_encoder_set_weight runs after all work already issued on the device and has finished
 * reading the caller's data on return; om_index_reserve synchronises the device when it grows the shard;
 * a search of a host-resident index (om_index_create_host) also uploads rows on a stream the index owns, ordered after
 * the caller's earlier work on `stream` and finished on return;
 * om_index_reset touches no device memory (the error-norm maxima are zeroed on the stream of the next
 * commit or search).  One handle must not be used from two streams at once.  The loss workspace is
 * process-global: loss calls must not overlap across streams.
 */
#ifndef OPENMATCH_B200_H_
#define OPENMATCH_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OM_ABI_VERSION 2

enum { OM_OK = 0, OM_EINVAL = -1, OM_ECUDA = -2, OM_ENOMEM = -3, OM_ENODEVICE = -4, OM_ESTATE = -5, OM_EFAULT = -6 };

typedef enum { OM_F32 = 0, OM_BF16 = 1, OM_F16 = 2, OM_I8 = 3 } om_dtype;
typedef enum { OM_HOST = 0, OM_DEVICE = 1 } om_memkind;
/* OM_ARCH_ROBERTA: RoBERTa / XLM-RoBERTa / CamemBERT, BERT's encoder (same parameter names, optionally prefixed
 * "roberta.") whose position ids come from the token ids, as HF's create_position_ids_from_input_ids computes them with
 * padding_idx = pad_token_id = 1 (the value of every such config; fixed here): a token with id != 1 gets position
 * 1 + (number of ids != 1 up to and including it in its sequence), a token with id 1 gets position 1, whatever the
 * attention mask says.  Sequences are at most max_position_embeddings - 2 tokens long (8194 positions, as in
 * XLM-RoBERTa-based bge-m3: 8192 tokens, the longest om_encode_packed takes).
 * OM_ARCH_MPNET: MPNet (all-mpnet-base-v2, multi-qa-mpnet), BERT's post-LN encoder with 64-wide heads only (any other
 * width returns OM_EINVAL), no token-type embeddings (token_type_ids are ignored, as for T5), RoBERTa's position ids
 * (padding_idx 1, whatever pad_token_id says) and a relative position bias shared by all layers, added to the scaled
 * logits: T5's bidirectional bucket of (key index - query index) in the sequence, rel_buckets = 32 and
 * rel_max_distance = 128 (both required, as MPNetEncoder.compute_position_bias fixes them).  Names, optionally prefixed
 * "mpnet.": embeddings.{word_embeddings, position_embeddings, LayerNorm}, encoder.layer.<i>.attention.attn.{q, k, v, o},
 * encoder.layer.<i>.attention.LayerNorm, encoder.layer.<i>.intermediate.dense, encoder.layer.<i>.output.{dense,
 * LayerNorm}, encoder.relative_attention_bias.weight [32, heads].  Sequences are at most min(512,
 * max_position_embeddings - 2) tokens long (the relative-bias tables cover 512).
 * OM_ARCH_DISTILBERT: DistilBERT (TAS-B, msmarco-distilbert, multi-qa-distilbert), BERT's encoder and arithmetic with
 * no token-type embeddings (token_type_ids are ignored) and positions 0 .. L-1; every LayerNorm eps is 1e-12 in HF, so
 * pass ln_eps = 1e-12.  Names, optionally prefixed "distilbert.": embeddings.{word_embeddings, position_embeddings,
 * LayerNorm}, transformer.layer.<i>.attention.{q_lin, k_lin, v_lin, out_lin}, transformer.layer.<i>.sa_layer_norm,
 * transformer.layer.<i>.ffn.{lin1, lin2}, transformer.layer.<i>.output_layer_norm.  Sequences are at most min(8192,
 * max_position_embeddings) tokens long, as for BERT. */
typedef enum {
  OM_ARCH_BERT = 0,
  OM_ARCH_T5ENC = 1,
  OM_ARCH_ROBERTA = 2,
  OM_ARCH_MPNET = 3,
  OM_ARCH_DISTILBERT = 4
} om_arch;
typedef enum { OM_POOL_FIRST = 0, OM_POOL_MEAN = 1 } om_pooling;
typedef enum { OM_REDUCE_MEAN = 0, OM_REDUCE_SUM = 1 } om_reduction;

typedef struct om_encoder om_encoder;
typedef struct om_index om_index;
typedef struct om_comm om_comm;

/* ---- library ------------------------------------------------------------------------------------- */
int om_abi_version(void);
const char* om_last_error(void);
/* number of SMs of the current device, or a negative error (OM_ENODEVICE without a GPU) */
int om_device_sm_count(void);

/* ---- encoder: replaces HF BertModel / T5EncoderModel forward + pooling + head + normalise ---------- */
typedef struct om_encoder_desc {
  int32_t arch;             /* om_arch */
  int32_t layers;           /* num_hidden_layers / num_layers */
  int32_t hidden;           /* hidden_size / d_model (multiple of 128, at most 1024) */
  int32_t heads;            /* attention heads.  Head width: BERT hidden / heads, 64 (bert-base/large) or 32 (MiniLM,
                               bge-small, e5-small, gte-small); T5 d_kv = 64.  heads * width: a multiple of 128, at
                               most 2048.  Any other width returns OM_EINVAL */
  int32_t ffn;              /* intermediate_size / d_ff (multiple of 64) */
  int32_t vocab;            /* vocab_size */
  int32_t max_pos;          /* max_position_embeddings (BERT; RoBERTa, MPNet: including their offset of 2, e.g. 514,
                               at least 3); ignored for T5 */
  int32_t type_vocab;       /* type_vocab_size (BERT; RoBERTa: normally 1); ignored for T5, MPNet and DistilBERT */
  float ln_eps;             /* layer_norm_eps (1e-12 BERT) / layer_norm_epsilon (1e-6 T5) */
  int32_t pooling;          /* om_pooling: DRModel.pooling 'first' | 'mean' */
  int32_t has_head;         /* 1: bias-free LinearHead follows pooling */
  int32_t head_out;         /* LinearHead output_dim (any positive width) */
  int32_t normalize;        /* 1: F.normalize(reps, dim=1) */
  int32_t rel_buckets;      /* T5 relative_attention_num_buckets (32); MPNet: must be 32 */
  int32_t rel_max_distance; /* T5 relative_attention_max_distance (128); MPNet: must be 128 */
  int32_t max_batch_tokens; /* workspace sizing: max B*L per om_encode call (e.g. 256*128) */
} om_encoder_desc;

int om_encoder_create(const om_encoder_desc* desc, om_encoder** out);
/* Parameter by its HuggingFace state_dict name (e.g. "encoder.layer.3.attention.self.query.weight",
 * "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight", or "head.linear.weight" for
 * the LinearHead).  Data is fp32, row-major, host or device; the library keeps its own packed copy, the
 * caller's tensor may be freed afterwards.  Unknown names (e.g. "pooler.*", which OpenMatch never uses)
 * are ignored and reported through the return value 1.  Names are matched exactly.  Every parameter must be set
 * before om_encoder_finalize: once it has folded the weights, om_encoder_set_weight returns OM_ESTATE and changes
 * nothing (the handle stays finalized). */
int om_encoder_set_weight(om_encoder* enc, const char* name, const void* data, om_memkind kind,
                          const int64_t* shape, int ndim);
/* Verifies that every required parameter was supplied and builds derived tables. */
int om_encoder_finalize(om_encoder* enc);
/* input_ids / attention_mask / token_type_ids (nullable => zeros; ignored for T5, MPNet and DistilBERT): int64 [B, L]
 * device, row-major, exactly what DRInferenceCollator / QPCollator hand to the model; L <= 128 or 256 / 384 / 512, and
 * L <= max_position_embeddings (BERT, DistilBERT) / max_position_embeddings - 2 (RoBERTa, MPNet).
 * out_reps: device [B, rep_dim] fp32, bf16 or fp16 with row pitch out_row_stride (elements) — may point into an
 * index shard obtained from om_index_reserve() / om_index_reserve_rows().  fp16 output is the round-to-nearest-even
 * of the fp32 output of the same call (values beyond the half range become inf).  OM_I8 output: rows of an int8 index
 * (see om_index_create_typed), the fp32 output of the same call quantised by the index's rule: out_reps 4-byte aligned,
 * out_row_stride (bytes) a multiple of 4 and at least dpad + 16 (dpad = rep_dim rounded up to 16); a row holding inf
 * or NaN gets a NaN scale (om_index_commit counts it).  out_hidden: nullable device fp32 [B, L, hidden]
 * (last_hidden_state).  Asynchronous on `stream`. */
int om_encode(om_encoder* enc, const int64_t* input_ids, const int64_t* attention_mask,
              const int64_t* token_type_ids, int B, int L, void* out_reps, om_dtype out_dtype,
              int64_t out_row_stride, float* out_hidden, void* stream);
/* Variable-length batch, no padding.  tokens / token_type_ids (nullable => zeros; ignored for T5, MPNet and DistilBERT):
 * int64 [T] device, the B sequences back to back; seqlens: int32 [B] HOST, 1 <= seqlens[i] <= 8192 for BERT and
 * DistilBERT (and <= max_position_embeddings) and RoBERTa (and <= max_position_embeddings - 2, positions computed from
 * each sequence's own ids), <= 512 for T5 and MPNet (their relative-bias tables cover 512 tokens; MPNet also <=
 * max_position_embeddings - 2); and <= max_batch_tokens; T = sum(seqlens).  Result: what om_encode returns
 * for the same sequences padded to any L it takes with attention_mask = 1 on their tokens, up to the order of
 * floating-point sums in attention and pooling (longer sequences have no padded counterpart).  out_reps as in
 * om_encode (row i = sequence i).  out_hidden: nullable fp32 [T, hidden], packed like tokens.  seqlens may be reused on
 * return; no device synchronisation; asynchronous on `stream`.
 * Layout: sequences of <= 128 tokens are bin-packed whole into 128-row attention tiles (first-fit decreasing, ties by
 * input index: a deterministic function of seqlens); the longer ones come first, in input order, each starting on a
 * tile boundary and taking ceil(l / 128) tiles (a pipelined attention kernel), then the bins.  A layout of more than max_batch_tokens rows is encoded as consecutive groups of tiles on `stream`.
 * Invalid input (a null pointer, B < 0, a length outside the range above) returns OM_EINVAL and writes nothing. */
int om_encode_packed(om_encoder* enc, const int64_t* tokens, const int64_t* token_type_ids, const int32_t* seqlens,
                     int B, void* out_reps, om_dtype out_dtype, int64_t out_row_stride, float* out_hidden, void* stream);
/* Cross-encoder pairs (re-ranking, OpenMatch's RRModel.encode on encode_pair's sequences).  Sequence i =
 *   prefix ++ a_tokens[a_start_i : a_start_i + a_len_i] ++ b_tokens[b_start_i : b_start_i + b_len_i] ++ suffix,
 * token types all 0.  a_tokens [a_total] / b_tokens [b_total]: int32 DEVICE token stores (e.g. the queries and the
 * passages of a run, uploaded once); spans: int64 [B, 4] HOST (a_start, a_len, b_start, b_len); prefix / suffix: HOST,
 * 0..4 ids each (NULL when empty).  The pair tokens are assembled on the device, straight into the packed layout.
 * Result: bitwise what om_encode_packed returns for the same sequences given as an int64 token stream with
 * token_type_ids = NULL (the layout is the same function of the lengths, the same kernels run on it); out_reps as there,
 * no out_hidden.  A cross-encoder is an encoder with pooling first / mean, has_head = 1, head_out = 1 and normalize = 0:
 * out_reps then holds one score per pair.  spans, prefix and suffix may be reused on return; no device synchronisation;
 * asynchronous on `stream`.  Workspace for the assembled tokens (max_batch_tokens int64 + one span table) is allocated
 * on a handle's first call.  Invalid input returns OM_EINVAL and writes nothing: a null pointer, B < 0, n_prefix or
 * n_suffix outside [0, 4], a negative start or length, start + len beyond a_total / b_total, an assembled length
 * n_prefix + a_len + b_len + n_suffix outside the om_encode_packed range.  a_len = 0 and b_len = 0 are legal; B = 0 does
 * nothing. */
int om_encode_pairs(om_encoder* enc, const int32_t* a_tokens, int64_t a_total, const int32_t* b_tokens, int64_t b_total,
                    const int64_t* spans, int B, const int32_t* prefix, int n_prefix, const int32_t* suffix, int n_suffix,
                    void* out_reps, om_dtype out_dtype, int64_t out_row_stride, void* stream);
int om_encoder_rep_dim(const om_encoder* enc);
void om_encoder_destroy(om_encoder* enc);

/* ---- index: replaces faiss.IndexFlatIP (exact inner-product top-k) -------------------------------- */
int om_index_create(int d, om_index** out); /* faiss.IndexFlatIP(d); lives on the current device */
/* Index with a chosen row storage.  OM_F32 (= om_index_create): fp32 master rows + an fp16 scan copy, 6 bytes per
 * element.  OM_F16: the fp16 rows [n, dpad] (dpad = d rounded up to 8) only, 2 bytes per element; they are the scan
 * operand and the row store.  Search on an fp16 index is exact with respect to the STORED values: the exact top-k by
 * fp32 inner product of the fp32 query with the fp16 rows, in the summation order of the fp32 re-score, ties by
 * ascending id — bitwise what an fp32 index of the fp16-rounded rows returns.  Input fp16 cannot hold is refused:
 * om_index_add of a NaN or of a value that rounds to +-inf in fp16 (|x| >= 65520) returns OM_EINVAL and adds nothing;
 * rows written in place and committed with such values make every search return OM_EINVAL until om_index_reset (stat
 * "nonfinite_rows").
 * OM_I8: one byte per element and a per-row fp32 scale, rows of dpad + 16 bytes (dpad = d rounded up to 16): the codes
 * [0, d), zeros to dpad, the scale s at byte dpad, zeros to the end.  A row x (fp32; bf16 / fp16 converted exactly) is
 * stored as s = amax / 127 (amax = max |x_j|, IEEE division) and c_j = clamp(rint(x_j / s), -127, 127) (IEEE division,
 * half to even); a zero row gets s = 0 and codes 0; element j then holds fp32(s * c_j).  Search is exact with respect to
 * those values, bitwise what an fp32 index of them returns (same summation order, ties by ascending id).  om_index_add of
 * a row holding inf or NaN returns OM_EINVAL and adds nothing; rows written in place and committed with a non-finite
 * scale make every search return OM_EINVAL until om_index_reset (stat "nonfinite_rows").  The scan runs on s8 tensor
 * cores with a two-level int8 split of the query; "pair_scan" and "scan_cluster_*" do not apply.
 * OM_BF16 storage returns OM_EINVAL.  Every shard of a sharded search has the same storage. */
int om_index_create_typed(int d, om_dtype storage, om_index** out);
/* Host-resident index: the stored rows (same storages, row format and add rules as om_index_create_typed; fp32 storage
 * keeps the master rows only) live in pinned host memory, in chunks of window_rows rows, so a corpus larger than the
 * device memory can be searched on one GPU.  window_rows: a positive multiple of 256, or 0 = automatic (the largest
 * multiple of 256 rows, at least 256, for which two device windows take at most a quarter of the device memory free at
 * creation; a window row is the fp32 row plus its fp16 scan copy, dpad halves, or dpad + 16 bytes).
 * om_index_search / om_index_search_filtered search the rows one partition of window_rows rows at a time: the partition is
 * uploaded into one of two device windows while the previous one is searched, searched exactly, and merged into the
 * running top-k.  D and I are bitwise what a device index given the same adds returns (ties by ascending id across
 * partitions too); the stats that count work ("uncertified", "uncertified_wide", "exact_queries", "rounds", "launches")
 * are summed over the partitions; "partitions" is the number searched and, with "profile" on, "upload_wait_ns" the device
 * time the search waited for uploads.
 * Streams: the uploads run on a non-blocking stream the index owns, ordered after the work issued on `stream` before the
 * call, and the call returns with them finished — the one exception to "the work of a call runs on `stream` only".
 * om_index_add converts on the device (through a window) and synchronises `stream`; a failed pinned allocation returns
 * OM_ENOMEM and adds nothing.  om_index_reset keeps the host chunks; om_index_destroy frees them.
 * Limits: om_index_reserve, om_index_reserve_rows and om_index_commit return OM_ESTATE (there are no device rows to write
 * in place); om_index_search_sharded(_filtered) and om_index_range_search(_sharded)(_filtered) return OM_EINVAL; none
 * writes anything. */
int om_index_create_host(int d, om_dtype storage, int64_t window_rows, om_index** out);
int om_index_storage(const om_index* idx); /* the om_dtype given at creation */
/* index.add(x): x [n, d] row-major, fp32, bf16 or fp16 (host or device).  Rows get ids ntotal .. ntotal+n-1.
 * fp16 storage: converted to fp16 with round-to-nearest-even; int8 storage: quantised by the OM_I8 rule; both synchronise
 * `stream`. */
int om_index_add(om_index* idx, const void* x, om_memkind kind, om_dtype dtype, int64_t n, void* stream);
/* Zero-copy ingest: reserve room for n more rows and get the device address of the fp32 row block
 * (row pitch = d floats) so the encoder can write embeddings in place; om_index_commit(n) publishes
 * them (builds the fp16 scan copy and updates the error-norm maxima the exactness certificate uses).  */
int om_index_reserve(om_index* idx, int64_t n, float** dev_rows); /* fp32 storage only (OM_ESTATE otherwise) */
/* Any storage: the device address of the next n rows, fp32 at pitch d, fp16 at pitch dpad (elements) or int8 rows at
 * pitch dpad + 16 (bytes).  For fp16 / int8 rows om_index_commit updates the error-norm maxima and counts rows with a
 * non-finite element (fp16) or scale (int8). */
int om_index_reserve_rows(om_index* idx, int64_t n, void** dev_rows, int64_t* row_pitch_elems);
int om_index_commit(om_index* idx, int64_t n, void* stream);
int64_t om_index_ntotal(const om_index* idx);
int om_index_dim(const om_index* idx);
int om_index_reset(om_index* idx);
/* D, I = index.search(q, k): q [nq, d] fp32 (host or device); D fp32 [nq, k], I int64 [nq, k] written to
 * host or device memory (out_kind).  Rows are ordered by (score descending, id ascending); missing
 * slots (k > ntotal) hold id -1 and score -FLT_MAX, as faiss does.  Reported ids are id_offset + local
 * row, so a rank of a row-sharded index passes the global id of its first row.  k <= 4096.
 * Exactness: candidates (k + slack per query) are selected on fp16 tensor-core scores and re-scored in fp32;
 * an a-posteriori certificate (measured quantisation-error norms of corpus and query, see csrc/search.cu
 * certify_kernel) then PROVES per query that no row outside the candidate list can reach the k-th fp32 score.
 * Queries that fail it are re-run with the widest candidate list (4096) and, if still unproven (e.g. thousands
 * of near-duplicate rows), answered by an exact fp32 scan with the same summation order as the re-score.  The
 * result is therefore always the exact top-k by fp32 inner product with ties by ascending id.
 * Synchronous with respect to `stream` on return. */
int om_index_search(om_index* idx, const void* q, om_memkind q_kind, int nq, int k, float* D, int64_t* I,
                    om_memkind out_kind, int64_t id_offset, void* stream);
/* Row-sharded search with the exchange inside the library — replaces faiss.index_cpu_to_gpu_multiple(shard=True) +
 * IndexShards (src/openmatch/retriever/dense_retriever.py:43-58).  One process per GPU; every rank holds a contiguous
 * row shard and calls om_index_search_sharded with the same queries and its own id_offset; every rank receives the
 * same global (D, I).  Each shard keeps a candidate list sized for its share of the answer (m + 6 sqrt(m) + 32 with m = (k + slack) / world
 * rows), re-scores it in fp32 and ships it whole together with the list's stage-score floor and the shard's error-norm
 * maxima in ONE packed NCCL all-gather per query chunk (issued on `stream` between the kernels, single host
 * synchronisation at the end of a level); every rank merges the lists and runs the exactness certificate of
 * om_index_search with tau = the largest floor.  Skewed shards fail the certificate and are answered by the wider levels.
 *   om_comm_unique_id : rank 0 obtains 128 opaque bytes (ncclGetUniqueId) and ships them to the other ranks
 *                       (e.g. torch.distributed.broadcast_object_list)
 *   om_comm_init      : collective over the `world` ranks (ncclCommInitRank) on the current device
 * NCCL is bound at run time (dlopen of libnccl.so.2; inside PyTorch that is the copy torch already loaded). */
int om_comm_unique_id(char* out128);
int om_comm_init(const char* unique_id128, int rank, int world, om_comm** out);
void om_comm_destroy(om_comm* comm);
int om_index_search_sharded(om_index* idx, om_comm* comm, const void* q, om_memkind q_kind, int nq, int k, float* D,
                            int64_t* I, om_memkind out_kind, int64_t id_offset, void* stream);

/* Filtered search: the exact top-k, by fp32 inner product over the stored rows, among the rows the bitmap allows and the
 * query does not exclude; ties by ascending id.  D and I are bitwise what om_index_search returns on an index built from
 * the eligible rows only, with ids mapped back; fewer than k eligible rows leave id -1 and score -FLT_MAX slots.
 *   allow_bits       nullable, device: bit (r & 31) of word r >> 5 set = local row r may be returned
 *   allow_words      >= ceil(ntotal / 32) when allow_bits is given; bits past ntotal are ignored
 *   exclude_offsets  nullable, device [nq + 1]: CSR over the queries, non-decreasing; at most 128 ids per query
 *   exclude_ids      device: ids in the result id space (id_offset + local row), >= 0, any order, duplicates allowed; an
 *                    id outside [id_offset, id_offset + ntotal) is ignored, so every rank of a sharded search takes the
 *                    same CSR
 * A rule broken returns OM_EINVAL before any output is written.  A null filter, or one with both parts null, is
 * om_index_search / om_index_search_sharded.  The filter buffers are read on `stream`; everything else (tunables, the
 * synchronous return, the refusal of non-finite rows) is as for the unfiltered calls.  Sharded: allow_bits covers this
 * rank's rows; every rank calls om_index_search_sharded_filtered, and a rank may pass a null or empty filter while others
 * pass one (with more than one rank the filters are always checked together, one all-reduce). */
typedef struct om_search_filter {
  const uint32_t* allow_bits;
  int64_t allow_words;
  const int64_t* exclude_offsets;
  const int64_t* exclude_ids;
} om_search_filter;
int om_index_search_filtered(om_index* idx, const void* q, om_memkind q_kind, int nq, int k, float* D, int64_t* I,
                             om_memkind out_kind, int64_t id_offset, const om_search_filter* filter, void* stream);
int om_index_search_sharded_filtered(om_index* idx, om_comm* comm, const void* q, om_memkind q_kind, int nq, int k,
                                     float* D, int64_t* I, om_memkind out_kind, int64_t id_offset,
                                     const om_search_filter* filter, void* stream);

/* Range search (faiss IndexFlatIP.range_search): for query i every row whose fp32 score, as om_index_search computes it,
 * is strictly greater than radius[i], ordered by (score desc, id asc).  For every j <= min(count, 4096) the first j results
 * of a query are bitwise om_index_search(q, j)'s D and I.  Exact on every storage (fp16 / int8: with respect to the stored
 * values) with no certificate to fail: one sweep at radius - E(q) (the certificate's error bound) collects a superset,
 * which is re-scored exactly and cut at the radius; queries without a finite bound take the exact fp32 scan.
 * radius: [nq] fp32, same memkind as q; NaN returns OM_EINVAL before any write.  radius -inf returns every row, +inf none.
 * lims: [nq + 1] int64 written to out_kind memory; query i's results are [lims[i], lims[i + 1]), lims[nq] = total results.
 * The results stay in the handle until its next search / range search / reset / destroy: the caller learns the total
 * before it allocates, and om_index_range_results copies them out.  Synchronous on return.
 * Sharded: every rank passes the same queries and radii and its own id_offset and receives the same lims and results,
 * bitwise the range search of one index over the concatenated shards.  Tunables that apply: "pair_scan",
 * "scan_cluster_q" / "_x", "exact_only" and "range_list" (first candidate list length per query, default 4096; a query
 * with more candidates is swept again with a list sized from its count); stats "range_candidates" (rows re-scored),
 * "range_resweeps" (queries swept again) and "exact_queries". */
int om_index_range_search(om_index* idx, const void* q, om_memkind q_kind, int nq, const float* radius, int64_t* lims,
                          om_memkind out_kind, int64_t id_offset, void* stream);
int om_index_range_search_sharded(om_index* idx, om_comm* comm, const void* q, om_memkind q_kind, int nq,
                                  const float* radius, int64_t* lims, om_memkind out_kind, int64_t id_offset, void* stream);
/* Filtered range search: for query i every row that the filter's bitmap allows and query i does not exclude, and whose
 * fp32 score is strictly greater than radius[i], ordered by (score desc, id asc).  The filter is om_search_filter with
 * the rules of om_index_search_filtered (bitmap over the local rows, allow_words >= ceil(ntotal / 32), at most 128
 * excluded ids per query in the result id space, >= 0, non-decreasing offsets; ids outside the shard are ignored and
 * duplicates are allowed).  lims and the results are bitwise what om_index_range_search returns on an index built from
 * the eligible rows only, with ids mapped back, on every storage; for every j <= min(count, 4096) the first j results of
 * a query are bitwise om_index_search_filtered(q, j)'s with the same filter.  Disallowed rows are never collected, so
 * their count does not send a query to a second sweep.  A broken rule, a NaN radius or non-finite fp16 / int8 rows
 * return OM_EINVAL before lims is written.  A null filter, or one with both parts null, is om_index_range_search /
 * om_index_range_search_sharded.  Sharded: allow_bits covers this rank's rows, exclusions are global ids; every rank
 * calls om_index_range_search_sharded_filtered, and a rank may pass a null or empty filter while others pass one (with
 * more than one rank the filters are always checked together, one all-reduce).  Everything else (results kept in the
 * handle, tunables, stats, the synchronous return) is as for the unfiltered calls. */
int om_index_range_search_filtered(om_index* idx, const void* q, om_memkind q_kind, int nq, const float* radius,
                                   int64_t* lims, om_memkind out_kind, int64_t id_offset, const om_search_filter* filter,
                                   void* stream);
int om_index_range_search_sharded_filtered(om_index* idx, om_comm* comm, const void* q, om_memkind q_kind, int nq,
                                           const float* radius, int64_t* lims, om_memkind out_kind, int64_t id_offset,
                                           const om_search_filter* filter, void* stream);
/* D fp32 [lims[nq]], I int64 [lims[nq]] of the last range search on idx; OM_ESTATE if there is none. */
int om_index_range_results(const om_index* idx, float* D, int64_t* I, om_memkind out_kind, void* stream);

/* Tunables: "rescore_slack" (extra candidate-stage rows kept per query; default max(128, k/5)),
 * "force_safe_rounds" (1 = always use the overflow-proof fixed-size round schedule; testing),
 * "round_growth" (2..8: each scan round covers (g-1) x the rows already seen; default 0 = auto: 2, or 8 for <= 256 queries),
 * "certify" (default 1; 0 = skip the exactness certificate and its escalation: top-k of the fp16 candidate stage),
 * "exact_only" (1 = answer every query with the exact fp32 CUDA-core scan; testing),
 * "debug_stage_scores" (1 = D holds candidate-stage scores instead of fp32 re-scores; error-model measurement),
 * "pair_scan" (default 1: after the first round, batches of > 128 queries scan on 2-CTA clusters with 256-row corpus
 *   tiles multicast to both CTAs and the top-k filter on the accumulator registers; 0 = single-CTA 128 x 128 tiles),
 * "profile" (1 = bracket every kernel launch of a search with CUDA events on the launching stream). */
int om_index_set_param(om_index* idx, const char* name, int64_t value);
/* Statistics of the last search: "rounds", "overflow_retries", "candidates" (per query capacity),
 * "launches" (kernels launched), "uncertified" (queries the first level could not prove exact),
 * "uncertified_wide" (still unproven with 4096 candidates), "exact_queries" (answered by the exact fp32 scan),
 * "nonfinite_rows" (fp16 / int8 storage: committed rows holding inf or NaN, as the last search read it; 0 after a reset),
 * and with "profile" on: "scan_ns", "select_ns",
 * "finalize_ns", "other_ns" (device time summed over the launches of each kind; other = exchange + merge + certify). */
int64_t om_index_get_stat(const om_index* idx, const char* name);
void om_index_destroy(om_index* idx);

/* Exchange step of the row-sharded search: merge `nparts` per-shard results laid out as
 * D_parts [nparts, nq, k_in], I_parts [nparts, nq, k_in] (device) into the global top-k_out by (score desc, id asc);
 * ids < 0 are padding.  Matches merge semantics of faiss IndexShards / utils.py:215-229.  Input lists may be
 * narrower than the output (k_in < k_out); more than 8192 entries per query (nparts * k_in) are merged
 * hierarchically. */
int om_topk_merge_n(const float* D_parts, const int64_t* I_parts, int nparts, int nq, int k_in, int k_out, float* D,
                    int64_t* I, void* stream);

/* ---- loss: replaces matmul + cross_entropy + autograd backward ------------------------------------ */
/* Q [nq, d], P [np, d] device, fp32 or bf16 (both the same dtype; any other returns OM_EINVAL), row-major.
 * target: nullable int64 [nq] device (NULL => i * (np / nq), loss.py:11-13).
 * loss_out: device fp32 scalar = loss_scale * reduce_i(logsumexp_j s_ij - s_i,target_i).
 * dQ [nq, d], dP [np, d]: nullable device fp32 gradients of loss_out.  scores_out: nullable device fp32
 * [nq, np] logits (DROutput.scores).  Asynchronous on `stream`. */
int om_contrastive_loss_fwd_bwd(const void* Q, const void* P, om_dtype dtype, int nq, int np, int d,
                                const int64_t* target, int reduction, float loss_scale, float* loss_out,
                                float* dQ, float* dP, float* scores_out, void* stream);
/* Diagnostics: device time (ns, %globaltimer) the most recent loss call spent in its four phases
 * {PREP, LOGITS, SOFTMAX, GRADS}.  Synchronises the device first, so it reads the last call on any stream. */
int om_debug_loss_phase_ns(uint64_t out[4]);

#ifdef __cplusplus
}
#endif
#endif /* OPENMATCH_B200_H_ */

/* libw2b — C ABI of the H100-native Word2Bits training path.
 *
 * The reference (agnusmaximus/Word2Bits, src/word2bits.cpp) has no FFI: it is one
 * executable whose hot path is `void *TrainModelThread(void *id)` (:363-516) reading and
 * writing file-scope globals (:45-61).  This header is the seam a maintainer would cut
 * there: every entry point below names the reference code it replaces.  Plain C types
 * only; the caller owns host buffers, the library owns device memory; one context is
 * driven by one host thread; all calls are synchronous; every function returns 0 on
 * success or a non-zero W2B_E* code, and w2b_last_error() gives the message (the
 * reference's convention is printf + exit(1), which the CLI wrapper reproduces).
 */
#ifndef W2B_H
#define W2B_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define W2B_OK 0
#define W2B_EINVAL 1   /* bad argument / unsupported configuration */
#define W2B_ECUDA 2    /* CUDA runtime error (no device, launch failure, OOM) */
#define W2B_EIO 3      /* file not found / unreadable / unwritable */
#define W2B_ESTATE 4   /* call sequence error (e.g. train before set_corpus) */
#define W2B_ENCCL 5    /* NCCL error / NCCL not loadable */
#define W2B_ENOMEM 6   /* host allocation failed (nothing is thrown across the ABI) */

#define W2B_TABLE_SIZE 100000000 /* table_size, :60 */
#define W2B_MAX_SENTENCE 1000    /* MAX_SENTENCE_LENGTH, :32 */
#define W2B_MAX_WINDOW 512   /* a sentence has at most 1000 words (:32): beyond ~500 every word is context anyway */
#define W2B_MAX_NEGATIVE 63   /* 1 + negative targets per position fit one 64-entry trace record / two lanes-worth of loss terms */

#define W2B_MODE_FAST 0   /* production: one warp per shard, all shards concurrent (Hogwild) */
#define W2B_MODE_STRICT 1 /* parity: shards one after another, sequential IEEE op order */

/* ------------------------------------------------------------------ host glue (no GPU)
 * Corpus reader + vocabulary: replaces ReadWord/SearchVocab/AddWordToVocab/SortVocab/
 * LearnVocabFromTrainFile (:131-301).  Results (word order, counts, train_words,
 * file_size) are identical; the text is tokenised ONCE into an int32 id stream. */
typedef struct w2b_corpus w2b_corpus;
int w2b_corpus_load(const char *train_file, int min_count, w2b_corpus **out);
void w2b_corpus_free(w2b_corpus *c);
int64_t w2b_corpus_vocab_size(const w2b_corpus *c);  /* vocab_size, :50 */
int64_t w2b_corpus_train_words(const w2b_corpus *c); /* train_words, :51 */
int64_t w2b_corpus_file_size(const w2b_corpus *c);   /* file_size, :299 */
const char *w2b_corpus_word(const w2b_corpus *c, int64_t i);
const int64_t *w2b_corpus_counts(const w2b_corpus *c); /* vocab[i].cn */
int64_t w2b_corpus_num_tokens(const w2b_corpus *c);    /* in-vocab tokens incl. </s> */
const int32_t *w2b_corpus_tokens(const w2b_corpus *c);
/* Shard i of n starts where the reference's fseek(file_size/n*i) (:377) puts thread i:
 * first[i] = id of the first token read there (a suffix fragment when the seek lands
 * mid-word; -1 if it is out of vocabulary), start[i] = index of the next regular token. */
int w2b_corpus_shards(const w2b_corpus *c, int n, int64_t *start, int32_t *first);
/* Vector file writer (:560-576): header "%lld %lld\n", then "<word> " + D values
 * ("%lf " text or raw float32) + "\n" per word. */
int w2b_write_vectors(const char *path, const w2b_corpus *c, const float *vectors, int64_t V,
                      int64_t D, int binary);

/* Packed vector file (SURVEY section 8(f).3: the README's storage claim is realised only by gzip in the
 * reference).  Header "<V> <D> <bitlevel>\n", then per word "<word> " + ceil(D*bitlevel/8) bytes
 * (value j occupies bits [j*bitlevel, (j+1)*bitlevel) little-endian: bit 0 = sign (1 = negative),
 * bit 1 (bitlevel 2) = magnitude (1 = .75)) + "\n".  bitlevel 1 and 2 only.  unpack restores the exact
 * float32 levels, so `unpack -> w2b_write_vectors(binary=1)` feeds compute_accuracy unchanged. */
int w2b_write_packed(const char *path, const w2b_corpus *c, const float *vectors, int64_t V, int64_t D,
                     int bitlevel);
int w2b_read_packed_header(const char *path, int64_t *V, int64_t *D, int *bitlevel);
int w2b_read_packed(const char *path, float *vectors /* V*D */, char *words /* V*max_word */, int max_word);

/* Vector file kinds, and the one rule that tells them apart.  A first line of three integers is a packed file.  A first
 * line of two integers "V D" is a text file (-binary 0: per word "<word> " then D values "%lf " then "\n") when (a) the
 * byte right after the 4 D bytes that follow the first name's ' ' is not '\n' and (b) the bytes from that ' ' to the
 * first '\n' are exactly D tokens of the grammar of w2b_host_parse_floats.  Every other file is word2vec binary (every
 * binary file has '\n' after its first row's 4 D bytes; a "%lf " value takes at least 9 bytes).
 * *V = the header's word count (at most threshold when threshold > 0), *D = its size, *bits = a packed file's bit level
 * (else 0).  W2B_EIO only when the file cannot be opened. */
#define W2B_VECTORS_BINARY 0
#define W2B_VECTORS_TEXT 1
#define W2B_VECTORS_PACKED 2
int w2b_vector_file_info(const char *path, int64_t threshold, int *kind, int64_t *V, int64_t *D, int *bits);
/* The names of the first V rows (w2b_vector_file_info) of any vector file as the evaluator compares them: up to the
 * first ' ', '\n' skipped, at most 50 characters, upper-cased; name i at names[i*max_word], NUL-terminated (cut to
 * max_word - 1 characters).  *n = the rows read. */
int w2b_vector_names(const char *path, int64_t threshold, char *names /* V*max_word */, int max_word, int64_t *n);
/* A text vector file parsed on the GPU `device`: vectors = V x D floats (V, D from w2b_vector_file_info), each value
 * the float strtof returns for its token; words as w2b_read_packed writes them.  The file is streamed through the
 * device in chunks; no V x D array or whole text is held on the host beyond `vectors`.  W2B_EIO names the row and token
 * of a row with too few or too many values or a token outside the grammar. */
int w2b_read_text_vectors(const char *path, int device, float *vectors /* V*D */, char *words /* V*max_word */,
                          int max_word);

/* Host-side arithmetic of the path, callable (and tested) without a GPU.  The device path uses exactly
 * these functions for what it uploads: unigram boundaries (InitUnigramTable :112-128 in boundary form:
 * start[i] = first of the 1e8 table slots owned by word i, start[V] = 1e8), expTable (:614-618, same libm
 * expf), the sub-sampling thresholds `ran` (:403-404, float32), and the k-step / 2^j-step jump constants
 * of the LCG r*25214903917+11 (:352,:405,:428,:455) that let 32 lanes take 32 draws at once
 * (ja/jc: 65 entries, r_k = r*ja[k]+jc[k]; pa/pc: 64 entries for 2^j steps). */
int w2b_host_unigram_bounds(const int64_t *cn, int64_t V, int32_t *start /* V+1 */);
int w2b_host_exptable(float *out /* 1000 */);
int w2b_host_keep_thresholds(const int64_t *cn, int64_t V, int64_t train_words, float sample, float *out /* V */);
int w2b_host_lcg_tables(uint64_t *ja /*65*/, uint64_t *jc /*65*/, uint64_t *pa /*64*/, uint64_t *pc /*64*/);
/* Decimal text to float32 exactly as glibc strtof rounds it (to nearest, ties to even, subnormals, +-inf past
 * FLT_MAX, +-0 below half the smallest subnormal), with the routine the GPU text reader runs.  Tokens are separated by
 * white space; a token is [+-]?(d+[.d*]|.d+)([eE][+-]?d+)? or, signed or not and in any case, nan, inf or infinity.
 * out[0..*n) = the values; W2B_EIO names a token outside the grammar, W2B_EINVAL more than cap tokens. */
int w2b_host_parse_floats(const char *text, int64_t n_bytes, float *out, int64_t cap, int64_t *n);

/* The host half of a streaming step (w2b_set_corpus resident = 0): the next L tokens of every unfinished shard are
 * gathered into one pinned staging buffer (slice i at stage[i*L]) by a few host threads before the single H2D copy.
 * xlate[i] = global token index - staging index, limit[i] = global end of the slice, limit_is_eof[i] = slice reaches
 * the end of the stream.  Outputs of finished shards are left untouched.  nthreads <= 0: chosen from the size. */
int w2b_host_gather_slices(const int32_t *ids, int64_t n_tokens, int64_t L, int nshards, const int64_t *cursor,
                           const int32_t *done, int32_t *stage /* nshards*L */, int64_t *xlate, int64_t *limit,
                           int32_t *limit_is_eof, int nthreads);

/* ------------------------------------------------------------------------ device path */
typedef struct w2b_ctx w2b_ctx;

typedef struct {
  int64_t vocab_size;  /* V, incl. </s> at 0 */
  int64_t layer1_size; /* -size */
  int32_t window;      /* -window */
  int32_t negative;    /* -negative */
  int32_t bitlevel;    /* -bitlevel */
  float alpha;         /* -alpha (starting_alpha, :524) */
  float sample;        /* -sample */
  float reg;           /* -reg */
  int64_t iter;        /* -iter: enters the learning-rate schedule (:391) */
  int32_t num_shards;  /* -threads: TOTAL number of corpus shards S */
  int32_t shard_begin; /* this context trains shards [shard_begin, shard_end) of S */
  int32_t shard_end;   /*   (0,0 = all; used to split S across GPUs) */
  int32_t device;      /* CUDA device ordinal */
  int32_t mode;        /* W2B_MODE_FAST | W2B_MODE_STRICT */
  int32_t group;       /* register kernel: target rows in flight per CTA step (0 = default) */
  int32_t plain_store; /* reserved, must be 0 (round 1's racy load/add/store variant of the register kernel is gone) */
  int32_t kernel;      /* fast mode: 0 = warp-per-shard kernel when applicable (default; csrc/w2b_warp.cuh),
                          1 = register kernel (one CTA per shard; also serves strict mode and D > 1024) */
  int32_t slots;       /* warp kernel: shared-memory row slots per warp (0 = as many as fit, at most 16) */
  int32_t prefetch;    /* warp kernel: 0 = the positions of a shard strictly one after another, like a reference
                          thread (default); 1 = rows of position p+1 are fetched before p's
                          updates have landed (a context row shared by neighbours is read one update stale) */
  int32_t sync_mode;   /* multi-GPU exchange (w2b_sync): 0 = replicas are averaged (default); 1 = every rank's
                          updates since the last exchange are summed onto the common base (needs two more tables;
                          call w2b_nccl_init after w2b_init_tables / w2b_checkpoint_load) */
} w2b_config;

typedef struct {
  double loss;            /* sum of shard losses accumulated by this call */
  int64_t words;          /* word_count advanced (reference semantics, :399) */
  int64_t positions;      /* trained positions (cw > 0) */
  int64_t context_rows;   /* sum of cw */
  int64_t target_rows;    /* processed targets (skips excluded) */
  int64_t shards_done;    /* shards that have reached their end */
  float alpha;            /* alpha after the call */
  int64_t word_count_actual;
  float kernel_ms;        /* CUDA-event time of the training kernel(s) in this call */
  int32_t launches;       /* kernels launched by this call */
  int64_t h2d_bytes;      /* host->device bytes copied by this call (token slices, shard states) */
  int64_t d2h_bytes;      /* device->host bytes copied by this call (shard states, alpha, counter) */
} w2b_step_stats;

/* One record per loop iteration that reaches the window draw (:428). */
typedef struct {
  int32_t center, b, cw, ntargets;
  int32_t targets[64];
  float alpha; /* the learning rate the position trains with (w2b_trace: as one shard alone would see it, from the
                  configured alpha and a counter of its own; w2b_train_step_traced: the shared value the shard read) */
} w2b_trace_rec;

const char *w2b_last_error(void);
int w2b_device_count(int *n);

/* Geometry the production (warp-per-shard) kernel would run with for a configuration: pure host arithmetic (no
 * CUDA call).  warp = 0: the configuration runs the register kernel instead (D > 1024, strict mode, kernel = 1). */
typedef struct {
  int32_t warp;           /* 1 = the warp kernel applies */
  int32_t slots;          /* K: shared-memory row slots of a warp's ring (K-2 loads in flight) */
  int32_t queue_entries;  /* job queue capacity (two positions) */
  int32_t warps_per_sm;   /* resident 1-warp CTAs per SM the registers are sized for */
  int32_t sentence_in_smem; /* 1: the shard's sentence buffer (4000 B) is part of smem_bytes; 0: global scratch */
  int32_t reserved;
  int64_t smem_bytes;     /* dynamic shared memory per warp */
} w2b_warp_plan;
int w2b_warp_plan_query(const w2b_config *cfg, w2b_warp_plan *out);

/* Number of shards that keeps every SM busy for this configuration (SMs x resident warps of the production kernel);
 * the CLI's default for -threads (the reference's default of 12 is a CPU core count). */
int w2b_suggest_shards(const w2b_config *cfg, int *out);
int w2b_create(const w2b_config *cfg, w2b_ctx **out); /* globals :45-61 -> context */
int w2b_destroy(w2b_ctx *ctx);

/* The kernel instantiations a context launches: its training launches (w2b_train_step, w2b_train_epoch) and its
 * single-position hook (w2b_apply_position).  Read-only. */
typedef struct {
  int32_t warp;        /* 1: train_warp_kernel<BM, NJ, MINB, REG> trains and serves the hook */
  int32_t nj;          /* warp kernel: float4 column groups per lane */
  int32_t minb;        /* warp kernel: resident warps per SM it is compiled for */
  int32_t bm;          /* bit level compiled in (0, 1, 2), or 9 = decided at run time */
  int32_t reg;         /* the -reg instantiation */
  int32_t vec;         /* register kernel: floats per thread (4 or 1) */
  int32_t threads;     /* register kernel: threads per CTA */
  int32_t wide;        /* register kernel, training: 1 = train_shards_wide_kernel (__launch_bounds__(1024, 1)), 0 =
                          the speed-tuned train_shards_kernel */
  int32_t group;       /* register kernel, training: targets per group G (strict mode: 1 target at a time) */
  int32_t apply_wide;  /* register kernel, hook: 1 = apply_position_wide_kernel, 0 = apply_position_kernel */
  int32_t apply_bm;    /* register kernel, hook: bit level compiled in, or 9 */
  int32_t apply_group; /* register kernel, hook: targets per group */
} w2b_kernel_info;
int w2b_kernel_query(w2b_ctx *ctx, w2b_kernel_info *out);

/* vocab[].cn + train_words -> sub-sampling thresholds (:403-404) and the 1e8-entry
 * unigram table (InitUnigramTable, :112-128; boundaries on the host with the same libm
 * pow(), expanded on the device). */
int w2b_set_vocab_counts(w2b_ctx *ctx, const int64_t *cn, int64_t V, int64_t train_words);
/* The id stream + shard starts (replaces each thread's fopen/fseek/ReadWordIndex,
 * :376-377,:396).  resident=1 uploads the whole stream once; resident=0 keeps the host
 * pointer (must stay valid) and w2b_train_step copies each shard's next slice. */
int w2b_set_corpus(w2b_ctx *ctx, const int32_t *ids, int64_t n, const int64_t *shard_start,
                   const int32_t *shard_first, int resident);
/* InitNet (:343-361) by LCG jump-ahead on the device + expTable (:614-618, host expf). */
int w2b_init_tables(w2b_ctx *ctx);

/* Re-arms every shard (seed = shard id :368, cursor = shard start :377) — what the
 * per-epoch pthread_create does (:532-535). */
int w2b_epoch_begin(w2b_ctx *ctx);
/* Advances every unfinished shard by >= words_per_shard words, whole sentences only
 * (<=0: to the end of the shard).  The per-step equivalent of TrainModelThread. */
int w2b_train_step(w2b_ctx *ctx, int64_t words_per_shard, w2b_step_stats *stats);
/* epoch_begin + steps until all shards are done; *loss = "Epoch Loss" (:537-539). */
int w2b_train_epoch(w2b_ctx *ctx, double *loss, w2b_step_stats *stats);

/* Parity hooks */
int w2b_trace(w2b_ctx *ctx, int shard, int64_t max_iterations, w2b_trace_rec *out, int64_t cap,
              int64_t *n_out); /* draws only; does not touch u/v or shard state */
/* Exactly w2b_train_step, and local shard i's draw records of the step, in order, at recs[i * cap_per_shard ...];
 * n_per_shard[i] = how many it made (may exceed the cap: only the first cap_per_shard are stored). */
int w2b_train_step_traced(w2b_ctx *ctx, int64_t words_per_shard, w2b_step_stats *stats, w2b_trace_rec *recs,
                          int64_t cap_per_shard, int64_t *n_per_shard);
int w2b_strict_prefix(w2b_ctx *ctx, int shard, int64_t max_iterations, double *loss); /* strict mode: first k iterations of a shard */
int w2b_apply_position(w2b_ctx *ctx, const int32_t *context_ids, int cw, const int32_t *targets,
                       int ntargets, float *f_out); /* Appendix-A steps 5-7 for explicit ids */
int w2b_get_state(w2b_ctx *ctx, float *alpha, int64_t *word_count_actual);
int w2b_set_state(w2b_ctx *ctx, float alpha, int64_t word_count_actual);
int w2b_download_raw(w2b_ctx *ctx, float *u, float *v);   /* fp32 master tables */
int w2b_upload_raw(w2b_ctx *ctx, const float *u, const float *v);
int w2b_download_table(w2b_ctx *ctx, int32_t *table);    /* 1e8 entries */
int w2b_download_exptable(w2b_ctx *ctx, float *t);       /* 1000 entries */

/* Resumable checkpoint (SURVEY section 8(f).4; -save-every-epoch only keeps the non-resumable quantized
 * sum, :540-557): fp32 master tables + learning rate + global word counter + epochs done. */
int w2b_checkpoint_save(w2b_ctx *ctx, const char *path, int64_t epochs_done);
int w2b_checkpoint_load(w2b_ctx *ctx, const char *path, int64_t *epochs_done);

/* quantize(u+v) (:568-569), V*D floats into host memory. */
int w2b_export(w2b_ctx *ctx, float *out);
/* quantize() itself on the device, for known-answer tests (:73-108). */
int w2b_quantize(w2b_ctx *ctx, const float *in, float *out, int64_t n, int bitlevel);

/* Analogy evaluator (SURVEY section 8(f).2), replaces src/compute-accuracy.c:63-189: same inputs
 * (word2vec-binary vector file, optional re-quantisation, vocabulary threshold, question stream),
 * same report text; all questions are scored on the GPU: one Q x V x D TF32 tensor-core contraction
 * (wgmma + TMA) as a filter with a proven error bound, then an fp32 re-score of the surviving candidates in the
 * reference's operation order, so the arg-max (ties included) is the reference's.  questions_file NULL = stdin.  report may be NULL. */
typedef struct {
  int64_t questions_total, questions_seen, correct;
  int64_t semantic_correct, semantic_seen, syntactic_correct, syntactic_seen;
  int64_t vocab, size;
  float gpu_ms; /* normalise + query build + scoring kernels, CUDA events */
  int64_t candidates; /* (question, word) pairs the tensor-core filter let through (within 2 eps of the running best) */
  int64_t rescored;   /* ... of which still within 2 eps of the final best: scored again in fp32, reference order */
} w2b_accuracy;
int w2b_compute_accuracy(const char *vectors_file, int bitlevel, int64_t threshold, const char *questions_file,
                         int device, w2b_accuracy *acc, char *report, int64_t report_cap);
/* The same evaluation, per question: answers[i] = index of the word chosen for the i-th question of the file (every
 * question line counts, in file order), -1 when the question is skipped (a word is not in the vocabulary) or no word
 * scores above 0.  At most answers_cap are written; *n_questions = the number of questions. */
int w2b_analogy_answers(const char *vectors_file, int bitlevel, int64_t threshold, const char *questions_file,
                        int device, int32_t *answers, int64_t answers_cap, int64_t *n_questions);
/* Test hook of the tensor-core filter: approx[q*words + c] = its TF32 score of Q row q against M row c (both used as
 * given, D floats per row), eps[q] = the error bound it uses for question q (eps may be NULL). */
int w2b_eval_filter_scores(const float *Q, int64_t nq, const float *M, int64_t words, int64_t D, int device,
                           float *approx, float *eps);

/* The evaluator on a packed vector file (w2b_write_packed / -binary 2): same questions, same report text and the
 * same chosen word per question as src/compute-accuracy.c gives on the unpacked file (w2b_read_packed ->
 * w2b_write_vectors(binary=1)) with <bitlevel> = the file's bit level.  The table stays packed on the device: scores
 * are exact integer dot products of bit planes (xor / popc), combined per question into a filter whose error bound
 * covers fp32 rounding only, then the same fp32 re-score.  acc->candidates and acc->rescored count what they count
 * above; acc->gpu_ms covers the plane, Gram, filter and re-score kernels. */
int w2b_compute_accuracy_packed(const char *packed_file, int64_t threshold, const char *questions_file,
                                int device, w2b_accuracy *acc, char *report, int64_t report_cap);
int w2b_analogy_answers_packed(const char *packed_file, int64_t threshold, const char *questions_file,
                               int device, int32_t *answers, int64_t answers_cap, int64_t *n_questions);
/* Test hook: rows = V packed rows as in the file (ceil(D*bitlevel/8) bytes each, no names); for query word ids
 * qid[0..W) gram[w*V + c] = the exact integer dot product of rows qid[w] and c in level units (1 bit: units of
 * 1/9, 2 bits: 1/16); for questions q3[0..3*nq) (indices into qid) approx[q*V + c] = the filter's score and
 * eps[q] the bound it uses on |approx - the reference's fp32 score|.  approx / eps may be NULL. */
int w2b_eval_packed_scores(const uint8_t *rows, int64_t V, int64_t D, int bitlevel, const int32_t *qid, int64_t W,
                           const int32_t *q3, int64_t nq, int device, int32_t *gram, float *approx, float *eps);

/* Top-k lists: the reference's top-N list (src/compute-accuracy.c:166-175) at N = k, for analogy questions and for
 * nearest neighbours.  A query is a question (b1, b2, b3), or a word w taken as the question (w, w, w), whose vec is
 * M[w] exactly and which skips only w.  Its list holds the k largest fp32 scores > 0 (each product rounded, then
 * added in index order, as the reference's build scores) of the words not in the query, in descending order, the
 * smaller index first on equal scores; ids[i*k + j] = the word of rank j + 1 of the i-th query (-1 past the end of
 * the list), scores[i*k + j] its score (0 with id -1).  A query with a word not in the vocabulary (only the first
 * threshold words are searched, upper-cased, first match) gets an all -1 row.  1 <= k <= W2B_MAX_TOPK.
 * Either file kind: a packed file (three integers on its first line) is scored in the bit domain, and bitlevel must
 * then be 0 or the file's level.  The scores pass a TF32 or bit-domain filter that keeps every word within 2 eps of
 * the query's running k-th best, then the survivors are scored exactly; a candidate list that overflows, and
 * W2B_EVAL_SIMT=1, score every word exactly on the SIMT cores instead.  Queries run in batches that keep the
 * candidate lists within 2 GB of device memory.  At most cap_queries rows are written; *n_queries = the number of
 * queries; st (may be NULL) reports the run.  cap_queries = 0 only counts the queries (ids and scores may then be
 * NULL; the vector file is not read). */
#define W2B_MAX_TOPK 1024
typedef struct {
  float gpu_ms;              /* all kernels of the call, CUDA events (uploads of the table and the queries excluded) */
  int64_t queries, skipped;  /* queries in the input; of which with a word not in the vocabulary */
  int64_t chunks;            /* vocabulary chunks the filter ran over */
  int64_t candidates;        /* (query, word) pairs the filter let through */
  int64_t rescored;          /* ... of which within 2 eps of the final k-th best: scored exactly */
  int32_t simt;              /* 1: the exact SIMT fall-back produced the lists (overflow or W2B_EVAL_SIMT=1) */
  int32_t packed;            /* 1: the file was a packed (-binary 2) file, scored in the bit domain */
} w2b_topk_stats;
/* top-k lists of every question of questions_file (file order, as w2b_analogy_answers counts them; NULL = stdin) */
int w2b_analogy_topk(const char *vectors_file, int bitlevel, int64_t threshold, const char *questions_file, int k,
                     int device, int32_t *ids, float *scores, int64_t cap_queries, int64_t *n_queries,
                     w2b_topk_stats *st);
/* nearest neighbours of every whitespace-separated word of words_file (NULL = stdin) */
int w2b_nearest(const char *vectors_file, int bitlevel, int64_t threshold, const char *words_file, int k,
                int device, int32_t *ids, float *scores, int64_t cap_queries, int64_t *n_queries,
                w2b_topk_stats *st);

/* The evaluator on a context's own tables: the vectors are quantize(u+v) as w2b_export computes them (the file
 * -binary 1 would write), with words[i] the name of row i (ctx's vocab_size names, the order of the rows).  Same
 * arguments, report text, answers, lists and statistics as the file-based calls on that file; nothing is copied to the
 * host and u, v, alpha, the word counter and the shard states are left untouched.
 * A name is read as the file's reader reads it (at most 50 characters, upper-cased); a name holding ' ' or '\n' cannot
 * survive the file and is W2B_EINVAL, as are a NULL ctx or words and a k outside 1..W2B_MAX_TOPK.  W2B_ESTATE before
 * w2b_init_tables / w2b_checkpoint_load.  The call runs on the context's device: it first waits for the context's
 * stream, and returns with nothing left running and every temporary device buffer freed (a failed allocation is
 * W2B_ECUDA; the context stays usable).  A 1-bit or 2-bit context evaluated with bitlevel 0 or its own level is scored
 * in the bit domain (st->packed = 1, as for its packed file), without an fp32 table; every other case forms the fp32
 * table on the device.  gpu_ms includes the kernel that builds the table or the bit planes from u and v. */
int w2b_ctx_compute_accuracy(w2b_ctx *ctx, const char *const *words, int bitlevel, int64_t threshold,
                             const char *questions_file, w2b_accuracy *acc, char *report, int64_t report_cap);
int w2b_ctx_analogy_answers(w2b_ctx *ctx, const char *const *words, int bitlevel, int64_t threshold,
                            const char *questions_file, int32_t *answers, int64_t answers_cap, int64_t *n_questions);
int w2b_ctx_analogy_topk(w2b_ctx *ctx, const char *const *words, int bitlevel, int64_t threshold,
                         const char *questions_file, int k, int32_t *ids, float *scores, int64_t cap_queries,
                         int64_t *n_queries, w2b_topk_stats *st);
int w2b_ctx_nearest(w2b_ctx *ctx, const char *const *words, int bitlevel, int64_t threshold, const char *words_file,
                    int k, int32_t *ids, float *scores, int64_t cap_queries, int64_t *n_queries, w2b_topk_stats *st);

/* Multi-GPU replica averaging (SURVEY §8(e)); G=1 contexts never touch NCCL. */
int w2b_device_ptrs(w2b_ctx *ctx, void **u, void **v, int64_t *elems);
int w2b_nccl_unique_id(void *id128);                                    /* ncclGetUniqueId */
int w2b_nccl_init(w2b_ctx *ctx, const void *id128, int rank, int nranks); /* ncclCommInitRank */
int w2b_sync(w2b_ctx *ctx); /* all-reduce-average u, v; exact global word_count_actual — one NCCL group, no host round trip */
int w2b_sync_timed(w2b_ctx *ctx, float *ms); /* same; *ms = device time of the exchange (CUDA events) */
/* Fingerprints of u and v (sum of the 32-bit patterns mod 2^64): equal on every rank right after w2b_sync. */
int w2b_table_checksum(w2b_ctx *ctx, uint64_t *u_sum, uint64_t *v_sum);
int w2b_scale_tables(w2b_ctx *ctx, float s); /* u*=s, v*=s (for host-driven all-reduce) */

#ifdef __cplusplus
}
#endif
#endif

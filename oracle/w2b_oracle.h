/* TEST INFRASTRUCTURE — CPU restatement ("oracle") of the Word2Bits training path.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load this library.  The product (libw2b.so + the word2bits_b200 CLI)
 * never links, loads or calls it.
 *
 * Every function cites the reference lines it restates (file = src/word2bits.cpp of
 * agnusmaximus/Word2Bits @ d029cca).  Arithmetic is sequential IEEE float32: this
 * file is compiled with -O2 -ffp-contract=off -fno-tree-vectorize so that it is
 * bit-comparable with oracle/_ref/libw2b_ref_strict.so (tests/test_oracle_vs_ref.py
 * pins it there; tests/golden/ holds vectors generated from the reference itself).
 */
#ifndef W2B_ORACLE_H
#define W2B_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define W2BO_TABLE_SIZE 100000000 /* :60 */
#define W2BO_MAX_SENTENCE 1000    /* :32 */
#define W2BO_EXP_TABLE 1000       /* :30 */

/* ---- scalar pieces -------------------------------------------------------------- */
float w2bo_quantize(float x, int bitlevel);           /* :73-108 */
void w2bo_quantize_n(const float *x, float *out, int64_t n, int bitlevel); /* w2bo_quantize per element */
float w2bo_sigmoid(float x);                          /* :67-71  */
uint64_t w2bo_lcg(uint64_t r);                        /* :352 et al. */
void w2bo_exptable(float *out /*1000*/);              /* :614-618 */
void w2bo_init_net(int64_t V, int64_t D, float *u, float *v);           /* :343-361 */
void w2bo_unigram_table(const int64_t *cn, int64_t V, int32_t *table);  /* :112-128, 1e8 entries */
/* Boundary form: start[i] = first slot owned by word i, start[V] = 1e8 (SURVEY App. A). */
void w2bo_unigram_bounds(const int64_t *cn, int64_t V, int64_t *start /*V+1*/);

/* ---- corpus + vocabulary (host glue; :131-301) ----------------------------------- */
typedef struct w2bo_corpus w2bo_corpus;
w2bo_corpus *w2bo_corpus_load(const char *path, int min_count);
void w2bo_corpus_free(w2bo_corpus *c);
int64_t w2bo_vocab_size(const w2bo_corpus *c);
int64_t w2bo_train_words(const w2bo_corpus *c);
int64_t w2bo_file_size(const w2bo_corpus *c);
const char *w2bo_word(const w2bo_corpus *c, int64_t i);
const int64_t *w2bo_counts(const w2bo_corpus *c);
int64_t w2bo_num_tokens(const w2bo_corpus *c);    /* in-vocab tokens incl. </s>, file order */
const int32_t *w2bo_tokens(const w2bo_corpus *c);
/* Shard `id` of `n`: the reference seeks to byte file_size/n*id (:377) and may land
 * mid-word.  *first = id of the (possibly fragment) first token or -1 if it is OOV /
 * absent; *start = index in tokens[] of the next regular token. */
void w2bo_shard_start(const w2bo_corpus *c, int id, int n, int64_t *start, int32_t *first);

/* ---- model + training (:363-516) -------------------------------------------------- */
typedef struct {
  int64_t V, D;
  int window, negative, bitlevel;
  float sample, reg, starting_alpha;
  int64_t iter, train_words;
  int num_shards;
  float *u, *v;            /* caller-owned, V*D each */
  const int32_t *table;    /* 1e8 entries */
  const int64_t *cn;       /* V counts */
  float alpha;             /* shared, mutated (:391) */
  int64_t word_count_actual; /* shared, mutated (:380,:415) */
} w2bo_model;

/* One record per loop iteration that reaches the window draw (:428), i.e. including the
 * "empty sentence" iterations (center = -1, cw = 0). */
typedef struct {
  int32_t center, b, cw, ntargets;
  int32_t targets[64]; /* processed targets in order, d=0 first (skips removed) */
  float alpha;
} w2bo_trace_rec;

typedef struct {
  w2bo_trace_rec *rec;
  int64_t cap, n;
} w2bo_trace;

/* Runs shard `id` to completion (or until max_positions window draws, <0 = no limit).
 * Returns the shard's total loss (the value stored in thread_losses[id], :511). */
double w2bo_train_shard(w2bo_model *m, const w2bo_corpus *c, int id, int64_t max_positions,
                        w2bo_trace *trace);
/* All shards concurrently on pthreads (Hogwild, :535-536); returns the epoch loss. */
double w2bo_train_epoch_threads(w2bo_model *m, const w2bo_corpus *c);

/* One position applied in place given explicit ids (used by the L1 single-step test).
 * Follows Appendix A steps 5-7; returns f of each processed target in f_out. */
void w2bo_apply_position(w2bo_model *m, const float *exptab, const int32_t *ctx, int cw,
                         const int32_t *targets, int ntargets, float *f_out, double *loss);

/* quantize(u+v) (:568-569) */
void w2bo_export(const w2bo_model *m, float *out);
/* Writes the vector file (:560-576). */
int w2bo_write_vectors(const w2bo_model *m, const w2bo_corpus *c, const char *path, int binary);

/* ---- analogy evaluator (src/compute-accuracy.c, fp32 operation order of its -O3 x86-64-v3 build) ---------- */
#define W2BO_AN_FUSED 1     /* negative control: fused multiply-add scoring */
#define W2BO_AN_LANE_NORM 2 /* negative control: 32 lane-strided fused partial sums + butterfly for |row| */
/* quantize + L2-normalise words rows of D in place (:106-110). */
void w2bo_analogy_normalize(float *M, int64_t words, int64_t D, int bitlevel, int flags);
/* The whole program on a vector file and a question file: its report text (stdout) into report, and per question
 * in file order the chosen word index, or -1 when the question is skipped or no word scores above 0.  flags = 0 is
 * the reference; nthreads threads share the questions.  Returns 0, or non-zero if a file cannot be read. */
int w2bo_analogy(const char *vectors_file, int bitlevel, int64_t threshold, const char *questions_file, int flags,
                 int nthreads, char *report, int64_t report_cap, int32_t *answers, int64_t answers_cap,
                 int64_t *n_questions);

#ifdef __cplusplus
}
#endif
#endif

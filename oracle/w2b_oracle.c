/* TEST INFRASTRUCTURE — see w2b_oracle.h.  CPU restatement of the reference's training
 * path in sequential float32 (build: -O2 -ffp-contract=off -fno-tree-vectorize).
 * Citations are to src/word2bits.cpp of the reference.  Parity of this file with the
 * reference itself is pinned by tests/test_oracle_vs_ref.py (bit-exact against the
 * strict-fp build of the unmodified source) and by tests/golden/.
 */
#define _GNU_SOURCE
#include "w2b_oracle.h"

#include <math.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* ================================================================== scalar pieces */

/* :73-108.  b==3 (and any b<0) matches no branch and yields sign*0. */
float w2bo_quantize(float x, int b) {
  if (b == 0) return x;
  float sgn = (x < 0) ? -1.0f : 1.0f; /* -0.0 and NaN take +1 (:82) */
  float mag = x * sgn;
  if (b == 1) return sgn / 3;
  float level = 0;
  if (b == 2) level = (mag >= 0 && mag <= .5) ? .25f : .75f;
  if (b >= 4) {
    int seg = (int)pow(2, b - 1);
    int k = (int)((mag * seg) + (float).5);
    if (k > seg) k = seg;
    level = k / (float)seg;
  }
  return sgn * level;
}

void w2bo_quantize_n(const float *x, float *out, int64_t n, int b) {
  for (int64_t i = 0; i < n; i++) out[i] = w2bo_quantize(x[i], b);
}

/* :67-71 */
float w2bo_sigmoid(float x) {
  if (x > 6) return 1;
  if (x < -6) return 1e-9;
  return 1 / (1 + expf(-x));
}

uint64_t w2bo_lcg(uint64_t r) { return r * 25214903917ULL + 11ULL; }

/* :614-618 — float expf, the table value is e/(e+1). */
void w2bo_exptable(float *out) {
  for (int i = 0; i < W2BO_EXP_TABLE; i++) {
    float e = expf((i / (float)W2BO_EXP_TABLE * 2 - 1) * 6);
    out[i] = e / (e + 1);
  }
}

/* :343-361 — one LCG stream from 1, v first, then u. */
void w2bo_init_net(int64_t V, int64_t D, float *u, float *v) {
  uint64_t r = 1;
  for (int64_t i = 0; i < V * D; i++) {
    r = w2bo_lcg(r);
    v[i] = ((r & 0xFFFF) / (float)65536) - 0.5;
  }
  for (int64_t i = 0; i < V * D; i++) {
    r = w2bo_lcg(r);
    u[i] = ((r & 0xFFFF) / (float)65536) - 0.5;
  }
}

/* :112-128 — the slot is assigned BEFORE the advance test; i is clamped to V-1. */
void w2bo_unigram_table(const int64_t *cn, int64_t V, int32_t *table) {
  double total = 0;
  for (int64_t a = 0; a < V; a++) total += pow((double)cn[a], 0.75);
  int64_t i = 0;
  double d1 = pow((double)cn[0], 0.75) / total;
  for (int64_t a = 0; a < W2BO_TABLE_SIZE; a++) {
    table[a] = (int32_t)i;
    if (a / (double)W2BO_TABLE_SIZE > d1) {
      i++;
      /* the reference reads vocab[V] here when i==V (one past the end, realloc'd
       * to V+1 entries at :236); the value is irrelevant because i is clamped next. */
      if (i < V) d1 += pow((double)cn[i], 0.75) / total;
    }
    if (i >= V) i = V - 1;
  }
}

void w2bo_unigram_bounds(const int64_t *cn, int64_t V, int64_t *start) {
  double total = 0;
  for (int64_t a = 0; a < V; a++) total += pow((double)cn[a], 0.75);
  double d1 = pow((double)cn[0], 0.75) / total;
  int64_t a = 0;
  start[0] = 0;
  for (int64_t i = 0; i + 1 < V; i++) {
    /* smallest a >= start[i] with a/1e8 > d1 */
    while (a < W2BO_TABLE_SIZE && !(a / (double)W2BO_TABLE_SIZE > d1)) a++;
    if (a >= W2BO_TABLE_SIZE) { /* table exhausted: remaining words own nothing */
      for (int64_t j = i + 1; j <= V; j++) start[j] = W2BO_TABLE_SIZE;
      return;
    }
    a++;
    start[i + 1] = a;
    d1 += pow((double)cn[i + 1], 0.75) / total;
  }
  start[V] = W2BO_TABLE_SIZE;
}

/* ======================================================= corpus + vocabulary (host) */

struct w2bo_corpus {
  int64_t vocab_size, train_words, file_size;
  char **words;
  int64_t *cn;
  int64_t n_tokens;
  int32_t *ids;
  int64_t *begin; /* byte offset where each in-vocab token starts */
  uint8_t *buf;   /* raw file bytes (kept for shard-start resolution) */
  /* string -> final id map */
  int64_t map_cap;
  int64_t *map_slot; /* index into pool entries, -1 empty */
  char **pool_word;
  int64_t *pool_final; /* final id or -1 */
  int64_t pool_n;
};

#define MAXW 4096 /* MAX_STRING :29 */

/* ReadWord (:131-155) over a memory image.  Returns 0 at EOF (a partially read
 * word is discarded by both callers, :279/:180), else 1 with the token in `word`. */
static int read_token(const uint8_t *buf, int64_t n, int64_t *pos, char *word, int64_t *begin) {
  int a = 0;
  for (;;) {
    if (*pos >= n) return 0;
    int ch = buf[(*pos)++];
    if (ch == 13) continue;
    if (ch == ' ' || ch == '\t' || ch == '\n') {
      if (a > 0) {
        if (ch == '\n') (*pos)--;
        break;
      }
      if (ch == '\n') {
        strcpy(word, "</s>");
        *begin = *pos - 1;
        return 1;
      }
      continue;
    }
    if (a == 0) *begin = *pos - 1;
    word[a++] = (char)ch;
    if (a >= MAXW - 1) a--;
  }
  word[a] = 0;
  return 1;
}

static uint64_t fnv(const char *s) {
  uint64_t h = 1469598103934665603ULL;
  for (; *s; s++) h = (h ^ (uint8_t)*s) * 1099511628211ULL;
  return h;
}

static int64_t map_find(const w2bo_corpus *c, const char *w) {
  uint64_t h = fnv(w) & (uint64_t)(c->map_cap - 1);
  for (;;) {
    int64_t s = c->map_slot[h];
    if (s < 0) return -1;
    if (!strcmp(c->pool_word[s], w)) return s;
    h = (h + 1) & (uint64_t)(c->map_cap - 1);
  }
}

static void map_grow(w2bo_corpus *c) {
  int64_t ncap = c->map_cap * 2;
  int64_t *ns = (int64_t *)malloc(sizeof(int64_t) * ncap);
  for (int64_t i = 0; i < ncap; i++) ns[i] = -1;
  for (int64_t e = 0; e < c->pool_n; e++) {
    uint64_t h = fnv(c->pool_word[e]) & (uint64_t)(ncap - 1);
    while (ns[h] >= 0) h = (h + 1) & (uint64_t)(ncap - 1);
    ns[h] = e;
  }
  free(c->map_slot);
  c->map_slot = ns;
  c->map_cap = ncap;
}

static int64_t map_insert(w2bo_corpus *c, const char *w, int64_t *pool_cap, int64_t **count) {
  if ((c->pool_n + 1) * 2 > c->map_cap) map_grow(c);
  if (c->pool_n == *pool_cap) {
    *pool_cap *= 2;
    c->pool_word = (char **)realloc(c->pool_word, sizeof(char *) * *pool_cap);
    *count = (int64_t *)realloc(*count, sizeof(int64_t) * *pool_cap);
  }
  int64_t e = c->pool_n++;
  c->pool_word[e] = strdup(w);
  (*count)[e] = 0;
  uint64_t h = fnv(w) & (uint64_t)(c->map_cap - 1);
  while (c->map_slot[h] >= 0) h = (h + 1) & (uint64_t)(c->map_cap - 1);
  c->map_slot[h] = e;
  return e;
}

/* stable merge sort of entry indices by count descending (glibc qsort + VocabCompare
 * :207-219 keeps ties in first-appearance order on this libc; asserted in tests). */
static void msort(int64_t *idx, int64_t *tmp, int64_t n, const int64_t *count) {
  if (n < 2) return;
  int64_t h = n / 2;
  msort(idx, tmp, h, count);
  msort(idx + h, tmp, n - h, count);
  int64_t i = 0, j = h, k = 0;
  while (i < h && j < n) tmp[k++] = (count[idx[j]] > count[idx[i]]) ? idx[j++] : idx[i++];
  while (i < h) tmp[k++] = idx[i++];
  while (j < n) tmp[k++] = idx[j++];
  memcpy(idx, tmp, sizeof(int64_t) * n);
}

w2bo_corpus *w2bo_corpus_load(const char *path, int min_count) {
  FILE *f = fopen(path, "rb");
  if (!f) return NULL;
  fseek(f, 0, SEEK_END);
  int64_t n = ftell(f);
  fseek(f, 0, SEEK_SET);
  w2bo_corpus *c = (w2bo_corpus *)calloc(1, sizeof(*c));
  c->buf = (uint8_t *)malloc(n > 0 ? n : 1);
  if (fread(c->buf, 1, n, f) != (size_t)n) { fclose(f); free(c->buf); free(c); return NULL; }
  fclose(f);
  c->file_size = n; /* :299 ftell at EOF */

  /* pass 1 (:265-293): count words in first-appearance order, </s> first (:276) */
  c->map_cap = 1 << 16;
  c->map_slot = (int64_t *)malloc(sizeof(int64_t) * c->map_cap);
  for (int64_t i = 0; i < c->map_cap; i++) c->map_slot[i] = -1;
  int64_t pool_cap = 1 << 12;
  c->pool_word = (char **)malloc(sizeof(char *) * pool_cap);
  int64_t *count = (int64_t *)malloc(sizeof(int64_t) * pool_cap);
  map_insert(c, "</s>", &pool_cap, &count);
  char word[MAXW];
  int64_t pos = 0, beg = 0;
  while (read_token(c->buf, n, &pos, word, &beg)) {
    int64_t e = map_find(c, word);
    if (e < 0) e = map_insert(c, word, &pool_cap, &count);
    count[e]++;
  }
  /* SortVocab (:215-242): entry 0 stays, the rest sorted by count desc, then
   * entries below min_count are dropped (a suffix, because of the sort). */
  int64_t m = c->pool_n;
  int64_t *idx = (int64_t *)malloc(sizeof(int64_t) * m);
  int64_t *tmp = (int64_t *)malloc(sizeof(int64_t) * m);
  for (int64_t i = 0; i < m; i++) idx[i] = i;
  msort(idx + 1, tmp, m - 1, count);
  c->pool_final = (int64_t *)malloc(sizeof(int64_t) * m);
  c->words = (char **)malloc(sizeof(char *) * m);
  c->cn = (int64_t *)malloc(sizeof(int64_t) * (m + 1));
  int64_t V = 0, tw = 0;
  for (int64_t k = 0; k < m; k++) {
    int64_t e = idx[k];
    if (count[e] < min_count && k != 0) {
      c->pool_final[e] = -1;
    } else {
      c->pool_final[e] = V;
      c->words[V] = c->pool_word[e];
      c->cn[V] = count[e];
      tw += count[e];
      V++;
    }
  }
  c->vocab_size = V;
  c->train_words = tw;
  free(idx);
  free(tmp);
  free(count);

  /* pass 2: the in-vocab token stream with byte offsets */
  int64_t cap = 1 << 16;
  c->ids = (int32_t *)malloc(sizeof(int32_t) * cap);
  c->begin = (int64_t *)malloc(sizeof(int64_t) * cap);
  pos = 0;
  while (read_token(c->buf, n, &pos, word, &beg)) {
    int64_t e = map_find(c, word);
    int64_t id = e < 0 ? -1 : c->pool_final[e];
    if (id < 0) continue;
    if (c->n_tokens == cap) {
      cap *= 2;
      c->ids = (int32_t *)realloc(c->ids, sizeof(int32_t) * cap);
      c->begin = (int64_t *)realloc(c->begin, sizeof(int64_t) * cap);
    }
    c->ids[c->n_tokens] = (int32_t)id;
    c->begin[c->n_tokens] = beg;
    c->n_tokens++;
  }
  return c;
}

void w2bo_corpus_free(w2bo_corpus *c) {
  if (!c) return;
  for (int64_t i = 0; i < c->pool_n; i++) free(c->pool_word[i]);
  free(c->pool_word); free(c->pool_final); free(c->map_slot);
  free(c->words); free(c->cn); free(c->ids); free(c->begin); free(c->buf);
  free(c);
}

int64_t w2bo_vocab_size(const w2bo_corpus *c) { return c->vocab_size; }
int64_t w2bo_train_words(const w2bo_corpus *c) { return c->train_words; }
int64_t w2bo_file_size(const w2bo_corpus *c) { return c->file_size; }
const char *w2bo_word(const w2bo_corpus *c, int64_t i) { return c->words[i]; }
const int64_t *w2bo_counts(const w2bo_corpus *c) { return c->cn; }
int64_t w2bo_num_tokens(const w2bo_corpus *c) { return c->n_tokens; }
const int32_t *w2bo_tokens(const w2bo_corpus *c) { return c->ids; }

/* :377 fseek(file_size / num_threads * id) followed by the first ReadWordIndex (:396). */
void w2bo_shard_start(const w2bo_corpus *c, int id, int n, int64_t *start, int32_t *first) {
  int64_t off = c->file_size / (int64_t)n * (int64_t)id;
  char word[MAXW];
  int64_t pos = off, beg = 0;
  *first = -1;
  if (!read_token(c->buf, c->file_size, &pos, word, &beg)) {
    *start = c->n_tokens;
    return;
  }
  int64_t e = map_find(c, word);
  if (e >= 0 && c->pool_final[e] >= 0) *first = (int32_t)c->pool_final[e];
  /* first regular token that begins at or after where the reader now stands */
  int64_t lo = 0, hi = c->n_tokens;
  while (lo < hi) {
    int64_t mid = (lo + hi) / 2;
    if (c->begin[mid] >= pos) hi = mid; else lo = mid + 1;
  }
  *start = lo;
}

/* ============================================================ training (:363-516) */

typedef struct {
  const w2bo_corpus *c;
  int64_t cur;
  int32_t first;
} tokstream;

static int next_id(tokstream *s, int32_t *out) {
  if (s->first >= 0) { *out = s->first; s->first = -1; return 1; }
  if (s->cur >= s->c->n_tokens) return 0;
  *out = s->c->ids[s->cur++];
  return 1;
}

/* Steps 5-7 of SURVEY Appendix A for one position; shared by the shard loop and the
 * single-step entry.  Returns through *loss the reported-loss contributions. */
static void apply_position(w2bo_model *m, const float *exptab, const int32_t *ctx, int cw,
                           const int32_t *targets, int ntargets, int first_is_positive,
                           float *avg, float *err, float *f_out, double *loss) {
  const int64_t D = m->D;
  const int b = m->bitlevel;
  for (int64_t c = 0; c < D; c++) avg[c] = 0;
  for (int64_t c = 0; c < D; c++) err[c] = 0;
  for (int k = 0; k < cw; k++) { /* :431-447 */
    const float *row = m->u + (int64_t)ctx[k] * D;
    float rl = 0;
    for (int64_t c = 0; c < D; c++) {
      float q = w2bo_quantize(row[c], b);
      avg[c] += q;
      rl += q * q;
    }
    rl = m->reg * rl;
    *loss += -rl;
  }
  if (!cw) return;
  for (int64_t c = 0; c < D; c++) avg[c] /= cw; /* :449 true division by (float)cw */
  for (int t = 0; t < ntargets; t++) {          /* :450-492 */
    int64_t label = (t == 0 && first_is_positive) ? 1 : 0;
    float *row = m->v + (int64_t)targets[t] * D;
    float f = 0, rl = 0;
    for (int64_t c = 0; c < D; c++) {
      float q = w2bo_quantize(row[c], b);
      f += avg[c] * q;
      rl += q * q;
    }
    rl = m->reg * rl;
    float g;
    if (f > 6) g = (label - 1) * m->alpha;
    else if (f < -6) g = (label - 0) * m->alpha;
    else g = (label - exptab[(int)((f + 6) * (W2BO_EXP_TABLE / 6 / 2))]) * m->alpha;
    float dp = (float)(f * pow(-1, 1 - label)); /* :480 */
    float ll = logf(w2bo_sigmoid(dp));           /* :481 */
    *loss += ll - rl;
    if (f_out) f_out[t] = f;
    for (int64_t c = 0; c < D; c++) err[c] += g * w2bo_quantize(row[c], b);            /* :487 old v */
    for (int64_t c = 0; c < D; c++) row[c] += g * avg[c] - 2 * m->alpha * m->reg * row[c]; /* :490 */
  }
  for (int k = 0; k < cw; k++) { /* :494-503, duplicates applied twice */
    float *row = m->u + (int64_t)ctx[k] * D;
    for (int64_t c = 0; c < D; c++) row[c] += err[c] - 2 * m->alpha * m->reg * row[c];
  }
}

void w2bo_apply_position(w2bo_model *m, const float *exptab, const int32_t *ctx, int cw,
                         const int32_t *targets, int ntargets, float *f_out, double *loss) {
  float *avg = (float *)malloc(sizeof(float) * m->D);
  float *err = (float *)malloc(sizeof(float) * m->D);
  double l = 0;
  apply_position(m, exptab, ctx, cw, targets, ntargets, 1, avg, err, f_out, &l);
  if (loss) *loss = l;
  free(avg);
  free(err);
}

double w2bo_train_shard(w2bo_model *m, const w2bo_corpus *c, int id, int64_t max_positions,
                        w2bo_trace *trace) {
  float exptab[W2BO_EXP_TABLE];
  w2bo_exptable(exptab);
  const int64_t D = m->D;
  float *avg = (float *)malloc(sizeof(float) * D);
  float *err = (float *)malloc(sizeof(float) * D);
  int32_t sen[W2BO_MAX_SENTENCE + 1];
  int32_t *tg_big = NULL;
  sen[0] = -1;
  int64_t len = 0, sp = 0, wc = 0, last = 0, npos = 0;
  uint64_t r = (uint64_t)(int64_t)id; /* :368 */
  int eof = 0;
  double total = 0;
  tokstream ts = {c, 0, -1};
  w2bo_shard_start(c, id, m->num_shards, &ts.cur, &ts.first);
  const int W = m->window;
  for (;;) {
    if (wc - last > 10000) { /* :379-393 */
      m->word_count_actual += wc - last;
      last = wc;
      m->alpha = m->starting_alpha * (1 - m->word_count_actual / (float)(m->iter * m->train_words + 1));
      if (m->alpha < m->starting_alpha * 0.0001) m->alpha = m->starting_alpha * 0.0001;
    }
    if (len == 0) { /* :394-413 */
      int32_t w;
      for (;;) {
        if (!next_id(&ts, &w)) { eof = 1; break; }
        wc++;
        if (w == 0) break;
        if (m->sample > 0) {
          float ran = (sqrtf(m->cn[w] / (m->sample * m->train_words)) + 1) * (m->sample * m->train_words) / m->cn[w];
          r = w2bo_lcg(r);
          if (ran < (r & 0xFFFF) / (float)65536) continue;
        }
        sen[len++] = w;
        if (len >= W2BO_MAX_SENTENCE) break;
      }
      sp = 0;
    }
    if (eof || wc > m->train_words / m->num_shards) { /* :414-423 */
      m->word_count_actual += wc - last;
      break;
    }
    if (max_positions >= 0 && npos >= max_positions) break; /* test-only early stop */
    npos++;
    r = w2bo_lcg(r); /* :428-429 — also drawn for an empty sentence (stale sen[0]) */
    int bshrink = (int)(r % (uint64_t)W);
    int32_t ctx[W2BO_MAX_SENTENCE + 1]; /* a window never holds more than the sentence (:32), whatever -window is */
    int cw = 0;
    int32_t center = len ? sen[sp] : -1;
    for (int a = bshrink; a < W * 2 + 1 - bshrink; a++) {
      if (a == W) continue;
      int64_t q = sp - W + a;
      if (q < 0 || q >= len) continue;
      ctx[cw++] = sen[q];
    }
    int32_t tg_fixed[64], *tg = tg_fixed; /* 1 + negative targets; the reference has no upper bound on -negative */
    if (m->negative + 1 > 64) tg = tg_big ? tg_big : (tg_big = (int32_t *)malloc(sizeof(int32_t) * (size_t)(m->negative + 1)));
    int nt = 0;
    if (cw) {
      tg[nt++] = center;
      for (int d = 1; d < m->negative + 1; d++) { /* :455-459 */
        r = w2bo_lcg(r);
        int64_t t = m->table[(r >> 16) % W2BO_TABLE_SIZE];
        if (t == 0) t = (int64_t)(r % (uint64_t)(m->V - 1)) + 1;
        if (t == center) continue;
        tg[nt++] = (int32_t)t;
      }
    }
    if (trace && trace->n < trace->cap) {
      w2bo_trace_rec *rec = &trace->rec[trace->n++];
      rec->center = center; rec->b = bshrink; rec->cw = cw; rec->ntargets = nt;
      for (int k = 0; k < nt && k < 64; k++) rec->targets[k] = tg[k];
      rec->alpha = m->alpha;
    }
    apply_position(m, exptab, ctx, cw, tg, nt, 1, avg, err, NULL, &total);
    sp++;
    if (sp >= len) len = 0; /* :505-509 */
  }
  free(avg);
  free(err);
  free(tg_big);
  return total;
}

typedef struct { w2bo_model *m; const w2bo_corpus *c; int id; double loss; } thr_arg;
static void *thr_main(void *p) {
  thr_arg *a = (thr_arg *)p;
  a->loss = w2bo_train_shard(a->m, a->c, a->id, -1, NULL);
  return NULL;
}

double w2bo_train_epoch_threads(w2bo_model *m, const w2bo_corpus *c) {
  int n = m->num_shards;
  pthread_t *t = (pthread_t *)malloc(sizeof(pthread_t) * n);
  thr_arg *a = (thr_arg *)malloc(sizeof(thr_arg) * n);
  for (int i = 0; i < n; i++) { a[i].m = m; a[i].c = c; a[i].id = i; a[i].loss = 0; pthread_create(&t[i], NULL, thr_main, &a[i]); }
  double s = 0;
  for (int i = 0; i < n; i++) { pthread_join(t[i], NULL); s += a[i].loss; }
  free(t);
  free(a);
  return s;
}

/* :568-569 */
void w2bo_export(const w2bo_model *m, float *out) {
  for (int64_t i = 0; i < m->V * m->D; i++) {
    float s = m->u[i] + m->v[i];
    out[i] = w2bo_quantize(s, m->bitlevel);
  }
}

/* :560-576 */
int w2bo_write_vectors(const w2bo_model *m, const w2bo_corpus *c, const char *path, int binary) {
  FILE *fo = fopen(path, "wb");
  if (!fo) return 1;
  fprintf(fo, "%lld %lld\n", (long long)m->V, (long long)m->D);
  for (int64_t a = 0; a < m->V; a++) {
    fprintf(fo, "%s ", c->words[a]);
    for (int64_t b = 0; b < m->D; b++) {
      float s = m->u[a * m->D + b] + m->v[a * m->D + b];
      s = w2bo_quantize(s, m->bitlevel);
      if (binary) fwrite(&s, sizeof(float), 1, fo);
      else fprintf(fo, "%lf ", s);
    }
    fprintf(fo, "\n");
  }
  fclose(fo);
  return 0;
}

/* ============================================================ analogy evaluator
 * src/compute-accuracy.c of the reference, with the floating-point operations of the build the stored reports come
 * from (gcc -O3 -march=x86-64-v3, oracle/Makefile).  Its compute-accuracy quantize() is the same function as
 * w2bo_quantize() (bit level 3 gives +-0, NaN takes the + sign).  Two orders are not what the C text suggests:
 *   len += M*M (:108)   the loop is split at 4*floor(D/4): the squares before it are rounded on their own (vmulps)
 *                       and added one by one in index order (vaddss); the last D mod 4 terms are fused (vfmadd231ss);
 *   dist += vec*M (:164) a rounded product, then a rounded add (vmulss, vaddss), in index order: never fused.
 * W2BO_AN_FUSED and W2BO_AN_LANE_NORM swap in other orders; tests use them to show the pin would notice. */
#include <ctype.h>

#define AN_MAX_W 50      /* :24 */
#define AN_MAX_SIZE 2000 /* :22 */

void w2bo_analogy_normalize(float *M, int64_t words, int64_t D, int bitlevel, int flags) {
  for (int64_t b = 0; b < words; b++) {
    float *r = M + b * D;
    for (int64_t a = 0; a < D; a++) r[a] = w2bo_quantize(r[a], bitlevel); /* :106 */
    float len = 0;
    if (flags & W2BO_AN_LANE_NORM) {
      /* 32 lane-strided fused partial sums, then an xor butterfly (what the GPU normalised with before) */
      float s[32];
      for (int l = 0; l < 32; l++) {
        s[l] = 0;
        for (int64_t a = l; a < D; a += 32) s[l] = fmaf(r[a], r[a], s[l]);
      }
      for (int o = 16; o > 0; o >>= 1) {
        float t[32];
        for (int l = 0; l < 32; l++) t[l] = s[l] + s[l ^ o];
        memcpy(s, t, sizeof s);
      }
      len = s[0];
    } else {
      const int64_t D4 = D & ~(int64_t)3;
      for (int64_t a = 0; a < D4; a++) {
        const float p = r[a] * r[a];
        len = len + p;
      }
      for (int64_t a = D4; a < D; a++) len = fmaf(r[a], r[a], len);
    }
    len = sqrtf(len); /* :109, correctly rounded either way */
    for (int64_t a = 0; a < D; a++) r[a] = r[a] / len; /* :110: a zero row becomes NaN */
  }
}

typedef struct {
  const float *M;
  int64_t words, D;
  const int64_t *q; /* b1, b2, b3 per scored question */
  int32_t *best;
  int64_t nq;
  int flags, nthreads, id;
} an_job;

static void *an_worker(void *p) {
  an_job *j = (an_job *)p;
  const int64_t D = j->D;
  float *vec = (float *)malloc(sizeof(float) * (size_t)(D ? D : 1));
  for (int64_t i = j->id; i < j->nq; i += j->nthreads) {
    const int64_t b1 = j->q[3 * i], b2 = j->q[3 * i + 1], b3 = j->q[3 * i + 2];
    for (int64_t a = 0; a < D; a++) vec[a] = (j->M[a + b2 * D] - j->M[a + b1 * D]) + j->M[a + b3 * D]; /* :155 */
    float bestd = 0; /* :146 */
    int32_t bestc = -1;
    for (int64_t c = 0; c < j->words; c++) { /* :158-177 */
      if (c == b1 || c == b2 || c == b3) continue;
      const float *m = j->M + c * D;
      float dist = 0;
      if (j->flags & W2BO_AN_FUSED) {
        for (int64_t a = 0; a < D; a++) dist = fmaf(vec[a], m[a], dist);
      } else {
        for (int64_t a = 0; a < D; a++) {
          const float p = vec[a] * m[a];
          dist = dist + p;
        }
      }
      if (dist > bestd) { bestd = dist; bestc = (int32_t)c; }
    }
    j->best[i] = bestc;
  }
  free(vec);
  return NULL;
}

typedef struct { char *p; int64_t n, cap; } an_text;
static void an_printf(an_text *t, const char *fmt, ...) __attribute__((format(printf, 2, 3)));
#include <stdarg.h>
static void an_printf(an_text *t, const char *fmt, ...) {
  char line[4096];
  va_list ap;
  va_start(ap, fmt);
  int k = vsnprintf(line, sizeof line, fmt, ap);
  va_end(ap);
  if (k < 0) return;
  if (k >= (int)sizeof line) k = (int)sizeof line - 1;
  if (t->n + k + 1 > t->cap) {
    t->cap = (t->n + k + 1) * 2;
    t->p = (char *)realloc(t->p, (size_t)t->cap);
  }
  memcpy(t->p + t->n, line, (size_t)k + 1);
  t->n += k;
}

static void an_upper(char *s) {
  for (size_t a = 0; a < strlen(s); a++) s[a] = (char)toupper((unsigned char)s[a]);
}

int w2bo_analogy(const char *vectors_file, int bitlevel, int64_t threshold, const char *questions_file, int flags,
                 int nthreads, char *report, int64_t report_cap, int32_t *answers, int64_t answers_cap,
                 int64_t *n_questions) {
  FILE *f = fopen(vectors_file, "rb");
  if (!f) return 1;
  long long words = 0, size = 0;
  if (fscanf(f, "%lld", &words) != 1) { fclose(f); return 2; } /* :85-87 */
  if (threshold) if (words > threshold) words = threshold;
  if (fscanf(f, "%lld", &size) != 1 || words < 1 || size < 1) { fclose(f); return 2; }
  char *vocab = (char *)calloc((size_t)(words + 1) * AN_MAX_W, 1);
  float *M = (float *)malloc(sizeof(float) * (size_t)words * (size_t)size);
  for (long long b = 0; b < words; b++) { /* :96-105 */
    long long a = 0;
    for (;;) {
      vocab[b * AN_MAX_W + a] = (char)fgetc(f);
      if (feof(f) || vocab[b * AN_MAX_W + a] == ' ') break;
      if (a < AN_MAX_W && vocab[b * AN_MAX_W + a] != '\n') a++;
    }
    vocab[b * AN_MAX_W + a] = 0;
    for (a = 0; a < AN_MAX_W; a++) vocab[b * AN_MAX_W + a] = (char)toupper((unsigned char)vocab[b * AN_MAX_W + a]);
    if (fread(M + b * size, sizeof(float), (size_t)size, f) != (size_t)size) { fclose(f); free(vocab); free(M); return 3; }
  }
  fclose(f);
  w2bo_analogy_normalize(M, words, size, bitlevel, flags); /* :106-110 */

  /* the question loop (:113-186), run twice: first to collect the questions, then to replay the counters */
  FILE *qf = fopen(questions_file, "rb");
  if (!qf) { free(vocab); free(M); return 1; }
  typedef struct { int kind; char name[AN_MAX_SIZE]; int64_t b1, b2, b3; char st4[AN_MAX_SIZE]; int64_t qi; } ev;
  int64_t nev = 0, evcap = 64, nq = 0, qcap = 64;
  ev *evs = (ev *)malloc(sizeof(ev) * (size_t)evcap);
  int64_t *q = (int64_t *)malloc(sizeof(int64_t) * 3 * (size_t)qcap);
  char st1[AN_MAX_SIZE] = "", st2[AN_MAX_SIZE] = "", st3[AN_MAX_SIZE] = "", st4[AN_MAX_SIZE] = "";
#define AN_SCAN(s) do { if (fscanf(qf, "%1999s", s) != 1) {} } while (0)
#define AN_FIND(s, out) do { for (out = 0; out < words; out++) if (!strcmp(&vocab[out * AN_MAX_W], s)) break; } while (0)
  for (;;) {
    if (nev == evcap) { evcap *= 2; evs = (ev *)realloc(evs, sizeof(ev) * (size_t)evcap); }
    ev *e = evs + nev;
    memset(e, 0, sizeof *e);
    e->qi = -1;
    AN_SCAN(st1);
    an_upper(st1);
    if (!strcmp(st1, ":") || !strcmp(st1, "EXIT") || feof(qf)) {
      e->kind = 0;
      AN_SCAN(st1);
      e->b1 = feof(qf) ? 1 : 0; /* the stream ended: stop after the counters */
      strcpy(e->name, st1);
      nev++;
      if (e->b1) break;
      continue;
    }
    AN_SCAN(st2); an_upper(st2);
    AN_SCAN(st3); an_upper(st3);
    AN_SCAN(st4); an_upper(st4);
    e->kind = 1;
    strcpy(e->st4, st4);
    int64_t b1, b2, b3, b4;
    AN_FIND(st1, b1); AN_FIND(st2, b2); AN_FIND(st3, b3);
    e->b1 = b1; e->b2 = b2; e->b3 = b3;
    if (b1 != words && b2 != words && b3 != words) {
      AN_FIND(st4, b4);
      if (b4 != words) {
        if (nq == qcap) { qcap *= 2; q = (int64_t *)realloc(q, sizeof(int64_t) * 3 * (size_t)qcap); }
        q[3 * nq] = b1; q[3 * nq + 1] = b2; q[3 * nq + 2] = b3;
        e->qi = nq++;
      }
    }
    nev++;
  }
#undef AN_SCAN
#undef AN_FIND
  fclose(qf);

  int32_t *best = (int32_t *)malloc(sizeof(int32_t) * (size_t)(nq ? nq : 1));
  if (nthreads < 1) nthreads = 1;
  pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nthreads);
  an_job *jobs = (an_job *)malloc(sizeof(an_job) * (size_t)nthreads);
  for (int i = 0; i < nthreads; i++) {
    jobs[i] = (an_job){M, words, size, q, best, nq, flags, nthreads, i};
    pthread_create(&th[i], NULL, an_worker, &jobs[i]);
  }
  for (int i = 0; i < nthreads; i++) pthread_join(th[i], NULL);

  an_text out = {NULL, 0, 0};
  an_printf(&out, "Starting eval...\n");
  int TCN = 0, CCN = 0, TACN = 0, CACN = 0, SECN = 0, SYCN = 0, SEAC = 0, SYAC = 0, QID = 0, TQ = 0, TQS = 0;
  int64_t na = 0;
  for (int64_t i = 0; i < nev; i++) {
    const ev *e = evs + i;
    if (e->kind == 0) {
      if (TCN == 0) TCN = 1;
      if (QID != 0) {
        an_printf(&out, "ACCURACY TOP1: %.2f %%  (%d / %d)\n", CCN / (float)TCN * 100, CCN, TCN);
        an_printf(&out, "Total accuracy: %.2f %%   Semantic accuracy: %.2f %%   Syntactic accuracy: %.2f %% \n",
                  CACN / (float)TACN * 100, SEAC / (float)SECN * 100, SYAC / (float)SYCN * 100);
      }
      QID++;
      if (e->b1) break;
      an_printf(&out, "%s:\n", e->name);
      TCN = 0;
      CCN = 0;
      continue;
    }
    TQ++;
    const int32_t c = e->qi >= 0 ? best[e->qi] : -1;
    if (answers && na < answers_cap) answers[na] = c;
    na++;
    if (e->qi < 0) continue;
    TQS++;
    if (c >= 0 && !strcmp(e->st4, &vocab[(int64_t)c * AN_MAX_W])) {
      CCN++;
      CACN++;
      if (QID <= 5) SEAC++; else SYAC++;
    }
    if (QID <= 5) SECN++; else SYCN++;
    TCN++;
    TACN++;
  }
  an_printf(&out, "Questions seen / total: %d %d   %.2f %% \n", TQS, TQ, TQS / (float)TQ * 100);
  if (report && report_cap > 0) {
    strncpy(report, out.p, (size_t)report_cap - 1);
    report[report_cap - 1] = 0;
  }
  if (n_questions) *n_questions = na;
  free(out.p); free(best); free(th); free(jobs); free(evs); free(q); free(vocab); free(M);
  return 0;
}

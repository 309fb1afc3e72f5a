// libw2b host side (no CUDA): corpus reader + vocabulary, shard-start resolution,
// unigram boundaries, expTable, vector-file writer.  These replace the reference's
// host glue (src/word2bits.cpp:112-301, :560-576, :614-618) with identical results;
// the text is read once through mmap and tokenised into an int32 id stream instead of
// being re-parsed with fgetc by every thread in every epoch (:396).
#include <ctype.h>
#include <fcntl.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <memory>
#include <functional>
#include <numeric>
#include <string>
#include <thread>
#include <vector>

#include "w2b.h"
#include "w2b_internal.h"
#include "w2b_text.cuh"

void w2b_unigram_bounds(const int64_t *cn, int64_t V, int32_t *start) {
  const double N = (double)W2B_TABLE_SIZE;
  double total = 0;
  for (int64_t a = 0; a < V; ++a) total += pow((double)cn[a], 0.75);
  double d1 = pow((double)cn[0], 0.75) / total;  // cumulative share of words 0..i
  int64_t a = 0;                                  // next table slot to examine
  start[0] = 0;
  int64_t i = 0;
  for (; i + 1 < V; ++i) {
    // The reference assigns slot a to word i and only then tests a/1e8 > d1 (:121-125):
    // word i keeps every slot up to and including the first one that passes the test.
    // Jump close with the closed form, then settle with the reference's own comparison.
    const int64_t guess = (int64_t)(d1 * N) - 2;  // the test is monotone in a
    if (guess > a) a = guess;
    while (a < W2B_TABLE_SIZE && !((double)a / N > d1)) ++a;
    if (a >= W2B_TABLE_SIZE) break;
    ++a;
    start[i + 1] = (int32_t)a;
    d1 += pow((double)cn[i + 1], 0.75) / total;
  }
  for (int64_t j = i + 1; j <= V; ++j) start[j] = W2B_TABLE_SIZE;
}

void w2b_exptable(float *out) {
  for (int i = 0; i < 1000; ++i) {
    float e = expf((i / (float)1000 * 2 - 1) * 6);
    out[i] = e / (e + 1);
  }
}

// Sub-sampling threshold `ran` of every word (:403-404), float32 throughout as in the reference:
// (sqrt(cn / (sample*train_words)) + 1) * (sample*train_words) / cn.
void w2b_keep_thresholds(const int64_t *cn, int64_t V, int64_t train_words, float sample, float *out) {
  const float S = sample * (float)train_words;
  for (int64_t w = 0; w < V; ++w) out[w] = (sqrtf((float)cn[w] / S) + 1.f) * S / (float)cn[w];
}

extern "C" int w2b_host_unigram_bounds(const int64_t *cn, int64_t V, int32_t *start) {
  if (!cn || !start || V < 1) { w2b_set_error("w2b_host_unigram_bounds: bad argument"); return W2B_EINVAL; }
  w2b_unigram_bounds(cn, V, start);
  return W2B_OK;
}
extern "C" int w2b_host_exptable(float *out) {
  if (!out) { w2b_set_error("w2b_host_exptable: null argument"); return W2B_EINVAL; }
  w2b_exptable(out);
  return W2B_OK;
}
extern "C" int w2b_host_keep_thresholds(const int64_t *cn, int64_t V, int64_t train_words, float sample, float *out) {
  if (!cn || !out || V < 1) { w2b_set_error("w2b_host_keep_thresholds: bad argument"); return W2B_EINVAL; }
  w2b_keep_thresholds(cn, V, train_words, sample, out);
  return W2B_OK;
}

void w2b_gather_slices(const int32_t *ids, long long n_tokens, long long L, int nshards, const long long *cursor,
                       const int *done, int32_t *stage, long long *xlate, long long *limit, int *limit_is_eof,
                       int nthreads) {
  auto gather = [=](int lo, int hi) {  // shard i only touches its own outputs and its own slice of the staging buffer
    for (int i = lo; i < hi; ++i) {
      if (done[i]) continue;
      const long long b = std::max<long long>(cursor[i], 0);  // cursor -1 = pending override token
      const long long e = std::min<long long>(b + L, n_tokens);
      if (e > b) memcpy(stage + (long long)i * L, ids + b, (size_t)(e - b) * sizeof(int32_t));
      xlate[i] = b - (long long)i * L;
      limit[i] = e;
      limit_is_eof[i] = (e == n_tokens);
    }
  };
  if (nthreads <= 0) {  // >= 1 M tokens per thread, at most 8 threads / half the host / one per shard
    const long long by_size = L * nshards / (1 << 20);
    const long long by_host = std::max(1u, std::thread::hardware_concurrency() / 2);
    nthreads = (int)std::min<long long>(std::min<long long>(8, by_host), std::min<long long>(nshards, by_size));
  }
  nthreads = std::min(nthreads, nshards);
  if (nthreads <= 1) {
    gather(0, nshards);
    return;
  }
  std::vector<std::thread> th;
  for (int t = 1; t < nthreads; ++t)
    th.emplace_back(gather, (int)((long long)nshards * t / nthreads), (int)((long long)nshards * (t + 1) / nthreads));
  gather(0, (int)((long long)nshards / nthreads));
  for (auto &x : th) x.join();
}

static int w2b_host_gather_slices_impl(const int32_t *ids, int64_t n_tokens, int64_t L, int nshards, const int64_t *cursor,
                                      const int32_t *done, int32_t *stage, int64_t *xlate, int64_t *limit,
                                      int32_t *limit_is_eof, int nthreads);
extern "C" int w2b_host_gather_slices(const int32_t *ids, int64_t n_tokens, int64_t L, int nshards, const int64_t *cursor,
                                      const int32_t *done, int32_t *stage, int64_t *xlate, int64_t *limit,
                                      int32_t *limit_is_eof, int nthreads) {
  return w2b_guarded("w2b_host_gather_slices", [&] { return w2b_host_gather_slices_impl(ids, n_tokens, L, nshards, cursor, done, stage, xlate, limit, limit_is_eof, nthreads); });
}
static int w2b_host_gather_slices_impl(const int32_t *ids, int64_t n_tokens, int64_t L, int nshards, const int64_t *cursor,
                                      const int32_t *done, int32_t *stage, int64_t *xlate, int64_t *limit,
                                      int32_t *limit_is_eof, int nthreads) {
  if (!ids || !cursor || !done || !stage || !xlate || !limit || !limit_is_eof || L < 1 || nshards < 1 || n_tokens < 0) {
    w2b_set_error("w2b_host_gather_slices: bad argument");
    return W2B_EINVAL;
  }
  std::vector<long long> cur(cursor, cursor + nshards), xl(nshards, 0), lim(nshards, 0);
  std::vector<int> dn(done, done + nshards), eof(nshards, 0);
  w2b_gather_slices(ids, n_tokens, L, nshards, cur.data(), dn.data(), stage, xl.data(), lim.data(), eof.data(), nthreads);
  for (int i = 0; i < nshards; ++i) {
    if (dn[i]) continue;
    xlate[i] = xl[i];
    limit[i] = lim[i];
    limit_is_eof[i] = eof[i];
  }
  return W2B_OK;
}

// ----------------------------------------------------------------------------- tokeniser
namespace {

constexpr int kMaxWord = 4096;  // MAX_STRING :29
constexpr int64_t kCkptEvery = 4096;

// One ReadWord call (:131-155) over the mapped file.  false at EOF; a word cut short by
// EOF is dropped, as both callers of the reference do (:279, :180).
inline bool next_token(const uint8_t *buf, int64_t n, int64_t &pos, char *word, int &len, int64_t &begin) {
  int a = 0;
  while (pos < n) {
    const int ch = buf[pos++];
    if (ch == 13) continue;
    if (ch == ' ' || ch == '\t' || ch == '\n') {
      if (a > 0) {
        if (ch == '\n') --pos;  // the newline is read again as </s>
        word[a] = 0;
        len = (int)strlen(word);  // an embedded NUL ends the C string, as in the reference
        return true;
      }
      if (ch == '\n') {
        memcpy(word, "</s>", 5);
        len = 4;
        begin = pos - 1;
        return true;
      }
      continue;
    }
    if (a == 0) begin = pos - 1;
    word[a++] = (char)ch;
    if (a >= kMaxWord - 1) --a;
  }
  return false;
}

inline uint64_t hash_bytes(const char *s, int len) {
  uint64_t h = 1469598103934665603ULL;
  for (int i = 0; i < len; ++i) h = (h ^ (uint8_t)s[i]) * 1099511628211ULL;
  return h;
}

// Open-addressing word table.  A slot holds (upper 32 hash bits << 32 | entry + 1), so a probe touches the
// entry / the string only when the tag matches; entries keep their hash (no re-hash on growth or merge).
struct WordMap {
  struct Entry {  // 32 bytes: a hit on a short word touches one cache line besides the slot
    uint64_t hash;
    int64_t count;
    uint32_t len;
    uint32_t aux;
    union {
      char inl[8];   // len <= 7: the NUL-terminated string itself
      uint64_t off;  // longer: arena offset of the NUL-terminated string
    };
  };
  std::vector<uint64_t> slot;
  std::vector<Entry> ent;
  std::string arena;
  uint64_t mask = 0;

  WordMap() { slot.assign(1u << 12, 0); mask = slot.size() - 1; }
  size_t size() const { return ent.size(); }
  const char *str(uint32_t e) const { return ent[e].len <= 7 ? ent[e].inl : arena.data() + ent[e].off; }
  void prefetch_slot(uint64_t h) const { __builtin_prefetch(&slot[h & mask]); }
  void prefetch_entry(uint64_t h) const {  // second stage: the entry the first slot of the probe points at
    const uint64_t sv = slot[h & mask];
    if (sv) __builtin_prefetch(&ent[(uint32_t)sv - 1]);
  }
  void grow() {
    std::vector<uint64_t> ns(slot.size() * 2, 0);
    const uint64_t m = ns.size() - 1;
    for (uint32_t e = 0; e < ent.size(); ++e) {
      uint64_t i = ent[e].hash & m;
      while (ns[i]) i = (i + 1) & m;
      ns[i] = (ent[e].hash & 0xffffffff00000000ULL) | (uint64_t)(e + 1);
    }
    slot.swap(ns);
    mask = m;
  }
  int64_t find(const char *w, int len, uint64_t h) const {
    const uint64_t tag = h & 0xffffffff00000000ULL;
    for (uint64_t i = h & mask; slot[i]; i = (i + 1) & mask) {
      if ((slot[i] & 0xffffffff00000000ULL) != tag) continue;
      const uint32_t e = (uint32_t)slot[i] - 1;
      if ((int)ent[e].len == len && !memcmp(str(e), w, len)) return e;
    }
    return -1;
  }
  int64_t find(const char *w, int len) const { return find(w, len, hash_bytes(w, len)); }
  uint32_t insert(const char *w, int len, uint64_t h) {
    if ((ent.size() + 1) * 2 > slot.size()) grow();
    const uint32_t e = (uint32_t)ent.size();
    Entry ne;
    ne.hash = h;
    ne.count = 0;
    ne.len = (uint32_t)len;
    ne.aux = 0;
    if (len <= 7) {
      memset(ne.inl, 0, sizeof ne.inl);
      memcpy(ne.inl, w, len);
    } else {
      ne.off = arena.size();
      arena.append(w, len);
      arena.push_back('\0');
    }
    ent.push_back(ne);
    uint64_t i = h & mask;
    while (slot[i]) i = (i + 1) & mask;
    slot[i] = (h & 0xffffffff00000000ULL) | (uint64_t)(e + 1);
    return e;
  }
};

constexpr int kParts = 64;  // merge partitions (by the top hash bits)
inline int part_of(uint64_t h) { return (int)(h >> 58); }

}  // namespace

struct w2b_corpus {
  const uint8_t *buf = nullptr;
  int64_t file_size = 0;
  int fd = -1;
  // vocabulary lookup after loading: kParts tables over all distinct words of the file
  std::vector<WordMap> parts;
  std::vector<std::vector<int32_t>> part_final;  // [partition][entry] -> vocab id or -1
  std::string eos_storage;
  std::vector<const char *> words;
  std::vector<int64_t> cn;
  int64_t train_words = 0;
  std::vector<int32_t> ids;
  // every kCkptEvery raw tokens: byte offset of the token and #in-vocab tokens before it
  std::vector<int64_t> ck_begin, ck_comp;

  int32_t lookup(const char *w, int len) const {  // vocab id of a word, -1 if absent / below min_count
    if (parts.empty()) return -1;
    const uint64_t h = hash_bytes(w, len);
    const int p = part_of(h);
    const int64_t e = parts[p].find(w, len, h);
    return e < 0 ? -1 : part_final[p][(size_t)e];
  }
};

namespace {

// Pass 1 over one chunk [begin, end) of the mapped file: chunk-local vocabulary in first-appearance
// order + the chunk's tokens as local ids.  Chunks start right after a whitespace byte, so the
// sequential reader would be in the same (empty-word) state there.
struct ChunkResult {
  WordMap map;
  std::vector<uint32_t> raw;        // local entry id per token
  std::vector<int64_t> ck_begin;    // byte offset of every kCkptEvery-th token of the chunk
  std::vector<uint32_t> by_part[kParts];  // local entries of every merge partition, in first-appearance order
  std::vector<uint32_t> l2g;        // local entry -> global entry (after the merge)
};

// byte classes of ReadWord (:131-155): 0 regular, 1 space / tab, 2 newline, 3 carriage return (skipped
// everywhere), 4 NUL (ends the C string the reference compares and hashes)
struct ByteClass {
  uint8_t c[256];
  ByteClass() {
    memset(c, 0, sizeof c);
    c[' '] = c['\t'] = 1;
    c['\n'] = 2;
    c[13] = 3;
    c[0] = 4;
  }
};
const ByteClass kClass;

void tokenize_chunk(const uint8_t *buf, int64_t begin, int64_t end, ChunkResult *out) {
  out->raw.reserve((size_t)((end - begin) / 5 + 16));
  WordMap &map = out->map;
  char word[kMaxWord];
  int64_t pos = begin;
  // Tokens are resolved in batches: the scanner only records (pointer, length, hash, offset); a batch is
  // looked up after its slots and entries have been prefetched, in token order (so first-appearance order
  // and the checkpoints are those of the sequential reader).  Pointers into `word` are copied: the buffer
  // is reused by the next slow-path token.
  constexpr int kBatch = 32;
  struct Pending { const char *w; int len; uint64_t h; int64_t tb; };
  Pending pend[kBatch];
  char slow[kBatch][64];  // slow-path tokens up to 63 bytes are parked here, longer ones flush the batch first
  int npend = 0;
  auto flush = [&] {
    for (int i = 0; i < npend; ++i) map.prefetch_slot(pend[i].h);
    for (int i = 0; i < npend; ++i) map.prefetch_entry(pend[i].h);
    for (int i = 0; i < npend; ++i) {
      const Pending &t = pend[i];
      int64_t e = map.find(t.w, t.len, t.h);
      if (e < 0) e = map.insert(t.w, t.len, t.h);
      map.ent[(size_t)e].count++;
      if ((int64_t)out->raw.size() % kCkptEvery == 0) out->ck_begin.push_back(t.tb);
      out->raw.push_back((uint32_t)e);
    }
    npend = 0;
  };
  auto emit = [&](const char *w, int len, uint64_t h, int64_t tb) {
    if (w == word) {  // slow-path token in the scratch buffer
      if (len < 64) {
        memcpy(slow[npend], w, len);
        w = slow[npend];
      } else {
        flush();
        pend[0] = Pending{w, len, h, tb};
        npend = 1;
        flush();
        return;
      }
    }
    pend[npend++] = Pending{w, len, h, tb};
    if (npend == kBatch) flush();
  };
  const uint64_t eos_hash = hash_bytes("</s>", 4);
  while (pos < end) {
    const uint8_t cls = kClass.c[buf[pos]];
    if (cls == 1 || cls == 3) { ++pos; continue; }
    if (cls == 2) {  // a newline outside a word is the token </s>
      emit("</s>", 4, eos_hash, pos);
      ++pos;
      continue;
    }
    // a word starts here.  Fast path: its bytes are contiguous in the file (no CR, no NUL, shorter than
    // MAX_STRING) — hash while scanning, look up straight from the mapping.
    const int64_t start = pos;
    uint64_t h = 1469598103934665603ULL;
    int64_t q = pos;
    uint8_t stop = 0;
    if (cls == 0) {
      while (q < end && (stop = kClass.c[buf[q]]) == 0) {
        h = (h ^ buf[q]) * 1099511628211ULL;
        ++q;
      }
    } else {
      stop = cls;  // the word starts with a NUL byte
    }
    if (q >= end) {
      if (q - start < kMaxWord - 1) break;  // cut short by the end of the file: dropped, as in the reference (:279,:180)
      stop = 3;                              // over-long word at EOF: let the reference-shaped reader decide
    }
    if (stop <= 2 && q - start < kMaxWord - 1) {
      emit((const char *)buf + start, (int)(q - start), h, start);
      pos = q;  // the delimiter is looked at again: a newline becomes </s>
      continue;
    }
    // slow path (CR or NUL inside the word, or 4095+ bytes): the byte-by-byte reader
    int len = 0;
    int64_t tb = 0, p2 = start;
    if (!next_token(buf, end, p2, word, len, tb)) break;
    emit(word, len, hash_bytes(word, len), tb);
    pos = p2;
  }
  flush();
}

}  // namespace

static int w2b_corpus_load_impl(const char *path, int min_count, w2b_corpus **out);
extern "C" int w2b_corpus_load(const char *path, int min_count, w2b_corpus **out) {
  return w2b_guarded("w2b_corpus_load", [&] { return w2b_corpus_load_impl(path, min_count, out); });
}
static int w2b_corpus_load_impl(const char *path, int min_count, w2b_corpus **out) {
  if (!out) {
    w2b_set_error("w2b_corpus_load: null out");
    return W2B_EINVAL;
  }
  *out = nullptr;
  int fd = path ? open(path, O_RDONLY) : -1;
  if (fd < 0) {
    w2b_set_error("ERROR: training data file not found!");  // :272
    return W2B_EIO;
  }
  struct stat st;
  if (fstat(fd, &st) != 0 || !S_ISREG(st.st_mode)) {  // a directory opens fine but cannot be mapped
    close(fd);
    w2b_set_error("ERROR: training data file not found!");
    return W2B_EIO;
  }
  // owned until the very end: an exception below (std::bad_alloc, std::system_error from a thread) unwinds through
  // this guard, which unmaps the file, closes the descriptor and frees the object (w2b_guarded turns it into a code)
  struct Owner {
    w2b_corpus *c;
    ~Owner() { if (c) w2b_corpus_free(c); }
  } owner{new w2b_corpus()};
  w2b_corpus *c = owner.c;
  c->fd = fd;
  c->file_size = st.st_size;  // == ftell at EOF, :299
  if (st.st_size > 0) {
    void *m = mmap(nullptr, st.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
    if (m == MAP_FAILED) {
      w2b_set_error("mmap failed for %s", path);
      return W2B_EIO;
    }
    c->buf = (const uint8_t *)m;
    madvise(m, st.st_size, MADV_SEQUENTIAL);
  }
  const bool dbg = getenv("W2B_TOKENIZER_DEBUG") != nullptr;
  auto t_start = std::chrono::steady_clock::now();
  auto lap = [&](const char *what) {
    if (!dbg) return;
    auto now = std::chrono::steady_clock::now();
    fprintf(stderr, "[tokenizer] %-10s %.3f s\n", what, std::chrono::duration<double>(now - t_start).count());
    t_start = now;
  };
  // ---- pass 1, parallel over chunks of the file (the reference's single fgetc loop, :277-293,
  // runs at ~7 M words/s; one GPU consumes 30 M words/s, eight consume 250 M)
  const int64_t n = c->file_size;
  int nthreads = (int)std::thread::hardware_concurrency();
  if (const char *e = getenv("W2B_TOKENIZER_THREADS")) nthreads = atoi(e);
  int64_t min_chunk = 4 << 20;
  if (const char *e = getenv("W2B_TOKENIZER_MIN_CHUNK")) min_chunk = atoll(e);
  nthreads = std::max(1, std::min(nthreads, 256));
  nthreads = (int)std::max<int64_t>(1, std::min<int64_t>(nthreads, n / std::max<int64_t>(min_chunk, 1)));
  std::vector<int64_t> cut(nthreads + 1, n);
  cut[0] = 0;
  for (int t = 1; t < nthreads; ++t) {
    int64_t p = n / nthreads * t;
    if (p < cut[t - 1]) p = cut[t - 1];
    // advance to just after the next whitespace byte: a clean token boundary
    while (p < n && !(c->buf[p] == ' ' || c->buf[p] == '\t' || c->buf[p] == '\n')) ++p;
    cut[t] = p < n ? p + 1 : n;
  }
  auto run_parallel = [](int count, int threads, const std::function<void(int)> &fn) {
    threads = std::max(1, std::min(threads, count));
    if (threads == 1) {
      for (int i = 0; i < count; ++i) fn(i);
      return;
    }
    std::atomic<int> next(0);
    auto work = [&] { for (int i; (i = next.fetch_add(1)) < count;) fn(i); };
    std::vector<std::thread> th;
    for (int t = 1; t < threads; ++t) th.emplace_back(work);
    work();
    for (auto &x : th) x.join();
  };
  std::vector<ChunkResult> chunks(nthreads);
  run_parallel(nthreads, nthreads, [&](int t) {
    ChunkResult &ch = chunks[t];
    tokenize_chunk(c->buf, cut[t], cut[t + 1], &ch);
    for (uint32_t e = 0; e < ch.map.size(); ++e) ch.by_part[part_of(ch.map.ent[e].hash)].push_back(e);
    ch.l2g.resize(ch.map.size());
  });
  lap("pass1");
  // ---- merge, one thread per partition of the hash space.  Global first-appearance order = chunk order,
  // then local order (what the reference's sequential pass produces): every global entry remembers the
  // (chunk, local entry) that introduced it, and that pair is the tie-break of the sort below.
  c->parts.resize(kParts);
  struct First { uint32_t chunk, local; };
  std::vector<std::vector<First>> first(kParts);
  run_parallel(kParts, nthreads, [&](int p) {
    WordMap &g = c->parts[p];
    size_t total = 0;
    for (int t = 0; t < nthreads; ++t) total += chunks[t].by_part[p].size();
    first[p].reserve(total / std::max(1, nthreads / 2) + 16);
    for (int t = 0; t < nthreads; ++t) {
      const WordMap &lm = chunks[t].map;
      for (uint32_t e : chunks[t].by_part[p]) {
        const WordMap::Entry &le = lm.ent[e];
        int64_t ge = g.find(lm.str(e), (int)le.len, le.hash);
        if (ge < 0) {
          ge = g.insert(lm.str(e), (int)le.len, le.hash);
          first[p].push_back(First{(uint32_t)t, e});
        }
        g.ent[(size_t)ge].count += le.count;
        chunks[t].l2g[e] = (uint32_t)ge;  // partition-local for now
      }
    }
  });
  std::vector<uint32_t> part_base(kParts + 1, 0);
  for (int p = 0; p < kParts; ++p) part_base[p + 1] = part_base[p] + (uint32_t)c->parts[p].size();
  lap("merge");
  // SortVocab (:215-242): </s> pinned at 0 (AddWordToVocab("</s>") comes first, :276, even when the file
  // has no newline), the rest by count descending, ties in first-appearance order (what glibc's qsort
  // yields here; asserted against the reference in tests), then the min_count cut.
  struct Key { int64_t count; uint32_t chunk, local, part, idx; };
  std::vector<Key> order;
  order.reserve(part_base[kParts]);
  const uint64_t eos_hash = hash_bytes("</s>", 4);
  const int eos_part = part_of(eos_hash);
  const int64_t eos_entry = c->parts[eos_part].find("</s>", 4, eos_hash);
  {  // the reference prunes its vocabulary in the middle of the scan once it holds more than 0.7 * 30 M words
     // (ReduceVocab, :245-263, :292) — an order-dependent cut this one-pass reader does not reproduce: refuse
    int64_t max_distinct = 21000000;
    if (const char *e = getenv("W2B_TOKENIZER_MAX_DISTINCT")) max_distinct = atoll(e);  // (tests)
    const int64_t distinct = (int64_t)part_base[kParts] + (eos_entry >= 0 ? 0 : 1);
    if (distinct > max_distinct) {  // (the guard above releases the corpus)
      w2b_set_error("%lld distinct words: above 21 M the reference prunes its vocabulary mid-scan (ReduceVocab), "
                    "which this reader does not reproduce", (long long)distinct);
      return W2B_EINVAL;
    }
  }
  for (int p = 0; p < kParts; ++p)
    for (uint32_t e = 0; e < c->parts[p].size(); ++e) {
      if (p == eos_part && (int64_t)e == eos_entry) continue;
      if (c->parts[p].ent[e].count < min_count) continue;  // never enters the vocabulary: no need to rank it
      order.push_back(Key{c->parts[p].ent[e].count, first[p][e].chunk, first[p][e].local, (uint32_t)p, e});
    }
  std::sort(order.begin(), order.end(), [](const Key &a, const Key &b) {
    if (a.count != b.count) return a.count > b.count;
    if (a.chunk != b.chunk) return a.chunk < b.chunk;
    return a.local < b.local;
  });
  c->part_final.resize(kParts);
  for (int p = 0; p < kParts; ++p) c->part_final[p].assign(c->parts[p].size(), -1);
  c->eos_storage = "</s>";
  c->words.push_back(eos_entry >= 0 ? c->parts[eos_part].str((uint32_t)eos_entry) : c->eos_storage.c_str());
  c->cn.push_back(eos_entry >= 0 ? c->parts[eos_part].ent[(size_t)eos_entry].count : 0);
  c->train_words += c->cn[0];
  if (eos_entry >= 0) c->part_final[eos_part][(size_t)eos_entry] = 0;
  for (const Key &k : order) {
    if (k.count < min_count) break;  // sorted by count: everything after is below the cut too
    c->part_final[k.part][k.idx] = (int32_t)c->words.size();
    c->words.push_back(c->parts[k.part].str(k.idx));
    c->cn.push_back(k.count);
    c->train_words += k.count;
  }
  lap("sort");
  // ---- compact to the in-vocab stream (parallel per chunk), remembering where every checkpoint lands
  std::vector<int64_t> kept(nthreads, 0), base(nthreads + 1, 0);
  std::vector<std::vector<int32_t>> lfinal(nthreads);  // chunk-local entry -> vocab id or -1
  run_parallel(nthreads, nthreads, [&](int t) {
    const ChunkResult &ch = chunks[t];
    lfinal[t].resize(ch.map.size());
    for (uint32_t e = 0; e < ch.map.size(); ++e)
      lfinal[t][e] = c->part_final[part_of(ch.map.ent[e].hash)][ch.l2g[e]];
    int64_t k = 0;
    for (uint32_t le : ch.raw) k += lfinal[t][le] >= 0;
    kept[t] = k;
  });
  for (int t = 0; t < nthreads; ++t) base[t + 1] = base[t] + kept[t];
  c->ids.resize((size_t)base[nthreads]);
  std::vector<std::vector<int64_t>> ck_comp(nthreads);
  run_parallel(nthreads, nthreads, [&](int t) {
    int64_t w = base[t];
    const auto &raw = chunks[t].raw;
    ck_comp[t].reserve(chunks[t].ck_begin.size());
    for (size_t k = 0; k < raw.size(); ++k) {
      if ((int64_t)k % kCkptEvery == 0) ck_comp[t].push_back(w);
      const int32_t id = lfinal[t][raw[k]];
      if (id >= 0) c->ids[(size_t)w++] = id;
    }
  });
  for (int t = 0; t < nthreads; ++t) {
    c->ck_begin.insert(c->ck_begin.end(), chunks[t].ck_begin.begin(), chunks[t].ck_begin.end());
    c->ck_comp.insert(c->ck_comp.end(), ck_comp[t].begin(), ck_comp[t].end());
  }
  lap("compact");
  *out = c;
  owner.c = nullptr;
  return W2B_OK;
}

extern "C" void w2b_corpus_free(w2b_corpus *c) {
  if (!c) return;
  if (c->buf) munmap((void *)c->buf, c->file_size);
  if (c->fd >= 0) close(c->fd);
  delete c;
}

extern "C" int64_t w2b_corpus_vocab_size(const w2b_corpus *c) { return (int64_t)c->words.size(); }
extern "C" int64_t w2b_corpus_train_words(const w2b_corpus *c) { return c->train_words; }
extern "C" int64_t w2b_corpus_file_size(const w2b_corpus *c) { return c->file_size; }
extern "C" const char *w2b_corpus_word(const w2b_corpus *c, int64_t i) { return c->words[i]; }
extern "C" const int64_t *w2b_corpus_counts(const w2b_corpus *c) { return c->cn.data(); }
extern "C" int64_t w2b_corpus_num_tokens(const w2b_corpus *c) { return (int64_t)c->ids.size(); }
extern "C" const int32_t *w2b_corpus_tokens(const w2b_corpus *c) { return c->ids.data(); }

static int w2b_corpus_shards_impl(const w2b_corpus *c, int n, int64_t *start, int32_t *first);
extern "C" int w2b_corpus_shards(const w2b_corpus *c, int n, int64_t *start, int32_t *first) {
  return w2b_guarded("w2b_corpus_shards", [&] { return w2b_corpus_shards_impl(c, n, start, first); });
}
static int w2b_corpus_shards_impl(const w2b_corpus *c, int n, int64_t *start, int32_t *first) {
  if (!c || !start || !first) {
    w2b_set_error("w2b_corpus_shards: null argument");
    return W2B_EINVAL;
  }
  if (n < 1) {
    w2b_set_error("shard count must be >= 1");
    return W2B_EINVAL;
  }
  char word[kMaxWord];
  for (int i = 0; i < n; ++i) {
    const int64_t off = c->file_size / (int64_t)n * (int64_t)i;  // :377
    int64_t pos = off, begin = 0;
    int len = 0;
    first[i] = -1;
    if (!next_token(c->buf, c->file_size, pos, word, len, begin)) {
      start[i] = (int64_t)c->ids.size();
      continue;
    }
    first[i] = c->lookup(word, len);
    // index of the first regular in-vocab token that begins at or after `pos`:
    // restart from the last checkpoint at or before it and count forward
    size_t k = std::upper_bound(c->ck_begin.begin(), c->ck_begin.end(), pos) - c->ck_begin.begin();
    if (k == 0) {
      start[i] = 0;
      continue;
    }
    --k;
    int64_t p2 = c->ck_begin[k], comp = c->ck_comp[k], b2 = 0;
    int l2 = 0;
    for (;;) {
      if (!next_token(c->buf, c->file_size, p2, word, l2, b2)) break;
      if (b2 >= pos) break;
      if (c->lookup(word, l2) >= 0) ++comp;
    }
    start[i] = comp;
  }
  return W2B_OK;
}

// "%lf " of a float, through a small direct-mapped cache keyed by the bit pattern: trained vectors hold
// 2^bitlevel distinct values (2 at bitlevel 1), so almost every value is a table hit; a miss is formatted by
// snprintf itself, which keeps the bytes identical to the reference's fprintf for every input (:571).
namespace {
struct FmtCache {
  struct Slot { uint32_t bits; uint8_t len, valid; char s[58]; };
  Slot slot[512];
  FmtCache() { memset(slot, 0, sizeof slot); }
  // "%lf " of one value.  A float times 10^6 is exact in double (24-bit x 20-bit significands), so rounding it
  // to the nearest integer, ties to even, is exactly the correctly rounded 6-decimal expansion printf produces
  // (round-to-nearest mode); everything that does not fit that scheme goes to snprintf itself.
  static int format(float x, char *out, size_t cap) {
    const double ax = fabs((double)x);
    if (!(ax < 1e12)) return snprintf(out, cap, "%lf ", (double)x);  // huge, inf, nan (<= 48 bytes for any float)
    const unsigned long long n = (unsigned long long)nearbyint(ax * 1e6);
    unsigned long long ip = n / 1000000ULL;
    unsigned fr = (unsigned)(n % 1000000ULL);
    char tmp[32];
    int k = 0;
    tmp[k++] = ' ';
    for (int i = 0; i < 6; ++i) { tmp[k++] = (char)('0' + fr % 10); fr /= 10; }
    tmp[k++] = '.';
    do { tmp[k++] = (char)('0' + ip % 10); ip /= 10; } while (ip);
    if (signbit(x)) tmp[k++] = '-';
    for (int i = 0; i < k; ++i) out[i] = tmp[k - 1 - i];
    return k;
  }
  inline void append(float x, std::string &out) {
    uint32_t b;
    memcpy(&b, &x, 4);
    Slot &e = slot[(b * 2654435761u) >> 23];
    if (!e.valid || e.bits != b) {
      e.len = (uint8_t)format(x, e.s, sizeof e.s);
      e.bits = b;
      e.valid = 1;
    }
    out.append(e.s, e.len);
  }
};
}  // namespace

static int w2b_write_vectors_impl(const char *path, const w2b_corpus *c, const float *vec, int64_t V, int64_t D,
                                 int binary);
extern "C" int w2b_write_vectors(const char *path, const w2b_corpus *c, const float *vec, int64_t V, int64_t D,
                                 int binary) {
  return w2b_guarded("w2b_write_vectors", [&] { return w2b_write_vectors_impl(path, c, vec, V, D, binary); });
}
static int w2b_write_vectors_impl(const char *path, const w2b_corpus *c, const float *vec, int64_t V, int64_t D,
                                 int binary) {
  if (!path || !c || !vec || V < 0 || V > (int64_t)c->words.size() || D < 1) {
    w2b_set_error("w2b_write_vectors: bad argument");
    return W2B_EINVAL;
  }
  FILE *fo = fopen(path, "wb");
  if (!fo) {
    w2b_set_error("cannot open %s for writing", path);
    return W2B_EIO;
  }
  std::vector<char> iobuf(4 << 20);  // per call: two writers may run on two host threads
  setvbuf(fo, iobuf.data(), _IOFBF, iobuf.size());
  fprintf(fo, "%lld %lld\n", (long long)V, (long long)D);
  if (binary) {
    for (int64_t a = 0; a < V; ++a) {
      fputs(c->words[a], fo);
      fputc(' ', fo);
      fwrite(vec + a * D, sizeof(float), D, fo);
      fputc('\n', fo);
    }
  } else {
    // text: V * D values (3.2 GB at V = 400 k, D = 800).  Blocks of rows are formatted by a few threads into
    // private buffers and written in order.
    int nthr = (int)std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
    if (const char *e = getenv("W2B_WRITER_THREADS")) nthr = std::max(1, atoi(e));
    const int64_t rows_per_task = std::max<int64_t>(1, (1 << 18) / (D * 10));  // ~256 KB of text per task
    nthr = (int)std::max<int64_t>(1, std::min<int64_t>(nthr, (V + rows_per_task - 1) / rows_per_task));
    std::vector<std::string> bufs(nthr);
    std::vector<FmtCache> caches(nthr);
    auto format_rows = [&](int t, int64_t lo, int64_t hi) {
      std::string &out = bufs[t];
      out.clear();
      for (int64_t a = lo; a < hi; ++a) {
        out.append(c->words[a]);
        out.push_back(' ');
        const float *row = vec + a * D;
        for (int64_t b = 0; b < D; ++b) caches[t].append(row[b], out);
        out.push_back('\n');
      }
    };
    for (int64_t base = 0; base < V; base += rows_per_task * nthr) {
      std::vector<std::thread> th;
      for (int t = 1; t < nthr; ++t) {
        const int64_t lo = std::min(V, base + t * rows_per_task), hi = std::min(V, lo + rows_per_task);
        th.emplace_back(format_rows, t, lo, hi);
      }
      format_rows(0, base, std::min(V, base + rows_per_task));
      for (auto &x : th) x.join();
      for (int t = 0; t < nthr; ++t) fwrite(bufs[t].data(), 1, bufs[t].size(), fo);
    }
  }
  const bool bad = ferror(fo) != 0;
  if (fclose(fo) != 0 || bad) {  // the reference ignores write errors; a truncated vector file is worse
    w2b_set_error("short write to %s (disk full?)", path);
    return W2B_EIO;
  }
  return W2B_OK;
}

// ------------------------------------------------------------------------- packed vector files
static inline int level_code(float x, int bits) {  // inverse of quantize() for bitlevel 1 / 2
  const int neg = x < 0.f;
  if (bits == 1) return neg;
  return neg | ((fabsf(x) > 0.5f) ? 2 : 0);
}
static inline float level_value(int code, int bits) {
  const float m = (bits == 1) ? (1.0f / 3) : ((code & 2) ? 0.75f : 0.25f);
  return (code & 1) ? -m : m;
}

static int w2b_write_packed_impl(const char *path, const w2b_corpus *c, const float *vec, int64_t V, int64_t D,
                                int bitlevel);
extern "C" int w2b_write_packed(const char *path, const w2b_corpus *c, const float *vec, int64_t V, int64_t D,
                                int bitlevel) {
  return w2b_guarded("w2b_write_packed", [&] { return w2b_write_packed_impl(path, c, vec, V, D, bitlevel); });
}
static int w2b_write_packed_impl(const char *path, const w2b_corpus *c, const float *vec, int64_t V, int64_t D,
                                int bitlevel) {
  if (bitlevel != 1 && bitlevel != 2) {
    w2b_set_error("packed format supports bitlevel 1 and 2");
    return W2B_EINVAL;
  }
  if (!path || !c || !vec || V < 0 || V > (int64_t)c->words.size() || D < 1) {
    w2b_set_error("w2b_write_packed: bad argument");
    return W2B_EINVAL;
  }
  FILE *fo = fopen(path, "wb");
  if (!fo) {
    w2b_set_error("cannot open %s for writing", path);
    return W2B_EIO;
  }
  fprintf(fo, "%lld %lld %d\n", (long long)V, (long long)D, bitlevel);
  const int64_t nbytes = (D * bitlevel + 7) / 8;
  std::vector<uint8_t> row(nbytes);
  for (int64_t a = 0; a < V; ++a) {
    fprintf(fo, "%s ", c->words[a]);
    std::fill(row.begin(), row.end(), 0);
    for (int64_t j = 0; j < D; ++j) {
      const int code = level_code(vec[a * D + j], bitlevel);
      const int64_t bit = j * bitlevel;
      row[bit >> 3] |= (uint8_t)(code << (bit & 7));  // bitlevel divides 8: a value never straddles bytes
    }
    fwrite(row.data(), 1, nbytes, fo);
    fputc('\n', fo);
  }
  const bool bad = ferror(fo) != 0;
  if (fclose(fo) != 0 || bad) {
    w2b_set_error("short write to %s (disk full?)", path);
    return W2B_EIO;
  }
  return W2B_OK;
}

int w2b_packed_open(const char *path, w2b_packed_file *pf) {
  pf->f = fopen(path, "rb");
  if (!pf->f) {
    w2b_set_error("cannot open %s", path);
    return W2B_EIO;
  }
  char line[128];
  long long v = 0, d = 0, b = 0;
  char extra;
  // three integers and nothing else on the first line: a word2vec-binary file has two
  if (!fgets(line, sizeof line, pf->f) || !strchr(line, '\n') ||
      sscanf(line, "%lld %lld %lld %c", &v, &d, &b, &extra) != 3 || (b != 1 && b != 2) || v < 0 || d < 1 ||
      d > (INT64_MAX - 7) / 2) {
    w2b_set_error("%s is not a packed vector file", path);
    return W2B_EIO;
  }
  pf->V = v; pf->D = d; pf->bits = (int)b;
  pf->nbytes = (d * b + 7) / 8;
  return W2B_OK;
}

int w2b_packed_next(w2b_packed_file *pf, char *name, int name_cap, uint8_t *row) {
  int ch, k = 0;
  while ((ch = fgetc(pf->f)) != EOF && ch != ' ')
    if (name && k < name_cap - 1) name[k++] = (char)ch;
  if (name) name[k] = 0;
  if (fread(row, 1, pf->nbytes, pf->f) != (size_t)pf->nbytes) {
    w2b_set_error("packed vector file is truncated");
    return W2B_EIO;
  }
  fgetc(pf->f);  // '\n'
  return W2B_OK;
}

extern "C" int w2b_read_packed_header(const char *path, int64_t *V, int64_t *D, int *bitlevel) {
  if (!path || !V || !D || !bitlevel) { w2b_set_error("w2b_read_packed_header: null argument"); return W2B_EINVAL; }
  w2b_packed_file pf;
  const int rc = w2b_packed_open(path, &pf);
  if (rc) return rc;
  *V = pf.V; *D = pf.D; *bitlevel = pf.bits;
  return W2B_OK;
}

static int w2b_read_packed_impl(const char *path, float *vec, char *words, int max_word);
extern "C" int w2b_read_packed(const char *path, float *vec, char *words, int max_word) {
  return w2b_guarded("w2b_read_packed", [&] { return w2b_read_packed_impl(path, vec, words, max_word); });
}
static int w2b_read_packed_impl(const char *path, float *vec, char *words, int max_word) {
  if (!path || !vec || (words && max_word < 1)) { w2b_set_error("w2b_read_packed: bad argument"); return W2B_EINVAL; }
  w2b_packed_file pf;
  int rc = w2b_packed_open(path, &pf);
  if (rc) return rc;
  const int64_t D = pf.D;
  const int bits = pf.bits;
  std::vector<uint8_t> row(pf.nbytes);
  for (int64_t a = 0; a < pf.V; ++a) {
    rc = w2b_packed_next(&pf, words ? words + a * max_word : nullptr, max_word, row.data());
    if (rc) return rc;
    for (int64_t j = 0; j < D; ++j) {
      const int64_t bit = j * bits;
      vec[a * D + j] = level_value((row[bit >> 3] >> (bit & 7)) & ((1 << bits) - 1), bits);
    }
  }
  return W2B_OK;
}

// ------------------------------------------------------------------------- text vector files (-binary 0)
extern "C" int w2b_host_parse_floats(const char *text, int64_t n_bytes, float *out, int64_t cap, int64_t *n) {
  if ((!text && n_bytes > 0) || n_bytes < 0 || (!out && cap > 0) || cap < 0 || !n) {
    w2b_set_error("w2b_host_parse_floats: bad argument");
    return W2B_EINVAL;
  }
  const char *p = text, *end = text + n_bytes;
  int64_t k = 0;
  for (;;) {
    while (p < end && w2b::text::is_space(*p)) ++p;
    if (p == end) break;
    const char *e = w2b::text::token_end(p, end);
    if (k >= cap) {
      w2b_set_error("w2b_host_parse_floats: more than %lld tokens", (long long)cap);
      return W2B_EINVAL;
    }
    if (!w2b::text::parse_token(p, e, out + k)) {
      w2b_set_error("token %lld '%.*s' is not a number", (long long)k, (int)std::min<long long>(e - p, 64), p);
      *n = k;
      return W2B_EIO;
    }
    ++k;
    p = e;
  }
  *n = k;
  return W2B_OK;
}

namespace {
// A FILE read through a large buffer, for walking the rows of a vector file.
struct ByteReader {
  FILE *f;
  std::vector<char> buf = std::vector<char>(1 << 20);
  size_t pos = 0, len = 0;
  bool fill() {
    pos = 0;
    len = fread(buf.data(), 1, buf.size(), f);
    return len > 0;
  }
  int get() { return (pos < len || fill()) ? (unsigned char)buf[pos++] : EOF; }
  // past the next '\n' (or to the end); the bytes before it are appended to *line when line is set
  void line_rest(std::string *line) {
    for (;;) {
      if (pos == len && !fill()) return;
      const char *s = buf.data() + pos, *nl = (const char *)memchr(s, '\n', len - pos);
      const size_t k = nl ? (size_t)(nl - s) : len - pos;
      if (line) line->append(s, k);
      pos += k + (nl ? 1 : 0);
      if (nl) return;
    }
  }
  void skip(int64_t k) {
    for (; k > 0;) {
      if (pos == len && !fill()) return;
      const size_t t = (size_t)std::min<int64_t>(k, (int64_t)(len - pos));
      pos += t;
      k -= t;
    }
  }
  // a name as read_vectors reads it: up to the first ' ' (not kept), '\n' skipped.  false at the end of the file.
  bool name(std::string &w) {
    w.clear();
    int ch = get();
    if (ch == EOF) return false;
    for (; ch != EOF && ch != ' '; ch = get())
      if (ch != '\n') w.push_back((char)ch);
    return true;
  }
};

// the header "V D" as fscanf reads it (read_vectors); the file is left right after D
bool header2(FILE *f, long long &V, long long &D) { return fscanf(f, "%lld", &V) == 1 && fscanf(f, "%lld", &D) == 1; }
}  // namespace

// The one decision on a vector file's format (w2b.h w2b_vector_file_info).
extern "C" int w2b_vector_file_info(const char *path, int64_t threshold, int *kind, int64_t *V, int64_t *D, int *bits) {
  if (!path || !kind || !V || !D || !bits) { w2b_set_error("w2b_vector_file_info: null argument"); return W2B_EINVAL; }
  return w2b_guarded("w2b_vector_file_info", [&]() -> int {
    FILE *f = fopen(path, "rb");
    if (!f) {
      w2b_set_error("Input file not found");
      return W2B_EIO;
    }
    std::unique_ptr<FILE, int (*)(FILE *)> closer(f, fclose);
    *kind = W2B_VECTORS_BINARY;
    *V = *D = 0;
    *bits = 0;
    char line[128], extra;
    long long v = 0, d = 0, b = 0;
    if (fgets(line, sizeof line, f) && sscanf(line, "%lld %lld %lld %c", &v, &d, &b, &extra) == 3) {
      *kind = W2B_VECTORS_PACKED;  // three integers on the first line
      *bits = (int)b;
    } else {
      rewind(f);
      if (!header2(f, v, d)) return W2B_OK;  // read_vectors reports the bad header
      if (d >= 1 && d <= (1LL << 20)) {
        // (a) a binary row has '\n' right after its 4 D value bytes; (b) a text row is D tokens up to its '\n'
        int ch;
        while ((ch = fgetc(f)) != EOF && ch != ' ') {}
        const long long sp = ftell(f) - 1;
        if (ch == ' ' && sp >= 0 && fseek(f, sp + 1 + 4 * d, SEEK_SET) == 0 && fgetc(f) != '\n' &&
            fseek(f, sp + 1, SEEK_SET) == 0) {
          ByteReader r{f};
          std::string row;
          r.line_rest(&row);
          const char *p = row.data(), *end = p + row.size();
          long long tokens = 0;
          bool ok = true;
          for (;;) {
            while (p < end && w2b::text::is_space(*p)) ++p;
            if (p == end) break;
            const char *e = w2b::text::token_end(p, end);
            float x;
            ok = ok && w2b::text::parse_token(p, e, &x) && ++tokens <= d;
            if (!ok) break;
            p = e;
          }
          if (ok && tokens == d) *kind = W2B_VECTORS_TEXT;
        }
      }
    }
    *V = (threshold > 0 && v > threshold) ? threshold : v;
    *D = d;
    return W2B_OK;
  });
}

// The names of a vector file's rows, each as the evaluator compares it (w2b.h w2b_vector_names).
extern "C" int w2b_vector_names(const char *path, int64_t threshold, char *names, int max_word, int64_t *n) {
  if (!path || !names || max_word < 1 || !n) { w2b_set_error("w2b_vector_names: bad argument"); return W2B_EINVAL; }
  return w2b_guarded("w2b_vector_names", [&]() -> int {
    int kind, bits;
    int64_t V, D;
    int rc = w2b_vector_file_info(path, threshold, &kind, &V, &D, &bits);
    if (rc) return rc;
    FILE *f = fopen(path, "rb");
    if (!f) {
      w2b_set_error("Input file not found");
      return W2B_EIO;
    }
    std::unique_ptr<FILE, int (*)(FILE *)> closer(f, fclose);
    long long v, d;
    char line[128];
    if (kind == W2B_VECTORS_PACKED ? !fgets(line, sizeof line, f) : !header2(f, v, d)) {
      w2b_set_error("bad header");
      return W2B_EIO;
    }
    const int64_t row = kind == W2B_VECTORS_PACKED ? (D * bits + 7) / 8 + 1 : 4 * D;  // a packed row ends with '\n'
    ByteReader r{f};
    std::string w;
    int64_t k = 0;
    for (; k < V && r.name(w); ++k) {
      char *out = names + k * max_word;
      int j = 0;
      for (; j < (int)w.size() && j < 50 && j < max_word - 1; ++j) out[j] = (char)toupper((unsigned char)w[j]);
      out[j] = 0;
      if (kind == W2B_VECTORS_TEXT)
        r.line_rest(nullptr);
      else
        r.skip(row);
    }
    *n = k;
    return W2B_OK;
  });
}

// Row `row` of a text vector file: its name and the bytes of its values (w2b_internal.h).
int w2b_text_row(const char *path, int64_t row, std::string &name, std::string &values) {
  FILE *f = fopen(path, "rb");
  if (!f) return W2B_EIO;
  std::unique_ptr<FILE, int (*)(FILE *)> closer(f, fclose);
  long long v, d;
  if (!header2(f, v, d)) return W2B_EIO;
  ByteReader r{f};
  for (int64_t k = 0; k <= row; ++k) {
    if (!r.name(name)) return W2B_EIO;
    values.clear();
    r.line_rest(k == row ? &values : nullptr);
  }
  return W2B_OK;
}

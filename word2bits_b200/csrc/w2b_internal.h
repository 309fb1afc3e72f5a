// Internal helpers shared by the host and device halves of libw2b (not part of the ABI).
#pragma once
#include <stdint.h>
#include <stdio.h>

#include <exception>
#include <new>
#include <string>
#include <vector>

void w2b_set_error(const char *fmt, ...);

// Nothing is thrown across the C ABI: entry points that allocate host memory or start threads run their body
// through this guard (std::bad_alloc -> W2B_ENOMEM, anything else -> W2B_EINVAL, message in w2b_last_error()).
template <class F>
static inline int w2b_guarded(const char *name, F &&body) {
  try {
    return body();
  } catch (const std::bad_alloc &) {
    w2b_set_error("%s: out of host memory", name);
    return 6;  // W2B_ENOMEM
  } catch (const std::exception &ex) {
    w2b_set_error("%s: %s", name, ex.what());
    return 1;  // W2B_EINVAL
  } catch (...) {
    w2b_set_error("%s: unexpected exception", name);
    return 1;
  }
}
// The one parser of the packed vector format (w2b_write_packed): a header line "V D bitlevel", then per word its
// name, ' ', nbytes = ceil(D * bitlevel / 8) bytes (value j in bits [j * bitlevel, (j + 1) * bitlevel), sign in the
// low bit, for 2 bits the magnitude in the high bit) and '\n'.  w2b_read_packed expands rows to floats; the
// evaluator keeps them packed.
struct w2b_packed_file {
  FILE *f = nullptr;
  int64_t V = 0, D = 0, nbytes = 0;
  int bits = 0;
  ~w2b_packed_file() { if (f) fclose(f); }
};
// W2B_EIO unless the first line holds exactly three integers with V >= 0, D >= 1 and bitlevel 1 or 2; on success the
// file is positioned at the first word.
int w2b_packed_open(const char *path, w2b_packed_file *pf);
// The next word: at most name_cap - 1 characters of its name (NUL-terminated; name may be NULL) and its nbytes
// packed bytes.  W2B_EIO when the file ends inside the row.
int w2b_packed_next(w2b_packed_file *pf, char *name, int name_cap, uint8_t *row);
// What the evaluator reads of a training context (w2b_ctx_compute_accuracy and friends): the fp32 master tables u
// and v, V rows of `pitch` floats of which the first D are the row (the rest is padding), the training bit level,
// the context's device and its stream (a cudaStream_t).  W2B_ESTATE before w2b_init_tables / w2b_checkpoint_load.
struct w2b_ctx;
struct w2b_ctx_tables {
  const float *u = nullptr, *v = nullptr;
  int64_t V = 0, D = 0, pitch = 0;
  int bitlevel = 0, device = 0;
  void *stream = nullptr;
};
int w2b_ctx_tables_of(w2b_ctx *ctx, w2b_ctx_tables *out);
// InitUnigramTable (src/word2bits.cpp:112-128) in boundary form: start[i] = first table
// slot owned by word i, start[V] = 1e8.  Same libm pow() and the same double arithmetic
// as the reference loop, so expanding it reproduces the 1e8-entry table bit for bit.
void w2b_unigram_bounds(const int64_t *cn, int64_t V, int32_t *start);
// expTable (:614-618), host expf.
void w2b_exptable(float *out /*1000*/);
// Sub-sampling thresholds `ran` (:403-404), float32.
void w2b_keep_thresholds(const int64_t *cn, int64_t V, int64_t train_words, float sample, float *out /*V*/);
// Streaming mode: copy tokens [max(cursor,0), +L) of every unfinished shard into its slice stage[i*L ..) and
// report where the slice sits (xlate = global index - staging index, limit = global end, eof flag).  A plain
// memcpy of tens of MB per step, spread over a few host threads (nthreads <= 0: pick from the size).
void w2b_gather_slices(const int32_t *ids, long long n_tokens, long long L, int nshards, const long long *cursor,
                       const int *done, int32_t *stage, long long *xlate, long long *limit, int *limit_is_eof,
                       int nthreads);
// Text vector files (-binary 0, w2b_write_vectors(binary = 0)).  w2b_text_parse streams the first V rows of the file,
// whose first row holds D values (w2b_vector_file_info said W2B_VECTORS_TEXT), into the device table M (zeroed by the
// caller, rows Dp floats apart) on the current device, and returns each row's name as written ('\n' skipped).
// W2B_EIO names the row and token of a malformed file.  W2B_TEXT_CHUNK_BYTES (test hook) sets the chunk size.
int w2b_text_parse(const char *path, int64_t V, int64_t D, float *M, int64_t Dp, std::vector<std::string> &names);
// Row `row` of a text vector file, read on the host: its name and the bytes of its values (for error messages).
int w2b_text_row(const char *path, int64_t row, std::string &name, std::string &values);

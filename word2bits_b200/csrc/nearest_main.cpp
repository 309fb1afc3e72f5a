// nearest — the nearest word vectors of every word read from stdin, on the GPU (w2b_nearest).
//   ./nearest <FILE> [k=40] [bitlevel] [threshold] < words.txt
// FILE is a word2vec-binary vector file, a text one (`word2bits -binary 0`, parsed on the GPU) or a packed one
// (`word2bits -binary 2`).  Per query word it prints
// "<WORD>:" and then up to k lines "<rank>\t<WORD>\t<score>", or "<WORD>: not in vocabulary".
#include <ctype.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <unordered_map>
#include <vector>

#include "w2b.h"

// the names as the evaluator compares them: up to the first ' ', '\n' skipped, at most 50 characters, upper-cased
static bool read_names(const char *path, long long threshold, std::vector<std::string> &names) {
  int kind, bits;
  int64_t V, D, n = 0;
  if (w2b_vector_file_info(path, threshold, &kind, &V, &D, &bits) || V < 0) return false;
  std::vector<char> buf((size_t)(V > 0 ? V : 1) * 51);
  if (w2b_vector_names(path, threshold, buf.data(), 51, &n)) return false;
  for (int64_t i = 0; i < n; ++i) names.push_back(&buf[(size_t)i * 51]);
  return true;
}

int main(int argc, char **argv) {
  if (argc < 2) {
    printf("Usage: ./nearest <FILE> [k=40] [bitlevel] [threshold] < words.txt\nwhere FILE contains word projections "
           "(word2vec binary, text or packed), k is the length of every list (1..%d), bitlevel re-quantises an fp32 file "
           "as compute_accuracy does, and threshold restricts the vocabulary to its first words (0 = off)\n",
           W2B_MAX_TOPK);
    return 0;
  }
  const int k = argc > 2 ? atoi(argv[2]) : 40;
  const int bitlevel = argc > 3 ? atoi(argv[3]) : 0;
  const long long threshold = argc > 4 ? atoll(argv[4]) : 0;
  // the query words, kept to print them back (w2b_nearest reads them from a file)
  std::vector<std::string> words;
  char buf[2048];
  while (scanf("%2000s", buf) == 1) words.push_back(buf);
  char tmpl[] = "/tmp/nearest_wordsXXXXXX";
  const int fd = mkstemp(tmpl);
  FILE *tf = fd >= 0 ? fdopen(fd, "w") : nullptr;
  if (!tf) {
    printf("cannot create a temporary file\n");
    return -1;
  }
  for (const std::string &w : words) fprintf(tf, "%s\n", w.c_str());
  fclose(tf);
  std::vector<int32_t> ids(words.size() * (k > 0 ? k : 1));
  std::vector<float> scores(ids.size());
  int64_t n = 0;
  const int rc = w2b_nearest(argv[1], bitlevel, threshold, tmpl, k, 0, ids.data(), scores.data(), (int64_t)words.size(), &n,
                             nullptr);
  remove(tmpl);
  if (rc) {
    printf("%s\n", w2b_last_error());  // "Input file not found", as compute_accuracy prints it
    return -1;
  }
  std::vector<std::string> names;
  if (!read_names(argv[1], threshold, names)) {
    printf("Input file not found\n");
    return -1;
  }
  for (size_t i = 0; i < words.size(); ++i) {
    std::string w = words[i];
    for (auto &ch : w) ch = (char)toupper((unsigned char)ch);
    if (ids[i * k] < 0) {
      bool known = false;
      for (const std::string &v : names) known |= v == w;
      if (!known) {
        printf("%s: not in vocabulary\n", w.c_str());
        continue;
      }
    }
    printf("%s:\n", w.c_str());
    for (int j = 0; j < k && ids[i * k + j] >= 0; ++j)
      printf("%d\t%s\t%f\n", j + 1, names[ids[i * k + j]].c_str(), scores[i * k + j]);
  }
  return 0;
}

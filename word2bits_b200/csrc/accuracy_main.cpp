// compute_accuracy — drop-in for the reference's evaluator (src/compute-accuracy.c), scored on the GPU.
//   ./compute_accuracy <FILE> <bitlevel> <threshold> < questions-words.txt
// FILE is a word2vec-binary vector file (first line "words size"), a text one (`word2bits -binary 0`, the same first
// line, then "%lf " values; parsed on the GPU) or a packed one (`word2bits -binary 2`, first line "words size
// bitlevel"), which is scored as it is, in the bit domain; <bitlevel> is then the file's or absent.  Which of the three
// a file is, w2b_vector_file_info decides.
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "w2b.h"

int main(int argc, char **argv) {
  if (argc < 2) {  // :74-77
    printf("Usage: ./compute-accuracy <FILE> <bitlevel> <threshold>\nwhere FILE contains word projections (word2vec binary, text or packed), and threshold is used to reduce vocabulary of the model for fast approximate evaluation (0 = off, otherwise typical value is 30000)\n");
    return 0;
  }
  const int bitlevel = argc > 2 ? atoi(argv[2]) : 0;
  const long long threshold = argc > 3 ? atoll(argv[3]) : 0;
  std::vector<char> report(1 << 20);
  w2b_accuracy acc;
  int kind = W2B_VECTORS_BINARY, bits = 0;
  int64_t words, size;
  if (w2b_vector_file_info(argv[1], threshold, &kind, &words, &size, &bits)) kind = W2B_VECTORS_BINARY;  // not found: below
  const long long packed_bits = kind == W2B_VECTORS_PACKED ? bits : 0;
  if (packed_bits && bitlevel != 0 && bitlevel != packed_bits) {
    printf("%s holds %lld-bit vectors: <bitlevel> must be %lld, 0 or absent\n", argv[1], packed_bits, packed_bits);
    return -1;
  }
  const int rc = packed_bits
                     ? w2b_compute_accuracy_packed(argv[1], threshold, nullptr, 0, &acc, report.data(), (long long)report.size())
                     : w2b_compute_accuracy(argv[1], bitlevel, threshold, nullptr, 0, &acc, report.data(), (long long)report.size());
  if (rc) {
    printf("%s\n", w2b_last_error());  // "Input file not found" (:83)
    return -1;
  }
  fputs(report.data(), stdout);
  return 0;
}

// word2bits — drop-in command line for the H100 training path.
//
// Same flags, defaults, progress lines, exit codes and output files as the reference's main()
// / TrainModel() (src/word2bits.cpp:518-621).  Differences, all additive:
//   -threads N   number of corpus shards (one CUDA CTA each).  When the flag is absent the
//                shard count that fills the GPU is used instead of the reference's 12.
//   -gpu N       first CUDA device ordinal (default 0).
//   -gpus G      train on G GPUs (devices gpu..gpu+G-1): shards split in G blocks, full replicas,
//                NCCL all-reduce-average every -sync-every steps (default 4) and at every epoch end;
//                -sync-mode 1 sums every GPU's updates onto the common base instead of averaging.
//   -strict 1    parity mode: shards one after another, sequential IEEE arithmetic.
//   -binary 2    packed output: bitlevel bits per value (bitlevel 1 and 2), see w2b_write_packed.
//   -checkpoint F  write a resumable checkpoint (fp32 u, v, alpha, word counter) to F after every epoch.
//   -resume F      continue from checkpoint F at the epoch it was written after.
//   -eval FILE     after every epoch, evaluate the model as it stands on the analogy questions of FILE (the
//                  evaluator on the context's own tables, bitlevel 0) and print the last two lines of the report
//                  compute_accuracy prints on the epoch's vector file; -eval-threshold N = its <threshold> (default 0).
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <time.h>

#include <condition_variable>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "w2b.h"

// reusable barrier for the per-GPU host threads
class Barrier {
 public:
  explicit Barrier(int n) : n_(n) {}
  void wait() {
    std::unique_lock<std::mutex> lk(m_);
    const long gen = gen_;
    if (++count_ == n_) {
      count_ = 0;
      ++gen_;
      cv_.notify_all();
    } else {
      cv_.wait(lk, [&] { return gen_ != gen; });
    }
  }

 private:
  std::mutex m_;
  std::condition_variable cv_;
  int n_, count_ = 0;
  long gen_ = 0;
};

static int arg_pos(const char *str, int argc, char **argv) {  // ArgPos, :579-589
  for (int a = 1; a < argc; a++)
    if (!strcmp(str, argv[a])) {
      if (a == argc - 1) {
        printf("Argument missing for %s\n", str);
        exit(1);
      }
      return a;
    }
  return -1;
}

static void die(const char *what) {
  printf("%s: %s\n", what, w2b_last_error());
  exit(1);
}

static int g_bitlevel = 1;
static int write_vectors(const std::string &path, w2b_ctx *ctx, w2b_corpus *corpus, long long V, long long D,
                         int binary, std::vector<float> &buf) {
  if (w2b_export(ctx, buf.data())) return 1;
  if (binary == 2) return w2b_write_packed(path.c_str(), corpus, buf.data(), V, D, g_bitlevel);
  return w2b_write_vectors(path.c_str(), corpus, buf.data(), V, D, binary);
}

int main(int argc, char **argv) {
  int i;
  std::string train_file, output_file;
  int binary = 0, debug_mode = 2, window = 5, min_count = 5, num_threads = 0, bitlevel = 1, negative = 5;
  long long layer1_size = 100, iter = 5, classes = 0;
  bool save_every_epoch = false;
  float alpha = 0.05f, sample = 1e-3f, reg = 0;
  int device = 0, strict = 0;
  if ((i = arg_pos("-save-every-epoch", argc, argv)) > 0) save_every_epoch = atoi(argv[i + 1]);
  if ((i = arg_pos("-bitlevel", argc, argv)) > 0) bitlevel = atoi(argv[i + 1]);
  if ((i = arg_pos("-size", argc, argv)) > 0) layer1_size = atoi(argv[i + 1]);
  if ((i = arg_pos("-reg", argc, argv)) > 0) reg = atof(argv[i + 1]);
  if ((i = arg_pos("-train", argc, argv)) > 0) train_file = argv[i + 1];
  if ((i = arg_pos("-debug", argc, argv)) > 0) debug_mode = atoi(argv[i + 1]);
  if ((i = arg_pos("-binary", argc, argv)) > 0) binary = atoi(argv[i + 1]);
  if ((i = arg_pos("-alpha", argc, argv)) > 0) alpha = atof(argv[i + 1]);
  if ((i = arg_pos("-output", argc, argv)) > 0) output_file = argv[i + 1];
  if ((i = arg_pos("-window", argc, argv)) > 0) window = atoi(argv[i + 1]);
  if ((i = arg_pos("-sample", argc, argv)) > 0) sample = atof(argv[i + 1]);
  if ((i = arg_pos("-negative", argc, argv)) > 0) negative = atoi(argv[i + 1]);
  if ((i = arg_pos("-threads", argc, argv)) > 0) num_threads = atoi(argv[i + 1]);
  if ((i = arg_pos("-iter", argc, argv)) > 0) iter = atoi(argv[i + 1]);
  if ((i = arg_pos("-min-count", argc, argv)) > 0) min_count = atoi(argv[i + 1]);
  if ((i = arg_pos("-classes", argc, argv)) > 0) classes = atoi(argv[i + 1]);
  if ((i = arg_pos("-gpu", argc, argv)) > 0) device = atoi(argv[i + 1]);
  if ((i = arg_pos("-strict", argc, argv)) > 0) strict = atoi(argv[i + 1]);
  std::string ckpt_file, resume_file;
  if ((i = arg_pos("-checkpoint", argc, argv)) > 0) ckpt_file = argv[i + 1];
  if ((i = arg_pos("-resume", argc, argv)) > 0) resume_file = argv[i + 1];
  g_bitlevel = bitlevel;
  int ngpus = 1, sync_every = 4;
  if ((i = arg_pos("-gpus", argc, argv)) > 0) ngpus = atoi(argv[i + 1]);
  if ((i = arg_pos("-sync-every", argc, argv)) > 0) sync_every = atoi(argv[i + 1]);
  int sync_mode = 0;  // 0 = average the replicas, 1 = sum every GPU's updates onto the common base
  if ((i = arg_pos("-sync-mode", argc, argv)) > 0) sync_mode = atoi(argv[i + 1]);
  if (ngpus < 1) ngpus = 1;
  if (sync_every < 1) sync_every = 1;
  std::string eval_file;
  long long eval_threshold = 0;
  if ((i = arg_pos("-eval", argc, argv)) > 0) eval_file = argv[i + 1];
  if ((i = arg_pos("-eval-threshold", argc, argv)) > 0) eval_threshold = atoll(argv[i + 1]);
  if (!eval_file.empty()) {  // checked now rather than after an epoch of training
    FILE *f = fopen(eval_file.c_str(), "rb");
    if (!f) {
      printf("ERROR: questions file %s not found!\n", eval_file.c_str());
      exit(1);
    }
    fclose(f);
  }

  printf("Starting training using file %s\n", train_file.c_str());  // :523
  w2b_corpus *corpus = nullptr;
  if (w2b_corpus_load(train_file.c_str(), min_count, &corpus)) {
    printf("%s\n", w2b_last_error());  // "ERROR: training data file not found!" (:272)
    exit(1);
  }
  const long long V = w2b_corpus_vocab_size(corpus);
  const long long train_words = w2b_corpus_train_words(corpus);
  if (debug_mode > 0) {  // :295-298
    printf("Vocab size: %lld\n", V);
    printf("Words in train file: %lld\n", train_words);
  }
  if (output_file.empty()) return 0;  // :527

  w2b_config cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.vocab_size = V;
  cfg.layer1_size = layer1_size;
  cfg.window = window;
  cfg.negative = negative;
  cfg.bitlevel = bitlevel;
  cfg.alpha = alpha;
  cfg.sample = sample;
  cfg.reg = reg;
  cfg.iter = iter;
  cfg.device = device;
  cfg.mode = strict ? W2B_MODE_STRICT : W2B_MODE_FAST;
  cfg.sync_mode = sync_mode == 1 ? 1 : 0;
  cfg.num_shards = num_threads > 0 ? num_threads : 1;
  if (num_threads <= 0) {
    int s = 0;
    if (w2b_suggest_shards(&cfg, &s)) die("w2b_suggest_shards");
    // every shard is a concurrent Hogwild worker: on a small corpus too many of them cost quality (tests/tools/
    // quality_planted.py measures kNN purity against the shard count), so keep at least ~20 k words per shard
    s *= ngpus;
    while (s > ngpus && train_words / s < 20000) s /= 2;
    cfg.num_shards = s;
  }
  if (strict && ngpus > 1) {
    printf("-strict 1 runs on one GPU\n");
    exit(1);
  }
  if (cfg.num_shards < ngpus) {
    printf("-threads must be at least -gpus\n");
    exit(1);
  }
  // ---- one host thread per GPU (rank); each owns a contiguous block of shards on a full replica of
  // u/v; replicas are all-reduce-averaged every `sync_every` steps and at every epoch end (w2b_sync)
  const int G = ngpus;
  std::vector<int64_t> start(cfg.num_shards);
  std::vector<int32_t> first(cfg.num_shards);
  if (w2b_corpus_shards(corpus, cfg.num_shards, start.data(), first.data())) die("w2b_corpus_shards");
  unsigned char uid[128] = {0};
  if (G > 1 && w2b_nccl_unique_id(uid)) die("w2b_nccl_unique_id");
  Barrier bar(G);
  std::mutex mu;
  double epoch_loss = 0;
  long long words_done = 0, words_at_start = 0, step_words = 0;
  int ranks_busy = 0;
  struct timespec t0;
  clock_gettime(CLOCK_MONOTONIC, &t0);

  auto worker = [&](int rank) {
    w2b_config c = cfg;
    c.device = device + rank;
    c.shard_begin = (int)((long long)cfg.num_shards * rank / G);
    c.shard_end = (int)((long long)cfg.num_shards * (rank + 1) / G);
    const int nlocal = c.shard_end - c.shard_begin;
    w2b_ctx *ctx = nullptr;
    if (w2b_create(&c, &ctx)) {
      if (strstr(w2b_last_error(), "cudaMalloc")) printf("Memory allocation failed\n");  // :347
      die("w2b_create");
    }
    if (w2b_set_vocab_counts(ctx, w2b_corpus_counts(corpus), V, train_words)) die("w2b_set_vocab_counts");
    if (w2b_set_corpus(ctx, w2b_corpus_tokens(corpus), w2b_corpus_num_tokens(corpus), start.data(), first.data(), 1))
      die("w2b_set_corpus");
    if (w2b_init_tables(ctx)) die("w2b_init_tables");
    long long first_epoch = 0;
    if (!resume_file.empty()) {
      int64_t done = 0;
      if (w2b_checkpoint_load(ctx, resume_file.c_str(), &done)) die("w2b_checkpoint_load");
      first_epoch = done;
      if (rank == 0) {  // Progress % continues from the checkpoint's word counter
        float a0 = 0;
        int64_t wca = 0;
        if (w2b_get_state(ctx, &a0, &wca)) die("w2b_get_state");
        std::lock_guard<std::mutex> lk(mu);
        words_done = words_at_start = wca;
      }
    }
    if (G > 1 && w2b_nccl_init(ctx, uid, rank, G)) die("w2b_nccl_init");  // (after the tables hold their starting point)
    std::vector<float> buf;
    if (rank == 0) buf.resize((size_t)V * layer1_size);
    std::vector<const char *> names;  // row names for -eval
    std::vector<char> report;
    if (rank == 0 && !eval_file.empty()) {
      for (long long w = 0; w < V; ++w) names.push_back(w2b_corpus_word(corpus, w));
      report.resize(1 << 20);  // compute_accuracy's report buffer
    }
    for (int iteration = (int)first_epoch; iteration < iter; iteration++) {
      if (rank == 0) {
        printf("Starting epoch: %d\n", iteration);  // :533
        epoch_loss = 0;
      }
      if (w2b_epoch_begin(ctx)) die("w2b_epoch_begin");
      bar.wait();
      for (long long step = 1;; ++step) {
        w2b_step_stats st;
        // 50k words per shard per step: progress lines 5x less often than the reference (:379), steps
        // long enough that the whole-sentence overshoot at a step boundary (<= ~1.2k words) stays ~1 %.
        // Several GPUs: replicas must meet often enough to stay one model — at least ~32 steps per epoch
        // (sync_every of them between two averages), but never steps shorter than a couple of sentences.
        long long per_step = 50000;
        if (G > 1) per_step = std::max<long long>(2000, std::min<long long>(50000, train_words / cfg.num_shards / 32));
        if (w2b_train_step(ctx, (debug_mode > 1 || G > 1) ? per_step : 0, &st)) die("w2b_train_step");
        {
          std::lock_guard<std::mutex> lk(mu);
          epoch_loss += st.loss;
          words_done += st.words;
          step_words += st.words;
          if (st.shards_done < nlocal) ++ranks_busy;
        }
        bar.wait();  // every rank sees the same ranks_busy: collectives stay aligned
        const bool more = ranks_busy > 0;
        if (G > 1 && (step % sync_every == 0 || !more) && w2b_sync(ctx)) die("w2b_sync");
        if (rank == 0 && debug_mode > 1) {
          // :384-387, same line format.  The reference divides by clock(), the CPU time of ALL its threads, i.e. it
          // prints words per worker-second; here a worker is a shard: words / (wall seconds x shards)
          struct timespec now;
          clock_gettime(CLOCK_MONOTONIC, &now);
          double secs = (now.tv_sec - t0.tv_sec) + (now.tv_nsec - t0.tv_nsec) * 1e-9;
          printf("%cAlpha: %f  Progress: %.2f%%  Cost: %f Words/thread/sec: %.2fk  ", 13, st.alpha,
                 words_done / (float)(iter * train_words + 1) * 100, st.loss,
                 (words_done - words_at_start) / (secs + 1e-9) / 1000 / cfg.num_shards);
          fflush(stdout);
        }
        bar.wait();
        if (rank == 0) ranks_busy = 0;
        bar.wait();
        if (!more) break;
      }
      if (rank == 0) {
        printf("Epoch Loss: %lf\n", epoch_loss);  // :539
        if (!eval_file.empty()) {  // (several GPUs: the epoch's last exchange has made the replicas equal)
          w2b_accuracy acc;
          if (w2b_ctx_compute_accuracy(ctx, names.data(), 0, eval_threshold, eval_file.c_str(), &acc, report.data(),
                                       (int64_t)report.size()))
            die("w2b_ctx_compute_accuracy");
          // the report's last two lines: "Total accuracy: ..." and "Questions seen / total: ..."
          const std::string text(report.data());
          size_t from = text.size();
          int newlines = 0;
          while (from > 0 && !(text[from - 1] == '\n' && ++newlines == 3)) --from;
          fputs(text.c_str() + from, stdout);
          fflush(stdout);
        }
        if (!ckpt_file.empty() && w2b_checkpoint_save(ctx, ckpt_file.c_str(), iteration + 1)) die("w2b_checkpoint_save");
        if (classes == 0 && save_every_epoch) {  // :540-557
          char name[4200];
          snprintf(name, sizeof name, "%s_epoch%d", output_file.c_str(), iteration);
          if (write_vectors(name, ctx, corpus, V, layer1_size, binary, buf)) die("write");
        }
      }
      bar.wait();
    }
    if (rank == 0) {
      if (classes == 0) {  // :560-576
        if (write_vectors(output_file, ctx, corpus, V, layer1_size, binary, buf)) die("write");
      } else {
        FILE *fo = fopen(output_file.c_str(), "wb");  // the reference creates an empty file (:561-562)
        if (fo) fclose(fo);
      }
    }
    bar.wait();
    w2b_destroy(ctx);
  };
  std::vector<std::thread> threads;
  for (int r = 1; r < G; ++r) threads.emplace_back(worker, r);
  worker(0);
  for (auto &t : threads) t.join();
  w2b_corpus_free(corpus);
  return 0;
}

// TEST INFRASTRUCTURE — runs the product's production kernel (train_warp_kernel, compiled from
// word2bits_b200/csrc/w2b_warp.cuh with -DW2B_EMULATE) on the CPU: one fiber per CUDA thread, one CTA (= one
// corpus shard) after another.  Purpose: functional verification of the kernel without a GPU — same
// source, same control flow, same index arithmetic and protocol; only the PTX wrappers and the intrinsics are
// host code.  It is not a timing model and not a fallback: nothing under word2bits_b200/ references it.
#include <stdio.h>
#include <stdlib.h>
#include <sys/mman.h>

#include <algorithm>
#include <random>
#include <vector>

#include "w2b_warp.cuh"

uint3 threadIdx, blockIdx;
dim3 blockDim, gridDim;
namespace w2b {
alignas(128) unsigned char smem[256 * 1024];
}

// ------------------------------------------------------------------------------ fibers
extern "C" void emu_switch(void **save_sp, void *load_sp);
asm(R"(
.text
.globl emu_switch
.type emu_switch,@function
emu_switch:
  pushq %rbp
  pushq %rbx
  pushq %r12
  pushq %r13
  pushq %r14
  pushq %r15
  movq %rsp, (%rdi)
  movq %rsi, %rsp
  popq %r15
  popq %r14
  popq %r13
  popq %r12
  popq %rbx
  popq %rbp
  ret
.size emu_switch,.-emu_switch
)");

namespace {

struct BulkOp { float *dst; unsigned src_off, bytes; };
struct Fiber {
  void *sp = nullptr;
  char *stack = nullptr;
  bool done = false;
  std::vector<BulkOp> open;
  std::vector<std::vector<BulkOp>> groups;
  std::vector<unsigned> unfenced;  // 16-byte chunks this thread stored to since its last fence.proxy.async
};
constexpr size_t kStack = 256 * 1024;
std::vector<Fiber> g_fib;
void *g_sched_sp = nullptr;
int g_cur = -1;
void (*g_entry)() = nullptr;
std::mt19937_64 g_rng;
int g_async_mode = 0;
int g_fault = 0;  // negative controls of the checkers: 1 = fence.proxy.async dropped, 2 = wait_group.read returns early
const char *g_error = nullptr;
unsigned long long g_progress = 0;  // bumped by everything except spinning: lets the scheduler tell a dead-lock from work

struct WarpX { unsigned long long gen = 0; int arrived = 0, op = -1, arg = 0; uint64_t val[32], res[32]; };
std::vector<WarpX> g_warp;
struct BlockBar { unsigned long long gen = 0; int arrived = 0; };
BlockBar g_bar[16];
struct MBar { int count = 0, pending = 0; long long tx = 0; unsigned phase = 0; bool init = false, unobserved = false; };
std::vector<MBar> g_mbar(sizeof(w2b::smem) / 8);
struct Load { unsigned dst_off, bytes, bar_off; const void *src; };
std::vector<Load> g_loads;

void fail(const char *msg) {
  if (!g_error) g_error = msg;
}

// planned carve-up of the running CTA (ring_layout of the launch geometry): bounds of the checked accesses
size_t g_smem_total = sizeof(w2b::smem), g_rows_end = 0, g_ring_end = 0;
unsigned g_rowb = 0;
// per 16-byte chunk: 1 + id of the thread whose generic-proxy store has not been fenced yet (0 = none)
std::vector<unsigned short> g_unfenced(sizeof(w2b::smem) / 16, 0);
// per row of the row regions: bulk reduces issued or committed whose source it is and that have not executed
std::vector<int> g_pending_rows;
void pending_rows_add(const BulkOp &op, int delta) {
  if (!g_rowb) return;
  for (unsigned r = op.src_off / g_rowb; r <= (op.src_off + op.bytes - 1) / g_rowb && r < g_pending_rows.size(); ++r)
    g_pending_rows[r] += delta;
}

void fiber_trampoline() {
  g_entry();
  g_fib[g_cur].done = true;
  emu_switch(&g_fib[g_cur].sp, g_sched_sp);
  abort();  // a finished fiber is never resumed
}

void make_fiber(Fiber &f) {
  if (!f.stack) f.stack = (char *)mmap(nullptr, kStack, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
  f.done = false;
  f.open.clear();
  f.groups.clear();
  f.unfenced.clear();
  // initial frame: six callee-saved registers, then the return address of emu_switch's `ret`; the stack is
  // 16-byte aligned at the trampoline's entry as the ABI wants after a call
  void **top = (void **)(f.stack + kStack - 64);
  top = (void **)((uintptr_t)top & ~(uintptr_t)15);
  *--top = nullptr;                       // fake return address of the trampoline (alignment)
  *--top = (void *)fiber_trampoline;      // `ret` target
  for (int i = 0; i < 6; ++i) *--top = nullptr;
  f.sp = top;
}

void complete_tx(unsigned bar_off, unsigned bytes) {
  MBar &m = g_mbar[bar_off / 8];
  m.tx -= bytes;
  if (m.pending == 0 && m.tx == 0) { m.phase ^= 1; m.pending = m.count; m.unobserved = true; }
}
void land(const Load &l) {
  ++g_progress;
  memcpy(w2b::smem + l.dst_off, l.src, l.bytes);
  complete_tx(l.bar_off, l.bytes);
}
void exec_group(std::vector<BulkOp> &g) {
  ++g_progress;
  for (const BulkOp &op : g) {  // the source is read NOW: whatever the slot holds at this moment is what gets added
    const float *src = (const float *)(w2b::smem + op.src_off);
    for (unsigned i = 0; i < op.bytes / 4; ++i) op.dst[i] += src[i];
    pending_rows_add(op, -1);
  }
  g.clear();
}

}  // namespace

void emu_yield() {
  Fiber &f = g_fib[g_cur];
  emu_switch(&f.sp, g_sched_sp);
}

uint64_t emu_warp_exchange(uint64_t v, int op, int arg) {
  const int tid = (int)threadIdx.x, lane = tid & 31;
  WarpX &w = g_warp[tid >> 5];
  if (w.arrived == 0) { w.op = op; w.arg = arg; }
  else if (w.op != op || (op != EMU_SHFL_IDX && w.arg != arg)) fail("lanes of a warp reached different collectives");
  w.val[lane] = v;
  const unsigned long long my = w.gen;
  if (++w.arrived == 32) {
    ++g_progress;
    unsigned ballot = 0;
    for (int l = 0; l < 32; ++l) ballot |= (w.val[l] ? 1u : 0u) << l;
    for (int l = 0; l < 32; ++l) {
      switch (op) {
        case EMU_SHFL_XOR: w.res[l] = w.val[l ^ arg]; break;
        case EMU_SHFL_IDX: w.res[l] = w.val[arg & 31]; break;  // all call sites use a warp-uniform source lane
        case EMU_BALLOT: w.res[l] = ballot; break;
        default: w.res[l] = 0;
      }
    }
    w.arrived = 0;
    ++w.gen;
  } else {
    while (w.gen == my) emu_yield();
  }
  return w.res[lane];
}

void emu_block_barrier(int id, int nthreads) {
  BlockBar &b = g_bar[id];
  const unsigned long long my = b.gen;
  if (++b.arrived == nthreads) { b.arrived = 0; ++b.gen; ++g_progress; }
  else while (b.gen == my) emu_yield();
}

namespace w2b {
void emu_check_smem(unsigned off, unsigned bytes, const char *what) {
  static char msg[160];
  if (g_error) return;  // keep the first report
  if ((size_t)off + bytes > g_smem_total) {
    snprintf(msg, sizeof msg, "%s at shared offset %u (+%u) beyond the planned %zu bytes", what, off, bytes, g_smem_total);
    fail(msg);
  } else if (off < g_rows_end && g_rowb && off % g_rowb + bytes > g_rowb) {
    snprintf(msg, sizeof msg, "%s at shared offset %u (+%u) crosses a row boundary (rows of %u bytes)", what, off, bytes, g_rowb);
    fail(msg);
  }
}
static bool pending_reduce_reads(unsigned off, unsigned bytes) {  // issued or committed, not yet executed
  if (!g_rowb || off >= g_rows_end) return false;
  for (unsigned r = off / g_rowb; r <= (off + bytes - 1) / g_rowb && r < g_pending_rows.size(); ++r)
    if (g_pending_rows[r] > 0) return true;
  return false;
}
void emu_generic_store(unsigned off, unsigned bytes) {
  if (g_error) return;
  if (pending_reduce_reads(off, bytes)) { fail("store into the source of a bulk reduce that has not been confirmed read (wait_group.read)"); return; }
  Fiber &f = g_fib[g_cur];
  for (unsigned c = off / 16; c <= (off + bytes - 1) / 16; ++c) {
    g_unfenced[c] = (unsigned short)(g_cur + 1);
    f.unfenced.push_back(c);
  }
}
void emu_fence_async() {
  if (g_fault == 1) return;
  Fiber &f = g_fib[g_cur];
  for (unsigned c : f.unfenced)
    if (g_unfenced[c] == (unsigned short)(g_cur + 1)) g_unfenced[c] = 0;
  f.unfenced.clear();
}
void emu_mbar_init(unsigned off, int count) {
  emu_check_smem(off, 8, "mbarrier.init");
  if (off < g_rows_end) fail("mbarrier inside the row regions");
  MBar &m = g_mbar[off / 8];
  m = MBar();
  m.count = m.pending = count;
  m.init = true;
}
void emu_mbar_expect_tx(unsigned off, unsigned bytes) {
  MBar &m = g_mbar[off / 8];
  if (!m.init) fail("expect_tx on an uninitialised mbarrier");
  if (m.pending <= 0) fail("mbarrier armed twice in one phase");
  // what compute-sanitizer's synccheck calls "Missing wait": a phase completed and the barrier is armed for the next
  // one although no thread ever waited for it (harmless for the hardware, but every job is expected to wait)
  if (m.unobserved) fail("mbarrier armed again although no thread waited for its previous phase");
  ++g_progress;
  m.tx += bytes;
  m.pending -= 1;
  if (m.pending == 0 && m.tx == 0) { m.phase ^= 1; m.pending = m.count; m.unobserved = true; }
}
bool emu_mbar_try_wait(unsigned off, unsigned parity) {
  MBar &m = g_mbar[off / 8];
  const bool done = (m.phase & 1u) != (parity & 1u);  // the phase with this parity has completed
  if (done) m.unobserved = false;
  return done;
}
void emu_bulk_load(unsigned dst_off, const void *src, unsigned bytes, unsigned bar_off) {
  if (bytes % 16 || dst_off % 16 || ((uintptr_t)src) % 16) fail("bulk copy operands must be 16-byte aligned");
  emu_check_smem(dst_off, bytes, "cp.async.bulk (load)");
  emu_check_smem(bar_off, 8, "cp.async.bulk mbarrier");
  if (dst_off >= g_ring_end || dst_off % g_rowb || bytes != g_rowb) fail("bulk load is not one whole row into a ring slot");
  if (pending_reduce_reads(dst_off, bytes)) fail("bulk load into the source of a bulk reduce that has not been confirmed read");
  Load l{dst_off, bytes, bar_off, src};
  if (g_async_mode == 0) land(l);
  else g_loads.push_back(l);
}
void emu_bulk_reduce_add(void *dst, unsigned src_off, unsigned bytes) {
  if (bytes % 16 || src_off % 16 || ((uintptr_t)dst) % 16) fail("bulk reduce operands must be 16-byte aligned");
  emu_check_smem(src_off, bytes, "cp.reduce.async.bulk");
  if (src_off >= g_rows_end) fail("bulk reduce source outside the row regions");
  for (unsigned c = src_off / 16; c < (src_off + bytes) / 16 && !g_error; ++c)
    if (g_unfenced[c]) fail("bulk reduce reads bytes stored through the generic proxy without the storing thread's fence.proxy.async");
  ++g_progress;
  g_fib[g_cur].open.push_back(BulkOp{(float *)dst, src_off, bytes});
  pending_rows_add(g_fib[g_cur].open.back(), +1);
}
void emu_bulk_commit() {
  Fiber &f = g_fib[g_cur];
  f.groups.push_back(std::move(f.open));
  f.open.clear();
}
void emu_bulk_wait(int keep) {
  if (g_fault == 2) return;
  Fiber &f = g_fib[g_cur];
  while ((int)f.groups.size() > keep) {
    exec_group(f.groups.front());
    f.groups.erase(f.groups.begin());
  }
}
}  // namespace w2b

namespace {

// runs one CTA to completion; false on deadlock / protocol error
bool run_block(int nthreads, void (*entry)()) {
  g_entry = entry;
  g_fib.resize(std::max<size_t>(g_fib.size(), nthreads));
  g_warp.assign((nthreads + 31) / 32, WarpX());
  for (auto &b : g_bar) b = BlockBar();
  for (auto &m : g_mbar) m = MBar();
  std::fill(g_unfenced.begin(), g_unfenced.end(), 0);
  g_pending_rows.assign(g_rowb ? g_rows_end / g_rowb + 1 : 0, 0);
  g_loads.clear();
  for (int t = 0; t < nthreads; ++t) make_fiber(g_fib[t]);
  blockDim.x = nthreads;
  int live = nthreads;
  unsigned long long idle_rounds = 0, seen = g_progress;
  std::vector<int> order(nthreads);
  for (int t = 0; t < nthreads; ++t) order[t] = t;
  while (live > 0) {
    if (g_error) return false;
    if (g_progress != seen) { seen = g_progress; idle_rounds = 0; }
    else if (++idle_rounds > 20000) { fail("no progress: the CTA dead-locked"); return false; }
    if (g_async_mode) {  // asynchronous engines: a pending load lands, a committed reduce group is executed early
      for (size_t i = 0; i < g_loads.size();)
        if (g_rng() % 4 == 0) { land(g_loads[i]); g_loads[i] = g_loads.back(); g_loads.pop_back(); }
        else ++i;
      if (g_rng() % 8 == 0) {
        Fiber &f = g_fib[g_rng() % nthreads];
        if (!f.groups.empty()) { exec_group(f.groups.front()); f.groups.erase(f.groups.begin()); }
      }
      if (g_async_mode == 2)  // shuffled scheduling order as well
        for (int t = nthreads - 1; t > 0; --t) std::swap(order[t], order[g_rng() % (t + 1)]);
    }
    for (int k = 0; k < nthreads; ++k) {
      const int t = order[k];
      Fiber &f = g_fib[t];
      if (f.done) continue;
      g_cur = t;
      threadIdx.x = t; threadIdx.y = threadIdx.z = 0;
      emu_switch(&g_sched_sp, f.sp);
      if (f.done) {
        --live;
        ++g_progress;
        if (!f.open.empty()) fail("thread exited with uncommitted bulk operations");
        for (auto &g : f.groups) exec_group(g);  // (the kernel ends with wait_group 0; harmless otherwise)
        f.groups.clear();
      }
    }
  }
  if (!g_loads.empty()) fail("bulk loads still in flight at kernel end");
  return g_error == nullptr;
}

w2b::TrainParams g_p;
int g_nu, g_nv, g_sen_smem = 1;
typedef void (*entry_fn)();
template <int BM, int NJ>
void warp_entry() {
  w2b::ApplyArgs none;
  memset(&none, 0, sizeof none);
  if (g_p.reg != 0.f) w2b::train_warp_kernel<9, NJ, 8, 1>(g_p, g_nv, g_nu | (g_sen_smem << 31), none);
  else w2b::train_warp_kernel<BM, NJ, 12>(g_p, g_nv, g_nu | (g_sen_smem << 31), none);
}
template <int BM>
entry_fn warp_by_nj(int nj) {
  switch (nj) {
    case 1: return warp_entry<BM, 1>;
    case 2: return warp_entry<BM, 2>;
    case 3: return warp_entry<BM, 3>;
    case 4: return warp_entry<BM, 4>;
    case 5: return warp_entry<BM, 5>;
    case 6: return warp_entry<BM, 6>;
    case 7: return warp_entry<BM, 7>;
    case 8: return warp_entry<BM, 8>;
    case 10: return warp_entry<BM, 10>;
    case 12: return warp_entry<BM, 12>;
    case 16: return warp_entry<9, 16>;
  }
  return nullptr;
}

}  // namespace

extern "C" {

struct EmuRun {
  int64_t V, D;
  int32_t window, negative, bitlevel;
  float sample, alpha0;
  int64_t iter, train_words;
  int32_t num_shards;
  int32_t opt, lpr, xw, nu, nv, G, threads, serial;
  float *u, *v;
  const int32_t *table;
  const float *keep, *exptab;
  const int32_t *tokens;
  int64_t n_tokens;
  const int64_t *shard_start;
  const int32_t *shard_first;
  float *alpha;
  uint64_t *wca;
  int64_t word_budget, max_iters;
  uint64_t seed;
  int32_t async_mode, train;
  double *loss;
  int64_t *words, *n_pos, *n_ctx, *n_tgt;
  int32_t *done;
  w2b_trace_rec *trace;  // per shard, as w2b_train_step_traced lays it out: shard i's records at trace[i * trace_cap ..),
  int64_t trace_cap;     // their count in trace_n[i] (num_shards entries)
  uint64_t *trace_n;
  int32_t only_shard;  // >= 0: run just this shard
  int32_t fault;       // 0; 1 / 2: injected protocol faults (negative controls, see g_fault)
  float reg;           // -reg
};

const char *emu_last_error() { return g_error ? g_error : ""; }

// the kernel's division-free context average (w2b::div_by_count) on n numerators: out[i] = a[i] / cw
void emu_div_by_count(const float *a, int n, int cw, float *out) {
  const float fcw = (float)cw, rc = __frcp_rn(fcw);
  for (int i = 0; i + 1 < n; i += 2) {
    const w2b::F2 q = w2b::div_by_count(w2b::F2{a[i], a[i + 1]}, fcw, rc);
    out[i] = q.x;
    out[i + 1] = q.y;
  }
}

// negative control of the shared-memory checks: would an access of `bytes` at `off` be reported under the
// carve-up of the last run?  (returns the planned total through *total)
int emu_check_probe(unsigned off, unsigned bytes, uint64_t *total) {
  g_error = nullptr;
  w2b::emu_check_smem(off, bytes, "probe");
  if (total) *total = g_smem_total;
  const int bad = g_error != nullptr;
  g_error = nullptr;
  return bad;
}

static void emu_setup(const EmuRun *r, std::vector<w2b::ShardState> &shards, w2b::TrainParams &p) {
  using namespace w2b;
  g_error = nullptr;
  g_rng.seed(r->seed);
  g_async_mode = r->async_mode;
  g_fault = r->fault;
  // LCG jump tables (csrc/w2b_cuda.cu: lcg_tables)
  c_JA[0] = 1; c_JC[0] = 0;
  for (int k = 1; k <= 64; ++k) { c_JA[k] = c_JA[k - 1] * kLcgA; c_JC[k] = c_JC[k - 1] * kLcgA + kLcgC; }
  c_PA[0] = kLcgA; c_PC[0] = kLcgC;
  for (int j = 1; j < 64; ++j) { c_PA[j] = c_PA[j - 1] * c_PA[j - 1]; c_PC[j] = c_PA[j - 1] * c_PC[j - 1] + c_PC[j - 1]; }
  memcpy(c_exptab, r->exptab, sizeof(float) * kExpN);
  shards.assign(r->num_shards, ShardState());
  for (int i = 0; i < r->num_shards; ++i) {  // csrc/w2b_cuda.cu: w2b_epoch_begin
    ShardState &s = shards[i];
    memset(&s, 0, sizeof s);
    s.rng = (unsigned long long)(long long)i;
    const bool ovr = r->shard_first[i] >= 0;
    s.cursor = ovr ? r->shard_start[i] - 1 : r->shard_start[i];
    s.ovr_idx = ovr ? r->shard_start[i] - 1 : -2;
    s.ovr_tok = ovr ? r->shard_first[i] : -1;
    s.limit = r->n_tokens;
    s.limit_is_eof = 1;
  }
  memset(&p, 0, sizeof p);
  p.u = r->u; p.v = r->v; p.table = r->table; p.keep_thr = r->keep; p.exptab = r->exptab; p.tokens = r->tokens;
  p.shards = shards.data(); p.alpha = r->alpha; p.wca = (unsigned long long *)r->wca;
  p.D = r->D; p.V = r->V; p.pitch = (r->D + 3) & ~3LL; p.ncol = (int)(p.pitch / 4); p.window = r->window; p.negative = r->negative; p.bitlevel = r->bitlevel;
  p.sample = r->sample; p.reg = r->reg; p.starting_alpha = r->alpha0;
  p.alpha_denom = (float)(r->iter * r->train_words + 1);
  p.shard_word_limit = r->train_words / r->num_shards;
  p.word_budget = r->word_budget; p.max_iters = r->max_iters; p.shard_base = 0; p.train = r->train;
  p.serial = r->serial; p.wca_scale = 1;
  p.trace = r->trace; p.trace_cap = r->trace_cap; p.trace_n = (unsigned long long *)r->trace_n; p.trace_per_shard = 1;
}

static void emu_results(const EmuRun *r, const std::vector<w2b::ShardState> &shards) {
  for (int i = 0; i < r->num_shards; ++i) {
    r->loss[i] = shards[i].loss; r->words[i] = shards[i].word_count; r->n_pos[i] = (int64_t)shards[i].n_pos;
    r->n_ctx[i] = (int64_t)shards[i].n_ctx; r->n_tgt[i] = (int64_t)shards[i].n_tgt; r->done[i] = shards[i].done;
  }
}

// The warp-per-shard kernel (csrc/w2b_warp.cuh): r->nv = ring slots K, r->nu = job queue capacity; one 32-thread
// CTA per shard, one after another.
int emu_run_warp(const EmuRun *r) {
  using namespace w2b;
  std::vector<ShardState> shards;
  TrainParams p;
  emu_setup(r, shards, p);
  const int nj = ((int)(p.pitch / 4) + 31) / 32;  // (u, v: rows of p.pitch floats, padding zero)
  entry_fn fn = nullptr;
  switch (r->bitlevel) {
    case 0: fn = warp_by_nj<0>(nj); break;
    case 1: fn = warp_by_nj<1>(nj); break;
    case 2: fn = warp_by_nj<2>(nj); break;
    default: fn = warp_by_nj<9>(nj); break;
  }
  if (!fn) { fail("no emulated instantiation for this shape"); return 1; }
  std::vector<int> sen((size_t)kMaxS * (r->num_shards + 1));
  p.sen = sen.data();
  g_sen_smem = r->lpr == 32 ? 1 : 0;  // r->lpr: 32 = sentence buffer in shared memory, anything else = global
  g_p = p; g_nv = r->nv; g_nu = r->nu;
  {
    const WarpLayout L = warp_layout(p.pitch, r->nv, r->nu, g_sen_smem);
    if (L.total > sizeof(w2b::smem)) { fail("planned shared memory exceeds the emulator's buffer"); return 1; }
    g_smem_total = L.total;
    g_rows_end = (size_t)r->nv * L.rowb;  // the ring: rows of 4*D bytes from offset 0
    g_ring_end = g_rows_end;
    g_rowb = (unsigned)L.rowb;
  }
  gridDim.x = r->num_shards;
  for (int b = 0; b < r->num_shards; ++b) {
    if (r->only_shard >= 0 && b != r->only_shard) continue;
    blockIdx.x = b; blockIdx.y = blockIdx.z = 0;
    if (!run_block(32, fn)) return 2;
  }
  emu_results(r, shards);
  return 0;
}
}

// Shared definitions for the visdial_b200 engine (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <functional>
#include <string>
#include <stdexcept>
#include <vector>
#include <map>

namespace vd {

struct CudaError : std::runtime_error {
  int code;
  CudaError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define VD_CUDA_CHECK(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      char _buf[512];                                                                    \
      snprintf(_buf, sizeof(_buf), "%s:%d: %s -> %s", __FILE__, __LINE__, #expr,         \
               cudaGetErrorString(_e));                                                  \
      (void)cudaGetLastError(); /* a refused call must not fail the next check_launch */ \
      throw vd::CudaError(_e == cudaErrorMemoryAllocation ? -5 : -3, _buf);              \
    }                                                                                    \
  } while (0)

#define VD_REQUIRE(cond, code, msg)                                                      \
  do {                                                                                   \
    if (!(cond)) {                                                                       \
      char _buf[512];                                                                    \
      snprintf(_buf, sizeof(_buf), "%s:%d: %s (%s)", __FILE__, __LINE__, msg, #cond);    \
      throw vd::CudaError(code, _buf);                                                   \
    }                                                                                    \
  } while (0)

// ---------------------------------------------------------------------------------------------
// Dropout RNG: Philox4x32-10, counter = (q_lo, q_hi, site, iteration), key = (seed_lo, seed_hi),
// q = element_index / 4, word = element_index % 4.  keep <=> word >= thresh (thresh = p * 2^32).
// The numpy twin used by the tests is oracle/philox.py.
// ---------------------------------------------------------------------------------------------
struct DropCfg {
  uint32_t seed_lo, seed_hi, iter, thresh;  // thresh == 0 -> dropout disabled (identity)
  float scale;                              // 1 / (1 - p)
};

__host__ __device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2,
                                                       uint32_t c3, uint32_t k0, uint32_t k1,
                                                       uint32_t out[4]) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = (uint64_t)M0 * c0, p1 = (uint64_t)M1 * c2;
    uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
    uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += W0; k1 += W1;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// multiplicative factor (0 or scale) of element `idx` at dropout site `site`
__device__ __forceinline__ float drop_factor(const DropCfg& d, uint32_t site, uint64_t idx) {
  if (d.thresh == 0) return 1.f;
  uint64_t q = idx >> 2;
  uint32_t o[4];
  philox4x32_10((uint32_t)q, (uint32_t)(q >> 32), site, d.iter, d.seed_lo, d.seed_hi, o);
  return o[idx & 3] >= d.thresh ? d.scale : 0.f;
}
// factors of the 4 elements idx4*4 .. idx4*4+3 with one Philox call
__device__ __forceinline__ void drop_factor4(const DropCfg& d, uint32_t site, uint64_t idx4, float f[4]) {
  if (d.thresh == 0) { f[0] = f[1] = f[2] = f[3] = 1.f; return; }
  uint32_t o[4];
  philox4x32_10((uint32_t)idx4, (uint32_t)(idx4 >> 32), site, d.iter, d.seed_lo, d.seed_hi, o);
#pragma unroll
  for (int i = 0; i < 4; ++i) f[i] = o[i] >= d.thresh ? d.scale : 0.f;
}

// Dropout sites (mirrors oracle/visdial_oracle.py)
enum : uint32_t {
  SITE_QEMBED = 0, SITE_HEMBED = 1, SITE_HATT = 2, SITE_IMG_TR = 3, SITE_U_OUT = 5,
  SITE_FUSION = 6, SITE_IMG_FC7 = 7, SITE_HOP0 = 16,
  SITE_SAMPLE = 64          // generateAnswers' sampling draws (not a dropout site)
};

// ---------------------------------------------------------------------------------------------
// Sampling (Engine::gen_sample, model.lua:584-602) by the Gumbel-max trick: the token drawn from step `step`'s row r is
// 1 + argmax_j (x_j / T + g_j), x = the vocabulary logits with bias, ties to the lower class.  g_j = -log(-log(u_j)),
// u_j = ((w >> 8) + 0.5) 2^-24, w = Philox4x32-10 word idx % 4 at counter (idx/4 lo, idx/4 hi, SITE_SAMPLE, step), key =
// seed, idx = (row_offset + r row_stride) V + j: the element index of the step's (rows, V) decOut over the whole split, so a
// draw depends only on (seed, global round, step, class).  row_stride = 1 when the rows are consecutive rounds; the dialog
// loop (Engine::gen_dialog) samples round r of B dialogs, rows b R + r, with row_offset = first round + r and stride R.  Exactly a draw from softmax(x / T) = exp(logp / T) / sum.  Every
// device route evaluates the key with these full-precision functions, so equal logits give equal tokens on every route.
// The numpy twin is tests/sampling_twin.py.
// ---------------------------------------------------------------------------------------------
struct SampleCfg {
  uint32_t seed_lo, seed_hi, step;
  float temperature;
  int64_t row_offset;       // global round of row 0
  int64_t row_stride;       // global rounds between consecutive rows
  // device (rows): row r's global round, replacing row_offset + r row_stride (a dialog pool's ask, whose rows are
  // conversations at their own rounds); null: the affine rule
  const int64_t* row_round = nullptr;
};
__device__ __forceinline__ int64_t sample_round(const SampleCfg& s, int64_t r) {
  return s.row_round ? s.row_round[r] : s.row_offset + r * s.row_stride;
}
// largest Gumbel value the rule can produce (u = 1 - 2^-25: -log(-log u) = 17.33): an element whose x / T + GUMBEL_MAX is
// below the best key so far cannot win, so its Philox word and logarithms need not be computed
constexpr float GUMBEL_MAX = 17.5f;

// g of one Philox word.  u has 25 significant bits, so -log(u) is formed from an exact operand: u itself below 1/2,
// 1 - u (through log1p) above it.
__device__ __forceinline__ float gumbel_of_word(uint32_t w) {
  const uint32_t m = w >> 8;
  const float t = m < (1u << 23) ? -logf(((float)m + 0.5f) * 0x1p-24f)
                                 : -log1pf(-(((float)((1u << 24) - m) - 0.5f) * 0x1p-24f));
  return -logf(t);
}
__device__ __forceinline__ void sample_words(const SampleCfg& s, uint64_t q, uint32_t o[4]) {
  philox4x32_10((uint32_t)q, (uint32_t)(q >> 32), SITE_SAMPLE, s.step, s.seed_lo, s.seed_hi, o);
}
// (key, class) beats (key2, class2): key descending, class ascending
__device__ __forceinline__ bool sample_before(float k, int c, float k2, int c2) { return k > k2 || (k == k2 && c < c2); }

// Truncated sampling (DESIGN §23): the draw above restricted to a prefix of the classes in the order
// (y desc, class asc), y_j = x_j / T (the key's own fp32 division).  Active when 1 <= top_k < V or top_p < 1.
//  1. top-k: the first top_k classes (all V when top_k is 0 or >= V).
//  2. top-p over the classes step 1 kept: m = max y, w_j = expf(y_j - m), integer mass q_j = rint(w_j 2^32) (uint64),
//     S = the kept classes' sum of q, tau = (uint64)ceil((double)top_p * (double)S); keep the shortest prefix whose
//     cumulative q reaches tau (at least the first class).  Integer masses make S and every prefix sum independent of the
//     summation order.  top_p = 1 skips the step.
//  3. the token is 1 + argmax of y_j + g_j over the kept classes, g_j the SAME Philox Gumbel value as the untruncated draw
//     (idx, SITE_SAMPLE, step): an exact draw from the renormalised truncated softmax, and equal to the untruncated draw
//     whenever that draw's class is kept.  logp stays x_tok - lse of the untempered, untruncated LogSoftMax.
// The numpy twin is tests/truncation_twin.py.
struct TruncCfg {
  int32_t top_k = 0;        // 0: no top-k
  float top_p = 1.f;        // in (0, 1]; 1: no top-p
};
__host__ __device__ __forceinline__ bool trunc_active(const TruncCfg& t, int V) {
  return (t.top_k >= 1 && t.top_k < V) || t.top_p < 1.f;
}
// the widest vocabulary whose row (4 V bytes of y) fits the truncated sampler's shared-memory stage beside its histograms
constexpr int TRUNC_MAX_V = 49152;

// Answer rules (DESIGN §25): classes barred from a generation step's choice, in beam search and sampling alike.  At step stp
// of row r, t[1 .. stp-1] are the row's own earlier tokens (t[0] = <START>), read from hist + r * ld.
//  1. banned: the n_banned ids in [1, V] are never candidates.
//  2. min_words m: end_token is barred while stp <= m (the answer so far has stp - 1 words).
//  3. no_repeat_ngram n (0 = off): w is barred if for some j >= 1 with j + n - 1 <= stp - 1, t[j .. j+n-2] equals
//     t[stp-n+1 .. stp-1] and t[j+n-1] == w; a window holding a 0 (a pad) matches nothing; end_token is never barred here.
//     n = 1 bars every token already in the answer.
//  4. fallback: if every class is barred, end_token is allowed.
// Scores are untouched: logp stays the unconstrained LogSoftMax.  The numpy twin is tests/answer_rules_twin.py.
struct AnswerRules {
  int32_t min_words = 0, no_repeat_ngram = 0, n_banned = 0;
  const int32_t* banned = nullptr;   // device (n_banned)
  int32_t end_token = 0;
  int32_t step = 0;
  const int32_t* hist = nullptr;     // device: row r's tokens at hist + r * ld (beam search: the pre-merge beams (rows, L);
  int64_t ld = 0;                    // sampling: the answer (rows, L + 1))
};
__host__ __device__ __forceinline__ bool rules_active(int32_t min_words, int32_t no_repeat_ngram, int32_t n_banned) {
  return min_words > 0 || no_repeat_ngram > 0 || n_banned > 0;
}
// one bit per class: the barred set of a row lives in shared memory
constexpr int RULES_MASK_WORDS = TRUNC_MAX_V / 32;

// ---------------------------------------------------------------------------------------------
// Launch context: stream + launch accounting + optional per-class event bracketing.
// ---------------------------------------------------------------------------------------------
struct KStat {
  int64_t launches = 0;
  double flops = 0, bytes = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
  double ms = 0;
};

struct LaunchCtx {
  cudaStream_t stream = nullptr;
  int64_t launches = 0;
  int profiling = 0;          // 0 off, 1 every class, 2 only the roofline class (big lstm_step / lstm_step_bwd launches)
  int sm_count = 132;
  int sm_budget = 0;          // > 0: persistent / single-wave kernels size their grids to this many SMs (the rest stay free
                              // for a concurrent higher-priority stream); 0 = all of them
  int sms() const { return sm_budget > 0 ? sm_budget : sm_count; }
  // deterministic mode (DESIGN §27): the launchers of the gradient reductions take their routes without float atomics, whose
  // split counts and chunkings follow from the shapes alone; their partial sums live in `scratch` (device memory that stays
  // valid until the engine's next forward) and are added in a fixed order
  bool deterministic = false;
  std::function<void*(size_t)> scratch;
  template <typename T> T* scratch_get(int64_t n) {
    VD_REQUIRE(scratch, -3, "deterministic route without a scratch allocator");
    return static_cast<T*>(scratch((size_t)n * sizeof(T)));
  }
  std::map<std::string, KStat> stats;
  std::vector<cudaEvent_t> free_events;

  cudaEvent_t get_event() {
    if (!free_events.empty()) { cudaEvent_t e = free_events.back(); free_events.pop_back(); return e; }
    cudaEvent_t e; VD_CUDA_CHECK(cudaEventCreate(&e)); return e;
  }
  // bracket one launch (or a short group) of class `name`
  struct Scope {
    LaunchCtx* cx; KStat* st; cudaEvent_t a = nullptr, b = nullptr;
    Scope(LaunchCtx* c, const char* name, double flops, double bytes) : cx(c), st(nullptr) {
      if (!cx->profiling) return;
      if (cx->profiling == 2 && strcmp(name, "lstm_step") != 0 && strcmp(name, "lstm_step_bwd") != 0) return;
      st = &cx->stats[name];
      st->launches++; st->flops += flops; st->bytes += bytes;
      a = cx->get_event(); b = cx->get_event();
      cudaEventRecord(a, cx->stream);
    }
    ~Scope() {
      if (!st) return;
      cudaEventRecord(b, cx->stream);
      st->pending.emplace_back(a, b);
    }
  };
  void collect() {
    for (auto& kv : stats) {
      for (auto& p : kv.second.pending) {
        cudaEventSynchronize(p.second);
        float ms = 0; cudaEventElapsedTime(&ms, p.first, p.second);
        kv.second.ms += ms;
        free_events.push_back(p.first); free_events.push_back(p.second);
      }
      kv.second.pending.clear();
    }
  }
};

// counts the launch; with profiling 1 also under its own name in stats (launch count only, no events)
inline void check_launch(LaunchCtx& cx, const char* what) {
  cx.launches++;
  if (cx.profiling == 1) cx.stats[what].launches++;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    char buf[512];
    snprintf(buf, sizeof(buf), "kernel launch failed: %s -> %s", what, cudaGetErrorString(e));
    throw CudaError(-3, buf);
  }
}

static inline int cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

}  // namespace vd

// C ABI of libdwt_b200.so (declared in include/dwt_b200.h): argument validation, workspace
// carving, kernel-family selection by group size, launches.  No host synchronisation, no
// allocation, no CPU fallback.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include <atomic>
#include <mutex>
#include <string>
#include <vector>
#include <string.h>

#include "norm_launch.h"

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int check_launch(const char* what) {
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(DWT_E_LAUNCH, "%s: %s", what, cudaGetErrorString(e));
  }
  return DWT_OK;
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;   // H100 SXM
  }
  return n;
}

// ---- launch accounting / optional per-kernel event timing ------------------------------------
std::atomic<int64_t> g_launches{0};
std::mutex g_prof_mu;
bool g_prof_on = false;
struct ProfRec { char name[48]; cudaEvent_t a, b; double bytes; };
std::vector<ProfRec> g_prof;
std::vector<cudaEvent_t> g_event_pool;

cudaEvent_t take_event() {
  if (!g_event_pool.empty()) { cudaEvent_t e = g_event_pool.back(); g_event_pool.pop_back(); return e; }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}

// RAII bracket around one kernel launch
struct Launch {
  cudaStream_t st; ProfRec rec; bool on;
  // name = "<kernel family>|C|HW|GS|D|N" so the bench can break time down by norm site
  Launch(const char* family, const dwt::Geom* gm, double bytes, cudaStream_t s) : st(s), on(false) {
    rec.a = rec.b = nullptr; rec.bytes = bytes;
    if (gm) snprintf(rec.name, sizeof(rec.name), "%s|%d|%d|%d|%d|%d", family, gm->C, gm->HW, gm->GS, gm->D, gm->N);
    else snprintf(rec.name, sizeof(rec.name), "%s", family);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    std::lock_guard<std::mutex> lk(g_prof_mu);
    if (g_prof_on && g_prof.size() < (1u << 18)) {
      on = true; rec.a = take_event(); rec.b = take_event();
      cudaEventRecord(rec.a, st);
    }
  }
  ~Launch() {
    if (!on) return;
    cudaEventRecord(rec.b, st);
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof.push_back(rec);
  }
};

std::once_flag g_tiled_once;
int g_tiled_rc = 0;
int ensure_tiled() {
  std::call_once(g_tiled_once, [] { g_tiled_rc = dwt::tiled_init(); });
  return g_tiled_rc;
}

std::once_flag g_tc_once;
int g_tc_rc = 0;
int ensure_tc() {
  std::call_once(g_tc_once, [] { g_tc_rc = dwt::tc_init(); });
  return g_tc_rc;
}

// CTAs per (domain, super-block) of the tensor-core contraction: one full wave of 2 CTAs per SM
int tc_chunks(const dwt::Geom& g) {
  const int problems = dwt::tc_superblocks(g) * g.D;
  int n = 2 * sm_count() / problems;
  const int64_t tiles = (int64_t)g.N * ((g.HW + 31) / 32);
  if (n > tiles) n = (int)tiles;
  return n < 1 ? 1 : n;
}

// persistent CTAs per (domain, super-block) of the tensor-core apply kernels: per_sm CTAs per SM
int tc_apply_ctas(const dwt::Geom& g, int per_sm, int tile_px) {
  const int problems = dwt::tc_superblocks(g) * g.D;
  int n = per_sm * sm_count() / problems;
  const int64_t tiles = (int64_t)g.N * ((g.HW + tile_px - 1) / tile_px);
  if (n > tiles) n = (int)tiles;
  return n < 1 ? 1 : n;
}

int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return (v && *v) ? atoi(v) : dflt;
}

// channels-last launch shaping.  Every kernel is ONE wave of persistent CTAs sweeping 32-row chunks (norm_cl.cu):
// grid.x CTAs per (domain, column slab), grid.y slabs, grid.z = D domains side by side.  (grid.z = 1 -- all CTAs
// sweeping the domains one after the other, so that the whole grid moves through the tensor as a single window --
// writes three times the partial rows for no extra L2 hits;
// the kernels still accept it, DWT_CL_SEQ_MB=<tensor MB threshold> turns it on for experiments.)
struct ClPlan { int nred, new_, S, gridy, gz_red, gz_ew; };
ClPlan cl_plan(const dwt::Geom& g, int slots_red, int slots_ew, int unroll_red, int unroll_ew) {
  static const int seq_mb = env_int("DWT_CL_SEQ_MB", 1 << 30);  // experiment switch, off by default
  const int C4 = g.C / 4, CW = C4 < 256 ? C4 : 256, rpi = 256 / CW, gridy = C4 / CW;
  const long long rows = (long long)g.N * g.HW;
  const double mbytes = 4.0 * (double)g.D * (double)rows * (double)g.C / 1048576.0;
  const bool seq = g.D > 1 && mbytes >= (double)seq_mb;
  ClPlan p;
  p.gridy = gridy;
  p.gz_red = p.gz_ew = seq ? 1 : g.D;
  auto shape = [&](int slots, int unroll, int gz) {
    long long by_work = rows / ((long long)rpi * unroll * 2);      // >= two load batches per CTA and domain
    if (by_work < 1) by_work = 1;
    int cap = slots * sm_count() / (gridy * gz);
    if (cap < 1) cap = 1;
    return (int)(by_work < cap ? by_work : cap);
  };
  p.nred = shape(slots_red, unroll_red, p.gz_red);
  p.new_ = shape(slots_ew, unroll_ew, p.gz_ew);
  p.S = p.nred < 8 ? p.nred : 8;
  return p;
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Launch shaping.  Every norm kernel is a single wave of long-lived CTAs: `target` CTAs in total
// (a small multiple of the SM count, set by the kernel's register footprint), reached either by
// splitting each (domain, group) problem over `nchunks` CTAs (few large problems) or by serving
// `ppc` problems per CTA (thousands of small ones).
enum KernelKind { K_STATS, K_APPLY, K_BWD_REDUCE, K_BWD_APPLY };

// Resident CTAs per SM of each kernel (its __launch_bounds__ minimum); reductions launch at most
// one full wave of equal-work CTAs (no tail), elementwise kernels many short CTAs (>= 4 waves).
int slots_per_sm(KernelKind k, int GS) {
  if (GS > 4) return 2;                                    // tiled path: limited by shared memory
  return ((k == K_STATS || k == K_APPLY) && GS < 4) ? 4 : 3;
}

// Largest split any kernel may use for one problem: sizes the partials area of the workspace.
int chunk_cap(int GS, int G, int D) {
  (void)GS;
  const int target = 16 * sm_count();
  int cap = (target + G * D - 1) / (G * D);
  return cap < 1 ? 1 : cap;
}

struct Workspace {
  int* status;
  int* counters;      // [D*G]
  int* dom_counter;   // [G]   (forward)
  int* dom_counter2;  // [G]   (backward)
  float* partial;     // [D*G*cap*(GS*GS+GS)]
  float* save_cov;    // [D*G*GS*GS]
  float* coef;        // [D*G*(2*GS*GS+GS)]
  float* dgb_part;    // [D*2*C]
  float* gram;        // [D*SB*(64*64+64)]  reduced moments of the tensor-core contraction
  float* shift;       // [D*SB*64]          pilot shift of every channel
  float* red;         // [D*8*W]            channels-last path: split-reduced partial moments
  int* bad;           // [D*G]              per (domain, group): batch covariance not positive definite
  size_t bytes;
};

// The head of the workspace holds ONLY the status word and the arrival counters, at offsets
// that do not depend on the geometry: every call leaves its counters at zero, so calls with
// different shapes can share one zero-initialised buffer.  Scratch (any content) follows.
constexpr size_t kMaxGroups = 65536;
constexpr size_t kOffCounters = 256;
constexpr size_t kOffDom1 = kOffCounters + sizeof(int) * DWT_MAX_DOMAINS * kMaxGroups;
constexpr size_t kOffDom2 = kOffDom1 + sizeof(int) * kMaxGroups;
constexpr size_t kOffScratch = kOffDom2 + sizeof(int) * kMaxGroups;

Workspace carve(void* base, int64_t C, int GS, int D) {
  const int G = (int)(C / GS);
  const int cap = chunk_cap(GS, G, D);
  size_t off = kOffScratch;
  auto take = [&](size_t nbytes) { size_t o = off; off = align_up(off + nbytes, 256); return o; };
  char* b = static_cast<char*>(base);
  Workspace w;
  w.status = reinterpret_cast<int*>(b);
  w.counters = reinterpret_cast<int*>(b + kOffCounters);
  w.dom_counter = reinterpret_cast<int*>(b + kOffDom1);
  w.dom_counter2 = reinterpret_cast<int*>(b + kOffDom2);
  size_t partial_floats = (size_t)D * G * cap * (GS * GS + GS);
  if (GS >= 8 && 64 % GS == 0) {                           // tensor-core contraction: per super-block partials
    const size_t tc = ((size_t)2 * sm_count() + (size_t)((C + 63) / 64) * D) * (64 * 64 + 64);
    if (tc > partial_floats) partial_floats = tc;
  }
  size_t red_floats = 1;
  if (dwt::cl_supports((int)C, GS)) {                      // channels-last path: per-CTA rows of C/4-column vectors
    const size_t W = (size_t)dwt::cl_bwd_width((int)C, GS);
    const int C4 = (int)C / 4, gridy = C4 <= 256 ? 1 : C4 / 256;
    const size_t cl = (size_t)D * (3 * sm_count() / gridy + 1) * W;     // one row per (domain, CTA of grid.x)
    if (cl > partial_floats) partial_floats = cl;
    red_floats = (size_t)D * 8 * W;
  }
  w.partial = reinterpret_cast<float*>(b + take(sizeof(float) * partial_floats));
  w.red = reinterpret_cast<float*>(b + take(sizeof(float) * red_floats));
  w.save_cov = reinterpret_cast<float*>(b + take(sizeof(float) * (size_t)D * G * GS * GS));
  w.coef = reinterpret_cast<float*>(b + take(sizeof(float) * (size_t)D * G * dwt::coef_stride(GS)));
  w.dgb_part = reinterpret_cast<float*>(b + take(sizeof(float) * (size_t)D * 2 * C));
  const size_t SBn = (size_t)((C + 63) / 64);
  w.gram = reinterpret_cast<float*>(b + take(sizeof(float) * (size_t)D * SBn * (64 * 64 + 64)));
  w.shift = reinterpret_cast<float*>(b + take(sizeof(float) * (size_t)D * SBn * 64));
  w.bad = reinterpret_cast<int*>(b + take(sizeof(int) * (size_t)D * G));
  w.bytes = off;
  return w;
}

struct Plan {
  dwt::Geom gm;       // gm.nchunks / gm.ppc shaped for the REDUCTION kernel of this call
  dwt::Geom gm_ew;    // same geometry shaped for the elementwise kernel of this call
  int vec;            // 4 when rows can be read as float4
  int chunks_ew;      // grid.x of the elementwise (apply) kernel
  bool small;
};

void shape(dwt::Geom& g, int64_t work_units, KernelKind kind, bool small, int* chunks) {
  const bool reduce = (kind == K_STATS || kind == K_BWD_REDUCE);
  const int slots = slots_per_sm(kind, g.GS) * sm_count();
  const int target = reduce ? slots : 4 * slots;
  g.ppc = 1;
  if (small) {
    // smallest team split that fits the problems of this site into `target` CTAs
    while (g.ppc < 8 && (int64_t)((g.G + g.ppc - 1) / g.ppc) * g.D > target) g.ppc <<= 1;
  }
  int n = 1;
  if (g.ppc == 1) {
    n = target / (g.G * g.D);                              // floor: never spill into a second wave
    const int cap = chunk_cap(g.GS, g.G, g.D);
    if (n > cap) n = cap;
    if (n > work_units) n = (int)work_units;
    if (n < 1) n = 1;
  }
  *chunks = n;
}

int make_plan(Plan& p, KernelKind reduce_kind, KernelKind ew_kind, const void* a0, const void* a1, const void* a2,
              int64_t N, int64_t C, int64_t HW, int GS, int D) {
  if (N <= 0 || C <= 0 || HW <= 0) return fail(DWT_E_INVALID, "empty tensor (N=%lld C=%lld HW=%lld)", (long long)N,
                                               (long long)C, (long long)HW);
  if (GS < 1 || GS > DWT_MAX_GROUP_SIZE) return fail(DWT_E_UNSUPPORTED, "group_size %d outside [1,%d]", GS,
                                                     DWT_MAX_GROUP_SIZE);
  if (C % GS != 0) return fail(DWT_E_INVALID, "channels %lld not divisible by group_size %d", (long long)C, GS);
  if (D < 1 || D > DWT_MAX_DOMAINS) return fail(DWT_E_INVALID, "n_domains %d outside [1,%d]", D, DWT_MAX_DOMAINS);
  if (N * C * HW >= (int64_t)1 << 31 || C / GS > 65535)
    return fail(DWT_E_UNSUPPORTED, "shape too large for 32-bit item indexing");
  dwt::Geom& g = p.gm;
  g.N = (int)N; g.C = (int)C; g.HW = (int)HW; g.GS = GS; g.G = (int)(C / GS); g.D = D;
  g.M = (float)((double)N * (double)HW);
  const uintptr_t bits = (uintptr_t)a0 | (uintptr_t)a1 | (uintptr_t)a2;
  p.vec = (HW % 4 == 0 && bits % 16 == 0) ? 4 : 1;
  p.small = dwt::small_supports(GS);
  int64_t work_units;   // CTA-sized pieces of work available per (domain, group)
  if (p.small) work_units = (N * (HW / p.vec) + dwt::kThreads * 2 - 1) / (dwt::kThreads * 2);
  else work_units = (N * HW + 127) / 128;
  if (work_units < 1) work_units = 1;
  shape(g, work_units, reduce_kind, p.small, &g.nchunks);
  p.gm_ew = g;
  shape(p.gm_ew, work_units, ew_kind, p.small, &p.chunks_ew);
  p.gm_ew.nchunks = g.nchunks;
  return DWT_OK;
}

int whiten_like_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int GS, int D, int mode, float a,
                    float b, float momentum, float unbias, int update_running, float* const* rmean,
                    float* const* rcov, const float* gamma, const float* beta, const float* residual,
                    uint8_t* relu_mask, int epi, float* save_mean, float* save_w, void* ws, size_t ws_bytes,
                    cudaStream_t st) {
  const bool nhwc = (mode & DWT_LAYOUT_NHWC) != 0;
  mode &= 0xFF;
  Plan p;
  if (int rc = make_plan(p, K_STATS, K_APPLY, x, y, nullptr, N, C, HW, GS, D)) return rc;
  if (!x || !y || !save_mean || !save_w || !ws) return fail(DWT_E_INVALID, "null pointer argument");
  if (nhwc && !dwt::cl_supports((int)C, GS))
    return fail(DWT_E_UNSUPPORTED, "channels-last layout is built for group_size 1, 2, 4 with C/4 a power of two (C=%lld gs=%d)", (long long)C, GS);
  if (nhwc && (((uintptr_t)x | (uintptr_t)y) % 16 != 0)) return fail(DWT_E_INVALID, "channels-last tensors must be 16-byte aligned");
  if (mode != DWT_MODE_TRAIN && mode != DWT_MODE_EVAL) return fail(DWT_E_INVALID, "bad mode %d", mode);
  if ((epi & DWT_EPI_RELU) && !(epi & DWT_EPI_AFFINE)) return fail(DWT_E_INVALID, "RELU epilogue needs AFFINE");
  if ((epi & DWT_EPI_AFFINE) && (!gamma || !beta)) return fail(DWT_E_INVALID, "AFFINE epilogue needs gamma and beta");
  if ((epi & DWT_EPI_RESIDUAL) && ((epi & 3) != 3 || !residual)) return fail(DWT_E_INVALID, "RESIDUAL epilogue needs AFFINE|RELU and a residual tensor");
  if ((epi & DWT_EPI_RESIDUAL) && (uintptr_t)residual % 16 != 0) return fail(DWT_E_INVALID, "residual must be 16-byte aligned");
  if (relu_mask && !((epi & DWT_EPI_RESIDUAL) && nhwc))
    return fail(DWT_E_UNSUPPORTED, "the ReLU byte map is written by the channels-last RESIDUAL epilogue only");
  if (epi != 0 && !p.small)
    return fail(DWT_E_UNSUPPORTED, "fused gamma/beta/ReLU epilogue is built for group_size 1, 2, 4 (got %d)", GS);
  const bool need_running = (mode == DWT_MODE_EVAL) || update_running;
  if (need_running) {
    if (!rmean || !rcov) return fail(DWT_E_INVALID, "running buffers required");
    for (int d = 0; d < D; ++d)
      if (!rmean[d] || !rcov[d]) return fail(DWT_E_INVALID, "running buffer of domain %d is null", d);
  }
  Workspace w = carve(ws, C, GS, D);
  if (w.bytes > ws_bytes) return fail(DWT_E_WORKSPACE, "workspace too small: need %zu bytes, got %zu", w.bytes, ws_bytes);
  if ((uintptr_t)ws % 256 != 0) return fail(DWT_E_WORKSPACE, "workspace must be 256-byte aligned");
  if (!p.small && ensure_tiled() != 0) return fail(DWT_E_LAUNCH, "cudaFuncSetAttribute failed (%d)", g_tiled_rc);

  dwt::FwdFin fin{};
  fin.a = a; fin.b = b; fin.momentum = momentum; fin.unbias = unbias;
  fin.update_running = (mode == DWT_MODE_TRAIN) ? update_running : 0;
  fin.save_mean = save_mean; fin.save_w = save_w; fin.save_cov = w.save_cov;
  for (int d = 0; d < D; ++d) { fin.rmean[d] = need_running ? rmean[d] : nullptr; fin.rcov[d] = need_running ? rcov[d] : nullptr; }
  fin.dom_counter = w.dom_counter; fin.status = w.status; fin.bad = w.bad;
  if (need_running && D > 1) {
    bool all_same = true, all_distinct = true;
    for (int d = 1; d < D; ++d) {
      if (rmean[d] != rmean[0] || rcov[d] != rcov[0]) all_same = false;
      for (int e = 0; e < d; ++e)
        if (rmean[d] == rmean[e] || rcov[d] == rcov[e]) all_distinct = false;
    }
    fin.aliased = all_same ? 1 : (all_distinct ? 0 : -1);
  }

  const double E = 4.0 * (double)D * (double)N * (double)C * (double)HW;   // bytes of one activation tensor
  if (nhwc) {
    const ClPlan cp = cl_plan(p.gm, 3, 3, 8, (epi & DWT_EPI_RESIDUAL) ? 4 : 8);
    if (mode == DWT_MODE_TRAIN) {
      {
        Launch l("cl_stats", &p.gm, E, st);
        dwt::cl_stats(x, p.gm, cp.nred, cp.gz_red, w.partial, w.shift, st);
      }
      if (int rc = check_launch("channels-last statistics kernel")) return rc;
      Launch l("cl_fwd_finalize", &p.gm, 0.0, st);
      dwt::cl_fwd_finalize(w.partial, cp.nred, w.shift, p.gm, fin, st);
    } else {
      Launch l("eval_prep", &p.gm, 0.0, st);
      dwt::small_eval_prep(p.gm, fin, st);
    }
    if (int rc = check_launch("channels-last finalize kernel")) return rc;
    {
      Launch l("cl_apply", &p.gm, ((epi & DWT_EPI_RESIDUAL) ? (relu_mask ? 3.0625 : 3.0) : 2.0) * E, st);
      dwt::cl_apply(x, y, p.gm, cp.new_, cp.gz_ew, epi, save_mean, save_w, gamma, beta, residual, relu_mask, st);
    }
    return check_launch("channels-last apply kernel");
  }
  const bool tc = !p.small && dwt::tc_supports(p.gm, p.vec) && ensure_tc() == 0;
  if (mode == DWT_MODE_TRAIN) {
    Launch l(p.small ? "small_stats" : (tc ? "tc_stats" : "tiled_stats"), &p.gm, E, st);
    if (p.small) dwt::small_stats(x, p.gm, p.vec, fin, w.partial, w.counters, st);
    else if (tc) {
      if (int cr = dwt::tc_stats(x, p.gm, tc_chunks(p.gm), w.shift, w.partial, st))
        return fail(DWT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d) x=%p N=%d C=%d HW=%d D=%d", cr, (const void*)x, p.gm.N, p.gm.C, p.gm.HW, p.gm.D);
    } else dwt::tiled_stats(x, p.gm, p.vec, fin, w.partial, w.counters, st);
  } else {
    Launch l("eval_prep", &p.gm, 0.0, st);
    if (p.small) dwt::small_eval_prep(p.gm, fin, st);
    else if (tc) dwt::dense_fwd_factor(nullptr, nullptr, p.gm, fin, st);
    else dwt::tiled_eval_prep(p.gm, fin, st);
  }
  if (tc && mode == DWT_MODE_TRAIN) {
    if (int rc = check_launch("tensor-core statistics kernel")) return rc;
    Launch l("dense_fwd_finalize", &p.gm, 0.0, st);
    dwt::dense_partial_reduce(w.partial, tc_chunks(p.gm), dwt::tc_superblocks(p.gm) * D, w.gram, st);
    dwt::dense_fwd_factor(w.gram, w.shift, p.gm, fin, st);
  }
  if (int rc = check_launch("whitening statistics kernel")) return rc;
  {
    Launch l(p.small ? "small_apply" : (tc ? "tc_apply" : "tiled_apply"), &p.gm, ((epi & DWT_EPI_RESIDUAL) ? 3 : 2) * E, st);
    if (p.small) dwt::small_apply(x, y, p.gm_ew, p.vec, p.chunks_ew, epi, save_mean, save_w, gamma, beta, residual, st);
    else if (tc) {
      if (int cr = dwt::tc_apply(x, y, p.gm, tc_apply_ctas(p.gm, 1, 64), save_mean, save_w, st))
        return fail(DWT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d)", cr);
    } else dwt::tiled_apply(x, y, p.gm_ew, p.vec, p.chunks_ew, save_mean, save_w, st);
  }
  return check_launch("whitening apply kernel");
}

int whiten_like_bwd(const float* x, const float* dout, const float* dout2, float* dx, int64_t N, int64_t C, int64_t HW, int GS, int D,
                    int mode, float a, const float* save_mean, const float* save_w, const float* gamma,
                    const float* beta, const uint8_t* relu_mask, float* dresidual, int epi, float* dgamma,
                    float* dbeta, void* ws, size_t ws_bytes, cudaStream_t st) {
  const bool nhwc = (mode & DWT_LAYOUT_NHWC) != 0;
  mode &= 0xFF;
  Plan p;
  if (int rc = make_plan(p, K_BWD_REDUCE, K_BWD_APPLY, x, dout, dx, N, C, HW, GS, D)) return rc;
  if (!x || !dout || !dx || !save_mean || !save_w || !ws) return fail(DWT_E_INVALID, "null pointer argument");
  if (dout2 && (!nhwc || (uintptr_t)dout2 % 16 != 0))
    return fail(nhwc ? DWT_E_INVALID : DWT_E_UNSUPPORTED, "a second gradient addend (dout2) is built for the channels-last "
                "kernels (16-byte aligned tensor); add it to dout otherwise");
  if (nhwc && !dwt::cl_supports((int)C, GS))
    return fail(DWT_E_UNSUPPORTED, "channels-last layout is built for group_size 1, 2, 4 with C/4 a power of two (C=%lld gs=%d)", (long long)C, GS);
  if (nhwc && (((uintptr_t)x | (uintptr_t)dout | (uintptr_t)dx) % 16 != 0)) return fail(DWT_E_INVALID, "channels-last tensors must be 16-byte aligned");
  if (mode != DWT_MODE_TRAIN && mode != DWT_MODE_EVAL) return fail(DWT_E_INVALID, "bad mode %d", mode);
  if ((epi & DWT_EPI_RELU) && !(epi & DWT_EPI_AFFINE)) return fail(DWT_E_INVALID, "RELU epilogue needs AFFINE");
  if ((epi & DWT_EPI_AFFINE) && (!gamma || !beta)) return fail(DWT_E_INVALID, "AFFINE epilogue needs gamma and beta");
  if (epi & DWT_EPI_RESIDUAL) {
    // backward of out = relu(z + residual): the ReLU mask comes from the byte map the forward wrote
    if (!nhwc || !relu_mask || (epi & 3) != 3)
      return fail(DWT_E_INVALID, "backward of a RESIDUAL forward needs the channels-last layout, AFFINE|RELU and the forward's "
                                 "ReLU byte map (or pass dout already masked by (out > 0) with epilogue AFFINE)");
    if (dresidual && (uintptr_t)dresidual % 16 != 0) return fail(DWT_E_INVALID, "dresidual must be 16-byte aligned");
  } else if (relu_mask || dresidual) {
    return fail(DWT_E_INVALID, "relu_mask / dresidual belong to the RESIDUAL epilogue");
  }
  if ((dgamma == nullptr) != (dbeta == nullptr)) return fail(DWT_E_INVALID, "dgamma and dbeta go together");
  if (epi != 0 && !p.small)
    return fail(DWT_E_UNSUPPORTED, "fused gamma/beta/ReLU epilogue is built for group_size 1, 2, 4 (got %d)", GS);
  Workspace w = carve(ws, C, GS, D);
  if (w.bytes > ws_bytes) return fail(DWT_E_WORKSPACE, "workspace too small: need %zu bytes, got %zu", w.bytes, ws_bytes);
  if ((uintptr_t)ws % 256 != 0) return fail(DWT_E_WORKSPACE, "workspace must be 256-byte aligned");
  if (!p.small && ensure_tiled() != 0) return fail(DWT_E_LAUNCH, "cudaFuncSetAttribute failed (%d)", g_tiled_rc);

  dwt::BwdFin fin{};
  fin.a = a; fin.mode = mode; fin.epi = epi;
  fin.save_mean = save_mean; fin.save_w = save_w; fin.gamma = gamma;
  fin.coef = w.coef; fin.dgb_part = w.dgb_part;
  fin.dgamma = (epi & DWT_EPI_AFFINE) ? dgamma : nullptr;
  fin.dbeta = (epi & DWT_EPI_AFFINE) ? dbeta : nullptr;
  fin.dom_counter = w.dom_counter2;

  const bool need_reduce = (mode == DWT_MODE_TRAIN) || (fin.dgamma != nullptr);
  const double E = 4.0 * (double)D * (double)N * (double)C * (double)HW;
  if (nhwc) {
    const ClPlan cp = cl_plan(p.gm, 2, 2, 4, 4);
    const bool masked = (epi & DWT_EPI_RESIDUAL) != 0;
    if (need_reduce) {
      {
        Launch l("cl_bwd_reduce", &p.gm, ((masked ? 2.0625 : 2.0) + (dout2 ? 1.0 : 0.0)) * E, st);
        dwt::cl_bwd_reduce(x, dout, dout2, p.gm, cp.nred, cp.gz_red, epi, save_mean, save_w, gamma, beta, relu_mask, w.partial, st);
      }
      if (int rc = check_launch("channels-last backward reduction kernel")) return rc;
      Launch l("cl_bwd_finalize", &p.gm, 0.0, st);
      dwt::cl_bwd_finalize(w.partial, cp.nred, p.gm, fin, st);
    } else {
      Launch l("bwd_prep", &p.gm, 0.0, st);
      dwt::small_bwd_prep(p.gm, fin, st);
    }
    if (int rc = check_launch("channels-last backward finalize kernel")) return rc;
    {
      Launch l("cl_bwd_apply", &p.gm, ((masked ? (dresidual ? 4.0625 : 3.0625) : 3.0) + (dout2 ? 1.0 : 0.0)) * E, st);
      dwt::cl_bwd_apply(x, dout, dout2, dx, p.gm, cp.new_, cp.gz_ew, epi, w.coef, save_mean, save_w, gamma, beta, relu_mask, dresidual, st);
    }
    return check_launch("channels-last backward apply kernel");
  }
  const bool tc = !p.small && dwt::tc_supports(p.gm, p.vec) && ensure_tc() == 0;
  if (need_reduce) {
    Launch l(p.small ? "small_bwd_reduce" : (tc ? "tc_bwd_reduce" : "tiled_bwd_reduce"), &p.gm, 2 * E, st);
    if (p.small) dwt::small_bwd_reduce(x, dout, p.gm, p.vec, fin, beta, w.partial, w.counters, st);
    else if (tc) {
      if (int cr = dwt::tc_bwd_reduce(x, dout, p.gm, tc_chunks(p.gm), save_mean, w.partial, st))
        return fail(DWT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d) x=%p dout=%p N=%d C=%d HW=%d D=%d", cr, (const void*)x, (const void*)dout, p.gm.N, p.gm.C, p.gm.HW, p.gm.D);
    } else dwt::tiled_bwd_reduce(x, dout, p.gm, p.vec, fin, w.partial, w.counters, st);
  } else {
    Launch l("bwd_prep", &p.gm, 0.0, st);
    if (p.small) dwt::small_bwd_prep(p.gm, fin, st);
    else if (tc) dwt::dense_bwd_coef(nullptr, p.gm, fin, w.shift, st);
    else dwt::tiled_bwd_prep(p.gm, fin, st);
  }
  if (tc && need_reduce) {
    if (int rc = check_launch("tensor-core backward reduction kernel")) return rc;
    Launch l("dense_bwd_finalize", &p.gm, 0.0, st);
    dwt::dense_partial_reduce(w.partial, tc_chunks(p.gm), dwt::tc_superblocks(p.gm) * D, w.gram, st);
    dwt::dense_bwd_coef(w.gram, p.gm, fin, w.shift, st);
  }
  if (int rc = check_launch("whitening backward reduction kernel")) return rc;
  {
    Launch l(p.small ? "small_bwd_apply" : (tc ? "tc_bwd_apply" : "tiled_bwd_apply"), &p.gm, 3 * E, st);
    if (p.small) dwt::small_bwd_apply(x, dout, dx, p.gm_ew, p.vec, p.chunks_ew, epi, w.coef, save_mean, save_w, gamma, beta, st);
    else if (tc) {
      if (int cr = dwt::tc_bwd_apply(x, dout, dx, p.gm, tc_apply_ctas(p.gm, 1, 64), w.coef, save_mean, w.shift, st))
        return fail(DWT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d)", cr);
    } else dwt::tiled_bwd_apply(x, dout, dx, p.gm_ew, p.vec, p.chunks_ew, w.coef, st);
  }
  return check_launch("whitening backward apply kernel");
}

}  // namespace

extern "C" {

int dwt_abi_version(void) { return DWT_B200_ABI_VERSION; }

const char* dwt_last_error(void) { return g_err; }

size_t dwt_workspace_bytes(int64_t N, int64_t C, int64_t HW, int group_size, int n_domains) {
  (void)N; (void)HW;
  if (C <= 0 || group_size < 1 || group_size > DWT_MAX_GROUP_SIZE || C % group_size != 0 || n_domains < 1 ||
      n_domains > DWT_MAX_DOMAINS)
    return 0;
  return carve(nullptr, C, group_size, n_domains).bytes;
}

int dwt_whiten_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains,
                   int mode, float eps, float momentum, int update_running, float* const* running_mean,
                   float* const* running_cov, const float* gamma, const float* beta, const float* residual,
                   uint8_t* relu_mask, int epilogue, float* save_mean, float* save_w, void* workspace,
                   size_t workspace_bytes, dwt_stream_t stream) {
  return whiten_like_fwd(x, y, N, C, HW, group_size, n_domains, mode, 1.f - eps, eps, momentum, 1.f, update_running,
                         running_mean, running_cov, gamma, beta, residual, relu_mask, epilogue, save_mean, save_w,
                         workspace, workspace_bytes, (cudaStream_t)stream);
}

int dwt_whiten_bwd(const float* x, const float* dout, const float* dout2, float* dx, int64_t N, int64_t C, int64_t HW, int group_size,
                   int n_domains, int mode, float eps, const float* save_mean, const float* save_w,
                   const float* gamma, const float* beta, const uint8_t* relu_mask, float* dresidual, int epilogue,
                   float* dgamma, float* dbeta, void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  return whiten_like_bwd(x, dout, dout2, dx, N, C, HW, group_size, n_domains, mode, 1.f - eps, save_mean, save_w, gamma,
                         beta, relu_mask, dresidual, epilogue, dgamma, dbeta, workspace, workspace_bytes,
                         (cudaStream_t)stream);
}

// Batch norm is the group-size-1 member of the same family: "covariance" = biased variance,
// S = var + eps, W = 1/sqrt(S) = invstd; only the EMA differs (unbiased variance).
int dwt_bn_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int n_domains, int mode, float eps,
               float factor, int update_running, float* const* running_mean, float* const* running_var,
               const float* weight, const float* bias, const float* residual, uint8_t* relu_mask, int epilogue,
               float* save_mean, float* save_invstd, void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  const double M = (double)N * (double)HW;
  const float unbias = M > 1.0 ? (float)(M / (M - 1.0)) : 1.f;
  return whiten_like_fwd(x, y, N, C, HW, 1, n_domains, mode, 1.f, eps, factor, unbias, update_running, running_mean,
                         running_var, weight, bias, residual, relu_mask, epilogue, save_mean, save_invstd, workspace,
                         workspace_bytes, (cudaStream_t)stream);
}

int dwt_bn_bwd(const float* x, const float* dout, const float* dout2, float* dx, int64_t N, int64_t C, int64_t HW, int n_domains,
               int mode, const float* save_mean, const float* save_invstd, const float* weight, const float* bias,
               const uint8_t* relu_mask, float* dresidual, int epilogue, float* dweight, float* dbias, void* workspace,
               size_t workspace_bytes, dwt_stream_t stream) {
  return whiten_like_bwd(x, dout, dout2, dx, N, C, HW, 1, n_domains, mode, 1.f, save_mean, save_invstd, weight, bias,
                         relu_mask, dresidual, epilogue, dweight, dbias, workspace, workspace_bytes,
                         (cudaStream_t)stream);
}

int dwt_mec_fwd_bwd(const float* x, const float* y, int64_t N, int64_t K, float* loss, float* gx, float* gy,
                    dwt_stream_t stream) {
  if (!x || !y || !loss || !gx || !gy) return fail(DWT_E_INVALID, "null pointer argument");
  if (N <= 0 || K <= 0 || N >= (1 << 24) || K >= (1 << 24)) return fail(DWT_E_INVALID, "bad logits shape [%lld,%lld]", (long long)N, (long long)K);
  {
    Launch l("mec", nullptr, 16.0 * (double)N * (double)K, (cudaStream_t)stream);
    dwt::mec_launch(x, y, (int)N, (int)K, loss, gx, gy, (cudaStream_t)stream);
  }
  return check_launch("MEC kernel");
}

int dwt_head_loss_fwd_bwd(const float* logits, const int64_t* labels, int64_t B, int64_t K, float lambda, float* losses,
                          float* grad, int* status, dwt_stream_t stream) {
  if (!logits || !labels || !losses || !grad) return fail(DWT_E_INVALID, "null pointer argument");
  if (B <= 0 || K <= 0 || B >= (1 << 22) || K >= (1 << 24)) return fail(DWT_E_INVALID, "bad logits shape [3*%lld,%lld]", (long long)B, (long long)K);
  {
    Launch l("head_loss", nullptr, 4.0 * 3 * (double)B * (double)K * 2, (cudaStream_t)stream);
    dwt::head_loss_launch(logits, reinterpret_cast<const long long*>(labels), (int)B, (int)K, lambda, losses, grad, status,
                          (cudaStream_t)stream);
  }
  return check_launch("head loss kernel");
}

int dwt_augment_pair(const uint8_t* images, int64_t B, int src_h, int src_w, int crop, const int32_t* crop_plain,
                     const int32_t* crop_aug, const uint8_t* flip, const float* affine, const float* mean,
                     const float* stdv, float* out_plain, float* out_aug, int layout, dwt_stream_t stream) {
  if (!images || !mean || !stdv) return fail(DWT_E_INVALID, "null pointer argument");
  if (!out_plain && !out_aug) return fail(DWT_E_INVALID, "at least one of out_plain / out_aug is needed");
  if (out_plain && !crop_plain) return fail(DWT_E_INVALID, "out_plain needs crop_plain");
  if (out_aug && (!crop_aug || !flip || !affine)) return fail(DWT_E_INVALID, "out_aug needs crop_aug, flip and affine");
  if (B <= 0 || B > 65535 || src_h <= 0 || src_w <= 0 || src_h > 16384 || src_w > 16384)
    return fail(DWT_E_INVALID, "bad image batch [%lld,%d,%d,3]", (long long)B, src_h, src_w);
  if (crop <= 0 || crop > src_h || crop > src_w) return fail(DWT_E_INVALID, "crop %d does not fit %dx%d", crop, src_h, src_w);
  if (layout != 0 && layout != DWT_LAYOUT_NHWC) return fail(DWT_E_INVALID, "layout must be 0 (NCHW) or DWT_LAYOUT_NHWC");
  for (int c = 0; c < 3; ++c)
    if (!(stdv[c] != 0.f)) return fail(DWT_E_INVALID, "std[%d] must be non-zero", c);
  {
    const double px = (double)B * crop * crop;
    Launch l("augment_pair", nullptr, px * 3 * ((out_plain ? 5.0 : 0.0) + (out_aug ? 5.0 : 0.0)), (cudaStream_t)stream);
    dwt::augment_pair_launch(images, (int)B, src_h, src_w, crop, crop_plain, crop_aug, flip, affine, mean, stdv, out_plain,
                             out_aug, layout != 0, (cudaStream_t)stream);
  }
  return check_launch("augmentation kernel");
}

namespace {
int pool_check(int64_t N, int64_t H, int64_t W, int64_t C, int k, int s, int p, int* OH, int* OW) {
  if (N <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 4 != 0) return fail(DWT_E_INVALID, "bad pooling input [%lld,%lld,%lld,%lld] (C must be a multiple of 4)", (long long)N, (long long)H, (long long)W, (long long)C);
  if (k < 1 || k > 15 || s < 1 || p < 0 || 2 * p > k) return fail(DWT_E_INVALID, "bad pooling window k=%d s=%d p=%d (k <= 15, pad <= k/2)", k, s, p);
  if (H + 2 * p < k || W + 2 * p < k) return fail(DWT_E_INVALID, "pooling window larger than the padded image");
  *OH = (int)((H + 2 * p - k) / s + 1);
  *OW = (int)((W + 2 * p - k) / s + 1);
  if (N * H * W * C >= ((int64_t)1 << 40)) return fail(DWT_E_UNSUPPORTED, "tensor too large");
  return DWT_OK;
}
}  // namespace

int dwt_maxpool_fwd(const float* x, float* y, uint8_t* argmax, int64_t N, int64_t H, int64_t W, int64_t C, int kernel,
                    int stride, int padding, dwt_stream_t stream) {
  int OH = 0, OW = 0;
  if (int rc = pool_check(N, H, W, C, kernel, stride, padding, &OH, &OW)) return rc;
  if (!x || !y || !argmax) return fail(DWT_E_INVALID, "null pointer argument");
  if ((((uintptr_t)x | (uintptr_t)y) % 16) != 0 || (uintptr_t)argmax % 4 != 0) return fail(DWT_E_INVALID, "pooling tensors must be 16-byte aligned");
  {
    const double in = (double)N * H * W * C, out = (double)N * OH * OW * C;
    Launch l("maxpool_fwd", nullptr, 4.0 * (in + out) + out, (cudaStream_t)stream);
    dwt::maxpool_fwd_launch(x, y, argmax, (int)N, (int)H, (int)W, (int)C, OH, OW, kernel, stride, padding, (cudaStream_t)stream);
  }
  return check_launch("max-pool forward kernel");
}

int dwt_maxpool_bwd(const float* dy, const uint8_t* argmax, float* dx, int64_t N, int64_t H, int64_t W, int64_t C, int kernel,
                    int stride, int padding, dwt_stream_t stream) {
  int OH = 0, OW = 0;
  if (int rc = pool_check(N, H, W, C, kernel, stride, padding, &OH, &OW)) return rc;
  if (!dy || !dx || !argmax) return fail(DWT_E_INVALID, "null pointer argument");
  if ((((uintptr_t)dy | (uintptr_t)dx) % 16) != 0 || (uintptr_t)argmax % 4 != 0) return fail(DWT_E_INVALID, "pooling tensors must be 16-byte aligned");
  {
    const double in = (double)N * H * W * C, out = (double)N * OH * OW * C;
    Launch l("maxpool_bwd", nullptr, 4.0 * (in + out) + out, (cudaStream_t)stream);
    dwt::maxpool_bwd_launch(dy, argmax, dx, (int)N, (int)H, (int)W, (int)C, OH, OW, kernel, stride, padding, (cudaStream_t)stream);
  }
  return check_launch("max-pool backward kernel");
}

int64_t dwt_launch_count(void) { return g_launches.load(); }

void dwt_profile_begin(void) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  for (auto& r : g_prof) { g_event_pool.push_back(r.a); g_event_pool.push_back(r.b); }
  g_prof.clear();
  g_prof_on = true;
}

int dwt_profile_end(dwt_profile_entry* out, int max_entries) {
  std::vector<ProfRec> recs;
  {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof_on = false;
    recs.swap(g_prof);
  }
  int n = 0;
  for (auto& r : recs) {
    float ms = 0.f;
    if (cudaEventSynchronize(r.b) == cudaSuccess && cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
      int k = 0;
      for (; k < n; ++k)
        if (strcmp(out[k].name, r.name) == 0) break;
      if (k == n && n < max_entries) {
        memset(&out[n], 0, sizeof(out[n]));
        strncpy(out[n].name, r.name, sizeof(out[n].name) - 1);
        ++n;
      }
      if (k < n) { out[k].launches += 1; out[k].ms += ms; out[k].bytes += r.bytes; }
    }
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_event_pool.push_back(r.a); g_event_pool.push_back(r.b);
  }
  return n;
}

}  // extern "C"

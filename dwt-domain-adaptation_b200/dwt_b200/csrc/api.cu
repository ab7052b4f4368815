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

// what: printf-style name of the kernel, formatted only when the launch failed
int check_launch(const char* what, ...) {
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    cudaGetLastError();
    char name[128];
    va_list ap;
    va_start(ap, what);
    vsnprintf(name, sizeof(name), what, ap);
    va_end(ap);
    return fail(DWT_E_LAUNCH, "%s: %s", name, cudaGetErrorString(e));
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

// CTAs per problem of a tensor-core contraction: one full wave of 2 CTAs per SM.  Problems: (domain, super-block);
// at group size 128 also (domain, group) of the off-diagonal Gram block and (domain, block of R), see tc_pair_chunks
int tc_chunks(const dwt::Geom& g, int problems = 0) {
  if (problems == 0) problems = dwt::tc_superblocks(g) * g.D;
  int n = 2 * sm_count() / problems;
  const int64_t tiles = (int64_t)g.N * ((g.HW + 31) / 32);
  if (n > tiles) n = (int)tiles;
  return n < 1 ? 1 : n;
}
// group size 128: the forward's off-diagonal Gram blocks (SB/2 per domain) and the backward's four blocks of R per group
int tc_pair_chunks(const dwt::Geom& g, bool bwd) {
  const int SB = dwt::tc_superblocks(g);
  return tc_chunks(g, (bwd ? 2 * SB : SB / 2) * g.D);
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

int check_align(bool bf16, uintptr_t bits, const char* what) {
  if (bits % (bf16 ? 8 : 16) == 0) return DWT_OK;
  return bf16 ? fail(DWT_E_INVALID, "%s must be 8-byte aligned (bf16)", what) : fail(DWT_E_INVALID, "%s must be 16-byte aligned", what);
}
// family name of a launch in the profile: bf16 calls report under their own names (algorithmic bytes at 2 B/element)
inline const char* fam(bool bf16, const char* f32, const char* b16) { return bf16 ? b16 : f32; }

// channels-last launch shaping.  Every kernel is ONE wave of persistent CTAs sweeping 32-row chunks (norm_cl.cu):
// grid.x CTAs per (domain, column slab), grid.y slabs, grid.z = D domains side by side.  (grid.z = 1 -- all CTAs
// sweeping the domains one after the other, so that the whole grid moves through the tensor as a single window --
// writes three times the partial rows for no extra L2 hits;
// the kernels still accept it, DWT_CL_SEQ_MB=<tensor MB threshold> turns it on for experiments.)
struct ClPlan { int nred, new_, S, gridy, gz_red, gz_ew; };
ClPlan cl_plan(const dwt::Geom& g, int slots_red, int slots_ew, int unroll_red, int unroll_ew) {
  static const int seq_mb = env_int("DWT_CL_SEQ_MB", 1 << 30);  // experiment switch, off by default
  const int C4 = g.C / 4, gridy = dwt::cl_slabs(g.C), CW = (C4 + gridy - 1) / gridy,
            rpi = 256 / dwt::cl_lane(g.C, CW);
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
// different shapes can share one zero-initialised buffer.  Scratch (any content) follows; the two-site tail carves
// a second site's scratch behind the first (carve(..., start = first.bytes)), sharing the head.
constexpr size_t kMaxGroups = 65536;
constexpr size_t kOffCounters = 256;
constexpr size_t kOffDom1 = kOffCounters + sizeof(int) * DWT_MAX_DOMAINS * kMaxGroups;
constexpr size_t kOffDom2 = kOffDom1 + sizeof(int) * kMaxGroups;
constexpr size_t kOffScratch = kOffDom2 + sizeof(int) * kMaxGroups;

Workspace carve(void* base, int64_t C, int GS, int D, size_t start = kOffScratch) {
  const int G = (int)(C / GS);
  const int cap = chunk_cap(GS, G, D);
  size_t off = start;
  auto take = [&](size_t nbytes) { size_t o = off; off = align_up(off + nbytes, 256); return o; };
  char* b = static_cast<char*>(base);
  Workspace w;
  w.status = reinterpret_cast<int*>(b);
  w.counters = reinterpret_cast<int*>(b + kOffCounters);
  w.dom_counter = reinterpret_cast<int*>(b + kOffDom1);
  w.dom_counter2 = reinterpret_cast<int*>(b + kOffDom2);
  const bool gs128 = GS == DWT_TC_MAX_GROUP_SIZE;         // tensor-core kernels only: no tiled partials
  size_t partial_floats = gs128 ? 0 : (size_t)D * G * cap * (GS * GS + GS);
  if (GS >= 8 && 64 % GS == 0) {                           // tensor-core contraction: per super-block partials
    const size_t tc = ((size_t)2 * sm_count() + (size_t)((C + 63) / 64) * D) * (64 * 64 + 64);
    if (tc > partial_floats) partial_floats = tc;
  }
  if (gs128) {
    // tc_chunks(g, problems) * problems <= max(2 SMs, problems).  Forward: SB diagonal blocks, then SB/2 off-diagonal
    // blocks behind them; backward: 2 SB blocks of R -- per domain.  This stays within the partials of the group-size-64
    // call on 2C channels, whose workspace therefore covers this one (dwt_workspace_bytes, dwt_b200.h).
    const size_t S2 = (size_t)2 * sm_count(), P = (size_t)(C / 64) * D;
    auto wave = [&](size_t problems) { return problems > S2 ? problems : S2; };
    const size_t fwd = wave(P) + wave(P / 2), bwd = wave(2 * P);
    partial_floats = (fwd > bwd ? fwd : bwd) * (64 * 64 + 64);
  }
  size_t red_floats = 1;
  if (dwt::cl_supports((int)C, GS)) {                      // channels-last path: per-CTA rows of C/4-column vectors
    const size_t W = (size_t)dwt::cl_bwd_width((int)C, GS);
    const int gridy = dwt::cl_slabs((int)C);                // cl_plan's grid.x <= 3 SMs / grid.y
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
  // group size 128: forward SB diagonal + SB/2 off-diagonal blocks, backward 2 SB blocks of R, per domain
  w.gram = reinterpret_cast<float*>(b + take(sizeof(float) * (size_t)D * (gs128 ? 2 : 1) * SBn * (64 * 64 + 64)));
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

// vec = 4 when rows can be read as 4-element vectors: HW % 4 == 0 and a0..a2 aligned to 4 elements of elem_bytes each
// (16 bytes in fp32, 8 in bf16), so an aligned bf16 call gets the plan of the fp32 call of its shape
int make_plan(Plan& p, KernelKind reduce_kind, KernelKind ew_kind, const void* a0, const void* a1, const void* a2,
              int64_t N, int64_t C, int64_t HW, int GS, int D, int elem_bytes) {
  if (N <= 0 || C <= 0 || HW <= 0) return fail(DWT_E_INVALID, "empty tensor (N=%lld C=%lld HW=%lld)", (long long)N,
                                               (long long)C, (long long)HW);
  if (GS < 1 || (GS > DWT_MAX_GROUP_SIZE && GS != DWT_TC_MAX_GROUP_SIZE))
    return fail(DWT_E_UNSUPPORTED, "group_size %d outside [1,%d] and not %d", GS, DWT_MAX_GROUP_SIZE, DWT_TC_MAX_GROUP_SIZE);
  if (C % GS != 0) return fail(DWT_E_INVALID, "channels %lld not divisible by group_size %d", (long long)C, GS);
  if (D < 1 || D > DWT_MAX_DOMAINS) return fail(DWT_E_INVALID, "n_domains %d outside [1,%d]", D, DWT_MAX_DOMAINS);
  if (N * C * HW >= (int64_t)1 << 31 || C / GS > 65535)
    return fail(DWT_E_UNSUPPORTED, "shape too large for 32-bit item indexing");
  dwt::Geom& g = p.gm;
  g.N = (int)N; g.C = (int)C; g.HW = (int)HW; g.GS = GS; g.G = (int)(C / GS); g.D = D;
  g.M = (float)((double)N * (double)HW);
  const uintptr_t bits = (uintptr_t)a0 | (uintptr_t)a1 | (uintptr_t)a2;
  p.vec = (HW % 4 == 0 && bits % (4 * elem_bytes) == 0) ? 4 : 1;
  const bool small = dwt::small_supports(GS);
  int64_t work_units;   // CTA-sized pieces of work available per (domain, group)
  if (small) work_units = (N * (HW / p.vec) + dwt::kThreads * 2 - 1) / (dwt::kThreads * 2);
  else work_units = (N * HW + 127) / 128;
  if (work_units < 1) work_units = 1;
  shape(g, work_units, reduce_kind, small, &g.nchunks);
  p.gm_ew = g;
  shape(p.gm_ew, work_units, ew_kind, small, &p.chunks_ew);
  p.gm_ew.nchunks = g.nchunks;
  return DWT_OK;
}

// ---- which kernel family runs a norm call ------------------------------------------------------------------
// CL: channels-last (DWT_LAYOUT_NHWC) register-resident kernels, group sizes 1, 2, 4.  SMALL: their NCHW counterparts
// (bf16: a thread's four pixels of a channel row are 8 bytes, the fp32 plan with vec == 4).  TC: TMA + wgmma kernels,
// group sizes 8..64 and 128 (fp32 only, no other kernel is that wide); NCHW fp32 when geometry and alignment allow and
// the kernels could be set up.  TILED: NCHW fp32 shared-memory kernels, any group size up to 64, any alignment.
enum Family { CL, SMALL, TC, TILED };
enum Pass { REDUCE, FINALIZE, PREP, APPLY };

struct Route {
  Family fam;
  int align;            // bytes the activation tensors' addresses must be a multiple of; 0: any (the plan's vec adapts)
  bool inputs_only;     // the rule covers the tensors the kernels read through TMA (x, dout), not the one they write
  const char* what;     // how a refusal names the tensors (nullptr: by name)
  const char* why;      // what it says after "N-byte aligned"
};

#define DWT_CL_RULE "group_size 1, 2, 4 with C a multiple of 4, C/4 <= 16384"

// Family and alignment rule of a call with plan p, or the refusal of its geometry or of its second gradient addend
// (dout2, backward only: the channels-last kernels read it).  No device or driver call: the tensor-core kernels are
// set up (ensure_tc) only once the call has passed every check.
int route(const Plan& p, bool nhwc, bool bf16, const void* dout2, Route* r) {
  const dwt::Geom& g = p.gm;
  const bool cl = dwt::cl_supports(g.C, g.GS), tc_nhwc = dwt::tc_supports(g, 4) && g.HW % 4 == 0, small = dwt::small_supports(g.GS);
  if (g.GS == DWT_TC_MAX_GROUP_SIZE) {
    if (bf16) return fail(DWT_E_UNSUPPORTED, "group_size 128 is built for fp32 activations (C=%d HW=%d N=%d)", g.C, g.HW, g.N);
    if (!(nhwc ? tc_nhwc : dwt::tc_supports(g, p.vec)))
      return fail(DWT_E_UNSUPPORTED, "group_size 128 runs on the tensor-core kernels only: HW >= 32 and a multiple of 4, "
                  "N*HW >= 4096 per domain, NCHW tensors 16-byte aligned (C=%d HW=%d N=%d)", g.C, g.HW, g.N);
  }
  auto fail_nhwc = [&] {
    return fail(DWT_E_UNSUPPORTED, "channels-last %s built for " DWT_CL_RULE ", and for the tensor-core kernels: group_size "
                "8, 16, 32, 64, HW >= 32 and a multiple of 4, N*HW >= 4096 per domain (C=%d HW=%d N=%d gs=%d)",
                bf16 ? "bf16 activations are" : "layout is", g.C, g.HW, g.N, g.GS);
  };
  if (bf16 && nhwc && !cl && !tc_nhwc) return fail_nhwc();
  if (bf16 && !nhwc && !(small ? g.HW % 4 == 0 : dwt::tc_supports(g, 4) && g.HW % 8 == 0))
    return fail(DWT_E_UNSUPPORTED, "NCHW bf16 activations are built for group_size 1, 2, 4 and batch norm with HW a multiple "
                "of 4, and for the tensor-core kernels: group_size 8, 16, 32, 64, HW >= 32 and a multiple of 8, N*HW >= 4096 "
                "per domain (C=%d HW=%d N=%d gs=%d)", g.C, g.HW, g.N, g.GS);
  if (dout2 && (!nhwc || tc_nhwc || (uintptr_t)dout2 % (bf16 ? 8 : 16) != 0))
    return fail(nhwc && !tc_nhwc ? DWT_E_INVALID : DWT_E_UNSUPPORTED, "a second gradient addend (dout2) is built for the "
                "channels-last kernels of group sizes 1, 2, 4 (16-byte aligned tensor, 8 for bf16); add it to dout otherwise");
  if (nhwc) {
    if (!cl && !tc_nhwc) return fail_nhwc();
    *r = cl ? Route{CL, bf16 ? 8 : 16, false, "channels-last tensors", bf16 ? " (bf16)" : ""}
            : Route{TC, 16, false, nullptr, " (channels-last tensor-core kernels: TMA)"};
    return DWT_OK;
  }
  if (small) *r = Route{SMALL, bf16 ? 8 : 0, false, nullptr, " (bf16)"};
  else if (bf16) *r = Route{TC, 16, true, nullptr, " (bf16 NCHW: TMA)"};
  else *r = Route{g.GS > DWT_MAX_GROUP_SIZE || dwt::tc_supports(g, p.vec) ? TC : TILED, 0, false, nullptr, ""};
  return DWT_OK;
}

// Profile family name of a launch: [backward][family][pass][channels-last * 2 + bf16].  bf16 launches report under
// their own names (algorithmic bytes at 2 B/element); fp32 channels-last prep runs, and is named as, the NCHW one.
const char* const kProfName[2][4][4][4] = {
    {{{"", "", "cl_stats", "cl_stats_bf16"}, {"", "", "cl_fwd_finalize", "cl_fwd_finalize_bf16"},
      {"", "", "eval_prep", "cl_eval_prep_bf16"}, {"", "", "cl_apply", "cl_apply_bf16"}},
     {{"small_stats", "small_stats_bf16", "", ""}, {"", "", "", ""}, {"eval_prep", "eval_prep_bf16", "", ""},
      {"small_apply", "small_apply_bf16", "", ""}},
     {{"tc_stats", "tc_stats_bf16", "tc_stats_nhwc", "tc_stats_nhwc_bf16"},
      {"dense_fwd_finalize", "dense_fwd_finalize_bf16", "dense_fwd_finalize", "dense_fwd_finalize_bf16"},
      {"eval_prep", "eval_prep_bf16", "eval_prep", "eval_prep_bf16"},
      {"tc_apply", "tc_apply_bf16", "tc_apply_nhwc", "tc_apply_nhwc_bf16"}},
     {{"tiled_stats", "", "", ""}, {"", "", "", ""}, {"eval_prep", "", "", ""}, {"tiled_apply", "", "", ""}}},
    {{{"", "", "cl_bwd_reduce", "cl_bwd_reduce_bf16"}, {"", "", "cl_bwd_finalize", "cl_bwd_finalize_bf16"},
      {"", "", "bwd_prep", "cl_bwd_prep_bf16"}, {"", "", "cl_bwd_apply", "cl_bwd_apply_bf16"}},
     {{"small_bwd_reduce", "small_bwd_reduce_bf16", "", ""}, {"", "", "", ""}, {"bwd_prep", "bwd_prep_bf16", "", ""},
      {"small_bwd_apply", "small_bwd_apply_bf16", "", ""}},
     {{"tc_bwd_reduce", "tc_bwd_reduce_bf16", "tc_bwd_reduce_nhwc", "tc_bwd_reduce_nhwc_bf16"},
      {"dense_bwd_finalize", "dense_bwd_finalize_bf16", "dense_bwd_finalize", "dense_bwd_finalize_bf16"},
      {"bwd_prep", "bwd_prep_bf16", "bwd_prep", "bwd_prep_bf16"},
      {"tc_bwd_apply", "tc_bwd_apply_bf16", "tc_bwd_apply_nhwc", "tc_bwd_apply_nhwc_bf16"}},
     {{"tiled_bwd_reduce", "", "", ""}, {"", "", "", ""}, {"bwd_prep", "", "", ""}, {"tiled_bwd_apply", "", "", ""}}}};

int check_running(bool need_running, float* const* rmean, float* const* rcov, int D) {
  if (!need_running) return DWT_OK;
  if (!rmean || !rcov) return fail(DWT_E_INVALID, "running buffers required");
  for (int d = 0; d < D; ++d)
    if (!rmean[d] || !rcov[d]) return fail(DWT_E_INVALID, "running buffer of domain %d is null", d);
  return DWT_OK;
}

dwt::FwdFin make_fwd_fin(float a, float b, float momentum, float unbias, int update_running, bool need_running,
                         float* const* rmean, float* const* rcov, float* save_mean, float* save_w, const Workspace& w, int D) {
  dwt::FwdFin fin{};
  fin.a = a; fin.b = b; fin.momentum = momentum; fin.unbias = unbias;
  fin.update_running = update_running;
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
  return fin;
}

dwt::BwdFin make_bwd_fin(float a, int mode, int epi, const float* save_mean, const float* save_w, const float* gamma,
                         float* dgamma, float* dbeta, const Workspace& w) {
  dwt::BwdFin fin{};
  fin.a = a; fin.mode = mode; fin.epi = epi;
  fin.save_mean = save_mean; fin.save_w = save_w; fin.gamma = gamma;
  fin.coef = w.coef; fin.dgb_part = w.dgb_part;
  fin.dgamma = (epi & DWT_EPI_AFFINE) ? dgamma : nullptr;
  fin.dbeta = (epi & DWT_EPI_AFFINE) ? dbeta : nullptr;
  fin.dom_counter = w.dom_counter2;
  return fin;
}

// A norm call past its checks: plan, route, workspace, and its mode with the layout and dtype bits stripped
struct Call {
  Plan p;
  Route r;
  Workspace w;
  bool nhwc, bf16;
  int mode;
  const char* name(bool bwd, Pass ps) const { return kProfName[bwd][r.fam][ps][2 * nhwc + bf16]; }
};

// The whitening basis of a call, and the per-group matrices its forward saves for the backward:
//   CHOLESKY       dwt_whiten_*, dwt_bn_* (nothing saved beyond save_w)
//   NEWTON_SCHULZ  dwt_whiten_zca_*: `iters` iterations, save = save_p [D][C/gs][iters][gs][gs]
//   EIGH           dwt_whiten_eigh_*: the exact ZCA basis, save = save_e [D][C/gs][gs+1][gs] (U, then lambda)
//   COLOR          dwt_whiten_color_*: the Cholesky basis coloured, y = color W (x - mean) + bias; color W goes to the
//                  workspace's coefficient area (w.coef, unused by a forward), bias into the apply's accumulator
// All but CHOLESKY run their own dense pair in place of fwd_factor / bwd_coef; every other pass is the Cholesky basis's.
struct Basis {
  enum Kind { CHOLESKY, NEWTON_SCHULZ, EIGH, COLOR } kind = CHOLESKY;
  int iters = 0;
  const float* save = nullptr;     // written by the forward, read by the backward
  const float* color = nullptr;    // COLOR: [C/gs][gs][gs] and [C]
  const float* bias = nullptr;
  float* dcolor = nullptr;         // COLOR backward: both or neither
  float* dbias = nullptr;
  bool own() const { return kind != CHOLESKY; }
};

int basis_refuse(const Basis& z, int64_t N, int64_t C, int64_t HW, int GS) {
  return fail(DWT_E_UNSUPPORTED, "the %s is built for the tensor-core kernels only: group_size 8, 16, 32, 64, HW >= 32 "
              "and a multiple of 4 (NCHW bf16: of 8), N*HW >= 4096 per domain, tensors 16-byte aligned (C=%lld HW=%lld N=%lld gs=%d)",
              z.kind == Basis::EIGH ? "exact ZCA basis (eigendecomposition)" : z.kind == Basis::COLOR ? "colouring transform" : "ZCA basis",
              (long long)C, (long long)HW, (long long)N, GS);
}

int check_param(const float* p, const char* name) {
  if (!p) return fail(DWT_E_INVALID, "null pointer argument (%s)", name);
  if ((uintptr_t)p % 16 != 0) return fail(DWT_E_INVALID, "%s must be 16-byte aligned", name);
  return DWT_OK;
}

// a call's own basis arguments, and its family: validate()'s route, which must be the tensor-core one
int basis_check(const Call& c, const Basis& z, bool bwd) {
  if (z.kind == Basis::COLOR) {
    if (int rc = check_param(z.color, "color")) return rc;
    if (!bwd) { if (int rc = check_param(z.bias, "bias")) return rc; }
    if ((z.dcolor == nullptr) != (z.dbias == nullptr)) return fail(DWT_E_INVALID, "dcolor and dbias go together");
    if (z.dcolor) {
      if (int rc = check_param(z.dcolor, "dcolor")) return rc;
      if (int rc = check_param(z.dbias, "dbias")) return rc;
    }
  } else {
    const char* name = z.kind == Basis::EIGH ? "save_e" : "save_p";
    if (z.kind == Basis::NEWTON_SCHULZ && (z.iters < 1 || z.iters > DWT_ZCA_MAX_ITERATIONS))
      return fail(DWT_E_INVALID, "iterations %d outside [1,%d]", z.iters, DWT_ZCA_MAX_ITERATIONS);
    if (int rc = check_param(z.save, name)) return rc;
  }
  const dwt::Geom& g = c.p.gm;
  if (g.GS > DWT_MAX_GROUP_SIZE || c.r.fam != TC) return basis_refuse(z, g.N, g.C, g.HW, g.GS);
  return DWT_OK;
}

const char* basis_family(const Basis& z, bool bwd, bool bf16) {
  if (z.kind == Basis::EIGH) return bwd ? fam(bf16, "dense_bwd_eigh", "dense_bwd_eigh_bf16") : fam(bf16, "dense_fwd_eigh", "dense_fwd_eigh_bf16");
  if (z.kind == Basis::COLOR) return bwd ? fam(bf16, "dense_bwd_color", "dense_bwd_color_bf16") : fam(bf16, "dense_fwd_color", "dense_fwd_color_bf16");
  return bwd ? fam(bf16, "dense_bwd_zca", "dense_bwd_zca_bf16") : fam(bf16, "dense_fwd_zca", "dense_fwd_zca_bf16");
}

void basis_fwd(const float* gram, const float* shift, const dwt::Geom& gm, const dwt::FwdFin& fin, const Basis& z, const Workspace& w,
               cudaStream_t st) {
  if (z.kind == Basis::EIGH) dwt::dense_fwd_eigh(gram, shift, gm, fin, const_cast<float*>(z.save), st);
  else if (z.kind == Basis::COLOR) dwt::dense_fwd_color(gram, shift, gm, fin, z.color, w.coef, st);
  else dwt::dense_fwd_zca(gram, shift, gm, fin, z.iters, const_cast<float*>(z.save), st);
}

void basis_bwd(const float* rgram, const dwt::Geom& gm, const dwt::BwdFin& fin, const Basis& z, float* dybar, cudaStream_t st) {
  if (z.kind == Basis::EIGH) dwt::dense_bwd_eigh(rgram, gm, fin, z.save, dybar, st);
  else if (z.kind == Basis::COLOR) dwt::dense_bwd_color(rgram, gm, fin, z.color, z.dcolor, z.dbias, dybar, st);
  else dwt::dense_bwd_zca(rgram, gm, fin, z.iters, z.save, dybar, st);
}

// The checks both directions make, in order; `own` holds the direction's own (residual, running buffers, gradient
// outputs, basis arguments), checked before the epilogue's family rule.  in0, in1: the tensors the kernels read (x, x or
// x, dout); out: the one they write (y or dx); dout2: the backward's second gradient addend; z: the call's basis, which,
// when it is not Cholesky, must end up on the tensor-core kernels.
template <class Own>
int validate(Call& c, const Basis& z, bool bwd, const void* in0, const void* in1, const void* out, const void* dout2, int64_t N,
             int64_t C, int64_t HW, int GS, int D, int mode, int epi, const float* gamma, const float* beta,
             const float* save_mean, const float* save_w, void* ws, size_t ws_bytes, Own own) {
  c.nhwc = (mode & DWT_LAYOUT_NHWC) != 0, c.bf16 = (mode & DWT_DTYPE_BF16) != 0, c.mode = mode & 0xFF;
  const int elem_bytes = c.bf16 && !c.nhwc ? 2 : 4;
  // colouring names itself in every refusal of its geometry, make_plan()'s and route()'s included
  auto geometry = [&](int rc) { return rc == DWT_E_UNSUPPORTED && z.kind == Basis::COLOR ? basis_refuse(z, N, C, HW, GS) : rc; };
  if (int rc = geometry(make_plan(c.p, bwd ? K_BWD_REDUCE : K_STATS, bwd ? K_BWD_APPLY : K_APPLY, in0, in1, out, N, C, HW,
                                  GS, D, elem_bytes)))
    return rc;
  if (!in0 || !in1 || !out || !save_mean || !save_w || !ws) return fail(DWT_E_INVALID, "null pointer argument");
  if (int rc = geometry(route(c.p, c.nhwc, c.bf16, dout2, &c.r))) return rc;
  const uintptr_t bits = (uintptr_t)in0 | (uintptr_t)in1 | (c.r.inputs_only ? 0 : (uintptr_t)out);
  if (c.r.align && bits % c.r.align != 0)
    return fail(DWT_E_INVALID, "%s must be %d-byte aligned%s", c.r.what ? c.r.what : bwd ? (c.r.inputs_only ? "x and dout" : "x, dout and dx")
                : (c.r.inputs_only ? "x" : "x and y"), c.r.align, c.r.why);
  if (c.mode != DWT_MODE_TRAIN && c.mode != DWT_MODE_EVAL) return fail(DWT_E_INVALID, "bad mode %d", c.mode);
  if ((epi & DWT_EPI_RELU) && !(epi & DWT_EPI_AFFINE)) return fail(DWT_E_INVALID, "RELU epilogue needs AFFINE");
  if ((epi & DWT_EPI_AFFINE) && (!gamma || !beta)) return fail(DWT_E_INVALID, "AFFINE epilogue needs gamma and beta");
  if (int rc = own()) return rc;
  if (epi != 0 && c.r.fam != CL && c.r.fam != SMALL)
    return fail(DWT_E_UNSUPPORTED, "fused gamma/beta/ReLU epilogue is built for group_size 1, 2, 4 (got %d)", GS);
  c.w = carve(ws, C, GS, D);
  if (c.w.bytes > ws_bytes) return fail(DWT_E_WORKSPACE, "workspace too small: need %zu bytes, got %zu", c.w.bytes, ws_bytes);
  if ((uintptr_t)ws % 256 != 0) return fail(DWT_E_WORKSPACE, "workspace must be 256-byte aligned");
  if ((c.r.fam == TC || c.r.fam == TILED) && ensure_tiled() != 0)
    return fail(DWT_E_LAUNCH, "cudaFuncSetAttribute failed (%d)", g_tiled_rc);
  if (c.r.fam == TC && ensure_tc() != 0) {
    if (c.bf16 || c.nhwc || GS > DWT_MAX_GROUP_SIZE) return fail(DWT_E_LAUNCH, "tensor-core kernel set-up failed (%d)", g_tc_rc);
    if (z.own()) return basis_refuse(z, N, C, HW, GS);                // no other kernels take it
    c.r.fam = TILED;      // fp32 NCHW up to group size 64: the tiled kernels take every geometry
  }
  return DWT_OK;
}

int whiten_like_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int GS, int D, int mode, float a,
                    float b, float momentum, float unbias, int update_running, float* const* rmean,
                    float* const* rcov, const float* gamma, const float* beta, const float* residual,
                    uint8_t* relu_mask, int epi, float* save_mean, float* save_w, void* ws, size_t ws_bytes,
                    cudaStream_t st, const Basis& basis = Basis{}) {
  Call c;
  const bool need_running = ((mode & 0xFF) == DWT_MODE_EVAL) || update_running;
  const int rc = validate(c, basis, false, x, x, y, nullptr, N, C, HW, GS, D, mode, epi, gamma, beta, save_mean, save_w, ws, ws_bytes, [&] {
    if ((epi & DWT_EPI_RESIDUAL) && ((epi & 3) != 3 || !residual)) return fail(DWT_E_INVALID, "RESIDUAL epilogue needs AFFINE|RELU and a residual tensor");
    if (epi & DWT_EPI_RESIDUAL) if (int rc = check_align(c.bf16, (uintptr_t)residual, "residual")) return rc;
    if (relu_mask && !((epi & DWT_EPI_RESIDUAL) && c.nhwc))
      return fail(DWT_E_UNSUPPORTED, "the ReLU byte map is written by the channels-last RESIDUAL epilogue only");
    if (basis.own()) if (int rc = basis_check(c, basis, false)) return rc;
    return check_running(need_running, rmean, rcov, D);
  });
  if (rc) return rc;
  const Plan& p = c.p; const Workspace& w = c.w;
  const bool bf16 = c.bf16, nhwc = c.nhwc, train = c.mode == DWT_MODE_TRAIN;
  const dwt::FwdFin fin = make_fwd_fin(a, b, momentum, unbias, train ? update_running : 0, need_running, rmean, rcov,
                                       save_mean, save_w, w, D);
  const double n_el = (double)D * (double)N * (double)C * (double)HW;
  const double E = (bf16 ? 2.0 : 4.0) * n_el, Mb = 0.25 * n_el;   // bytes of one activation tensor, of the ReLU byte map
  const ClPlan cp = c.r.fam == CL ? cl_plan(p.gm, 3, 3, 8, (epi & DWT_EPI_RESIDUAL) ? 4 : 8) : ClPlan{};
  const bool gs128 = GS == DWT_TC_MAX_GROUP_SIZE;
  const size_t pair_part = (size_t)tc_chunks(p.gm) * dwt::tc_superblocks(p.gm) * D * (64 * 64 + 64);   // behind the diagonal partials
  // reduce: batch statistics (train) or the eval coefficients from the running buffers
  if (train) {
    {
      Launch l(c.name(false, REDUCE), &p.gm, E, st);
      switch (c.r.fam) {
        case CL: dwt::cl_stats(x, bf16, p.gm, cp.nred, cp.gz_red, w.partial, w.shift, st); break;
        case SMALL: dwt::small_stats(x, bf16, p.gm, p.vec, fin, w.partial, w.counters, st); break;
        case TILED: dwt::tiled_stats(x, p.gm, p.vec, fin, w.partial, w.counters, st); break;
        case TC: {
          int cr = dwt::tc_stats(x, bf16, nhwc, p.gm, tc_chunks(p.gm), w.shift, w.partial, st);
          // group size 128: the off-diagonal blocks behind the diagonal ones (a second read of x, counted once above)
          if (cr == 0 && gs128)
            cr = dwt::tc_gram_pair(x, nhwc, p.gm, tc_pair_chunks(p.gm, false), w.shift, w.partial + pair_part, st);
          if (cr) return fail(DWT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d) x=%p N=%d C=%d HW=%d D=%d", cr, (const void*)x, p.gm.N, p.gm.C, p.gm.HW, p.gm.D);
        }
      }
    }
    if (c.r.fam == CL || c.r.fam == TC) {   // the small and tiled kernels finalize in their last CTA
      if (int rc = check_launch(c.r.fam == CL ? "channels-last statistics kernel" : "tensor-core statistics kernel")) return rc;
      Launch l(basis.own() ? basis_family(basis, false, bf16) : c.name(false, FINALIZE), &p.gm, 0.0, st);
      if (c.r.fam == CL) {
        dwt::cl_fwd_finalize(w.partial, cp.nred, w.shift, p.gm, fin, st);
      } else {
        dwt::dense_partial_reduce(w.partial, tc_chunks(p.gm), dwt::tc_superblocks(p.gm) * D, w.gram, st);
        if (gs128)
          dwt::dense_partial_reduce(w.partial + pair_part, tc_pair_chunks(p.gm, false), dwt::tc_superblocks(p.gm) / 2 * D,
                                    w.gram + (size_t)dwt::tc_superblocks(p.gm) * D * (64 * 64 + 64), st);
        if (basis.own()) basis_fwd(w.gram, w.shift, p.gm, fin, basis, w, st);
        else dwt::dense_fwd_factor(w.gram, w.shift, p.gm, fin, st);
      }
    }
  } else if (basis.own()) {
    Launch l(basis_family(basis, false, bf16), &p.gm, 0.0, st);
    basis_fwd(nullptr, nullptr, p.gm, fin, basis, w, st);
  } else {
    Launch l(c.name(false, PREP), &p.gm, 0.0, st);
    if (c.r.fam == TC) dwt::dense_fwd_factor(nullptr, nullptr, p.gm, fin, st);
    else if (c.r.fam == TILED) dwt::tiled_eval_prep(p.gm, fin, st);
    else dwt::small_eval_prep(p.gm, fin, st);
  }
  if (int rc = check_launch(c.r.fam == CL ? "channels-last finalize kernel" : "whitening statistics kernel")) return rc;
  {
    Launch l(c.name(false, APPLY), &p.gm, (epi & DWT_EPI_RESIDUAL) ? 3.0 * E + (relu_mask ? Mb : 0.0) : 2.0 * E, st);
    switch (c.r.fam) {
      case CL: dwt::cl_apply(x, y, bf16, p.gm, cp.new_, cp.gz_ew, epi, save_mean, save_w, gamma, beta, residual, relu_mask, st); break;
      case SMALL: dwt::small_apply(x, y, bf16, p.gm_ew, p.vec, p.chunks_ew, epi, save_mean, save_w, gamma, beta, residual, st); break;
      case TILED: dwt::tiled_apply(x, y, p.gm_ew, p.vec, p.chunks_ew, save_mean, save_w, st); break;
      case TC:   // colouring: color W from the workspace, and the bias
        if (int cr = basis.kind == Basis::COLOR
                         ? dwt::tc_apply(x, y, bf16, nhwc, p.gm, tc_apply_ctas(p.gm, 1, 64), save_mean, w.coef, st, basis.bias)
                         : dwt::tc_apply(x, y, bf16, nhwc, p.gm, tc_apply_ctas(p.gm, 1, 64), save_mean, save_w, st))
          return fail(DWT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d)", cr);
    }
  }
  return check_launch(c.r.fam == CL ? "channels-last apply kernel" : "whitening apply kernel");
}

int whiten_like_bwd(const float* x, const float* dout, const float* dout2, float* dx, int64_t N, int64_t C, int64_t HW, int GS, int D,
                    int mode, float a, const float* save_mean, const float* save_w, const float* gamma,
                    const float* beta, const uint8_t* relu_mask, float* dresidual, int epi, float* dgamma,
                    float* dbeta, void* ws, size_t ws_bytes, cudaStream_t st, const Basis& basis = Basis{}) {
  Call c;
  const int rc = validate(c, basis, true, x, dout, dx, dout2, N, C, HW, GS, D, mode, epi, gamma, beta, save_mean, save_w, ws, ws_bytes, [&] {
    if (epi & DWT_EPI_RESIDUAL) {
      // backward of out = relu(z + residual): the ReLU mask comes from the byte map the forward wrote, the masked
      // gradient goes to dresidual and is what the apply pass reads
      if (!c.nhwc || !relu_mask || (epi & 3) != 3 || !dresidual)
        return fail(DWT_E_INVALID, "backward of a RESIDUAL forward needs the channels-last layout, AFFINE|RELU, the forward's "
                                   "ReLU byte map and dresidual (or pass dout already masked by (out > 0) with epilogue AFFINE)");
      if (int rc = check_align(c.bf16, (uintptr_t)dresidual, "dresidual")) return rc;
    } else if (relu_mask || dresidual) {
      return fail(DWT_E_INVALID, "relu_mask / dresidual belong to the RESIDUAL epilogue");
    }
    if ((dgamma == nullptr) != (dbeta == nullptr)) return fail(DWT_E_INVALID, "dgamma and dbeta go together");
    if (basis.own()) return basis_check(c, basis, true);
    return DWT_OK;
  });
  if (rc) return rc;
  const Plan& p = c.p; const Workspace& w = c.w;
  const bool bf16 = c.bf16, nhwc = c.nhwc;
  const dwt::BwdFin fin = make_bwd_fin(a, c.mode, epi, save_mean, save_w, gamma, dgamma, dbeta, w);
  const bool masked = nhwc && (epi & DWT_EPI_RESIDUAL) != 0;   // the reduction also writes the masked gradient
  const bool need_reduce = (c.mode == DWT_MODE_TRAIN) || (fin.dgamma != nullptr) || masked || (basis.dcolor != nullptr);
  const double n_el = (double)D * (double)N * (double)C * (double)HW;
  const double E = (bf16 ? 2.0 : 4.0) * n_el, Mb = 0.25 * n_el;
  const ClPlan cp = c.r.fam == CL ? cl_plan(p.gm, 2, 2, 4, 4) : ClPlan{};
  // group size 128: four blocks of R per group, 2 SB problems per domain
  const bool gs128 = GS == DWT_TC_MAX_GROUP_SIZE;
  const int rchunks = gs128 ? tc_pair_chunks(p.gm, true) : tc_chunks(p.gm);
  const int rproblems = (gs128 ? 2 : 1) * dwt::tc_superblocks(p.gm) * D;
  // reduce: the gradient moments (train, dgamma/dbeta or the masked gradient), or the eval coefficients
  if (need_reduce) {
    {
      Launch l(c.name(true, REDUCE), &p.gm, (masked ? 3.0 * E + Mb : 2.0 * E) + (dout2 ? E : 0.0), st);
      switch (c.r.fam) {
        case CL: dwt::cl_bwd_reduce(x, dout, dout2, bf16, p.gm, cp.nred, cp.gz_red, epi, save_mean, save_w, gamma, beta, relu_mask, dresidual, w.partial, st); break;
        case SMALL: dwt::small_bwd_reduce(x, dout, bf16, p.gm, p.vec, fin, beta, w.partial, w.counters, st); break;
        case TILED: dwt::tiled_bwd_reduce(x, dout, p.gm, p.vec, fin, w.partial, w.counters, st); break;
        case TC:
          // the pilot shift of dy needs save_mean to be the batch mean: not in eval (colouring's dcolor)
          if (int cr = dwt::tc_bwd_reduce(x, dout, bf16, nhwc, p.gm, rchunks, save_mean, w.partial, st, c.mode == DWT_MODE_TRAIN))
            return fail(DWT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d) x=%p dout=%p N=%d C=%d HW=%d D=%d", cr, (const void*)x, (const void*)dout, p.gm.N, p.gm.C, p.gm.HW, p.gm.D);
      }
    }
    if (c.r.fam == CL || c.r.fam == TC) {   // the small and tiled kernels finalize in their last CTA
      if (int rc = check_launch(c.r.fam == CL ? "channels-last backward reduction kernel" : "tensor-core backward reduction kernel")) return rc;
      Launch l(basis.own() ? basis_family(basis, true, bf16) : c.name(true, FINALIZE), &p.gm, 0.0, st);
      if (c.r.fam == CL) {
        dwt::cl_bwd_finalize(w.partial, cp.nred, p.gm, fin, st);
      } else {
        dwt::dense_partial_reduce(w.partial, rchunks, rproblems, w.gram, st);
        if (basis.own()) basis_bwd(w.gram, p.gm, fin, basis, w.shift, st);
        else dwt::dense_bwd_coef(w.gram, p.gm, fin, w.shift, st);
      }
    }
  } else if (basis.own()) {
    Launch l(basis_family(basis, true, bf16), &p.gm, 0.0, st);
    basis_bwd(nullptr, p.gm, fin, basis, w.shift, st);
  } else {
    Launch l(c.name(true, PREP), &p.gm, 0.0, st);
    if (c.r.fam == TC) dwt::dense_bwd_coef(nullptr, p.gm, fin, w.shift, st);
    else if (c.r.fam == TILED) dwt::tiled_bwd_prep(p.gm, fin, st);
    else dwt::small_bwd_prep(p.gm, fin, st);
  }
  if (int rc = check_launch(c.r.fam == CL ? "channels-last backward finalize kernel" : "whitening backward reduction kernel")) return rc;
  {
    Launch l(c.name(true, APPLY), &p.gm, (3.0 + (dout2 && !masked ? 1.0 : 0.0)) * E, st);
    switch (c.r.fam) {
      case CL:
        if (masked) dwt::cl_bwd_apply(x, dresidual, nullptr, dx, bf16, p.gm, cp.new_, cp.gz_ew, DWT_EPI_AFFINE, w.coef, save_mean, save_w, gamma, beta, st);
        else dwt::cl_bwd_apply(x, dout, dout2, dx, bf16, p.gm, cp.new_, cp.gz_ew, epi, w.coef, save_mean, save_w, gamma, beta, st);
        break;
      case SMALL: dwt::small_bwd_apply(x, dout, dx, bf16, p.gm_ew, p.vec, p.chunks_ew, epi, w.coef, save_mean, save_w, gamma, beta, st); break;
      case TILED: dwt::tiled_bwd_apply(x, dout, dx, p.gm_ew, p.vec, p.chunks_ew, w.coef, st); break;
      case TC:
        if (int cr = dwt::tc_bwd_apply(x, dout, dx, bf16, nhwc, p.gm, tc_apply_ctas(p.gm, 1, 64), w.coef, save_mean, w.shift, st))
          return fail(DWT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d)", cr);
    }
  }
  return check_launch(c.r.fam == CL ? "channels-last backward apply kernel" : "whitening backward apply kernel");
}

// ---- two-site residual tail (dwt_tail2_fwd / dwt_tail2_bwd) ----------------------------------------------
struct SiteConst { float a, b, unbias; };
SiteConst site_const(int kind, float eps, int64_t N, int64_t HW) {
  if (kind == DWT_KIND_BN) {                       // as dwt_bn_fwd: S = var + eps, unbiased variance into the EMA
    const double M = (double)N * (double)HW;
    return {1.f, eps, M > 1.0 ? (float)(M / (M - 1.0)) : 1.f};
  }
  return {1.f - eps, eps, 1.f};                    // as dwt_whiten_fwd
}

// checks shared by both directions; out is the tensor-sized output of the call (y, or dz)
int tail2_plan(Plan& p, int kind, bool bf16, const dwt_tail_site* s, const void* out, int64_t N, int64_t C, int64_t HW, int GS, int D) {
  if (kind != DWT_KIND_WHITEN && kind != DWT_KIND_BN) return fail(DWT_E_INVALID, "bad kind %d", kind);
  if (kind == DWT_KIND_BN && GS != 1) return fail(DWT_E_INVALID, "batch norm has group_size 1 (got %d)", GS);
  if (!s) return fail(DWT_E_INVALID, "null pointer argument");
  if (int rc = make_plan(p, K_STATS, K_APPLY, s[0].x, s[1].x, out, N, C, HW, GS, D, 4)) return rc;
  Route r;
  if (route(p, true, bf16, nullptr, &r) != DWT_OK || r.fam != CL)
    return fail(DWT_E_UNSUPPORTED, "the two-site tail runs on the channels-last kernels: " DWT_CL_RULE " (C=%lld gs=%d)",
                (long long)C, GS);
  for (int k = 0; k < 2; ++k)
    if (!s[k].x || !s[k].gamma || !s[k].beta || !s[k].save_mean || !s[k].save_w || !out) return fail(DWT_E_INVALID, "null pointer argument");
  return check_align(bf16, (uintptr_t)s[0].x | (uintptr_t)s[1].x | (uintptr_t)out, "channels-last tensors");
}

// the two sites' scratch: site 1 behind site 0, sharing the head (status word, counters)
int tail2_workspace(Workspace (&w)[2], void* ws, size_t ws_bytes, int64_t C, int GS, int D) {
  if (!ws) return fail(DWT_E_INVALID, "null pointer argument");
  w[0] = carve(ws, C, GS, D);
  w[1] = carve(ws, C, GS, D, w[0].bytes);
  if (w[1].bytes > ws_bytes) return fail(DWT_E_WORKSPACE, "workspace too small: need %zu bytes, got %zu", w[1].bytes, ws_bytes);
  if ((uintptr_t)ws % 256 != 0) return fail(DWT_E_WORKSPACE, "workspace must be 256-byte aligned");
  return DWT_OK;
}

int tail2_fwd(int kind, const dwt_tail_site* s, float* y, uint8_t* relu_mask, int64_t N, int64_t C, int64_t HW, int GS, int D,
              void* ws, size_t ws_bytes, cudaStream_t st) {
  const bool bf16 = (kind & DWT_DTYPE_BF16) != 0;
  kind &= ~DWT_DTYPE_BF16;
  Plan p;
  if (int rc = tail2_plan(p, kind, bf16, s, y, N, C, HW, GS, D)) return rc;
  if (!relu_mask) return fail(DWT_E_INVALID, "the two-site tail writes the ReLU byte map its backward reads");
  for (int k = 0; k < 2; ++k)
    if (int rc = check_running(s[k].update_running != 0, s[k].running_mean, s[k].running_cov, D)) return rc;
  Workspace w[2];
  if (int rc = tail2_workspace(w, ws, ws_bytes, C, GS, D)) return rc;
  dwt::FwdFin fin[2];
  for (int k = 0; k < 2; ++k) {
    const SiteConst sc = site_const(kind, s[k].eps, N, HW);
    fin[k] = make_fwd_fin(sc.a, sc.b, s[k].momentum, sc.unbias, s[k].update_running, s[k].update_running != 0, s[k].running_mean,
                          s[k].running_cov, s[k].save_mean, s[k].save_w, w[k], D);
  }
  const double n_el = (double)D * (double)N * (double)C * (double)HW;
  const double E = (bf16 ? 2.0 : 4.0) * n_el, Mb = 0.25 * n_el;
  const ClPlan cp = cl_plan(p.gm, 3, 3, 8, 4);
  for (int k = 0; k < 2; ++k) {            // the tail's input first: conv3 wrote it last, its end is still in L2
    Launch l(fam(bf16, "cl_stats", "cl_stats_bf16"), &p.gm, E, st);
    dwt::cl_stats(s[k].x, bf16, p.gm, cp.nred, cp.gz_red, w[k].partial, w[k].shift, st);
  }
  if (int rc = check_launch("channels-last statistics kernel")) return rc;
  {
    Launch l(fam(bf16, "cl_tail2_fwd_finalize", "cl_tail2_fwd_finalize_bf16"), &p.gm, 0.0, st);
    dwt::cl_fwd_finalize(w[0].partial, cp.nred, w[0].shift, p.gm, fin[0], st, &fin[1], (size_t)(w[1].partial - w[0].partial),
                         (size_t)(w[1].shift - w[0].shift));
  }
  if (int rc = check_launch("channels-last finalize kernel")) return rc;
  {
    Launch l(fam(bf16, "cl_tail2_apply", "cl_tail2_apply_bf16"), &p.gm, 3.0 * E + Mb, st);       // x, xd -> out + byte map
    dwt::cl_tail2_apply(s[0].x, s[1].x, y, bf16, p.gm, cp.new_, cp.gz_ew, s[0].save_mean, s[0].save_w, s[0].gamma, s[0].beta,
                        s[1].save_mean, s[1].save_w, s[1].gamma, s[1].beta, relu_mask, st);
  }
  return check_launch("channels-last two-site apply kernel");
}

int tail2_bwd(int kind, const dwt_tail_site* s, const float* dout, const float* dout2, const uint8_t* relu_mask, float* dz,
              int64_t N, int64_t C, int64_t HW, int GS, int D, void* ws, size_t ws_bytes, cudaStream_t st) {
  const bool bf16 = (kind & DWT_DTYPE_BF16) != 0;
  kind &= ~DWT_DTYPE_BF16;
  Plan p;
  if (int rc = tail2_plan(p, kind, bf16, s, dz, N, C, HW, GS, D)) return rc;
  if (!dout || !relu_mask || !s[0].dx || !s[1].dx) return fail(DWT_E_INVALID, "null pointer argument");
  if (int rc = check_align(bf16, (uintptr_t)dout | (uintptr_t)dout2 | (uintptr_t)s[0].dx | (uintptr_t)s[1].dx, "channels-last tensors")) return rc;
  for (int k = 0; k < 2; ++k)
    if ((s[k].dgamma == nullptr) != (s[k].dbeta == nullptr)) return fail(DWT_E_INVALID, "dgamma and dbeta go together");
  Workspace w[2];
  if (int rc = tail2_workspace(w, ws, ws_bytes, C, GS, D)) return rc;
  dwt::BwdFin fin[2];
  for (int k = 0; k < 2; ++k)
    fin[k] = make_bwd_fin(site_const(kind, s[k].eps, N, HW).a, DWT_MODE_TRAIN, k ? DWT_EPI_AFFINE : (DWT_EPI_AFFINE | DWT_EPI_RELU | DWT_EPI_RESIDUAL),
                          s[k].save_mean, s[k].save_w, s[k].gamma, s[k].dgamma, s[k].dbeta, w[k]);
  const double n_el = (double)D * (double)N * (double)C * (double)HW;
  const double E = (bf16 ? 2.0 : 4.0) * n_el, Mb = 0.25 * n_el;
  const ClPlan cp = cl_plan(p.gm, 2, 2, 4, 4);
  {
    Launch l(fam(bf16, "cl_tail2_bwd_reduce", "cl_tail2_bwd_reduce_bf16"), &p.gm, (4.0 + (dout2 ? 1.0 : 0.0)) * E + Mb, st);   // x, xd, dout (+ dout2), byte map -> dz
    dwt::cl_tail2_bwd_reduce(s[0].x, s[1].x, dout, dout2, bf16, p.gm, cp.nred, cp.gz_red, s[0].save_mean, s[1].save_mean, relu_mask, dz,
                             w[0].partial, (size_t)(w[1].partial - w[0].partial), st);
  }
  if (int rc = check_launch("channels-last two-site backward reduction kernel")) return rc;
  {
    Launch l(fam(bf16, "cl_tail2_bwd_finalize", "cl_tail2_bwd_finalize_bf16"), &p.gm, 0.0, st);
    dwt::cl_bwd_finalize(w[0].partial, cp.nred, p.gm, fin[0], st, &fin[1], (size_t)(w[1].partial - w[0].partial));
  }
  if (int rc = check_launch("channels-last backward finalize kernel")) return rc;
  {
    Launch l(fam(bf16, "cl_tail2_bwd_apply", "cl_tail2_bwd_apply_bf16"), &p.gm, 5.0 * E, st);       // x, xd, dz -> dx, dxd
    dwt::cl_tail2_bwd_apply(s[0].x, s[1].x, dz, s[0].dx, s[1].dx, bf16, p.gm, cp.new_, cp.gz_ew, w[0].coef, w[1].coef, st);
  }
  return check_launch("channels-last two-site backward apply kernel");
}

// ---- per-image whitening: instance (dwt_whiten_instance_*), switchable (dwt_whiten_switch_*) and latent-domain
// (dwt_whiten_latent_*) ------------------------------------------------------------------------------------------------
// Every image is its own problem.  The tensor-core kernels index their problems by (domain, super-block) and the dense
// ones by (domain, group); per-image whitening runs them with the images as the domains: Geom D = N images of N = 1 each,
// M = HW.  Statistics and the backward contraction are tc_stats / tc_bwd_reduce unchanged (tc_chunks splits an image over
// CTAs when there are fewer problems than two per SM, and gives a CTA a whole image otherwise -- then the partials are the
// reduced moments and the fixed-order reduction is skipped); apply and backward apply are tc_apply / tc_bwd_apply
// unchanged.  Between them each variant runs its own finalize:
//   instance    forward fwd_instance (fwd_factor serialises the domains of a group in one CTA for its ordered EMA);
//               backward bwd_coef unchanged (one CTA per (domain, group) already), tc_bwd_apply centred on save_mean.
//   switchable  forward sw_stats (save_stats: per-image rows and the batch row by the law of total covariance, no second
//               pass over x) -> sw_fwd_factor (mix, Cholesky + inverse, EMA); backward tc_bwd_reduce about the mixed mean
//               without the pilot centring (sum (x - m) is not zero) -> sw_bwd_coef / sw_bwd_sum / sw_dmix /
//               sw_bwd_apply_coef -> tc_bwd_apply centred on the images' own means, the per-image constant of dx in dybar.
//   latent      forward ld_stats (save_stats: per-image rows, each latent domain's weighted moments by the law of total
//               covariance, s_k) -> ld_fwd_factor (W_k per (domain, group), EMA) -> ld_mix (A_n = sum_k w_nk W_k and m~_n);
//               backward as switchable: tc_bwd_reduce about m~_n without the pilot -> ld_bwd_sum / ld_bwd_dom (per domain)
//               / ld_bwd_coef (per image) / ld_dw -> tc_bwd_apply centred on the images' own means.
// What a switchable or latent-domain call adds to an instance call (Mix{} is instance whitening)
enum MixKind { MIX_INSTANCE = 0, MIX_SWITCH = 1, MIX_LATENT = 2 };
struct Mix {
  int kind = MIX_INSTANCE;
  const float* mix = nullptr;          // switchable: [6];  latent: weights [N][K]
  const float* save_stats = nullptr;   // switchable: [N + 1][G][gs*gs + gs];  latent: dwt_b200.h.  Written by the forward
  int K = 0;                           // latent: domains
  float momentum = 0.f;
  int update_running = 0;
  float* rmean = nullptr;              // switchable: [C], [G][gs][gs];  latent: [K][C], [K][G][gs][gs]
  float* rcov = nullptr;
  float* dmix = nullptr;               // backward: switchable [6], latent dweights [N][K], or null
  const char* what() const {
    return kind == MIX_LATENT ? "latent-domain whitening" : kind == MIX_SWITCH ? "switchable whitening" : "instance whitening";
  }
};

int image_refuse(int64_t N, int64_t C, int64_t HW, int GS, int flags, const char* what) {
  return fail(DWT_E_UNSUPPORTED, "%s is built for the tensor-core kernels only: group_size 8, 16, 32, 64 "
              "dividing C, HW >= 256 and a multiple of 4 (NCHW bf16: of 8), N <= 65535 images, N*C*HW < 2^31 "
              "(C=%lld HW=%lld N=%lld gs=%d flags=%#x)", what, (long long)C, (long long)HW, (long long)N, GS, flags);
}

// flags (switchable, latent: the mode word, which may also hold DWT_MODE_EVAL) and geometry; fills gm (no device call)
int image_geom(dwt::Geom& gm, int64_t N, int64_t C, int64_t HW, int GS, int flags, const Mix& m) {
  const bool on = m.kind != MIX_INSTANCE;
  if (m.kind == MIX_LATENT && (m.K < 1 || m.K > DWT_MAX_LATENT_DOMAINS))
    return fail(DWT_E_INVALID, "n_domains %d outside [1,%d] (latent-domain whitening)", m.K, DWT_MAX_LATENT_DOMAINS);
  if (on && (flags & ~(DWT_MODE_EVAL | DWT_LAYOUT_NHWC | DWT_DTYPE_BF16)))
    return fail(DWT_E_INVALID, "bad mode %#x (DWT_MODE_TRAIN or DWT_MODE_EVAL | DWT_LAYOUT_NHWC | DWT_DTYPE_BF16)", flags);
  if (!on && (flags & ~(DWT_LAYOUT_NHWC | DWT_DTYPE_BF16)))
    return fail(DWT_E_INVALID, "bad flags %#x (DWT_LAYOUT_NHWC | DWT_DTYPE_BF16)", flags);
  flags &= ~DWT_MODE_EVAL;
  if (N <= 0 || C <= 0 || HW <= 0) return fail(DWT_E_INVALID, "empty tensor (N=%lld C=%lld HW=%lld)", (long long)N,
                                               (long long)C, (long long)HW);
  const bool nchw_bf16 = (flags & DWT_DTYPE_BF16) && !(flags & DWT_LAYOUT_NHWC);
  if ((GS != 8 && GS != 16 && GS != 32 && GS != 64) || C % GS != 0 || HW < 256 || HW % (nchw_bf16 ? 8 : 4) != 0 ||
      N > 65535 || N * C * HW >= (int64_t)1 << 31)
    return image_refuse(N, C, HW, GS, flags, m.what());
  gm = dwt::Geom{};
  gm.N = 1; gm.C = (int)C; gm.HW = (int)HW; gm.GS = GS; gm.G = (int)(C / GS); gm.D = (int)N; gm.ppc = 1;
  gm.M = (float)HW;
  gm.nchunks = tc_chunks(gm);
  return DWT_OK;
}

struct ImageWork {
  Workspace w;
  float* pd;       // switchable: [N][G][gs*gs + gs]  P_n | dm_n;         latent: [K][G][gs*gs + gs]  P_k | mubar_k
  float* part;     //             [N][G][8]           dmix terms per (image, group);  latent: [N][G][kLdMaxDomains] dweights terms
  float* sums;     //             [G][gs*gs + gs]     sum_n P_n | sum_n dm_n;  latent: [K][G][gs*gs + gs]  Wbar_k | sum w g
  float* mu;       //             [N][C]              the images' own means (the backward apply's centre)
  float* pc;       // latent:     [K][G]              <P_k, Sigma_k>
};

// Scratch behind the common head (the status word is shared with every other call on the stream's workspace):
// partials [N][SB][nchunks][64*64+64], reduced moments (only when nchunks > 1), pilot shifts / mean of dy / dybar
// [N][SB][64], backward coefficients [N][G][2 gs^2 + gs]; switchable and latent-domain whitening then pd, part, sums
// and mu (latent: and pc)
ImageWork carve_image(void* base, const dwt::Geom& gm, const Mix& m) {
  const size_t P = (size_t)dwt::tc_superblocks(gm) * gm.D, nacc = 64 * 64 + 64;
  const size_t rec = (size_t)gm.GS * gm.GS + gm.GS, PG = (size_t)gm.D * gm.G;
  size_t off = kOffScratch;
  auto take = [&](size_t nbytes) { size_t o = off; off = align_up(off + nbytes, 256); return o; };
  char* b = static_cast<char*>(base);
  ImageWork s{};
  Workspace& w = s.w;
  w.status = reinterpret_cast<int*>(b);
  w.counters = reinterpret_cast<int*>(b + kOffCounters);
  w.dom_counter = reinterpret_cast<int*>(b + kOffDom1);
  w.dom_counter2 = reinterpret_cast<int*>(b + kOffDom2);
  w.partial = reinterpret_cast<float*>(b + take(sizeof(float) * P * gm.nchunks * nacc));
  w.gram = gm.nchunks > 1 ? reinterpret_cast<float*>(b + take(sizeof(float) * P * nacc)) : w.partial;
  w.shift = reinterpret_cast<float*>(b + take(sizeof(float) * P * 64));
  w.coef = reinterpret_cast<float*>(b + take(sizeof(float) * PG * dwt::coef_stride(gm.GS)));
  if (m.kind == MIX_SWITCH) {
    s.pd = reinterpret_cast<float*>(b + take(sizeof(float) * PG * rec));
    s.part = reinterpret_cast<float*>(b + take(sizeof(float) * PG * 8));
    s.sums = reinterpret_cast<float*>(b + take(sizeof(float) * gm.G * rec));
    s.mu = reinterpret_cast<float*>(b + take(sizeof(float) * (size_t)gm.D * gm.C));
  } else if (m.kind == MIX_LATENT) {
    const size_t KG = (size_t)m.K * gm.G;
    s.pd = reinterpret_cast<float*>(b + take(sizeof(float) * KG * rec));
    s.part = reinterpret_cast<float*>(b + take(sizeof(float) * PG * dwt::kLdMaxDomains));
    s.sums = reinterpret_cast<float*>(b + take(sizeof(float) * KG * rec));
    s.mu = reinterpret_cast<float*>(b + take(sizeof(float) * (size_t)gm.D * gm.C));
    s.pc = reinterpret_cast<float*>(b + take(sizeof(float) * KG));
  }
  w.bytes = off;
  return s;
}

// A size query leaves the last error text alone
size_t image_workspace_bytes(int64_t N, int64_t C, int64_t HW, int GS, const Mix& m) {
  dwt::Geom gm;
  char saved[sizeof(g_err)];
  memcpy(saved, g_err, sizeof(g_err));
  const int rc = image_geom(gm, N, C, HW, GS, 0, m);
  memcpy(g_err, saved, sizeof(g_err));
  return rc ? 0 : carve_image(nullptr, gm, m).w.bytes;
}

// The workspace of the latent-domain bandwidth layers: the larger of the two layouts' plans, each bytes(mode) (0 where
// the layout does not run), leaving the last error text alone
template <class Bytes>
size_t larger_layout_workspace_bytes(Bytes bytes) {
  char saved[sizeof(g_err)];
  memcpy(saved, g_err, sizeof(g_err));
  size_t most = 0;
  for (int mode : {0, DWT_LAYOUT_NHWC}) {
    const size_t b = bytes(mode);
    if (b > most) most = b;
  }
  memcpy(g_err, saved, sizeof(g_err));
  return most;
}

// Profile family of a launch: [MixKind][pass][channels-last * 2 + bf16]
enum ImagePass { I_STATS, I_FWD_FINALIZE, I_APPLY, I_BWD_REDUCE, I_BWD_FINALIZE, I_BWD_APPLY };
const char* const kImageName[3][6][4] = {
    {{"iw_stats", "iw_stats_bf16", "iw_stats_nhwc", "iw_stats_nhwc_bf16"},
     {"iw_fwd_finalize", "iw_fwd_finalize_bf16", "iw_fwd_finalize", "iw_fwd_finalize_bf16"},
     {"iw_apply", "iw_apply_bf16", "iw_apply_nhwc", "iw_apply_nhwc_bf16"},
     {"iw_bwd_reduce", "iw_bwd_reduce_bf16", "iw_bwd_reduce_nhwc", "iw_bwd_reduce_nhwc_bf16"},
     {"iw_bwd_finalize", "iw_bwd_finalize_bf16", "iw_bwd_finalize", "iw_bwd_finalize_bf16"},
     {"iw_bwd_apply", "iw_bwd_apply_bf16", "iw_bwd_apply_nhwc", "iw_bwd_apply_nhwc_bf16"}},
    {{"sw_stats", "sw_stats_bf16", "sw_stats_nhwc", "sw_stats_nhwc_bf16"},
     {"sw_fwd_finalize", "sw_fwd_finalize_bf16", "sw_fwd_finalize", "sw_fwd_finalize_bf16"},
     {"sw_apply", "sw_apply_bf16", "sw_apply_nhwc", "sw_apply_nhwc_bf16"},
     {"sw_bwd_reduce", "sw_bwd_reduce_bf16", "sw_bwd_reduce_nhwc", "sw_bwd_reduce_nhwc_bf16"},
     {"sw_bwd_finalize", "sw_bwd_finalize_bf16", "sw_bwd_finalize", "sw_bwd_finalize_bf16"},
     {"sw_bwd_apply", "sw_bwd_apply_bf16", "sw_bwd_apply_nhwc", "sw_bwd_apply_nhwc_bf16"}},
    {{"ld_stats", "ld_stats_bf16", "ld_stats_nhwc", "ld_stats_nhwc_bf16"},
     {"ld_fwd_finalize", "ld_fwd_finalize_bf16", "ld_fwd_finalize", "ld_fwd_finalize_bf16"},
     {"ld_apply", "ld_apply_bf16", "ld_apply_nhwc", "ld_apply_nhwc_bf16"},
     {"ld_bwd_reduce", "ld_bwd_reduce_bf16", "ld_bwd_reduce_nhwc", "ld_bwd_reduce_nhwc_bf16"},
     {"ld_bwd_finalize", "ld_bwd_finalize_bf16", "ld_bwd_finalize", "ld_bwd_finalize_bf16"},
     {"ld_bwd_apply", "ld_bwd_apply_bf16", "ld_bwd_apply_nhwc", "ld_bwd_apply_nhwc_bf16"}}};

// The checks both directions make, in order: flags and geometry, pointers, running buffers (switchable, latent forward),
// alignment, workspace, kernel set-up.  in0, in1: what the kernels read (x; x and dout); out: what they write (y; dx).
int image_validate(dwt::Geom& gm, ImageWork& s, const Mix& m, const void* in0, const void* in1, const void* out, int64_t N,
                   int64_t C, int64_t HW, int GS, int flags, const float* save_mean, const float* save_w, void* ws,
                   size_t ws_bytes, bool running_missing = false) {
  if (int rc = image_geom(gm, N, C, HW, GS, flags, m)) return rc;
  const bool on = m.kind != MIX_INSTANCE;
  if (!in0 || !in1 || !out || !save_mean || !save_w || !ws || (on && (!m.mix || !m.save_stats)))
    return fail(DWT_E_INVALID, "null pointer argument");
  if (running_missing) return fail(DWT_E_INVALID, "running buffer is null (eval, or train with update_running)");
  // instance whitening: mix and save_stats are null
  if (((uintptr_t)in0 | (uintptr_t)in1 | (uintptr_t)out | (uintptr_t)save_w | (uintptr_t)m.save_stats | (uintptr_t)m.mix) % 16 != 0)
    return m.kind == MIX_LATENT ? fail(DWT_E_INVALID, "activation tensors, weights, save_w and save_stats must be 16-byte aligned (latent-domain whitening)")
         : on ? fail(DWT_E_INVALID, "activation tensors, mix, save_w and save_stats must be 16-byte aligned (switchable whitening)")
              : fail(DWT_E_INVALID, "activation tensors and save_w must be 16-byte aligned (instance whitening: TMA and vector stores)");
  s = carve_image(ws, gm, m);
  if (s.w.bytes > ws_bytes) return fail(DWT_E_WORKSPACE, "workspace too small: need %zu bytes, got %zu", s.w.bytes, ws_bytes);
  if ((uintptr_t)ws % 256 != 0) return fail(DWT_E_WORKSPACE, "workspace must be 256-byte aligned");
  if (ensure_tc() != 0) return image_refuse(N, C, HW, GS, flags & ~DWT_MODE_EVAL, m.what());   // the tensor-core kernels could not be set up
  return DWT_OK;
}

// The kernels only read save_mean, save_w and save_stats in the backward
dwt::SwFin make_sw_fin(int mode, float eps, const Mix& m, const float* save_mean, const float* save_w, int* status) {
  dwt::SwFin f{};
  f.a = 1.f - eps; f.b = eps; f.train = (mode & DWT_MODE_EVAL) == 0; f.mix = m.mix;
  f.save_mean = const_cast<float*>(save_mean); f.save_w = const_cast<float*>(save_w);
  f.save_stats = const_cast<float*>(m.save_stats); f.status = status;
  return f;
}

dwt::LdFin make_ld_fin(int mode, float eps, const Mix& m, const float* save_mean, const float* save_w, int* status) {
  dwt::LdFin f{};
  f.a = 1.f - eps; f.b = eps; f.train = (mode & DWT_MODE_EVAL) == 0; f.K = m.K; f.weights = m.mix;
  f.momentum = m.momentum; f.update_running = f.train && m.update_running; f.rmean = m.rmean; f.rcov = m.rcov;
  f.save_mean = const_cast<float*>(save_mean); f.save_w = const_cast<float*>(save_w);
  f.save_stats = const_cast<float*>(m.save_stats); f.status = status;
  return f;
}

int image_fwd(const Mix& m, const void* x, void* y, int64_t N, int64_t C, int64_t HW, int GS, int flags, float eps,
              float* save_mean, float* save_w, void* ws, size_t ws_bytes, cudaStream_t st) {
  dwt::Geom gm;
  ImageWork s;
  const bool train = (flags & DWT_MODE_EVAL) == 0;
  const bool running_missing = m.kind != MIX_INSTANCE && (!train || m.update_running) && (!m.rmean || !m.rcov);
  if (int rc = image_validate(gm, s, m, x, x, y, N, C, HW, GS, flags, save_mean, save_w, ws, ws_bytes, running_missing))
    return rc;
  const bool nhwc = (flags & DWT_LAYOUT_NHWC) != 0, bf16 = (flags & DWT_DTYPE_BF16) != 0;
  const int k = 2 * nhwc + bf16;
  const double E = (bf16 ? 2.0 : 4.0) * (double)N * (double)C * (double)HW;
  {
    Launch l(kImageName[m.kind][I_STATS][k], &gm, E, st);
    if (int cr = dwt::tc_stats(x, bf16, nhwc, gm, gm.nchunks, s.w.shift, s.w.partial, st))
      return fail(DWT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d) x=%p N=%lld C=%d HW=%d", cr, x, (long long)N, gm.C, gm.HW);
  }
  if (int rc = check_launch("%s statistics kernel", m.what())) return rc;
  {
    Launch l(kImageName[m.kind][I_FWD_FINALIZE][k], &gm, 0.0, st);
    if (gm.nchunks > 1) dwt::dense_partial_reduce(s.w.partial, gm.nchunks, dwt::tc_superblocks(gm) * gm.D, s.w.gram, st);
    if (m.kind == MIX_LATENT) {
      const dwt::LdFin fin = make_ld_fin(flags, eps, m, save_mean, save_w, s.w.status);
      dwt::dense_ld_stats(s.w.gram, s.w.shift, gm, fin, st);
      dwt::dense_ld_fwd(gm, fin, st);
    } else if (m.kind == MIX_SWITCH) {
      dwt::SwFin fin = make_sw_fin(flags, eps, m, save_mean, save_w, s.w.status);
      fin.momentum = m.momentum; fin.update_running = train && m.update_running;
      fin.rmean = m.rmean; fin.rcov = m.rcov;
      dwt::dense_sw_stats(s.w.gram, s.w.shift, gm, fin, st);
      dwt::dense_sw_fwd_factor(gm, fin, st);
    } else {
      dwt::FwdFin fin{};
      fin.a = 1.f - eps; fin.b = eps; fin.save_mean = save_mean; fin.save_w = save_w; fin.status = s.w.status;
      dwt::dense_fwd_instance(s.w.gram, s.w.shift, gm, fin, st);
    }
  }
  if (int rc = check_launch("%s finalize kernel", m.what())) return rc;
  {
    Launch l(kImageName[m.kind][I_APPLY][k], &gm, 2.0 * E, st);
    if (int cr = dwt::tc_apply(x, y, bf16, nhwc, gm, tc_apply_ctas(gm, 1, 64), save_mean, save_w, st))
      return fail(DWT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d)", cr);
  }
  return check_launch("%s apply kernel", m.what());
}

int image_bwd(const Mix& m, const void* x, const void* dout, void* dx, int64_t N, int64_t C, int64_t HW, int GS, int flags,
              float eps, const float* save_mean, const float* save_w, void* ws, size_t ws_bytes, cudaStream_t st) {
  dwt::Geom gm;
  ImageWork s;
  if (int rc = image_validate(gm, s, m, x, dout, dx, N, C, HW, GS, flags, save_mean, save_w, ws, ws_bytes)) return rc;
  const bool nhwc = (flags & DWT_LAYOUT_NHWC) != 0, bf16 = (flags & DWT_DTYPE_BF16) != 0;
  const int k = 2 * nhwc + bf16;
  const double E = (bf16 ? 2.0 : 4.0) * (double)N * (double)C * (double)HW;
  {
    Launch l(kImageName[m.kind][I_BWD_REDUCE][k], &gm, 2.0 * E, st);
    if (int cr = dwt::tc_bwd_reduce(x, dout, bf16, nhwc, gm, gm.nchunks, save_mean, s.w.partial, st, /*pilot=*/m.kind == MIX_INSTANCE))
      return fail(DWT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d) x=%p dout=%p N=%lld C=%d HW=%d", cr, x, dout,
                  (long long)N, gm.C, gm.HW);
  }
  if (int rc = check_launch("%s backward reduction kernel", m.what())) return rc;
  {
    Launch l(kImageName[m.kind][I_BWD_FINALIZE][k], &gm, 0.0, st);
    if (gm.nchunks > 1) dwt::dense_partial_reduce(s.w.partial, gm.nchunks, dwt::tc_superblocks(gm) * gm.D, s.w.gram, st);
    if (m.kind == MIX_LATENT) {
      const dwt::LdFin fin = make_ld_fin(flags, eps, m, save_mean, save_w, s.w.status);
      dwt::dense_ld_bwd(s.w.gram, gm, fin, s.sums, s.pd, s.pc, s.part, m.dmix, s.w.coef, s.w.shift, s.mu, st);
    } else if (m.kind == MIX_SWITCH) {
      const dwt::SwFin fin = make_sw_fin(flags, eps, m, save_mean, save_w, s.w.status);
      dwt::dense_sw_bwd(s.w.gram, gm, fin, s.pd, s.part, s.sums, m.dmix, s.w.coef, s.w.shift, s.mu, st);
    } else {
      dwt::BwdFin fin{};
      fin.a = 1.f - eps; fin.mode = DWT_MODE_TRAIN; fin.save_mean = save_mean; fin.save_w = save_w; fin.coef = s.w.coef;
      dwt::dense_bwd_coef(s.w.gram, gm, fin, s.w.shift, st);           // s.w.shift: mean_M dy per (image, channel)
    }
  }
  if (int rc = check_launch("%s backward finalize kernel", m.what())) return rc;
  {
    Launch l(kImageName[m.kind][I_BWD_APPLY][k], &gm, 3.0 * E, st);
    if (int cr = dwt::tc_bwd_apply(x, dout, dx, bf16, nhwc, gm, tc_apply_ctas(gm, 1, 64), s.w.coef,
                                   m.kind != MIX_INSTANCE ? s.mu : save_mean,
                                   s.w.shift, st))
      return fail(DWT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d)", cr);
  }
  return check_launch("%s backward apply kernel", m.what());
}

// ---- latent-domain batch norm (dwt_bn_latent_*) -----------------------------------------------------------------------
// Forward: ldbn_stats (train only) -> ldbn_fwd_finalize -> ldbn_apply; backward: ldbn_bwd_reduce -> ldbn_bwd_finalize
// (+ ldbn_dw when dweights is given) -> ldbn_bwd_apply (norm_ldbn.cu).  Scratch behind the common head: the segment
// partials (two arrays), the pilot shifts, three [N][C] coefficient arrays and the dweights shares.
struct LdbnWork { float *pa, *pb, *pilot, *c0, *c1, *c2, *dw; size_t bytes; };

LdbnWork carve_ldbn(void* base, const dwt::LdbnGeom& g) {
  size_t part, nc, dw;
  dwt::ldbn_scratch_floats(g, &part, &nc, &dw);
  size_t off = kOffScratch;
  char* b = static_cast<char*>(base);
  auto take = [&](size_t floats) { size_t o = off; off = align_up(off + sizeof(float) * floats, 256); return reinterpret_cast<float*>(b + o); };
  LdbnWork w;
  w.pa = take(part); w.pb = take(part); w.pilot = take(nc);
  w.c0 = take(nc); w.c1 = take(nc); w.c2 = take(nc); w.dw = take(dw);
  w.bytes = off;
  return w;
}

// n_domains, mode bits and geometry (no device call); fills the plan
int ldbn_geom(dwt::LdbnGeom& g, int64_t N, int64_t C, int64_t HW, int D, int mode) {
  if (D < 1 || D > DWT_MAX_LATENT_DOMAINS)
    return fail(DWT_E_INVALID, "n_domains %d outside [1,%d] (latent-domain batch norm)", D, DWT_MAX_LATENT_DOMAINS);
  if (mode & ~(DWT_MODE_EVAL | DWT_LAYOUT_NHWC | DWT_DTYPE_BF16))
    return fail(DWT_E_INVALID, "bad mode %#x (DWT_MODE_TRAIN or DWT_MODE_EVAL | DWT_LAYOUT_NHWC | DWT_DTYPE_BF16)", mode);
  if (N <= 0 || C <= 0 || HW <= 0) return fail(DWT_E_INVALID, "empty tensor (N=%lld C=%lld HW=%lld)", (long long)N,
                                               (long long)C, (long long)HW);
  const bool nhwc = (mode & DWT_LAYOUT_NHWC) != 0, bf16 = (mode & DWT_DTYPE_BF16) != 0;
  if ((double)N * (double)C * (double)HW >= 2147483648.0)
    return fail(DWT_E_UNSUPPORTED, "latent-domain batch norm needs N*C*HW < 2^31 (N=%lld C=%lld HW=%lld)", (long long)N,
                (long long)C, (long long)HW);
  if (nhwc && C % 4 != 0)
    return fail(DWT_E_UNSUPPORTED, "latent-domain batch norm runs channels-last at C %% 4 == 0 only (C=%lld)", (long long)C);
  if (bf16 && !nhwc && HW % 4 != 0)
    return fail(DWT_E_UNSUPPORTED, "latent-domain batch norm runs NCHW bf16 at HW %% 4 == 0 only (HW=%lld)", (long long)HW);
  g = dwt::ldbn_plan((int)N, (int)C, (int)HW, D, nhwc, bf16);
  return DWT_OK;
}

// The checks both directions make, in order: geometry, pointers, alignment, workspace.  act: the activation tensors.
int ldbn_validate(dwt::LdbnGeom& g, LdbnWork& w, int64_t N, int64_t C, int64_t HW, int D, int mode, const void* const (&act)[3],
                  const float* weights, const float* save, const float* gamma, const float* beta, void* ws, size_t ws_bytes) {
  if (int rc = ldbn_geom(g, N, C, HW, D, mode)) return rc;
  if (!act[0] || !act[1] || !act[2] || !weights || !save || !ws) return fail(DWT_E_INVALID, "null pointer argument");
  if (!gamma != !beta)
    return fail(DWT_E_INVALID, "gamma and beta (dgamma and dbeta) must be both given or both NULL (latent-domain batch norm)");
  const uintptr_t bits = (uintptr_t)act[0] | (uintptr_t)act[1] | (uintptr_t)act[2];
  if (bits % (g.bf16 ? 8 : 16) != 0)
    return fail(DWT_E_INVALID, "activation tensors must be %d-byte aligned (latent-domain batch norm)", g.bf16 ? 8 : 16);
  if (((uintptr_t)weights | (uintptr_t)gamma | (uintptr_t)beta) % 4 != 0 || (uintptr_t)save % 16 != 0)
    return fail(DWT_E_INVALID, "weights, gamma and beta must be 4-byte and save_stats 16-byte aligned (latent-domain batch norm)");
  w = carve_ldbn(ws, g);
  if (w.bytes > ws_bytes) return fail(DWT_E_WORKSPACE, "workspace too small: need %zu bytes, got %zu", w.bytes, ws_bytes);
  if ((uintptr_t)ws % 256 != 0) return fail(DWT_E_WORKSPACE, "workspace must be 256-byte aligned");
  return DWT_OK;
}

dwt::LdbnFin make_ldbn_fin(const dwt::LdbnGeom& g, int mode, float eps, const float* weights, const float* gamma,
                           const float* beta, const float* save, void* ws) {
  dwt::LdbnFin f{};
  f.N = g.N; f.C = g.C; f.D = g.D; f.S = g.S; f.M = (double)g.HW;
  f.eps = eps; f.train = (mode & DWT_MODE_EVAL) == 0;
  f.weights = weights; f.gamma = gamma; f.beta = beta; f.save = const_cast<float*>(save);
  f.status = static_cast<int*>(ws);
  return f;
}

// Profile family of a launch: [pass][channels-last * 2 + bf16]
const char* const kLdbnName[6][4] = {
    {"ldbn_stats", "ldbn_stats_bf16", "ldbn_stats_nhwc", "ldbn_stats_nhwc_bf16"},
    {"ldbn_fwd_finalize", "ldbn_fwd_finalize", "ldbn_fwd_finalize", "ldbn_fwd_finalize"},
    {"ldbn_apply", "ldbn_apply_bf16", "ldbn_apply_nhwc", "ldbn_apply_nhwc_bf16"},
    {"ldbn_bwd_reduce", "ldbn_bwd_reduce_bf16", "ldbn_bwd_reduce_nhwc", "ldbn_bwd_reduce_nhwc_bf16"},
    {"ldbn_bwd_finalize", "ldbn_bwd_finalize", "ldbn_bwd_finalize", "ldbn_bwd_finalize"},
    {"ldbn_bwd_apply", "ldbn_bwd_apply_bf16", "ldbn_bwd_apply_nhwc", "ldbn_bwd_apply_nhwc_bf16"}};

dwt::Geom ldbn_prof_geom(const dwt::LdbnGeom& g) {
  dwt::Geom gm{};
  gm.N = g.N; gm.C = g.C; gm.HW = g.HW; gm.GS = 1; gm.G = g.C; gm.D = g.D;
  return gm;
}

// ---- latent-domain whitening at group sizes 1, 2, 4 (dwt_whiten_latent_small_*) -----------------------------------------
// Forward: lds_stats -> lds_fwd_finalize (per-image moments, per-domain W_k + EMA, per-image A_n, m~_n) -> lds_apply;
// backward: lds_bwd_reduce about the images' own means -> lds_bwd_finalize (+ the dweights sum when it is given) ->
// lds_bwd_apply (norm_ldbn.cu, on latent-domain batch norm's segments).  Scratch behind the common head: the segment
// partials, the pilot shifts, the per-image fp64 moments, the backward's per-image sums, per-domain P_k | mubar_k and
// <P_k, Sigma_k>, the apply coefficients and the dweights shares.
struct LdsWork { float *part, *pilot, *red, *pd, *pc, *coef, *dw; double* im; size_t bytes; };

LdsWork carve_lds(void* base, const dwt::LdbnGeom& g, int GS, int K) {
  const size_t NG = (size_t)g.N * (g.C / GS), KG = (size_t)K * (g.C / GS);
  size_t off = kOffScratch;
  char* b = static_cast<char*>(base);
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return b + o; };
  LdsWork w;
  w.part = reinterpret_cast<float*>(take(sizeof(float) * NG * g.S * dwt::lds_partial_floats(GS)));
  w.pilot = reinterpret_cast<float*>(take(sizeof(float) * (size_t)g.N * g.C));
  w.im = reinterpret_cast<double*>(take(sizeof(double) * NG * (GS + GS * (GS + 1) / 2)));
  w.red = reinterpret_cast<float*>(take(sizeof(float) * NG * (GS + GS * GS)));
  w.pd = reinterpret_cast<float*>(take(sizeof(float) * KG * (GS * GS + GS)));
  w.pc = reinterpret_cast<float*>(take(sizeof(float) * KG));
  w.coef = reinterpret_cast<float*>(take(sizeof(float) * NG * dwt::lds_coef_floats(GS)));
  w.dw = reinterpret_cast<float*>(take(sizeof(float) * NG * dwt::kLdsMaxDomains));
  w.bytes = off;
  return w;
}

// n_domains, mode bits and geometry (no device call); fills the plan
int lds_geom(dwt::LdbnGeom& g, int64_t N, int64_t C, int64_t HW, int GS, int K, int mode) {
  if (K < 1 || K > DWT_MAX_LATENT_DOMAINS)
    return fail(DWT_E_INVALID, "n_domains %d outside [1,%d] (latent-domain whitening)", K, DWT_MAX_LATENT_DOMAINS);
  if (mode & ~(DWT_MODE_EVAL | DWT_LAYOUT_NHWC | DWT_DTYPE_BF16))
    return fail(DWT_E_INVALID, "bad mode %#x (DWT_MODE_TRAIN or DWT_MODE_EVAL | DWT_LAYOUT_NHWC | DWT_DTYPE_BF16)", mode);
  if (N <= 0 || C <= 0 || HW <= 0) return fail(DWT_E_INVALID, "empty tensor (N=%lld C=%lld HW=%lld)", (long long)N,
                                               (long long)C, (long long)HW);
  const bool nhwc = (mode & DWT_LAYOUT_NHWC) != 0, bf16 = (mode & DWT_DTYPE_BF16) != 0;
  if ((GS != 1 && GS != 2 && GS != 4) || C % GS != 0)
    return fail(DWT_E_UNSUPPORTED, "latent-domain whitening at group sizes 1, 2, 4 needs group_size 1, 2 or 4 dividing C "
                "(C=%lld gs=%d)", (long long)C, GS);
  if ((double)N * (double)C * (double)HW >= 2147483648.0)
    return fail(DWT_E_UNSUPPORTED, "latent-domain whitening at group sizes 1, 2, 4 needs N*C*HW < 2^31 (N=%lld C=%lld "
                "HW=%lld)", (long long)N, (long long)C, (long long)HW);
  if (nhwc && C % 4 != 0)
    return fail(DWT_E_UNSUPPORTED, "latent-domain whitening at group sizes 1, 2, 4 runs channels-last at C %% 4 == 0 only "
                "(C=%lld)", (long long)C);
  if (bf16 && !nhwc && HW % 4 != 0)
    return fail(DWT_E_UNSUPPORTED, "latent-domain whitening at group sizes 1, 2, 4 runs NCHW bf16 at HW %% 4 == 0 only "
                "(HW=%lld)", (long long)HW);
  g = dwt::lds_plan((int)N, (int)C, (int)HW, GS, K, nhwc, bf16);
  return DWT_OK;
}

// The checks both directions make, in order: geometry, pointers, alignment, workspace.  act: the activation tensors.
int lds_validate(dwt::LdbnGeom& g, LdsWork& w, int64_t N, int64_t C, int64_t HW, int GS, int K, int mode,
                 const void* const (&act)[3], const float* weights, const float* save_mean, const float* save_w,
                 const float* save_stats, void* ws, size_t ws_bytes) {
  if (int rc = lds_geom(g, N, C, HW, GS, K, mode)) return rc;
  if (!act[0] || !act[1] || !act[2] || !weights || !save_mean || !save_w || !save_stats || !ws)
    return fail(DWT_E_INVALID, "null pointer argument");
  const uintptr_t bits = (uintptr_t)act[0] | (uintptr_t)act[1] | (uintptr_t)act[2];
  if (bits % (g.bf16 ? 8 : 16) != 0)
    return fail(DWT_E_INVALID, "activation tensors must be %d-byte aligned (latent-domain whitening)", g.bf16 ? 8 : 16);
  if (((uintptr_t)weights | (uintptr_t)save_w | (uintptr_t)save_stats) % 16 != 0 || (uintptr_t)save_mean % 4 != 0)
    return fail(DWT_E_INVALID, "weights, save_w and save_stats must be 16-byte and save_mean 4-byte aligned "
                "(latent-domain whitening)");
  w = carve_lds(ws, g, GS, K);
  if (w.bytes > ws_bytes) return fail(DWT_E_WORKSPACE, "workspace too small: need %zu bytes, got %zu", w.bytes, ws_bytes);
  if ((uintptr_t)ws % 256 != 0) return fail(DWT_E_WORKSPACE, "workspace must be 256-byte aligned");
  return DWT_OK;
}

dwt::LdsFin make_lds_fin(const dwt::LdbnGeom& g, int GS, int K, int mode, float eps, const float* weights,
                         const float* save_mean, const float* save_w, const float* save_stats, void* ws) {
  dwt::LdsFin f{};
  f.N = g.N; f.C = g.C; f.GS = GS; f.G = g.C / GS; f.K = K; f.S = g.S; f.M = (double)g.HW;
  f.a = 1.f - eps; f.b = eps; f.train = (mode & DWT_MODE_EVAL) == 0; f.weights = weights;
  f.save_mean = const_cast<float*>(save_mean); f.save_w = const_cast<float*>(save_w);
  f.save_stats = const_cast<float*>(save_stats);
  f.status = static_cast<int*>(ws);
  return f;
}

// Profile family of a launch: [pass][channels-last * 2 + bf16]
const char* const kLdsName[6][4] = {
    {"lds_stats", "lds_stats_bf16", "lds_stats_nhwc", "lds_stats_nhwc_bf16"},
    {"lds_fwd_finalize", "lds_fwd_finalize", "lds_fwd_finalize", "lds_fwd_finalize"},
    {"lds_apply", "lds_apply_bf16", "lds_apply_nhwc", "lds_apply_nhwc_bf16"},
    {"lds_bwd_reduce", "lds_bwd_reduce_bf16", "lds_bwd_reduce_nhwc", "lds_bwd_reduce_nhwc_bf16"},
    {"lds_bwd_finalize", "lds_bwd_finalize", "lds_bwd_finalize", "lds_bwd_finalize"},
    {"lds_bwd_apply", "lds_bwd_apply_bf16", "lds_bwd_apply_nhwc", "lds_bwd_apply_nhwc_bf16"}};

dwt::Geom lds_prof_geom(const dwt::LdbnGeom& g, int GS, int K) {
  dwt::Geom gm{};
  gm.N = g.N; gm.C = g.C; gm.HW = g.HW; gm.GS = GS; gm.G = g.C / GS; gm.D = K;
  return gm;
}

// dwt_bn_latent_fwd, and dwt_latent_site_fwd with a site epilogue epi (checked by the caller)
int ldbn_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int n_domains, int mode, float eps, float momentum,
             int update_running, float* running_mean, float* running_var, const float* weights, const float* gamma,
             const float* beta, float* save_stats, void* workspace, size_t workspace_bytes, dwt_stream_t stream, int epi,
             const void* residual, uint8_t* relu_mask) {
  dwt::LdbnGeom g;
  LdbnWork w;
  const void* const act[3] = {x, x, y};
  if (int rc = ldbn_validate(g, w, N, C, HW, n_domains, mode, act, weights, save_stats, gamma, beta, workspace,
                             workspace_bytes))
    return rc;
  const bool train = (mode & DWT_MODE_EVAL) == 0;
  if ((!train || update_running) && (!running_mean || !running_var))
    return fail(DWT_E_INVALID, "running buffer is null (eval, or train with update_running)");
  cudaStream_t st = (cudaStream_t)stream;
  dwt::LdbnFin f = make_ldbn_fin(g, mode, eps, weights, gamma, beta, save_stats, workspace);
  f.momentum = momentum; f.update_running = train && update_running; f.rmean = running_mean; f.rvar = running_var;
  const float* save_a = save_stats + (size_t)2 * N * C;
  const dwt::LdEpi ep{gamma, beta, save_a, save_a + (size_t)N * C, residual, relu_mask, nullptr};
  const dwt::Geom pg = ldbn_prof_geom(g);
  const int k = 2 * g.nhwc + g.bf16;
  const double E = (g.bf16 ? 2.0 : 4.0) * (double)N * (double)C * (double)HW;
  if (train) {
    Launch l(kLdbnName[0][k], &pg, E, st);
    dwt::ldbn_stats(x, g, w.pa, w.pb, w.pilot, st);
  }
  if (int rc = check_launch("latent-domain batch norm statistics kernel")) return rc;
  {
    Launch l(kLdbnName[1][k], &pg, 0.0, st);
    dwt::ldbn_fwd_finalize(f, w.pa, w.pb, w.pilot, w.c0, w.c1, st);
  }
  if (int rc = check_launch("latent-domain batch norm finalize kernel")) return rc;
  {
    const bool res = (epi & DWT_EPI_RESIDUAL) != 0;
    Launch l(kLdbnName[2][k], &pg, (res ? 3.0 : 2.0) * E + (relu_mask ? E / (g.bf16 ? 8.0 : 16.0) : 0.0), st);
    dwt::ldbn_apply(x, y, g, w.c0, w.c1, epi, ep, st);
  }
  return check_launch("latent-domain batch norm apply kernel");
}

// dwt_bn_latent_bwd, and dwt_latent_site_bwd with a site epilogue epi (checked by the caller)
int ldbn_bwd(const float* x, const float* dout, float* dx, int64_t N, int64_t C, int64_t HW, int n_domains, int mode,
             float eps, const float* weights, const float* gamma, const float* save_stats, float* dweights, float* dgamma,
             float* dbeta, void* workspace, size_t workspace_bytes, dwt_stream_t stream, int epi, const float* beta,
             const uint8_t* relu_mask, float* dresidual) {
  dwt::LdbnGeom g;
  LdbnWork w;
  const void* const act[3] = {x, dout, dx};
  if (int rc = ldbn_validate(g, w, N, C, HW, n_domains, mode, act, weights, save_stats, dgamma, dbeta, workspace,
                             workspace_bytes))
    return rc;
  if (dgamma && !gamma) return fail(DWT_E_INVALID, "dgamma / dbeta given without gamma (latent-domain batch norm)");
  if ((uintptr_t)dweights % 4 != 0) return fail(DWT_E_INVALID, "dweights must be 4-byte aligned (latent-domain batch norm)");
  cudaStream_t st = (cudaStream_t)stream;
  dwt::LdbnFin f = make_ldbn_fin(g, mode, eps, weights, gamma, nullptr, save_stats, workspace);
  f.dgamma = dgamma; f.dbeta = dbeta;
  const dwt::Geom pg = ldbn_prof_geom(g);
  const int k = 2 * g.nhwc + g.bf16;
  const double E = (g.bf16 ? 2.0 : 4.0) * (double)N * (double)C * (double)HW;
  const float* centre = save_stats;                           // [N][C] first in save_stats
  const float* save_a = save_stats + (size_t)2 * N * C;
  const dwt::LdEpi ep{gamma, beta, save_a, save_a + (size_t)N * C, nullptr, const_cast<uint8_t*>(relu_mask), dresidual};
  {
    const bool mk = (epi & DWT_EPI_RESIDUAL) != 0;
    Launch l(kLdbnName[3][k], &pg, (mk ? 3.0 : 2.0) * E + (mk ? E / (g.bf16 ? 8.0 : 16.0) : 0.0), st);
    dwt::ldbn_bwd_reduce(x, dout, g, centre, w.pa, w.pb, epi, ep, st);
  }
  if (int rc = check_launch("latent-domain batch norm backward reduction kernel")) return rc;
  {
    Launch l(kLdbnName[4][k], &pg, 0.0, st);
    dwt::ldbn_bwd_finalize(f, w.pa, w.pb, w.c0, w.c1, w.c2, w.dw, dweights, st);
  }
  if (int rc = check_launch("latent-domain batch norm backward finalize kernel")) return rc;
  {
    Launch l(kLdbnName[5][k], &pg, 3.0 * E, st);
    // a residual's apply reads the masked gradient its reduction wrote
    const void* dz = (epi & DWT_EPI_RESIDUAL) ? static_cast<const void*>(dresidual) : dout;
    dwt::ldbn_bwd_apply(x, dz, dx, g, w.c0, w.c1, w.c2, centre, epi, ep, st);
  }
  return check_launch("latent-domain batch norm backward apply kernel");
}

// dwt_whiten_latent_small_fwd, and dwt_latent_site_fwd with a site epilogue epi (checked by the caller)
int lds_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains, int mode, float eps,
            float momentum, int update_running, float* running_mean, float* running_cov, const float* weights,
            float* save_mean, float* save_w, float* save_stats, void* workspace, size_t workspace_bytes,
            dwt_stream_t stream, int epi, const float* gamma, const float* beta, const void* residual,
            uint8_t* relu_mask) {
  dwt::LdbnGeom g;
  LdsWork w;
  const void* const act[3] = {x, x, y};
  if (int rc = lds_validate(g, w, N, C, HW, group_size, n_domains, mode, act, weights, save_mean, save_w, save_stats,
                            workspace, workspace_bytes))
    return rc;
  const bool train = (mode & DWT_MODE_EVAL) == 0;
  if ((!train || update_running) && (!running_mean || !running_cov))
    return fail(DWT_E_INVALID, "running buffer is null (eval, or train with update_running)");
  cudaStream_t st = (cudaStream_t)stream;
  const int GS = group_size;
  dwt::LdsFin f = make_lds_fin(g, GS, n_domains, mode, eps, weights, save_mean, save_w, save_stats, workspace);
  f.momentum = momentum; f.update_running = train && update_running; f.rmean = running_mean; f.rcov = running_cov;
  const dwt::LdEpi ep{gamma, beta, save_mean, save_w, residual, relu_mask, nullptr};
  const dwt::Geom pg = lds_prof_geom(g, GS, n_domains);
  const int k = 2 * g.nhwc + g.bf16;
  const double E = (g.bf16 ? 2.0 : 4.0) * (double)N * (double)C * (double)HW;
  {
    Launch l(kLdsName[0][k], &pg, E, st);
    dwt::lds_stats(x, g, GS, w.part, w.pilot, st);
  }
  if (int rc = check_launch("latent-domain whitening statistics kernel")) return rc;
  {
    Launch l(kLdsName[1][k], &pg, 0.0, st);
    dwt::lds_fwd_finalize(f, w.part, w.pilot, w.im, st);
  }
  if (int rc = check_launch("latent-domain whitening finalize kernel")) return rc;
  {
    const bool res = (epi & DWT_EPI_RESIDUAL) != 0;
    Launch l(kLdsName[2][k], &pg, (res ? 3.0 : 2.0) * E + (relu_mask ? E / (g.bf16 ? 8.0 : 16.0) : 0.0), st);
    dwt::lds_apply(x, y, g, GS, epi, ep, st);
  }
  return check_launch("latent-domain whitening apply kernel");
}

// dwt_whiten_latent_small_bwd, and dwt_latent_site_bwd with a site epilogue epi (checked by the caller)
int lds_bwd(const float* x, const float* dout, float* dx, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains,
            int mode, float eps, const float* weights, const float* save_mean, const float* save_w, const float* save_stats,
            float* dweights, void* workspace, size_t workspace_bytes, dwt_stream_t stream, int epi, const float* gamma,
            const float* beta, const uint8_t* relu_mask, float* dresidual, float* dgamma, float* dbeta) {
  dwt::LdbnGeom g;
  LdsWork w;
  const void* const act[3] = {x, dout, dx};
  if (int rc = lds_validate(g, w, N, C, HW, group_size, n_domains, mode, act, weights, save_mean, save_w, save_stats,
                            workspace, workspace_bytes))
    return rc;
  if ((uintptr_t)dweights % 4 != 0) return fail(DWT_E_INVALID, "dweights must be 4-byte aligned (latent-domain whitening)");
  cudaStream_t st = (cudaStream_t)stream;
  const int GS = group_size;
  const dwt::LdsFin f = make_lds_fin(g, GS, n_domains, mode, eps, weights, save_mean, save_w, save_stats, workspace);
  const dwt::Geom pg = lds_prof_geom(g, GS, n_domains);
  const dwt::LdEpi ep{gamma, beta, save_mean, save_w, nullptr, const_cast<uint8_t*>(relu_mask), dresidual};
  const int k = 2 * g.nhwc + g.bf16;
  const double E = (g.bf16 ? 2.0 : 4.0) * (double)N * (double)C * (double)HW;
  {
    const bool mk = (epi & DWT_EPI_RESIDUAL) != 0;
    Launch l(kLdsName[3][k], &pg, (mk ? 3.0 : 2.0) * E + (mk ? E / (g.bf16 ? 8.0 : 16.0) : 0.0), st);
    dwt::lds_bwd_reduce(x, dout, g, GS, save_stats, w.part, epi, ep, st);
  }
  if (int rc = check_launch("latent-domain whitening backward reduction kernel")) return rc;
  {
    Launch l(kLdsName[4][k], &pg, 0.0, st);
    // a site's per-image dgamma / dbeta shares reuse the forward's per-image moments (w.im, free in the backward)
    dwt::lds_bwd_finalize(f, w.part, w.red, w.pd, w.pc, w.coef, w.dw, dweights, gamma, reinterpret_cast<float*>(w.im),
                          dgamma, dbeta, st);
  }
  if (int rc = check_launch("latent-domain whitening backward finalize kernel")) return rc;
  {
    Launch l(kLdsName[5][k], &pg, 3.0 * E, st);
    // a residual's apply reads the masked gradient its reduction wrote
    const void* dz = (epi & DWT_EPI_RESIDUAL) ? static_cast<const void*>(dresidual) : dout;
    dwt::lds_bwd_apply(x, dz, dx, g, GS, w.coef, epi, ep, st);
  }
  return check_launch("latent-domain whitening backward apply kernel");
}


// ---- latent-domain sites (dwt_latent_site_*) ----------------------------------------------------------------------------
// The checks of a site call the layer's own entry points do not make: kind and group size, the epilogue bits and the
// pointers they need.  The drivers above check the rest.  bwd: dresidual / relu_mask of the backward.
int site_check(int kind, int GS, int mode, int epi, const float* gamma, const float* beta, const void* residual,
               const void* relu_mask, const void* dresidual, bool bwd, bool bf16_bytes) {
  if (kind != DWT_KIND_BN && kind != DWT_KIND_WHITEN)
    return fail(DWT_E_INVALID, "kind %d is neither DWT_KIND_BN nor DWT_KIND_WHITEN (latent-domain site)", kind);
  if (kind == DWT_KIND_BN && GS != 1)
    return fail(DWT_E_INVALID, "a batch-norm latent-domain site takes group_size 1 (got %d)", GS);
  if (kind == DWT_KIND_WHITEN && GS != 1 && GS != 2 && GS != 4)
    return fail(DWT_E_UNSUPPORTED, "a whitening latent-domain site runs at group sizes 1, 2, 4 only (got %d)", GS);
  if (epi & ~(DWT_EPI_AFFINE | DWT_EPI_RELU | DWT_EPI_RESIDUAL))
    return fail(DWT_E_INVALID, "bad epilogue %#x (latent-domain site)", epi);
  if ((epi & DWT_EPI_RELU) && !(epi & DWT_EPI_AFFINE))
    return fail(DWT_E_INVALID, "a latent-domain site's RELU epilogue needs AFFINE");
  if ((epi & DWT_EPI_RESIDUAL) && !(epi & DWT_EPI_RELU))
    return fail(DWT_E_INVALID, "a latent-domain site's RESIDUAL epilogue needs AFFINE|RELU");
  if (!(epi & DWT_EPI_AFFINE) != (!gamma || !beta) || !gamma != !beta)
    return fail(DWT_E_INVALID, "a latent-domain site takes gamma and beta exactly with the AFFINE epilogue");
  if (((uintptr_t)gamma | (uintptr_t)beta) % 4 != 0)
    return fail(DWT_E_INVALID, "gamma and beta must be 4-byte aligned (latent-domain site)");
  const bool nhwc = (mode & DWT_LAYOUT_NHWC) != 0, res = (epi & DWT_EPI_RESIDUAL) != 0;
  if (res && bwd && !nhwc)
    return fail(DWT_E_INVALID, "an NCHW latent-domain site's residual backward is the AFFINE one on dz = dout * (out > 0)");
  if (!relu_mask != !(res && nhwc))
    return fail(DWT_E_INVALID, "a latent-domain site takes a ReLU byte map exactly with the channels-last RESIDUAL epilogue");
  const void* t = bwd ? dresidual : residual;
  if (!t != !res)
    return fail(DWT_E_INVALID, "a latent-domain site takes %s exactly with the RESIDUAL epilogue", bwd ? "dresidual" : "residual");
  if ((uintptr_t)t % (bf16_bytes ? 8 : 16) != 0)
    return fail(DWT_E_INVALID, "%s must be %d-byte aligned (latent-domain site)", bwd ? "dresidual" : "residual",
                bf16_bytes ? 8 : 16);
  return DWT_OK;
}
}  // namespace

extern "C" {

int dwt_abi_version(void) { return DWT_B200_ABI_VERSION; }

size_t dwt_instance_workspace_bytes(int64_t N, int64_t C, int64_t HW, int group_size) {
  return image_workspace_bytes(N, C, HW, group_size, Mix{});
}

int dwt_whiten_instance_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int group_size, int flags, float eps,
                            float* save_mean, float* save_w, void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  return image_fwd(Mix{}, x, y, N, C, HW, group_size, flags, eps, save_mean, save_w, workspace, workspace_bytes,
                   (cudaStream_t)stream);
}

int dwt_whiten_instance_bwd(const float* x, const float* dout, float* dx, int64_t N, int64_t C, int64_t HW, int group_size,
                            int flags, float eps, const float* save_mean, const float* save_w, void* workspace,
                            size_t workspace_bytes, dwt_stream_t stream) {
  return image_bwd(Mix{}, x, dout, dx, N, C, HW, group_size, flags, eps, save_mean, save_w, workspace, workspace_bytes,
                   (cudaStream_t)stream);
}

size_t dwt_switch_workspace_bytes(int64_t N, int64_t C, int64_t HW, int group_size) {
  Mix m;
  m.kind = MIX_SWITCH;
  return image_workspace_bytes(N, C, HW, group_size, m);
}

int dwt_whiten_switch_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int group_size, int mode, float eps,
                          float momentum, int update_running, float* running_mean, float* running_cov, const float* mix,
                          float* save_mean, float* save_w, float* save_stats, void* workspace, size_t workspace_bytes,
                          dwt_stream_t stream) {
  Mix m;
  m.kind = MIX_SWITCH; m.mix = mix; m.save_stats = save_stats;
  m.momentum = momentum; m.update_running = update_running; m.rmean = running_mean; m.rcov = running_cov;
  return image_fwd(m, x, y, N, C, HW, group_size, mode, eps, save_mean, save_w, workspace, workspace_bytes, (cudaStream_t)stream);
}

int dwt_whiten_switch_bwd(const float* x, const float* dout, float* dx, int64_t N, int64_t C, int64_t HW, int group_size,
                          int mode, float eps, const float* mix, const float* save_mean, const float* save_w,
                          const float* save_stats, float* dmix, void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  Mix m;
  m.kind = MIX_SWITCH; m.mix = mix; m.save_stats = save_stats; m.dmix = dmix;
  return image_bwd(m, x, dout, dx, N, C, HW, group_size, mode, eps, save_mean, save_w, workspace, workspace_bytes,
                   (cudaStream_t)stream);
}

size_t dwt_latent_workspace_bytes(int64_t N, int64_t C, int64_t HW, int group_size, int n_domains) {
  Mix m;
  m.kind = MIX_LATENT; m.K = n_domains;
  return image_workspace_bytes(N, C, HW, group_size, m);
}

int dwt_whiten_latent_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains, int mode,
                          float eps, float momentum, int update_running, float* running_mean, float* running_cov,
                          const float* weights, float* save_mean, float* save_w, float* save_stats, void* workspace,
                          size_t workspace_bytes, dwt_stream_t stream) {
  Mix m;
  m.kind = MIX_LATENT; m.K = n_domains; m.mix = weights; m.save_stats = save_stats;
  m.momentum = momentum; m.update_running = update_running; m.rmean = running_mean; m.rcov = running_cov;
  return image_fwd(m, x, y, N, C, HW, group_size, mode, eps, save_mean, save_w, workspace, workspace_bytes, (cudaStream_t)stream);
}

int dwt_whiten_latent_bwd(const float* x, const float* dout, float* dx, int64_t N, int64_t C, int64_t HW, int group_size,
                          int n_domains, int mode, float eps, const float* weights, const float* save_mean, const float* save_w,
                          const float* save_stats, float* dweights, void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  Mix m;
  m.kind = MIX_LATENT; m.K = n_domains; m.mix = weights; m.save_stats = save_stats; m.dmix = dweights;
  return image_bwd(m, x, dout, dx, N, C, HW, group_size, mode, eps, save_mean, save_w, workspace, workspace_bytes,
                   (cudaStream_t)stream);
}

size_t dwt_bn_latent_workspace_bytes(int64_t N, int64_t C, int64_t HW, int n_domains) {
  return larger_layout_workspace_bytes([&](int mode) -> size_t {
    dwt::LdbnGeom g;
    return ldbn_geom(g, N, C, HW, n_domains, mode) == DWT_OK ? carve_ldbn(nullptr, g).bytes : 0;
  });
}

int dwt_bn_latent_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int n_domains, int mode, float eps,
                      float momentum, int update_running, float* running_mean, float* running_var, const float* weights,
                      const float* gamma, const float* beta, float* save_stats, void* workspace, size_t workspace_bytes,
                      dwt_stream_t stream) {
  return ldbn_fwd(x, y, N, C, HW, n_domains, mode, eps, momentum, update_running, running_mean, running_var, weights, gamma,
                  beta, save_stats, workspace, workspace_bytes, stream, 0, nullptr, nullptr);
}

int dwt_bn_latent_bwd(const float* x, const float* dout, float* dx, int64_t N, int64_t C, int64_t HW, int n_domains, int mode,
                      float eps, const float* weights, const float* gamma, const float* save_stats, float* dweights,
                      float* dgamma, float* dbeta, void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  return ldbn_bwd(x, dout, dx, N, C, HW, n_domains, mode, eps, weights, gamma, save_stats, dweights, dgamma, dbeta, workspace,
                  workspace_bytes, stream, 0, nullptr, nullptr, nullptr);
}

size_t dwt_latent_small_workspace_bytes(int64_t N, int64_t C, int64_t HW, int group_size, int n_domains) {
  return larger_layout_workspace_bytes([&](int mode) -> size_t {
    dwt::LdbnGeom g;
    return lds_geom(g, N, C, HW, group_size, n_domains, mode) == DWT_OK ? carve_lds(nullptr, g, group_size, n_domains).bytes
                                                                        : 0;
  });
}

int dwt_whiten_latent_small_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains,
                                int mode, float eps, float momentum, int update_running, float* running_mean,
                                float* running_cov, const float* weights, float* save_mean, float* save_w,
                                float* save_stats, void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  return lds_fwd(x, y, N, C, HW, group_size, n_domains, mode, eps, momentum, update_running, running_mean, running_cov,
                 weights, save_mean, save_w, save_stats, workspace, workspace_bytes, stream, 0, nullptr, nullptr, nullptr,
                 nullptr);
}

int dwt_whiten_latent_small_bwd(const float* x, const float* dout, float* dx, int64_t N, int64_t C, int64_t HW,
                                int group_size, int n_domains, int mode, float eps, const float* weights,
                                const float* save_mean, const float* save_w, const float* save_stats, float* dweights,
                                void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  return lds_bwd(x, dout, dx, N, C, HW, group_size, n_domains, mode, eps, weights, save_mean, save_w, save_stats, dweights,
                 workspace, workspace_bytes, stream, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
}

// a refusal of the layer's own checks or launches, passed through a site call: its text also names the site
static int site_rc(int rc) {
  if (rc != DWT_OK) {
    const size_t n = strlen(g_err);
    snprintf(g_err + n, sizeof(g_err) - n, " [latent-domain site]");
  }
  return rc;
}

int dwt_latent_site_fwd(int kind, const float* x, float* y, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains,
                        int mode, float eps, float momentum, int update_running, float* running_mean,
                        float* running_second, const float* weights, const float* gamma, const float* beta,
                        const float* residual, uint8_t* relu_mask, int epilogue, float* save_mean, float* save_w,
                        float* save_stats, void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  if (int rc = site_check(kind, group_size, mode, epilogue, gamma, beta, residual, relu_mask, nullptr, false,
                          (mode & DWT_DTYPE_BF16) != 0))
    return rc;
  if (kind == DWT_KIND_BN)
    return site_rc(ldbn_fwd(x, y, N, C, HW, n_domains, mode, eps, momentum, update_running, running_mean, running_second, weights,
                    gamma, beta, save_stats, workspace, workspace_bytes, stream, epilogue, residual, relu_mask));
  return site_rc(lds_fwd(x, y, N, C, HW, group_size, n_domains, mode, eps, momentum, update_running, running_mean, running_second,
                 weights, save_mean, save_w, save_stats, workspace, workspace_bytes, stream, epilogue, gamma, beta, residual,
                 relu_mask));
}

int dwt_latent_site_bwd(int kind, const float* x, const float* dout, float* dx, int64_t N, int64_t C, int64_t HW,
                        int group_size, int n_domains, int mode, float eps, const float* weights, const float* gamma,
                        const float* beta, const uint8_t* relu_mask, float* dresidual, int epilogue, const float* save_mean,
                        const float* save_w, const float* save_stats, float* dweights, float* dgamma, float* dbeta,
                        void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  if (int rc = site_check(kind, group_size, mode, epilogue, gamma, beta, nullptr, relu_mask, dresidual, true,
                          (mode & DWT_DTYPE_BF16) != 0))
    return rc;
  if (!dgamma != !dbeta || (dgamma && !gamma))
    return fail(DWT_E_INVALID, "dgamma and dbeta go together and need the AFFINE epilogue (latent-domain site)");
  if (((uintptr_t)dgamma | (uintptr_t)dbeta) % 4 != 0)
    return fail(DWT_E_INVALID, "dgamma and dbeta must be 4-byte aligned (latent-domain site)");
  if (kind == DWT_KIND_BN)
    return site_rc(ldbn_bwd(x, dout, dx, N, C, HW, n_domains, mode, eps, weights, gamma, save_stats, dweights, dgamma, dbeta,
                    workspace, workspace_bytes, stream, epilogue, beta, relu_mask, dresidual));
  return site_rc(lds_bwd(x, dout, dx, N, C, HW, group_size, n_domains, mode, eps, weights, save_mean, save_w, save_stats, dweights,
                 workspace, workspace_bytes, stream, epilogue, gamma, beta, relu_mask, dresidual, dgamma, dbeta));
}

const char* dwt_last_error(void) { return g_err; }

size_t dwt_workspace_bytes(int64_t N, int64_t C, int64_t HW, int group_size, int n_domains) {
  (void)N; (void)HW;
  // group size 128 is sized by the group-size-64 query on 2C channels (dwt_b200.h): this query keeps its range
  if (C <= 0 || group_size < 1 || group_size > DWT_MAX_GROUP_SIZE || C % group_size != 0 || n_domains < 1 ||
      n_domains > DWT_MAX_DOMAINS)
    return 0;
  return carve(nullptr, C, group_size, n_domains, carve(nullptr, C, group_size, n_domains).bytes).bytes;   // two sites
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

int dwt_whiten_zca_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains, int mode,
                       float eps, float momentum, int update_running, float* const* running_mean, float* const* running_cov,
                       int iterations, float* save_mean, float* save_w, float* save_p, void* workspace,
                       size_t workspace_bytes, dwt_stream_t stream) {
  return whiten_like_fwd(x, y, N, C, HW, group_size, n_domains, mode, 1.f - eps, eps, momentum, 1.f, update_running,
                         running_mean, running_cov, nullptr, nullptr, nullptr, nullptr, 0, save_mean, save_w, workspace,
                         workspace_bytes, (cudaStream_t)stream, Basis{Basis::NEWTON_SCHULZ, iterations, save_p});
}

int dwt_whiten_zca_bwd(const float* x, const float* dout, float* dx, int64_t N, int64_t C, int64_t HW, int group_size,
                       int n_domains, int mode, float eps, int iterations, const float* save_mean, const float* save_w,
                       const float* save_p, void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  return whiten_like_bwd(x, dout, nullptr, dx, N, C, HW, group_size, n_domains, mode, 1.f - eps, save_mean, save_w, nullptr,
                         nullptr, nullptr, nullptr, 0, nullptr, nullptr, workspace, workspace_bytes, (cudaStream_t)stream,
                         Basis{Basis::NEWTON_SCHULZ, iterations, save_p});
}

int dwt_whiten_eigh_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains, int mode,
                        float eps, float momentum, int update_running, float* const* running_mean, float* const* running_cov,
                        float* save_mean, float* save_w, float* save_e, void* workspace, size_t workspace_bytes,
                        dwt_stream_t stream) {
  return whiten_like_fwd(x, y, N, C, HW, group_size, n_domains, mode, 1.f - eps, eps, momentum, 1.f, update_running,
                         running_mean, running_cov, nullptr, nullptr, nullptr, nullptr, 0, save_mean, save_w, workspace,
                         workspace_bytes, (cudaStream_t)stream, Basis{Basis::EIGH, 0, save_e});
}

int dwt_whiten_eigh_bwd(const float* x, const float* dout, float* dx, int64_t N, int64_t C, int64_t HW, int group_size,
                        int n_domains, int mode, float eps, const float* save_mean, const float* save_w, const float* save_e,
                        void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  return whiten_like_bwd(x, dout, nullptr, dx, N, C, HW, group_size, n_domains, mode, 1.f - eps, save_mean, save_w, nullptr,
                         nullptr, nullptr, nullptr, 0, nullptr, nullptr, workspace, workspace_bytes, (cudaStream_t)stream,
                         Basis{Basis::EIGH, 0, save_e});
}

int dwt_whiten_color_fwd(const float* x, float* y, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains, int mode,
                         float eps, float momentum, int update_running, float* const* running_mean, float* const* running_cov,
                         const float* color, const float* bias, float* save_mean, float* save_w, void* workspace,
                         size_t workspace_bytes, dwt_stream_t stream) {
  Basis b;
  b.kind = Basis::COLOR; b.color = color; b.bias = bias;
  return whiten_like_fwd(x, y, N, C, HW, group_size, n_domains, mode, 1.f - eps, eps, momentum, 1.f, update_running,
                         running_mean, running_cov, nullptr, nullptr, nullptr, nullptr, 0, save_mean, save_w, workspace,
                         workspace_bytes, (cudaStream_t)stream, b);
}

int dwt_whiten_color_bwd(const float* x, const float* dout, float* dx, int64_t N, int64_t C, int64_t HW, int group_size,
                         int n_domains, int mode, float eps, const float* save_mean, const float* save_w, const float* color,
                         float* dcolor, float* dbias, void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  Basis b;
  b.kind = Basis::COLOR; b.color = color; b.dcolor = dcolor; b.dbias = dbias;
  return whiten_like_bwd(x, dout, nullptr, dx, N, C, HW, group_size, n_domains, mode, 1.f - eps, save_mean, save_w, nullptr,
                         nullptr, nullptr, nullptr, 0, nullptr, nullptr, workspace, workspace_bytes, (cudaStream_t)stream, b);
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

int dwt_tail2_fwd(int kind, const dwt_tail_site* sites, float* y, uint8_t* relu_mask, int64_t N, int64_t C, int64_t HW,
                  int group_size, int n_domains, void* workspace, size_t workspace_bytes, dwt_stream_t stream) {
  return tail2_fwd(kind, sites, y, relu_mask, N, C, HW, group_size, n_domains, workspace, workspace_bytes, (cudaStream_t)stream);
}

int dwt_tail2_bwd(int kind, const dwt_tail_site* sites, const float* dout, const float* dout2, const uint8_t* relu_mask, float* dz,
                  int64_t N, int64_t C, int64_t HW, int group_size, int n_domains, void* workspace, size_t workspace_bytes,
                  dwt_stream_t stream) {
  return tail2_bwd(kind, sites, dout, dout2, relu_mask, dz, N, C, HW, group_size, n_domains, workspace, workspace_bytes,
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
                    int stride, int padding, int flags, dwt_stream_t stream) {
  int OH = 0, OW = 0;
  if (int rc = pool_check(N, H, W, C, kernel, stride, padding, &OH, &OW)) return rc;
  if (flags != 0 && flags != DWT_DTYPE_BF16) return fail(DWT_E_INVALID, "bad flags %#x (0 or DWT_DTYPE_BF16)", flags);
  const bool bf16 = flags == DWT_DTYPE_BF16;
  if (!x || !y || !argmax) return fail(DWT_E_INVALID, "null pointer argument");
  if ((uintptr_t)argmax % 4 != 0) return fail(DWT_E_INVALID, "pooling tensors must be 16-byte aligned");
  if (int rc = check_align(bf16, (uintptr_t)x | (uintptr_t)y, "pooling tensors")) return rc;
  {
    const double in = (double)N * H * W * C, out = (double)N * OH * OW * C;
    Launch l(fam(bf16, "maxpool_fwd", "maxpool_fwd_bf16"), nullptr, (bf16 ? 2.0 : 4.0) * (in + out) + out, (cudaStream_t)stream);
    dwt::maxpool_fwd_launch(x, y, bf16, argmax, (int)N, (int)H, (int)W, (int)C, OH, OW, kernel, stride, padding, (cudaStream_t)stream);
  }
  return check_launch("max-pool forward kernel");
}

int dwt_maxpool_bwd(const float* dy, const uint8_t* argmax, float* dx, int64_t N, int64_t H, int64_t W, int64_t C, int kernel,
                    int stride, int padding, int flags, dwt_stream_t stream) {
  int OH = 0, OW = 0;
  if (int rc = pool_check(N, H, W, C, kernel, stride, padding, &OH, &OW)) return rc;
  if (flags != 0 && flags != DWT_DTYPE_BF16) return fail(DWT_E_INVALID, "bad flags %#x (0 or DWT_DTYPE_BF16)", flags);
  const bool bf16 = flags == DWT_DTYPE_BF16;
  if (!dy || !dx || !argmax) return fail(DWT_E_INVALID, "null pointer argument");
  if ((uintptr_t)argmax % 4 != 0) return fail(DWT_E_INVALID, "pooling tensors must be 16-byte aligned");
  if (int rc = check_align(bf16, (uintptr_t)dy | (uintptr_t)dx, "pooling tensors")) return rc;
  {
    const double in = (double)N * H * W * C, out = (double)N * OH * OW * C;
    Launch l(fam(bf16, "maxpool_bwd", "maxpool_bwd_bf16"), nullptr, (bf16 ? 2.0 : 4.0) * (in + out) + out, (cudaStream_t)stream);
    dwt::maxpool_bwd_launch(dy, argmax, dx, bf16, (int)N, (int)H, (int)W, (int)C, OH, OW, kernel, stride, padding, (cudaStream_t)stream);
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

// C-ABI of libteaser_b200.so: context, workspace, stage entry points and the fused batch solve.
// See include/teaser_b200.h for the contract and the reference functions each symbol replaces.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "tzr_internal.cuh"

using namespace tzr;

// A grow-only device buffer (ensure), freed with its context.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() {
    if (p) cudaFree(p);
  }
};

namespace {

// What a per-problem buffer of a Batch holds: the input points (in the workspace only when the call owns them, not for
// tzr_solve_batch_dev or a caller's bitsets), the clique state (carved again for the large route's compacted batch), or
// the rest of the pipeline's per-problem state.
enum BufKind { kPoints, kClique, kOther };

// Every per-problem buffer of bt, in a fixed order: f(field, elements per problem, kind).  A batch's buffer holds its B
// problems back to back, so problem b starts b * elements in.
template <class F>
void batch_buffers(Batch& bt, F&& f) {
  const size_t n = (size_t)bt.n, W32 = (size_t)pitch32(bt.n), rot = (size_t)bt.rot_cap, sort = (size_t)bt.sort_cap;
  f(bt.src, 3 * n, kPoints);
  f(bt.dst, 3 * n, kPoints);
  f(bt.sf, n, kOther);
  f(bt.df, n, kOther);
  f(bt.gq, 2 * n, kOther);
  f(bt.pk, 6 * (size_t)npad128(bt.n), kOther);
  f(bt.opnd, tc_operand_bytes(1, bt.n) / sizeof(float), kOther);
  f(bt.gc, 1, kOther);
  f(bt.adj, n * pitch64(bt.n), kClique);
  f(bt.deg, n, kClique);
  f(bt.n_edges2, 1, kClique);
  f(bt.hclq, kHeurRoots * n, kClique);
  f(bt.hsize, kHeurRoots, kClique);
  f(bt.clq, n, kClique);
  f(bt.L, 1, kClique);
  f(bt.alive, W32, kClique);
  f(bt.best_bits, W32, kClique);
  f(bt.alive_cnt, 1, kClique);
  f(bt.root_ctr, 1, kClique);
  f(bt.lock, 1, kClique);
  f(bt.flags, 1, kClique);
  f(bt.kcore_final, 1, kClique);
  f(bt.t_start, 1, kClique);
  f(bt.ps, 3 * n, kOther);
  f(bt.pd, 3 * n, kOther);
  f(bt.wgt, rot, kOther);
  f(bt.res, n, kOther);
  f(bt.skey, 3 * sort, kOther);
  f(bt.sidx, 3 * sort, kOther);
  f(bt.sorted_clq, n, kOther);
  f(bt.rot_mask, rot, kOther);
  f(bt.trans_mask, n, kOther);
  f(bt.sol, 1, kOther);
}
constexpr int kBatchBuffers = 33;  // the fields batch_buffers visits

// Point a buffer field at byte `at` of a workspace allocation.
template <class T>
void point_at(T*& field, void* base, size_t at) {
  field = (T*)((char*)base + at);
}

// Bytes of the exact phase's scratch (Batch::stack, cv, centry) for bt's persistent grid (exact_ctas, max_depth).
struct ExactScratch {
  size_t stack, cv, centry;
};
ExactScratch exact_scratch(const Batch& bt) {
  const size_t warps = (size_t)bt.exact_ctas * 8;
  return ExactScratch{warps * bt.max_depth * 2 * pitch32(bt.n) * sizeof(uint32_t),
                      std::max(warps, (size_t)4 * bt.B) * bt.n * sizeof(int32_t),
                      warps * bt.max_depth * sizeof(int32_t)};
}

// The retained result of the most recent solve or graph build: its size classes (one for a uniform solve or a graph
// build) and where each problem lies in them; problem b is sub_batch(cls[at[b].c], at[b].k, 1).  Cleared whenever the
// workspace is reused (forget_retained).
struct Retained {
  struct Problem {
    int c, k, n;  // class, index in the class, own correspondences (<= the class's n)
  };
  std::vector<Batch> cls;
  std::vector<Problem> at;  // per problem in the caller's order; empty: nothing retained
  bool is_solve = false;    // every problem's record, clique, masks and inputs are in the workspace (tzr_last_inliers,
                            // tzr_certify_last_solve); false after tzr_graph_build
  bool complete = false;    // its rotation ran on COMPLETE TIMs
  bool has_graph = false;   // false: the solve ran with inlier selection NONE (no graph was built)
  // clique route of every problem of the most recent clique stage, a solve's or tzr_max_clique(_batch)'s, in the
  // caller's order (tzr_ctx_clique_route); empty after NONE or a graph build
  std::vector<int32_t> route;
};

}  // namespace

struct tzr_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  std::string last_error;
  int64_t launches = 0;
  uint32_t flags = 0;
  int num_sms = 132;
  // the solve's workspace: one buffer per field of batch_buffers, in its order, then the buffers every size class
  // shares: the re-check queue, the exact-phase scratch and the debug counters
  DevBuf ws[kBatchBuffers];
  DevBuf tclist, stack, cv, centry, dbg;
  // the single-stage entry points, the unknown-scale stage, the front end and the certifier
  DevBuf misc, sc, m_in, m_scratch, m_out, certb;
  // large clique route (n > kMaxN or debug flag 524288): scratch on the full graph, and the compacted batch's buffers
  DevBuf lg, cq;
  // ragged batches (DESIGN.md §4.2): the size-class tables, and the flat inputs / outputs of host-pointer calls
  DevBuf rg;
  // tzr_icp(_batch): its own workspace, so that refinement leaves a retained solve intact
  DevBuf icp;
  // tzr_voxel_downsample(_batch): its own workspace, for the same reason
  DevBuf vox;
  // tzr_pose_graph_optimize: its own workspace, for the same reason
  DevBuf pg;
  int last_strip_blocks = 0;  // strip length of the most recent graph kernel launch (tzr_ctx_last_strip_blocks)
  int max_n = kMaxN;  // per-problem size limit of this context (tzr_ctx_set_max_n: kMaxN ... kMaxNLarge)
  // pinned host staging
  void* h_pin = nullptr;
  size_t h_pin_cap = 0;
  Retained last;
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // start | prep | graph tiles | clique (incl. degrees) | rot+trans
  std::vector<cudaEvent_t> graph_ev;  // pairs around every graph-kernel launch of the last call (roofline timing)
  int graph_ev_used = 0;
  std::vector<cudaEvent_t> stage_ev;  // 5 per chunk; [stage_first, stage_chunks) belong to the last pipelined call
  int stage_chunks = 0, stage_first = 0, graph_first = 0;
  bool stage_log = false;  // keep the events of every call since the last tzr_ctx_stage_log_read (bench.py: no sync per step)
  int stage_log_calls = 0;
  uint64_t generation = 0;   // bumped by every call that rebuilds or invalidates the retained graph (ctx->last)
  // chunked batches run on two lanes: the issue-bound graph kernels queue back to back on the low-priority gstream,
  // the latency-/HBM-bound degree, clique and rotation kernels of the previous chunk run on the high-priority hstream
  // and slot into the SMs as graph CTAs retire
  cudaStream_t gstream = nullptr, hstream = nullptr;
  cudaEvent_t join_ev = nullptr, join_ev2 = nullptr;
  std::vector<cudaEvent_t> gdone_ev;
  void* solver_handle = nullptr;  // cusolverDnHandle_t of the certifier, created on first use (certify.cu)
  cudaStream_t copy_stream = nullptr;  // H2D of chunk k+1 overlaps the kernels of chunk k (host-pointer batches)
  std::vector<cudaEvent_t> chunk_ev;
  // the batch of the most recent tzr_max_clique(_batch) call (tzr_ctx_clique_info); B = 0 once the workspace is reused
  Batch clique{};
};

namespace {

#define CK(call)                                                                  \
  do {                                                                            \
    cudaError_t _e = (call);                                                      \
    if (_e != cudaSuccess) {                                                      \
      ctx->last_error = std::string(#call) + ": " + cudaGetErrorString(_e);       \
      return TZR_ERR_CUDA;                                                        \
    }                                                                             \
  } while (0)

int ensure(tzr_ctx* ctx, DevBuf& b, size_t bytes) {
  if (bytes <= b.cap && b.p) return TZR_OK;
  if (b.p) {
    cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
  }
  size_t want = bytes + bytes / 8 + 256;
  cudaError_t e = cudaMalloc(&b.p, want);
  if (e != cudaSuccess) {
    cudaGetLastError();  // not sticky: keep it from surfacing as a launch error of a later call
    ctx->last_error = std::string("cudaMalloc of ") + std::to_string(want) + " bytes: " + cudaGetErrorString(e);
    return TZR_ERR_ALLOC;
  }
  b.cap = want;
  return TZR_OK;
}

int ensure_pinned(tzr_ctx* ctx, size_t bytes) {
  if (bytes <= ctx->h_pin_cap) return TZR_OK;
  if (ctx->h_pin) cudaFreeHost(ctx->h_pin);
  ctx->h_pin = nullptr;
  ctx->h_pin_cap = 0;
  cudaError_t e = cudaMallocHost(&ctx->h_pin, bytes + bytes / 8 + 256);
  if (e != cudaSuccess) {
    ctx->last_error = std::string("cudaMallocHost: ") + cudaGetErrorString(e);
    return TZR_ERR_ALLOC;
  }
  ctx->h_pin_cap = bytes + bytes / 8 + 256;
  return TZR_OK;
}

struct CopySpan {
  void* dst;
  const void* src;
  size_t bytes;
};

// Host memcpy of every span with a few host threads, each taking a contiguous share of the bytes (pageable host memory
// cannot be DMA'd asynchronously; one thread moves ~10 GB/s, which is slower than the GPU consumes it).
void parallel_copy(const std::vector<CopySpan>& spans) {
  size_t total = 0;
  for (const CopySpan& s : spans) total += s.bytes;
  int T = (int)std::min<size_t>(8, total / ((size_t)4 << 20));
  const unsigned hw = std::thread::hardware_concurrency();
  if (hw && (unsigned)T > hw) T = (int)hw;
  auto run = [&spans](size_t lo, size_t hi) {
    size_t at = 0;
    for (const CopySpan& s : spans) {
      const size_t a = std::max(lo, at), b = std::min(hi, at + s.bytes);
      if (a < b) memcpy((char*)s.dst + (a - at), (const char*)s.src + (a - at), b - a);
      at += s.bytes;
      if (at >= hi) break;
    }
  };
  if (T <= 1) {
    run(0, total);
    return;
  }
  std::vector<std::thread> th;
  for (int t = 0; t < T; ++t) th.emplace_back(run, total * t / T, total * (t + 1) / T);
  for (auto& x : th) x.join();
}

// Host -> device of spans whose dst lies in the pinned area h (mirrored at d); [tables, bytes) holds the library's own
// tables.  A batch is gathered into the pinned area and copied once; a single cloud or pair goes straight from the
// caller's memory, where the driver pipelines its own staging of pageable memory with the DMA, and the tables follow
// in one pinned copy.
cudaError_t stage_in(const std::vector<CopySpan>& spans, char* h, char* d, size_t tables, size_t bytes, bool direct,
                     cudaStream_t st) {
  if (!direct) {
    parallel_copy(spans);
    return cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st);
  }
  std::vector<CopySpan> own;
  for (const CopySpan& s : spans) {
    const size_t off = (size_t)((char*)s.dst - h);
    if (off >= tables) {
      own.push_back(s);
      continue;
    }
    const cudaError_t e = cudaMemcpyAsync(d + off, s.src, s.bytes, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return e;
  }
  parallel_copy(own);
  return cudaMemcpyAsync(d + tables, h + tables, bytes - tables, cudaMemcpyHostToDevice, st);
}

// Device -> host of spans whose src lies in the pinned area h (mirrored at d), then synchronise: one copy of `bytes`
// and host copies for a batch, a copy per span (spans with dst == src land in the pinned area itself) for one cloud.
cudaError_t stage_out(const std::vector<CopySpan>& spans, char* h, const char* d, size_t bytes, bool direct,
                      cudaStream_t st) {
  cudaError_t e = cudaSuccess;
  if (!direct) {
    e = cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, st);
  } else {
    for (const CopySpan& s : spans)
      if (e == cudaSuccess) e = cudaMemcpyAsync(s.dst, d + ((const char*)s.src - h), s.bytes, cudaMemcpyDeviceToHost, st);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e == cudaSuccess && !direct) {
    std::vector<CopySpan> host;
    for (const CopySpan& s : spans)
      if (s.dst != s.src) host.push_back(s);
    parallel_copy(host);
  }
  return e;
}

// Copy `count` caller buffers of `per` bytes each into a contiguous pinned area.
void parallel_stage(char* dst_base, const double* const* bufs, int first, int count, size_t per) {
  std::vector<CopySpan> spans((size_t)count);
  for (int b = 0; b < count; ++b) spans[b] = CopySpan{dst_base + per * b, bufs[first + b], per};
  parallel_copy(spans);
}

// effective inlier selection mode (registration.cc:574-583)
int effective_mode(const tzr_params& p) {
  int mode = p.inlier_selection_mode;
  if (!p.use_max_clique) mode = 3;
  if (!p.max_clique_exact_solution) mode = 1;
  return mode;
}

// Exact-phase geometry of a (B, n) batch: a persistent grid that fills the GPU, whose warps own the search scratch (any
// problem): *ctas, *depth (stack levels per warp), *conc (problems searched at a time).
void search_geometry(const tzr_ctx* ctx, int B, int n, int* ctas, int* depth_out, int* conc) {
  int G = clique_exact_grid(n, ctx->num_sms);
  {
    const long long roots = ((long long)B * n + 7) / 8;  // never more warps than root vertices
    if ((long long)G > roots) G = (int)std::max<long long>(1, roots);
  }
  const size_t warps = (size_t)G * 8;
  const size_t level_bytes = (size_t)2 * pitch32(n) * sizeof(uint32_t);
  size_t depth = ((size_t)4 << 30) / (warps * level_bytes);
  if (depth > 512) depth = 512;
  if (depth > (size_t)n) depth = (size_t)n;
  if (depth < 16) depth = 16;
  *ctas = G;
  *depth_out = (int)depth;
  // debug flag 65536: a search stack of 8 levels, so that the depth cap (result not proven) is reachable at test sizes
  if (ctx->flags & 65536u) *depth_out = 8;
  {
    // problems under search at a time: their bitsets should stay in the L2 together (~18 MB of the 50 MB: the
    // stacks, the other lane's graph kernel and the two L2 partitions take the rest)
    const size_t bits = (size_t)n * pitch32(n) * sizeof(uint32_t);
    const size_t c = ((size_t)18 << 20) / std::max<size_t>(bits, 1);
    *conc = (int)std::min<size_t>(std::max<size_t>(c, 1), (size_t)B);
  }
}

// Nothing is retained any more: the workspace is about to be reused, or a call solved nothing.
void forget_retained(tzr_ctx* ctx) {
  ctx->last = Retained{};
  ++ctx->generation;
}

// Retain the size classes of the call that just ran.  Problem s in class order (the classes' problems back to back) is
// problem order[s] of the caller, with n[order[s]] correspondences of its own; order and n are nullptr for one class in
// the caller's order.  route: the clique routes in class order.  p: the solve's parameters, nullptr for a graph without
// solution records (tzr_graph_build).
void retain(tzr_ctx* ctx, std::vector<Batch> cls, const int* order, const int32_t* n, const std::vector<int32_t>& route,
            const tzr_params* p) {
  Retained& r = ctx->last;
  r.cls = std::move(cls);
  r.is_solve = p != nullptr;
  r.complete = p && p->rotation_tim_graph == 1;
  r.has_graph = !p || effective_mode(*p) != 3;  // NONE: populateVertices is never called (registration.cc:607-650)
  int B = 0;
  for (const Batch& bt : r.cls) B += bt.B;
  r.at.assign((size_t)B, Retained::Problem{});
  r.route.assign(r.has_graph ? route.size() : 0, 0);
  for (int c = 0, s = 0; c < (int)r.cls.size(); ++c) {
    Batch& bt = r.cls[c];
    for (int k = 0; k < bt.B; ++k, ++s) {
      const int q = order ? order[s] : s;
      r.at[q] = Retained::Problem{c, k, n ? n[q] : bt.n};
      if (!r.route.empty()) r.route[q] = route[s];
    }
    bt.nb_host = nullptr;  // the call's own host copy, gone once it returns
  }
}

// Size the workspace for C size classes (class c: B[c] problems of n[c] correspondences) and fill one Batch descriptor
// per class (src/dst left to the caller unless own_points).  Per-problem buffers hold the classes back to back in class
// order; the re-check queue, the exact-phase scratch and the debug counters are shared (the classes' pipelines run in
// stream order on each lane).  A uniform batch is one class.
int setup_classes(tzr_ctx* ctx, int C, const int* Bs, const int* ns, bool own_points, Batch* out,
                  bool complete_graph = false) {
  for (int c = 0; c < C; ++c) {
    if (Bs[c] <= 0 || ns[c] <= 0) return TZR_ERR_INVALID_ARG;
    if (ns[c] > ctx->max_n) {
      ctx->last_error = "n = " + std::to_string(ns[c]) + " exceeds this context's limit of " + std::to_string(ctx->max_n) +
                        " correspondences (tzr_ctx_set_max_n raises it to " + std::to_string(kMaxNLarge) + ")";
      return TZR_ERR_TOO_LARGE;
    }
  }
  // the workspace is about to be re-used (and possibly re-allocated): the retained graph of the previous call is gone
  forget_retained(ctx);
  ctx->clique.B = 0;
  // per class: geometry, and the largest size of each shared buffer
  size_t tcl = 0;
  ExactScratch ex{0, 0, 0};
  for (int c = 0; c < C; ++c) {
    const int B = Bs[c], n = ns[c];
    Batch& bt = out[c];
    bt = Batch{};
    bt.B = B;
    bt.n = n;
    bt.tc_list_cap = (unsigned int)tc_list_entries(B, n);
    tcl = std::max(tcl, (size_t)bt.tc_list_cap * sizeof(uint2) + 256);
    // debug flag 16384: a re-check queue of 64 entries (the buffer keeps its full size), so that the queue-full path of
    // the graph kernels (void entries, in-place exact evaluation, the patch kernel's clamp) runs at test sizes
    if (ctx->flags & 16384u) bt.tc_list_cap = std::min(bt.tc_list_cap, 64u);
    // exact phase: above kMaxN the search runs on the large route's compacted batch, which has its own scratch
    if (n <= kMaxN) {
      search_geometry(ctx, B, n, &bt.exact_ctas, &bt.max_depth, &bt.exact_conc);
      const ExactScratch e = exact_scratch(bt);
      ex = ExactScratch{std::max(ex.stack, e.stack), std::max(ex.cv, e.cv), std::max(ex.centry, e.centry)};
    }
    bt.sort_cap = next_pow2(2 * n);
    // rotation TIM capacity: n for CHAIN; for COMPLETE min(n(n-1)/2, what a 4 GiB budget allows)
    bt.rot_cap = n;
    if (complete_graph) {
      const long long full = (long long)n * (n - 1) / 2;
      const long long budget = ((long long)4 << 30) / (9LL * B);
      bt.rot_cap = std::max<long long>(n, std::min(full, budget));
    }
  }
  // per-problem buffers: the classes back to back, each class's share 256-byte aligned.  The first pass sizes the
  // buffers, the second (after they are allocated) points every class at its share.
  size_t total[kBatchBuffers];
  auto lay_out = [&](bool point) {
    std::fill(total, total + kBatchBuffers, (size_t)0);
    for (int c = 0; c < C; ++c) {
      int k = 0;
      batch_buffers(out[c], [&](auto& field, size_t per, BufKind kind) {
        if (point) point_at(field, ctx->ws[k].p, total[k]);
        if (kind != kPoints || own_points) total[k] += al256((size_t)out[c].B * per * sizeof(*field));
        ++k;
      });
    }
  };
  lay_out(false);
  int rc;
  for (int k = 0; k < kBatchBuffers; ++k)
    if (total[k] && (rc = ensure(ctx, ctx->ws[k], total[k])) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->tclist, tcl)) != TZR_OK || (rc = ensure(ctx, ctx->stack, ex.stack)) != TZR_OK ||
      (rc = ensure(ctx, ctx->cv, ex.cv)) != TZR_OK || (rc = ensure(ctx, ctx->centry, ex.centry)) != TZR_OK ||
      (rc = ensure(ctx, ctx->dbg, 16 * sizeof(unsigned long long))) != TZR_OK)
    return rc;
  lay_out(true);
  static const double kappa_env = [] {
    const char* e = std::getenv("TZR_TC_KAPPA");
    return e ? std::atof(e) : 0.0;
  }();
  static const int swap_env = [] {
    const char* e = std::getenv("TZR_TC_SWAP");
    return e ? std::atoi(e) : 0;
  }();
  for (int c = 0; c < C; ++c) {
    Batch& bt = out[c];
    bt.tc_list_count = (unsigned int*)ctx->tclist.p;
    bt.tc_list = (uint2*)((char*)ctx->tclist.p + 256);
    bt.stack = (uint32_t*)ctx->stack.p;
    bt.cv = (int32_t*)ctx->cv.p;
    bt.centry = (int32_t*)ctx->centry.p;
    bt.mismatches = (unsigned long long*)ctx->dbg.p;
    bt.rechecks = (ctx->flags & 4u) ? (unsigned long long*)ctx->dbg.p + 1 : nullptr;
    bt.flags_dbg = ctx->flags;
    bt.tc_kappa = kappa_env;
    bt.tc_desc_swap = swap_env;
  }
  return TZR_OK;
}

// Size the workspace for a (B, n) batch and fill the Batch descriptor (src/dst left to the caller).
int setup_batch(tzr_ctx* ctx, int B, int n, bool own_points, Batch* out, bool complete_graph = false) {
  return setup_classes(ctx, 1, &B, &n, own_points, out, complete_graph);
}

int check_launch(tzr_ctx* ctx, const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    ctx->last_error = std::string(what) + ": " + cudaGetErrorString(e);
    return TZR_ERR_CUDA;
  }
  return TZR_OK;
}

// Caller-supplied bitsets (tzr_max_clique_batch): clear the diagonal bit and the bits at or beyond n of every row, which
// the header declares ignored.  The clique kernels rely on neither being set.
__global__ void sanitize_adj_kernel(uint64_t* adj, int B, int n) {
  const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= (size_t)B * n) return;
  const int v = (int)(r % (size_t)n);
  uint64_t* row = adj + r * pitch64(n);
  row[v >> 6] &= ~(1ull << (v & 63));
  if (n & 63) row[words64(n) - 1] &= (1ull << (n & 63)) - 1ull;
}

__global__ void init_solutions_kernel(tzr_solution* sol, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  tzr_solution s;
  memset(&s, 0, sizeof(s));
  s.valid = 1;
  s.scale = 1.0;  // ScaleInliersSelector: *scale = 1  (registration.cc:432)
  sol[b] = s;
}

// View of problems [b0, b0+Bc) of a batch: every per-problem buffer is offset, geometry is unchanged.
Batch sub_batch(const Batch& bt, int b0, int Bc) {
  Batch s = bt;
  const size_t o = (size_t)b0;
  s.B = Bc;
  batch_buffers(s, [o](auto& field, size_t per, BufKind) { field += o * per; });
  if (bt.nb) s.nb = bt.nb + o;
  if (bt.nb_host) s.nb_host = bt.nb_host + o;
  return s;
}

// Problem b (caller's order) of the retained record: a view of its slot in its class.
Batch retained_problem(const tzr_ctx* ctx, int b) {
  const Retained::Problem& q = ctx->last.at[b];
  return sub_batch(ctx->last.cls[q.c], q.k, 1);
}

// Problems per pipeline chunk: small enough that a chunk's adjacency bitsets (written by the graph kernel, then
// read by the degree / clique kernels) stay resident in the 50 MB L2 instead of making a round trip through HBM.
int l2_chunk(const tzr_ctx* ctx, int B, int n, const tzr_params& p) {
  (void)ctx;
  // Optional sub-chunking of graph+degree so the degree pass reads the bitsets from L2 (TZR_L2_CHUNK_MB = MB of
  // adjacency per sub-chunk).  Off by default: with the v5 graph kernel the tail of each small launch costs more
  // than the saved HBM read.
  static const long long budget_mb = [] {
    const char* e = std::getenv("TZR_L2_CHUNK_MB");
    return e ? std::atoll(e) : 0LL;
  }();
  if (budget_mb <= 0 || p.estimate_scaling) return B;
  const size_t per = (size_t)n * pitch64(n) * 8;
  long long c = (long long)((size_t)budget_mb << 20) / (long long)std::max<size_t>(per, 1);
  if (c < 1) c = 1;
  if (c >= B) return B;
  return (int)c;
}

// Large clique route (DESIGN.md §3.2), taken when n > kMaxN or under debug flag 524288: the heuristic on the full graph,
// its (L-1)-core on many CTAs, the cores compacted (order-preserving) into a batch of at most kMaxN vertices per problem
// (64 under debug flag 1048576), the small route's peel and exact passes on that batch, the cliques mapped back.  One
// host read-back: the core sizes, which size the compacted batch, with each problem's last change counter.  A problem
// whose last round still removed vertices holds a superset of its core (a pendant path loses one or two vertices per
// round); while such a problem would be searched or capped, further blocks of kCoreRounds rounds run on it, each with
// its own read-back, so that every decision below is made on the core.  Graphs that converge inside the first block
// take no extra launch.  route: B entries as tzr_ctx_clique_route reports them.
int run_clique_large(tzr_ctx* ctx, const Batch& bt, const tzr_params& p, int mode, cudaStream_t st, int* nl,
                     int32_t* route) {
  const int B = bt.B, n = bt.n;
  const size_t Bn = (size_t)B * n;
  size_t off = 0;
  auto carve = [&off](size_t bytes) {
    const size_t o = off;
    off = al256(off + bytes);
    return o;
  };
  const size_t o_lists = carve(Bn * kHeurRoots * 2 * sizeof(uint16_t)), o_chg = carve((size_t)B * kCoreSlots * 4),
               o_n2o = carve(Bn * 4), o_o2n = carve(Bn * 4), o_cnt = carve((size_t)B * 4), o_route = carve((size_t)B * 4);
  int rc = ensure(ctx, ctx->lg, off);
  if (rc) return rc;
  char* lg = (char*)ctx->lg.p;
  int32_t* n2o = (int32_t*)(lg + o_n2o);
  int32_t* o2n = (int32_t*)(lg + o_o2n);
  int32_t* cnt_d = (int32_t*)(lg + o_cnt);
  int32_t* route_d = (int32_t*)(lg + o_route);
  int32_t* chg_d = (int32_t*)(lg + o_chg);
  launch_clique_large_front(bt, p, mode, (uint16_t*)(lg + o_lists), st, nl);
  std::vector<int32_t> L(B), cnt(B, 0), last(B, 0);
  // the core sizes and each problem's last change counter (slot kCoreRounds: removals in the block's last round)
  auto read_core = [&]() -> int {
    CK(cudaMemcpyAsync(cnt.data(), cnt_d, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpy2DAsync(last.data(), 4, chg_d + kCoreRounds, (size_t)kCoreSlots * 4, 4, (size_t)B,
                         cudaMemcpyDeviceToHost, st));
    return TZR_OK;
  };
  if (mode == 0) launch_core(bt, chg_d, n2o, o2n, cnt_d, ctx->num_sms, st, nl);
  CK(cudaMemcpyAsync(L.data(), bt.L, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  if (mode == 0 && (rc = read_core())) return rc;
  CK(cudaStreamSynchronize(st));
  if (mode == 0) {
    // peel on while a problem that would be searched or capped still shrinks (L <= 1 and the shortcut are final: a
    // set of exactly L survivors is the incumbent itself)
    std::vector<int32_t> go((size_t)B * kCoreSlots);
    for (;;) {
      std::fill(go.begin(), go.end(), 0);
      bool more = false;
      for (int b = 0; b < B; ++b)
        if (L[b] > 1 && cnt[b] != L[b] && last[b] != 0) {
          go[(size_t)b * kCoreSlots] = 1;
          more = true;
        }
      if (!more) break;
      CK(cudaMemcpyAsync(chg_d, go.data(), go.size() * 4, cudaMemcpyHostToDevice, st));
      launch_core_rounds(bt, chg_d, n2o, o2n, cnt_d, ctx->num_sms, st, nl);
      if ((rc = read_core())) return rc;
      CK(cudaStreamSynchronize(st));
    }
  }
  // heuristic modes, L <= 1 and the uniqueness shortcut (only the incumbent survives its own core bound): the result is
  // final, reported as the clique size (at least 1)
  const int cap = (ctx->flags & 1048576u) ? 64 : kMaxN;
  std::vector<int32_t> search(B, 0);
  int n2 = 0;
  for (int b = 0; b < B; ++b) {
    if (mode != 0 || L[b] <= 1 || cnt[b] == L[b]) {
      route[b] = std::max(L[b], 1);
    } else if (cnt[b] > cap) {
      route[b] = -1;
      search[b] = -1;
    } else {
      route[b] = cnt[b];
      search[b] = 1;
      n2 = std::max(n2, cnt[b]);
    }
  }
  if (mode != 0) return TZR_OK;
  CK(cudaMemcpyAsync(route_d, search.data(), (size_t)B * 4, cudaMemcpyHostToDevice, st));
  Batch cb = bt;
  if (n2 > 0) {
    // the compacted batch: B problems of n2 vertices, its own clique state and exact-phase scratch carved from one
    // buffer.  The first pass sizes it, the second (after it is allocated) points the fields at their shares.
    cb.n = n2;
    search_geometry(ctx, B, n2, &cb.exact_ctas, &cb.max_depth, &cb.exact_conc);
    const ExactScratch ex = exact_scratch(cb);
    auto lay_out = [&](char* q) {
      off = 0;
      batch_buffers(cb, [&](auto& field, size_t per, BufKind kind) {
        if (kind != kClique) return;
        const size_t at = carve((size_t)B * per * sizeof(*field));
        if (q) point_at(field, q, at);
      });
      const size_t at[3] = {carve(ex.stack), carve(ex.cv), carve(ex.centry)};
      if (q) {
        point_at(cb.stack, q, at[0]);
        point_at(cb.cv, q, at[1]);
        point_at(cb.centry, q, at[2]);
      }
    };
    lay_out(nullptr);
    if ((rc = ensure(ctx, ctx->cq, off))) return rc;
    lay_out((char*)ctx->cq.p);
    cb.kcore_final = nullptr;
    launch_core_compact(bt, cb, n2o, o2n, cnt_d, route_d, st, nl);
    CK(cudaMemsetAsync(cb.n_edges2, 0, (size_t)B * 8, st));
    launch_degree(cb, st, true);
    launch_clique_search(cb, st, nl);
    *nl += 1;
  }
  launch_core_map_back(bt, cb, n2o, route_d, st, nl);
  return TZR_OK;
}

// The clique stage of a batch: the small route (launch_clique) or the large one.  route: B entries (tzr_ctx_clique_route).
int run_clique(tzr_ctx* ctx, const Batch& bt, const tzr_params& p, int mode, cudaStream_t st, int* nl, int32_t* route) {
  if (bt.n > kMaxN || (ctx->flags & 524288u)) return run_clique_large(ctx, bt, p, mode, st, nl, route);
  launch_clique(bt, p, mode, st, nl);
  std::fill(route, route + bt.B, 0);
  return TZR_OK;
}

// The fused device pipeline for one uniform batch.  src/dst must already be set in bt.
// st: stream of the clique / rotation stages; sg: stream of prep + graph (== st for the single-lane form, otherwise
// gdone is recorded on sg after the graph kernel and st waits for it).
// route: the batch's clique routes.
int run_pipeline(tzr_ctx* ctx, Batch& bt, const tzr_params& p, cudaEvent_t* ev, cudaStream_t st, int32_t* route,
                 cudaStream_t sg = nullptr, cudaEvent_t gdone = nullptr) {
  if (!sg) sg = st;
  if (p.rotation_estimation_algorithm < 0 || p.rotation_estimation_algorithm > 2 || p.rotation_tim_graph < 0 ||
      p.rotation_tim_graph > 1)
    return TZR_ERR_INVALID_ARG;
  const int mode = effective_mode(p);
  bt.beta = 2.0 * p.noise_bound * std::sqrt(p.cbar2);  // registration.cc:438
  // Params::max_clique_time_limit (seconds) -> device-side budget of the exact search
  bt.budget_ns = 0ull;
  if (mode == 0 && p.max_clique_time_limit > 0 && p.max_clique_time_limit < 1e7)
    bt.budget_ns = (unsigned long long)(p.max_clique_time_limit * 1e9);
  // unknown scale (Params default): TLS over the K TIM ratios first (registration.cc:603 -> :410-425)
  bt.scale_mode = p.estimate_scaling ? 1 : 0;
  if (bt.scale_mode) {
    const size_t bytes = scale_scratch_bytes(bt.B, bt.n, ctx->flags);
    if (!bytes) {
      ctx->last_error = "estimate_scaling: 2K end points exceed 2^31";
      return TZR_ERR_TOO_LARGE;
    }
    const int rc = ensure(ctx, ctx->sc, bytes);
    if (rc != TZR_OK) return rc;
  }
  cudaEventRecord(ev[0], sg);
  init_solutions_kernel<<<(bt.B + 127) / 128, 128, 0, sg>>>(bt.sol, bt.B);
  ctx->launches += 1;
  // before prep: the FP32 filter copies are pre-scaled by the estimate
  if (bt.scale_mode) ctx->launches += launch_scale_estimation(bt, ctx->flags, ctx->sc.p, sg);
  launch_prep(bt, sg);
  ctx->launches += 1;
  cudaEventRecord(ev[1], sg);
  int nl = 0;
  if (mode != 3) {
    // graph + degree, optionally in L2-sized sub-chunks (see l2_chunk); the graph kernel has its own event pair.
    const int gch = l2_chunk(ctx, bt.B, bt.n, p);
    for (int b0 = 0; b0 < bt.B; b0 += gch) {
      Batch sb = (gch < bt.B) ? sub_batch(bt, b0, std::min(gch, bt.B - b0)) : bt;
      while ((int)ctx->graph_ev.size() < ctx->graph_ev_used + 2) {
        cudaEvent_t e;
        if (cudaEventCreate(&e) != cudaSuccess) return TZR_ERR_CUDA;
        ctx->graph_ev.push_back(e);
      }
      cudaEventRecord(ctx->graph_ev[ctx->graph_ev_used], sg);
      nl += launch_graph(sb, sg, ctx->num_sms, &ctx->last_strip_blocks) - 1;
      cudaEventRecord(ctx->graph_ev[ctx->graph_ev_used + 1], sg);
      ctx->graph_ev_used += 2;
      if (sg != st) {  // two lanes (never combined with L2 sub-chunking: gch == B there)
        cudaEventRecord(gdone, sg);
        cudaStreamWaitEvent(st, gdone, 0);
      }
      launch_degree(sb, st);
      nl += 2;
    }
    cudaEventRecord(ev[2], st);
    const int rc = run_clique(ctx, bt, p, mode, st, &nl, route);
    if (rc) return rc;
  } else {
    if (sg != st) {
      cudaEventRecord(gdone, sg);
      cudaStreamWaitEvent(st, gdone, 0);
    }
    cudaEventRecord(ev[2], st);
  }
  cudaEventRecord(ev[3], st);
  launch_rot_trans(bt, p, mode != 3 ? 1 : 0, st);
  cudaEventRecord(ev[4], st);
  ctx->launches += nl + 1;
  return check_launch(ctx, "pipeline launch");
}

// Run the pipeline chunk by chunk on the compute stream.  chunks: views of consecutive problems, chunk c starting at
// problem bounds[c] of the call's B = bounds.back() (route: B entries).  ready[c] (optional) is an event the chunk's
// inputs wait for.  lanes_ok: several chunks may alternate between the two compute lanes.
int run_chunks(tzr_ctx* ctx, std::vector<Batch>& chunks, const std::vector<int>& bounds, const tzr_params& p,
               const cudaEvent_t* ready, const std::function<int(int)>& before_chunk, bool lanes_ok,
               std::vector<int32_t>& route) {
  const int n_chunks = (int)chunks.size();
  if (!ctx->stage_log) {
    ctx->graph_ev_used = 0;
    ctx->stage_chunks = 0;
  }
  ctx->stage_first = ctx->stage_chunks;
  ctx->graph_first = ctx->graph_ev_used;
  while ((int)ctx->stage_ev.size() < 5 * (ctx->stage_first + n_chunks)) {
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) return TZR_ERR_CUDA;
    ctx->stage_ev.push_back(e);
  }
  const bool lanes = n_chunks > 1 && ctx->gstream && ctx->hstream && lanes_ok;
  route.assign((size_t)bounds.back(), 0);
  // debug counters cover the whole call: zeroed once, ahead of every chunk on either lane (not per chunk, which would
  // keep only the last chunk's counts)
  if (ctx->flags & 6u) CK(cudaMemsetAsync((void*)ctx->dbg.p, 0, 16 * sizeof(unsigned long long), ctx->stream));
  if (lanes) {
    while ((int)ctx->gdone_ev.size() < n_chunks) {
      cudaEvent_t e;
      if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return TZR_ERR_CUDA;
      ctx->gdone_ev.push_back(e);
    }
    if (cudaEventRecord(ctx->join_ev, ctx->stream) != cudaSuccess) return TZR_ERR_CUDA;
    if (cudaStreamWaitEvent(ctx->gstream, ctx->join_ev, 0) != cudaSuccess) return TZR_ERR_CUDA;
    if (cudaStreamWaitEvent(ctx->hstream, ctx->join_ev, 0) != cudaSuccess) return TZR_ERR_CUDA;
  }
  for (int c = 0; c < n_chunks; ++c) {
    const int b0 = bounds[c];
    cudaStream_t st = lanes ? ctx->hstream : ctx->stream;
    cudaStream_t sg = lanes ? ctx->gstream : ctx->stream;
    if (before_chunk) {  // host-side work that produces this chunk's inputs (staging + H2D enqueue)
      const int rcb = before_chunk(c);
      if (rcb) return rcb;
    }
    if (ready) {
      if (cudaStreamWaitEvent(sg, ready[c], 0) != cudaSuccess) return TZR_ERR_CUDA;
    }
    int rc = run_pipeline(ctx, chunks[c], p, ctx->stage_ev.data() + 5 * (ctx->stage_first + c), st,
                          route.data() + b0, sg, lanes ? ctx->gdone_ev[c] : nullptr);
    if (rc) return rc;
  }
  if (lanes) {  // everything later on ctx->stream (D2H, the caller's work) is ordered after both lanes
    if (cudaEventRecord(ctx->join_ev, ctx->hstream) != cudaSuccess) return TZR_ERR_CUDA;
    if (cudaStreamWaitEvent(ctx->stream, ctx->join_ev, 0) != cudaSuccess) return TZR_ERR_CUDA;
    if (cudaEventRecord(ctx->join_ev2, ctx->gstream) != cudaSuccess) return TZR_ERR_CUDA;
    if (cudaStreamWaitEvent(ctx->stream, ctx->join_ev2, 0) != cudaSuccess) return TZR_ERR_CUDA;
  }
  ctx->stage_chunks = ctx->stage_first + n_chunks;
  if (ctx->stage_log) ++ctx->stage_log_calls;
  return TZR_OK;
}

// run_chunks over the chunks [bounds[c], bounds[c+1]) of one uniform batch; the batch becomes the retained graph.
int run_chunked(tzr_ctx* ctx, Batch& bt, const tzr_params& p, const std::vector<int>& bounds,
                const cudaEvent_t* ready, const std::function<int(int)>& before_chunk = nullptr) {
  const int n_chunks = (int)bounds.size() - 1;
  std::vector<Batch> chunks;
  for (int c = 0; c < n_chunks; ++c)
    chunks.push_back(n_chunks > 1 ? sub_batch(bt, bounds[c], bounds[c + 1] - bounds[c]) : bt);
  std::vector<int32_t> route;
  const int rc =
      run_chunks(ctx, chunks, bounds, p, ready, before_chunk, l2_chunk(ctx, bt.B, bt.n, p) >= bt.B, route);
  if (rc) return rc;
  if (n_chunks == 1) bt = chunks[0];  // keep fields filled in by run_pipeline (beta, scale_mode, ...)
  retain(ctx, {bt}, nullptr, nullptr, route, &p);  // every uniform solve entry (tzr_solve, tzr_solve_batch(_dev)) ends here
  return TZR_OK;
}

// Pipeline chunks of a (B, n) batch as n_chunks+1 ascending problem offsets.  The H2D copy of chunk k+1 overlaps the
// kernels of chunk k and the clique / rotation kernels of one chunk run under the graph kernel of the next: PCIe moves a
// problem ~3x faster than the kernels consume it, so only the first chunk's copy is exposed: it is kept small (B/32) and
// the later chunks grow (3B/32, B/8, then B/4 each) to keep launch tails few.
std::vector<int> chunk_bounds(int B, int n, const tzr_params& p) {
  std::vector<int> bounds{0};
  if (n > kMaxN) {  // one such problem fills the GPU (a 512 MiB bitset at n = 65536): one per chunk
    for (int b = 1; b <= B; ++b) bounds.push_back(b);
  } else if (B >= 64 && !p.estimate_scaling) {
    const int unit = std::max(8, B / 32);
    const int sizes[3] = {unit, 3 * unit, 4 * unit};
    for (int k = 0; bounds.back() < B; ++k) {
      const int sz = k < 3 ? sizes[k] : 8 * unit;
      bounds.push_back(std::min(B, bounds.back() + sz));
    }
  } else {
    bounds.push_back(B);
  }
  return bounds;
}

// ---- ragged batches (DESIGN.md §4.2) -----------------------------------------------------------------------------
// Problems ordered by n (largest first) are cut into size classes; a class runs as one padded device batch of its
// largest n, each problem's own n in Batch::nb.  One entry per problem in class order:
struct RaggedSlot {
  double* src;             // the problem's padded slot (n_pad rows; rows past n are zero)
  double* dst;
  const tzr_solution* sol; // its record in the class
  const int32_t* clq;      // its sorted clique row
  long long flat;          // first row of the problem in the caller's flat arrays
  int n, n_pad, q, pad_;   // own size, class size, index in the caller's order
};

__global__ void __launch_bounds__(256) ragged_gather_kernel(const RaggedSlot* slots, const double* src,
                                                            const double* dst) {
  const RaggedSlot sl = slots[blockIdx.x];
  const long long own = 3LL * sl.n, all = 3LL * sl.n_pad;
  const double* s = src + 3 * sl.flat;
  const double* d = dst + 3 * sl.flat;
  for (long long i = threadIdx.x; i < all; i += blockDim.x) {
    sl.src[i] = i < own ? s[i] : 0.0;
    sl.dst[i] = i < own ? d[i] : 0.0;
  }
}

// solutions[q] and the clique row at cliques + flat (n entries, -1 past the clique)
__global__ void __launch_bounds__(256) ragged_scatter_kernel(const RaggedSlot* slots, tzr_solution* solutions,
                                                             int32_t* cliques) {
  const RaggedSlot sl = slots[blockIdx.x];
  static_assert(sizeof(tzr_solution) % 4 == 0, "tzr_solution is copied in 4-byte words");
  const uint32_t* from = reinterpret_cast<const uint32_t*>(sl.sol);
  uint32_t* to = reinterpret_cast<uint32_t*>(solutions + sl.q);
  for (int i = threadIdx.x; i < (int)(sizeof(tzr_solution) / 4); i += blockDim.x) to[i] = from[i];
  if (!cliques) return;
  const int m = max(0, min(sl.n, sl.sol->clique_size));
  for (int i = threadIdx.x; i < sl.n; i += blockDim.x) cliques[sl.flat + i] = i < m ? sl.clq[i] : -1;
}

// Size classes over `order` (problem indices by n, largest first): [lo[c], lo[c+1]).  A class starts at its largest n and
// takes the next problems while n >= n_class / r, so that its padded bitset is at most r^2 times theirs.  Two rules keep
// every problem on the path it takes alone: a problem above kMaxN (the large clique route) is a class of its own, and
// with estimate_scaling a class never mixes the two scale paths.  Debug flag 16777216 drops the ratio rule (one class
// wherever the two path rules allow).
std::vector<int> ragged_classes(const int32_t* n, const std::vector<int>& order, const tzr_params& p, uint32_t flags,
                                double r) {
  std::vector<int> lo;
  const int B = (int)order.size();
  for (int s = 0; s < B;) {
    lo.push_back(s);
    const int nc = n[order[s]];
    int e = s + 1;
    while (e < B && nc <= kMaxN) {
      const int m = n[order[e]];
      if (!(flags & 16777216u) && (double)m * r < (double)nc) break;
      if (p.estimate_scaling && scale_large(nc, flags) != scale_large(m, flags)) break;
      ++e;
    }
    s = e;
  }
  lo.push_back(B);
  return lo;
}

// Padding ratio r of the size classes (DESIGN.md §4.2).  TZR_RAGGED_RATIO overrides it for measurements.
double ragged_ratio() {
  const char* e = std::getenv("TZR_RAGGED_RATIO");
  const double r = e ? std::atof(e) : 0.0;
  return r >= 1.0 ? r : std::sqrt(2.0);
}

// A ragged batch on the device.  src/dst: the caller's flat arrays (problem b's n[b] rows of 3 doubles at row
// sum_{c<b} n[c]); solutions: B records in the caller's order; cliques (may be NULL): sum n int32 at the same row
// offsets.  All device pointers; asynchronous on ctx->stream except where a large-route class reads back its core sizes.
int solve_ragged_dev(tzr_ctx* ctx, const tzr_params& p, int B, const int32_t* n, const double* src, const double* dst,
                     tzr_solution* solutions, int32_t* cliques) {
  for (int b = 0; b < B; ++b)
    if (n[b] <= 0) return TZR_ERR_INVALID_ARG;
  std::vector<int> order(B);
  for (int b = 0; b < B; ++b) order[b] = b;
  std::stable_sort(order.begin(), order.end(), [&](int a, int c) { return n[a] > n[c]; });
  const std::vector<int> lo = ragged_classes(n, order, p, ctx->flags, ragged_ratio());
  const int C = (int)lo.size() - 1;
  std::vector<int> Bs(C), ns(C);
  for (int c = 0; c < C; ++c) {
    Bs[c] = lo[c + 1] - lo[c];
    ns[c] = n[order[lo[c]]];
  }
  std::vector<Batch> cls(C);
  int rc = setup_classes(ctx, C, Bs.data(), ns.data(), true, cls.data(), p.rotation_tim_graph == 1);
  if (rc) return rc;
  std::vector<long long> flat(B + 1, 0);
  for (int b = 0; b < B; ++b) flat[b + 1] = flat[b] + n[b];
  std::vector<int32_t> nb(B);
  std::vector<RaggedSlot> slots(B);
  for (int c = 0; c < C; ++c)
    for (int s = lo[c]; s < lo[c + 1]; ++s) {
      const int q = order[s];
      nb[s] = n[q];
      const Batch v = sub_batch(cls[c], s - lo[c], 1);
      RaggedSlot& sl = slots[s];
      sl.src = const_cast<double*>(v.src);
      sl.dst = const_cast<double*>(v.dst);
      sl.sol = v.sol;
      sl.clq = v.sorted_clq;
      sl.flat = flat[q];
      sl.n = n[q];
      sl.n_pad = ns[c];
      sl.q = q;
      sl.pad_ = 0;
    }
  const size_t o_nb = al256((size_t)B * sizeof(RaggedSlot));
  if ((rc = ensure(ctx, ctx->rg, o_nb + (size_t)B * sizeof(int32_t))) != TZR_OK) return rc;
  RaggedSlot* d_slots = (RaggedSlot*)ctx->rg.p;
  int32_t* d_nb = (int32_t*)((char*)ctx->rg.p + o_nb);
  cudaStream_t st = ctx->stream;
  CK(cudaMemcpyAsync(d_slots, slots.data(), (size_t)B * sizeof(RaggedSlot), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_nb, nb.data(), (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  ragged_gather_kernel<<<B, 256, 0, st>>>(d_slots, src, dst);
  ctx->launches += 1;
  // chunks: every class as a uniform batch of its size would be cut, its own n per problem unless all are equal
  std::vector<Batch> chunks;
  std::vector<int> bounds{0};
  bool lanes_ok = true;
  size_t sc_bytes = 0;
  for (int c = 0; c < C; ++c) {
    if (nb[lo[c + 1] - 1] != ns[c]) {
      cls[c].nb = d_nb + lo[c];
      cls[c].nb_host = nb.data() + lo[c];
    }
    const std::vector<int> cb = chunk_bounds(Bs[c], ns[c], p);
    lanes_ok &= l2_chunk(ctx, Bs[c], ns[c], p) >= Bs[c];
    for (size_t k = 0; k + 1 < cb.size(); ++k) {
      const int Bc = cb[k + 1] - cb[k];
      chunks.push_back(cb.size() > 2 ? sub_batch(cls[c], cb[k], Bc) : cls[c]);
      bounds.push_back(lo[c] + cb[k + 1]);
      if (p.estimate_scaling) {
        // sized here for every chunk at once: run_pipeline must not re-allocate it under an earlier chunk's kernels
        const size_t bytes = scale_scratch_bytes(Bc, ns[c], ctx->flags);
        if (!bytes) {
          ctx->last_error = "estimate_scaling: 2K end points exceed 2^31";
          return TZR_ERR_TOO_LARGE;
        }
        sc_bytes = std::max(sc_bytes, bytes);
      }
    }
  }
  if (sc_bytes && (rc = ensure(ctx, ctx->sc, sc_bytes)) != TZR_OK) return rc;
  std::vector<int32_t> route;
  rc = run_chunks(ctx, chunks, bounds, p, nullptr, nullptr, lanes_ok, route);
  if (rc) return rc;
  ragged_scatter_kernel<<<B, 256, 0, st>>>(d_slots, solutions, cliques);
  ctx->launches += 1;
  if ((rc = check_launch(ctx, "ragged gather / scatter")) != TZR_OK) return rc;
  retain(ctx, std::move(cls), order.data(), n, route, &p);
  return TZR_OK;
}

// tzr_compute_fpfh(_batch): B clouds staged back to back in one pinned area, one H2D copy, the batched launches, one
// D2H copy of [overflow flags | descriptors | normals], then the caller's buffers are filled from the pinned copy.
// normals_only (tzr_estimate_normals(_batch)): fpfh_out and fpfh_radius are not used, every normals_out[b] is required,
// the grid is planned with both radii equal to the normal radius, and no descriptor pass runs.
int fpfh_run(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts, double normal_radius,
             double fpfh_radius, float* const* fpfh_out, float* const* normals_out, int32_t* status,
             bool normals_only = false) {
  if (normals_only) {
    fpfh_out = nullptr;
    fpfh_radius = normal_radius;
  }
  if (!ctx || B < 1 || !n || !pts || !(normals_only ? normals_out != nullptr : fpfh_out != nullptr) ||
      !(normal_radius > 0) || !(fpfh_radius > 0))
    return TZR_ERR_INVALID_ARG;
  bool want_normals = false;
  for (int b = 0; b < B; ++b) {
    if (n[b] <= 0 || !pts[b] || (normals_only ? !normals_out[b] : !fpfh_out[b])) return TZR_ERR_INVALID_ARG;
    want_normals |= normals_out && normals_out[b];
  }
  std::vector<FpfhCloud> clouds((size_t)B);
  FpfhPlan plan;
  const int route = search_route(ctx->flags, kFlagFpfhBrute, kFlagFpfhGrid);
  if (fpfh_plan(B, n, normal_radius, fpfh_radius, route, clouds.data(), &plan) != TZR_OK) {
    ctx->last_error = "the batch's points do not fit 32-bit indices";
    return TZR_ERR_TOO_LARGE;
  }
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)plan.N;
  const size_t pb = N * 12, cb = (size_t)B * sizeof(FpfhCloud), ob = (size_t)B * 4, hb = normals_only ? 0 : N * 33 * 4,
               nb = N * 16;
  const size_t in_bytes = al256(pb) + cb, out_bytes = al256(ob) + al256(hb) + (want_normals ? nb : 0);
  int rc;
  if ((rc = ensure(ctx, ctx->m_in, in_bytes)) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->m_scratch, al256(hb) + plan.grid_bytes)) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->m_out, al256(ob) + al256(hb) + nb)) != TZR_OK) return rc;
  if ((rc = ensure_pinned(ctx, al256(in_bytes) + out_bytes)) != TZR_OK) return rc;
  char* h_in = (char*)ctx->h_pin;
  char* h_out = h_in + al256(in_bytes);
  std::vector<CopySpan> spans;
  for (int b = 0; b < B; ++b) spans.push_back(CopySpan{h_in + (size_t)clouds[b].lo * 12, pts[b], (size_t)n[b] * 12});
  spans.push_back(CopySpan{h_in + al256(pb), clouds.data(), cb});
  char* d_in = (char*)ctx->m_in.p;
  char* d_out = (char*)ctx->m_out.p;
  CK(stage_in(spans, h_in, d_in, al256(pb), in_bytes, B == 1, st));
  float* d_spfh = (float*)ctx->m_scratch.p;
  void* d_grid = plan.grid_bytes ? (void*)((char*)ctx->m_scratch.p + al256(hb)) : nullptr;
  int* d_overflow = (int*)d_out;
  float* d_fpfh = (float*)(d_out + al256(ob));
  float4* d_normals = (float4*)(d_out + al256(ob) + al256(hb));
  ctx->launches += launch_fpfh(plan, (const float*)d_in, (FpfhCloud*)(d_in + al256(pb)), normal_radius, fpfh_radius,
                               d_normals, normals_only ? nullptr : d_spfh, normals_only ? nullptr : d_fpfh, d_overflow,
                               d_grid, st);
  if ((rc = check_launch(ctx, "fpfh launch")) != TZR_OK) return rc;
  spans.clear();
  spans.push_back(CopySpan{h_out, h_out, ob});  // the overflow flags stay in the pinned area
  for (int b = 0; b < B; ++b) {
    const size_t lo = (size_t)clouds[b].lo;
    if (!normals_only)
      spans.push_back(CopySpan{fpfh_out[b], h_out + al256(ob) + lo * 33 * 4, (size_t)n[b] * 33 * 4});
    if (normals_out && normals_out[b])
      spans.push_back(CopySpan{normals_out[b], h_out + al256(ob) + al256(hb) + lo * 16, (size_t)n[b] * 16});
  }
  CK(stage_out(spans, h_out, d_out, out_bytes, B == 1, st));
  const int* overflow = (const int*)h_out;
  bool any_overflow = false;
  for (int b = 0; b < B; ++b) {
    if (status) status[b] = overflow[b] ? TZR_ERR_TOO_LARGE : TZR_OK;
    any_overflow |= overflow[b] != 0;
  }
  if (any_overflow) {
    ctx->last_error = "a point has more than 4096 neighbours inside a search radius";
    return TZR_ERR_TOO_LARGE;
  }
  return TZR_OK;
}

// tzr_estimate_color_gradients(_batch): the front end's buffers as fpfh_run's.  m_in: [points | cloud table | normals
// | colours], one H2D copy; m_scratch: the grid; m_out: the gradients, one D2H copy.
int gradients_run(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts, const float* const* normals,
                  const float* const* colors, double radius, double* const* grad_out, int32_t* status) {
  if (!ctx || B < 1 || !n || !pts || !normals || !colors || !grad_out || !(radius > 0) || !std::isfinite(radius))
    return TZR_ERR_INVALID_ARG;
  for (int b = 0; b < B; ++b)
    if (n[b] <= 0 || !pts[b] || !normals[b] || !colors[b] || !grad_out[b]) return TZR_ERR_INVALID_ARG;
  std::vector<FpfhCloud> clouds((size_t)B);
  FpfhPlan plan;
  const int route = search_route(ctx->flags, kFlagFpfhBrute, kFlagFpfhGrid);
  if (fpfh_plan(B, n, radius, radius, route, clouds.data(), &plan) != TZR_OK) {
    ctx->last_error = "the batch's points do not fit 32-bit indices";
    return TZR_ERR_TOO_LARGE;
  }
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)plan.N;
  const size_t o_cl = al256(N * 12), o_nrm = o_cl + al256((size_t)B * sizeof(FpfhCloud)), o_col = o_nrm + al256(N * 16);
  const size_t in_bytes = o_col + N * 12, out_bytes = N * 24;
  int rc;
  if ((rc = ensure(ctx, ctx->m_in, in_bytes)) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->m_scratch, plan.grid_bytes + 256)) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->m_out, out_bytes)) != TZR_OK) return rc;
  if ((rc = ensure_pinned(ctx, al256(in_bytes) + out_bytes)) != TZR_OK) return rc;
  char* h_in = (char*)ctx->h_pin;
  char* h_out = h_in + al256(in_bytes);
  std::vector<CopySpan> spans;
  for (int b = 0; b < B; ++b) {
    const size_t lo = (size_t)clouds[b].lo;
    spans.push_back(CopySpan{h_in + lo * 12, pts[b], (size_t)n[b] * 12});
    spans.push_back(CopySpan{h_in + o_nrm + lo * 16, normals[b], (size_t)n[b] * 16});
    spans.push_back(CopySpan{h_in + o_col + lo * 12, colors[b], (size_t)n[b] * 12});
  }
  memcpy(h_in + o_cl, clouds.data(), (size_t)B * sizeof(FpfhCloud));
  parallel_copy(spans);
  char* d_in = (char*)ctx->m_in.p;
  CK(cudaMemcpyAsync(d_in, h_in, in_bytes, cudaMemcpyHostToDevice, st));
  double* d_grad = (double*)ctx->m_out.p;
  ctx->launches += launch_color_gradients(plan, (const float*)d_in, (FpfhCloud*)(d_in + o_cl), radius,
                                          (const float4*)(d_in + o_nrm), (const float*)(d_in + o_col), d_grad,
                                          plan.grid_bytes ? ctx->m_scratch.p : nullptr, st);
  if ((rc = check_launch(ctx, "color gradient launch")) != TZR_OK) return rc;
  spans.clear();
  for (int b = 0; b < B; ++b)
    spans.push_back(CopySpan{grad_out[b], h_out + (size_t)clouds[b].lo * 24, (size_t)n[b] * 24});
  CK(stage_out(spans, h_out, (const char*)d_grad, out_bytes, false, st));
  for (int b = 0; b < B && status; ++b) status[b] = TZR_OK;
  return TZR_OK;
}

// tzr_match_correspondences(_batch): B pairs staged back to back in one pinned area with the pair table and the NN
// work list, one H2D copy, the batched launches, one D2H copy of [counts | global scales | pairs].
int match_run(tzr_ctx* ctx, int B, const int32_t* ns, const float* const* src_pts, const int32_t* nd,
              const float* const* dst_pts, const float* const* src_feat, const float* const* dst_feat, int dim,
              int use_absolute_scale, int use_crosscheck, int use_tuple_test, float tuple_scale,
              const uint64_t* seeds, int32_t* const* pairs, const int64_t* capacity, int64_t* n_pairs,
              float* global_scale) {
  if (!ctx || B < 1 || !ns || !nd || !src_pts || !dst_pts || !src_feat || !dst_feat || !seeds || !pairs ||
      !capacity || !n_pairs || dim < 1 || dim > kMatchMaxDim)
    return TZR_ERR_INVALID_ARG;
  for (int b = 0; b < B; ++b)
    if (!src_pts[b] || !dst_pts[b] || !src_feat[b] || !dst_feat[b] || !pairs[b] || ns[b] <= 0 || nd[b] <= 0 ||
        capacity[b] < 0)
      return TZR_ERR_INVALID_ARG;
  for (int b = 0; b < B; ++b)
    if ((long long)ns[b] + nd[b] > (1ll << 30)) return TZR_ERR_TOO_LARGE;
  std::vector<MatchPair> P;
  std::vector<NnWork> W;
  MatchPlan plan;
  if (match_plan(B, ns, nd, seeds, ctx->num_sms, &P, &W, &plan) != TZR_OK) {
    ctx->last_error = "the batch's points do not fit 32-bit indices";
    return TZR_ERR_TOO_LARGE;
  }
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t C = (size_t)plan.NS + plan.ND;
  const size_t psb = (size_t)plan.NS * 12, pdb = (size_t)plan.ND * 12, fsb = (size_t)plan.NS * dim * 4,
               fdb = (size_t)plan.ND * dim * 4, tb = P.size() * sizeof(MatchPair), wb = W.size() * sizeof(NnWork);
  const size_t o_dp = al256(psb), o_sf = o_dp + al256(pdb), o_df = o_sf + al256(fsb), o_t = o_df + al256(fdb),
               o_w = o_t + al256(tb), in_bytes = o_w + wb;
  const size_t o_g = (size_t)B * 4, o_pairs = al256((size_t)B * 8), out_bytes = o_pairs + C * 8;
  int rc;
  if ((rc = ensure(ctx, ctx->m_in, in_bytes)) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->m_scratch, match_scratch_bytes(plan))) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->m_out, out_bytes)) != TZR_OK) return rc;
  if ((rc = ensure_pinned(ctx, al256(in_bytes) + out_bytes)) != TZR_OK) return rc;
  char* h_in = (char*)ctx->h_pin;
  char* h_out = h_in + al256(in_bytes);
  std::vector<CopySpan> spans;
  for (int b = 0; b < B; ++b) {
    const size_t so = (size_t)P[b].s_off, dof = (size_t)P[b].d_off;
    spans.push_back(CopySpan{h_in + so * 12, src_pts[b], (size_t)ns[b] * 12});
    spans.push_back(CopySpan{h_in + o_dp + dof * 12, dst_pts[b], (size_t)nd[b] * 12});
    spans.push_back(CopySpan{h_in + o_sf + so * dim * 4, src_feat[b], (size_t)ns[b] * dim * 4});
    spans.push_back(CopySpan{h_in + o_df + dof * dim * 4, dst_feat[b], (size_t)nd[b] * dim * 4});
  }
  spans.push_back(CopySpan{h_in + o_t, P.data(), tb});
  spans.push_back(CopySpan{h_in + o_w, W.data(), wb});
  char* d_in = (char*)ctx->m_in.p;
  char* d_out = (char*)ctx->m_out.p;
  CK(stage_in(spans, h_in, d_in, o_t, in_bytes, B == 1, st));
  const int nl = launch_match(plan, (const MatchPair*)(d_in + o_t), (const NnWork*)(d_in + o_w), (int)W.size(),
                              (float*)d_in, (float*)(d_in + o_dp), (const float*)(d_in + o_sf),
                              (const float*)(d_in + o_df), dim, use_absolute_scale, use_crosscheck, use_tuple_test,
                              tuple_scale, ctx->m_scratch.p, (int32_t*)(d_out + o_pairs), (int*)d_out,
                              (float*)(d_out + o_g), ctx->num_sms, st);
  ctx->launches += nl;
  if ((rc = check_launch(ctx, "matcher launch")) != TZR_OK) return rc;
  struct {
    int count;
    float g;
  } one;
  if (B == 1) {  // one pair: its count and scale, then only the rows it has, straight into the caller's buffer
    CK(cudaMemcpyAsync(&one, d_out, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (one.count > 0 && (int64_t)one.count <= capacity[0]) {
      CK(cudaMemcpyAsync(pairs[0], d_out + o_pairs, (size_t)one.count * 8, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
    }
  } else {
    CK(cudaMemcpyAsync(h_out, d_out, out_bytes, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  const int* counts = B == 1 ? &one.count : (const int*)h_out;
  const float* g = B == 1 ? &one.g : (const float*)(h_out + o_g);
  spans.clear();
  bool too_small = false;
  for (int b = 0; b < B; ++b) {
    n_pairs[b] = counts[b];
    if (global_scale) global_scale[b] = g[b];
    if ((int64_t)counts[b] > capacity[b]) {
      too_small = true;
      continue;
    }
    const size_t slot = (size_t)P[b].s_off + P[b].d_off;
    if (B > 1) spans.push_back(CopySpan{pairs[b], h_out + o_pairs + slot * 8, (size_t)counts[b] * 8});
  }
  parallel_copy(spans);
  if (too_small) {
    ctx->last_error = "pairs capacity too small";
    return TZR_ERR_INVALID_ARG;
  }
  return TZR_OK;
}

}  // namespace

// ================================================================================================
extern "C" {

int tzr_abi_version(void) { return TZR_ABI_VERSION; }

const char* tzr_status_string(int s) {
  switch (s) {
    case TZR_OK: return "ok";
    case TZR_ERR_INVALID_ARG: return "invalid argument";
    case TZR_ERR_NO_DEVICE: return "no usable CUDA device (the GPU path has no CPU fallback)";
    case TZR_ERR_CUDA: return "CUDA error";
    case TZR_ERR_ALLOC: return "allocation failed";
    case TZR_ERR_UNSUPPORTED: return "unsupported parameter combination";
    case TZR_ERR_TOO_LARGE: return "problem too large";
    default: return "unknown";
  }
}

const char* tzr_last_error(const tzr_ctx* ctx) { return ctx ? ctx->last_error.c_str() : ""; }

void tzr_params_default(tzr_params* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->noise_bound = 0.01;
  p->cbar2 = 1;
  p->estimate_scaling = 1;
  p->rotation_estimation_algorithm = 0;
  p->rotation_gnc_factor = 1.4;
  p->rotation_max_iterations = 100;
  p->rotation_cost_threshold = 1e-6;
  p->rotation_tim_graph = 0;
  p->inlier_selection_mode = 0;
  p->kcore_heuristic_threshold = 0.5;
  p->use_max_clique = 1;
  p->max_clique_exact_solution = 1;
  p->max_clique_time_limit = 3600;
  p->max_clique_num_threads = 0;
}

int tzr_words_per_row(int n) { return words64(n); }

int tzr_ctx_create(int device, tzr_ctx** out) {
  if (!out) return TZR_ERR_INVALID_ARG;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) return TZR_ERR_NO_DEVICE;
  if (device < 0) {
    if (cudaGetDevice(&device) != cudaSuccess) return TZR_ERR_NO_DEVICE;
  }
  if (device >= count) return TZR_ERR_INVALID_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return TZR_ERR_NO_DEVICE;
  tzr_ctx* ctx = new tzr_ctx();
  ctx->device = device;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ctx->num_sms = prop.multiProcessorCount;
  if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete ctx;
    return TZR_ERR_CUDA;
  }
  for (int i = 0; i < 5; ++i) cudaEventCreate(&ctx->ev[i]);
  cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking);
  {
    int least = 0, greatest = 0;
    cudaDeviceGetStreamPriorityRange(&least, &greatest);
    cudaStreamCreateWithPriority(&ctx->gstream, cudaStreamNonBlocking, least);
    cudaStreamCreateWithPriority(&ctx->hstream, cudaStreamNonBlocking, greatest);
  }
  cudaEventCreateWithFlags(&ctx->join_ev, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&ctx->join_ev2, cudaEventDisableTiming);
  *out = ctx;
  return TZR_OK;
}

int tzr_ctx_destroy(tzr_ctx* ctx) {
  if (!ctx) return TZR_OK;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->h_pin) cudaFreeHost(ctx->h_pin);
  for (int i = 0; i < 5; ++i)
    if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
  for (cudaEvent_t e : ctx->chunk_ev) cudaEventDestroy(e);
  for (cudaEvent_t e : ctx->stage_ev) cudaEventDestroy(e);
  for (cudaEvent_t e : ctx->graph_ev) cudaEventDestroy(e);
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  certify_release(ctx->solver_handle);
  if (ctx->gstream) cudaStreamDestroy(ctx->gstream);
  if (ctx->hstream) cudaStreamDestroy(ctx->hstream);
  if (ctx->join_ev) cudaEventDestroy(ctx->join_ev);
  if (ctx->join_ev2) cudaEventDestroy(ctx->join_ev2);
  for (cudaEvent_t e : ctx->gdone_ev) cudaEventDestroy(e);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
  return TZR_OK;
}

int tzr_ctx_set_stream(tzr_ctx* ctx, void* s) {
  if (!ctx) return TZR_ERR_INVALID_ARG;
  cudaStreamSynchronize(ctx->stream);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  ctx->stream = (cudaStream_t)s;
  ctx->own_stream = false;
  return TZR_OK;
}

int tzr_ctx_synchronize(tzr_ctx* ctx) {
  if (!ctx) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  CK(cudaStreamSynchronize(ctx->stream));
  return TZR_OK;
}

int64_t tzr_ctx_kernel_launches(const tzr_ctx* ctx) { return ctx ? ctx->launches : 0; }

int tzr_ctx_set_flags(tzr_ctx* ctx, uint32_t flags) {
  if (!ctx) return TZR_ERR_INVALID_ARG;
  ctx->flags = flags;
  return TZR_OK;
}

int64_t tzr_ctx_filter_mismatches(tzr_ctx* ctx) {
  if (!ctx || !ctx->dbg.p) return -1;
  unsigned long long v = 0;
  cudaStreamSynchronize(ctx->stream);
  if (cudaMemcpy(&v, ctx->dbg.p, sizeof(v), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  return (int64_t)v;
}

int tzr_ctx_debug_counters(tzr_ctx* ctx, int64_t* out16) {
  if (!ctx || !ctx->dbg.p || !out16) return TZR_ERR_INVALID_ARG;
  cudaStreamSynchronize(ctx->stream);
  if (cudaMemcpy(out16, ctx->dbg.p, 16 * sizeof(int64_t), cudaMemcpyDeviceToHost) != cudaSuccess) return TZR_ERR_CUDA;
  return TZR_OK;
}

int tzr_ctx_last_strip_blocks(const tzr_ctx* ctx) { return ctx ? ctx->last_strip_blocks : 0; }

int tzr_graph_strip_schedule(int nt, int L, int32_t* I, int32_t* J0) {
  if (nt < 1 || nt > kMaxNLarge / kTile || L < 1 || L > 15) return TZR_ERR_INVALID_ARG;
  return strip_schedule(nt, L, I, J0);
}

int64_t tzr_ctx_filter_rechecks(tzr_ctx* ctx) {
  if (!ctx || !ctx->dbg.p) return -1;
  unsigned long long v = 0;
  cudaStreamSynchronize(ctx->stream);
  if (cudaMemcpy(&v, (unsigned long long*)ctx->dbg.p + 1, sizeof(v), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  return (int64_t)v;
}

// ------------------------------------------------------------------------------------------------
// stage 1
// ------------------------------------------------------------------------------------------------
int tzr_graph_build(tzr_ctx* ctx, const double* src, const double* dst, int n, double beta, uint64_t* adj_bits,
                    int32_t* degree, int64_t* n_edges) {
  if (!ctx || !src || !dst || !adj_bits || n <= 0) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  Batch bt;
  int rc = setup_batch(ctx, 1, n, true, &bt);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  bt.beta = beta;
  CK(cudaMemcpyAsync((void*)bt.src, src, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync((void*)bt.dst, dst, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
  if (ctx->flags & 6u) cudaMemsetAsync((void*)ctx->dbg.p, 0, 16 * sizeof(unsigned long long), st);
  launch_prep(bt, st);
  ctx->launches += 2 + launch_graph(bt, st, ctx->num_sms, &ctx->last_strip_blocks);
  launch_degree(bt, st);
  rc = check_launch(ctx, "graph build");
  if (rc) return rc;
  CK(cudaMemcpy2DAsync(adj_bits, (size_t)words64(n) * 8, bt.adj, (size_t)pitch64(n) * 8, (size_t)words64(n) * 8, n,
                       cudaMemcpyDeviceToHost, st));
  if (degree) CK(cudaMemcpyAsync(degree, bt.deg, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  unsigned long long e2 = 0;
  CK(cudaMemcpyAsync(&e2, bt.n_edges2, sizeof(e2), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (n_edges) *n_edges = (int64_t)(e2 / 2);
  retain(ctx, {bt}, nullptr, nullptr, {}, nullptr);
  return TZR_OK;
}

// ------------------------------------------------------------------------------------------------
// stage 2
// ------------------------------------------------------------------------------------------------
int tzr_max_clique_batch(tzr_ctx* ctx, int B, int n, const uint64_t* adj_bits, int mode, double kcore_thr,
                         double time_limit_s, int32_t* cliques, int32_t* clique_sizes, int32_t* proven_optimal,
                         int32_t* search_flags) {
  if (!ctx || !adj_bits || !cliques || !clique_sizes || B <= 0 || n <= 0) return TZR_ERR_INVALID_ARG;
  if (mode < 0 || mode > 2) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  Batch bt;
  int rc = setup_batch(ctx, B, n, false, &bt);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  const size_t rows = (size_t)B * n;
  CK(cudaMemsetAsync(bt.adj, 0, rows * pitch64(n) * 8, st));
  CK(cudaMemcpy2DAsync(bt.adj, (size_t)pitch64(n) * 8, adj_bits, (size_t)words64(n) * 8, (size_t)words64(n) * 8, rows,
                       cudaMemcpyHostToDevice, st));
  sanitize_adj_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>(bt.adj, B, n);
  CK(cudaMemsetAsync(bt.n_edges2, 0, (size_t)B * sizeof(unsigned long long), st));
  launch_degree(bt, st, true);
  tzr_params p;
  tzr_params_default(&p);
  p.kcore_heuristic_threshold = kcore_thr;
  if (mode == 0 && time_limit_s > 0 && time_limit_s < 1e7) bt.budget_ns = (unsigned long long)(time_limit_s * 1e9);
  int nl = 2;
  std::vector<int32_t> route((size_t)B, 0);
  rc = run_clique(ctx, bt, p, mode, st, &nl, route.data());
  ctx->launches += nl;
  if (rc) return rc;
  rc = check_launch(ctx, "max clique");
  if (rc) return rc;
  ctx->clique = bt;
  ctx->last.route = std::move(route);  // no solve is retained, but the routes are readable
  std::vector<int32_t> L(B), fl(B);
  CK(cudaMemcpyAsync(L.data(), bt.L, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(fl.data(), bt.flags, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(cliques, bt.clq, rows * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  for (int b = 0; b < B; ++b) {
    int32_t* c = cliques + (size_t)b * n;
    std::sort(c, c + L[b]);  // registration.cc:636
    std::fill(c + L[b], c + n, -1);
    clique_sizes[b] = L[b];
    if (proven_optimal)  // as tzr_solution
      proven_optimal[b] = (mode == 0 && !(fl[b] & 1)) ? ((fl[b] & 12) ? 2 : 1) : 0;
    if (search_flags) search_flags[b] = fl[b];
  }
  return TZR_OK;
}

int tzr_max_clique(tzr_ctx* ctx, const uint64_t* adj_bits, int n, int mode, double kcore_thr, double time_limit_s,
                   int32_t* clique, int32_t* clique_size, int32_t* proven_optimal) {
  return tzr_max_clique_batch(ctx, 1, n, adj_bits, mode, kcore_thr, time_limit_s, clique, clique_size, proven_optimal,
                              nullptr);
}

int tzr_ctx_clique_info(tzr_ctx* ctx, int32_t* geometry3, int32_t* heuristic_best) {
  if (!ctx || !geometry3 || ctx->clique.B <= 0) return TZR_ERR_INVALID_ARG;
  const Batch& bt = ctx->clique;
  geometry3[0] = bt.exact_ctas;
  geometry3[1] = bt.exact_conc;
  geometry3[2] = bt.max_depth;
  if (heuristic_best) {
    cudaSetDevice(ctx->device);
    std::vector<int32_t> hs((size_t)bt.B * kHeurRoots);
    CK(cudaMemcpyAsync(hs.data(), bt.hsize, hs.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int b = 0; b < bt.B; ++b)
      heuristic_best[b] = *std::max_element(hs.begin() + (size_t)b * kHeurRoots, hs.begin() + (size_t)(b + 1) * kHeurRoots);
  }
  return TZR_OK;
}

int tzr_ctx_set_max_n(tzr_ctx* ctx, int max_n) {
  if (!ctx || max_n < kMaxN || max_n > kMaxNLarge) return TZR_ERR_INVALID_ARG;
  ctx->max_n = max_n;
  return TZR_OK;
}

int tzr_ctx_clique_route(tzr_ctx* ctx, int32_t* per_problem) {
  if (!ctx || !per_problem || ctx->last.route.empty()) return TZR_ERR_INVALID_ARG;
  std::copy(ctx->last.route.begin(), ctx->last.route.end(), per_problem);
  return TZR_OK;
}

// ------------------------------------------------------------------------------------------------
// stage 3 / 4 / scalar TLS
// ------------------------------------------------------------------------------------------------
int tzr_gnc_tls_rotation(tzr_ctx* ctx, const double* src, const double* dst, int m, double noise_bound,
                         double gnc_factor, uint64_t max_iterations, double cost_threshold, double* R,
                         uint8_t* inlier_mask, double* cost, int32_t* iterations) {
  return tzr_rotation_solve(ctx, 0, src, dst, m, noise_bound, gnc_factor, max_iterations, cost_threshold, R,
                            inlier_mask, cost, iterations);
}

int tzr_rotation_solve(tzr_ctx* ctx, int algorithm, const double* src, const double* dst, int m, double noise_bound,
                       double gnc_factor, uint64_t max_iterations, double cost_threshold, double* R,
                       uint8_t* inlier_mask, double* cost, int32_t* iterations) {
  if (!ctx || !src || !dst || !R || m <= 0 || algorithm < 0 || algorithm > 2) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t pts = (size_t)m * 3 * sizeof(double);
  int rc = ensure(ctx, ctx->misc, 2 * pts + 2 * (size_t)m * sizeof(double) + (size_t)m + 16 * sizeof(double) + 64);
  if (rc) return rc;
  char* base = (char*)ctx->misc.p;
  double* d_src = (double*)base;
  double* d_dst = d_src + (size_t)m * 3;
  double* d_w = d_dst + (size_t)m * 3;
  double* d_r = d_w + m;
  double* d_out = d_r + m;  // 9 R + 1 cost
  int* d_it = (int*)(d_out + 10);
  uint8_t* d_mask = (uint8_t*)(d_out + 12);
  CK(cudaMemcpyAsync(d_src, src, pts, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_dst, dst, pts, cudaMemcpyHostToDevice, st));
  launch_gnc_only(algorithm, d_src, d_dst, m, noise_bound, gnc_factor, max_iterations, cost_threshold, d_w, d_r, d_out, d_mask,
                  d_out + 9, d_it, st);
  ctx->launches += 1;
  rc = check_launch(ctx, "gnc");
  if (rc) return rc;
  double hout[10];
  int it = 0;
  CK(cudaMemcpyAsync(hout, d_out, sizeof(hout), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(&it, d_it, sizeof(int), cudaMemcpyDeviceToHost, st));
  if (inlier_mask) CK(cudaMemcpyAsync(inlier_mask, d_mask, m, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  memcpy(R, hout, 9 * sizeof(double));
  if (cost) *cost = hout[9];
  if (iterations) *iterations = it;
  return TZR_OK;
}

int tzr_tls_translation(tzr_ctx* ctx, const double* src, const double* dst, int m, double noise_bound, double cbar2,
                        double* t3, uint8_t* inlier_mask) {
  if (!ctx || !src || !dst || !t3 || m <= 0) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t pts = (size_t)m * 3 * sizeof(double);
  const size_t keys = (size_t)3 * next_pow2(2 * m);
  // layout: src[3m] dst[3m] raw[3m] key[keys] t[4] idx[keys] mask[m]
  const size_t bytes = 3 * pts + keys * sizeof(double) + 4 * sizeof(double) + keys * sizeof(int32_t) + (size_t)m;
  int rc = ensure(ctx, ctx->misc, bytes);
  if (rc) return rc;
  double* d_src = (double*)ctx->misc.p;
  double* d_dst = d_src + (size_t)m * 3;
  double* d_raw = d_dst + (size_t)m * 3;
  double* d_key = d_raw + (size_t)m * 3;
  double* d_t = d_key + keys;
  int32_t* d_idx = (int32_t*)(d_t + 4);
  uint8_t* d_mask = (uint8_t*)(d_idx + keys);
  CK(cudaMemcpyAsync(d_src, src, pts, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_dst, dst, pts, cudaMemcpyHostToDevice, st));
  const double beta = noise_bound * std::sqrt(cbar2);  // registration.cc:459
  launch_translation_only(d_src, d_dst, m, beta, d_key, d_idx, d_raw, d_t, d_mask, st);
  ctx->launches += 1;
  rc = check_launch(ctx, "translation");
  if (rc) return rc;
  CK(cudaMemcpyAsync(t3, d_t, 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (inlier_mask) CK(cudaMemcpyAsync(inlier_mask, d_mask, m, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return TZR_OK;
}

int tzr_scalar_tls(tzr_ctx* ctx, const double* x, const double* ranges, int64_t m, double* estimate,
                   uint8_t* inliers) {
  if (!ctx || !x || !ranges || !estimate || m <= 1) return TZR_ERR_INVALID_ARG;  // reference asserts m > 1
  if (m > ((int64_t)1 << 22)) return TZR_ERR_TOO_LARGE;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const bool large = (ctx->flags & 262144u) != 0;  // debug flag: the unknown-scale stage's large path
  // layout: sort scratch (at the allocation's 256-byte alignment), x[m] r[m] est[2] inliers[m]
  const size_t sort = (tls_scratch_bytes(m, 1, large) + 7) & ~(size_t)7;
  int rc = ensure(ctx, ctx->misc, sort + 2 * (size_t)m * 8 + 16 + (size_t)m);
  if (rc) return rc;
  void* d_sort = ctx->misc.p;
  double* d_x = (double*)((char*)d_sort + sort);
  double* d_r = d_x + m;
  double* d_est = d_r + m;
  uint8_t* d_inl = (uint8_t*)(d_est + 2);
  CK(cudaMemcpyAsync(d_x, x, (size_t)m * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_r, ranges, (size_t)m * 8, cudaMemcpyHostToDevice, st));
  ctx->launches += launch_scalar_tls(d_x, d_r, m, large, d_sort, d_est, d_inl, st);
  rc = check_launch(ctx, "scalar tls");
  if (rc) return rc;
  CK(cudaMemcpyAsync(estimate, d_est, sizeof(double), cudaMemcpyDeviceToHost, st));
  if (inliers) CK(cudaMemcpyAsync(inliers, d_inl, (size_t)m, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return TZR_OK;
}

// ------------------------------------------------------------------------------------------------
// whole path
// ------------------------------------------------------------------------------------------------
int tzr_solve_batch_dev(tzr_ctx* ctx, const tzr_params* params, int B, int n, const double* src_dev,
                        const double* dst_dev, tzr_solution* solutions_dev, int32_t* cliques_dev) {
  if (!ctx || !params || !src_dev || !dst_dev || !solutions_dev) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  Batch bt;
  int rc = setup_batch(ctx, B, n, false, &bt, params->rotation_tim_graph == 1);
  if (rc) return rc;
  bt.src = src_dev;
  bt.dst = dst_dev;
  // Sub-batches alternate between the two compute streams: the latency-bound clique / rotation kernels of one
  // sub-batch run under the issue-bound graph kernel of the next (TZR_DEV_CHUNKS overrides the count).
  static const int dev_chunks = [] {
    const char* e = std::getenv("TZR_DEV_CHUNKS");
    return e ? std::max(1, atoi(e)) : 1;
  }();
  std::vector<int> bounds{0};
  const int nch = (B >= 64 * dev_chunks && !params->estimate_scaling) ? dev_chunks : 1;
  for (int c = 1; c <= nch; ++c) bounds.push_back((int)((long long)B * c / nch));
  rc = run_chunked(ctx, bt, *params, bounds, nullptr);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  CK(cudaMemcpyAsync(solutions_dev, bt.sol, (size_t)B * sizeof(tzr_solution), cudaMemcpyDeviceToDevice, st));
  if (cliques_dev)
    CK(cudaMemcpyAsync(cliques_dev, bt.sorted_clq, (size_t)B * n * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  return TZR_OK;
}

static int solve_uniform_host(tzr_ctx* ctx, const tzr_params* params, int B, int n, const double* const* src,
                              const double* const* dst, tzr_solution* solutions, int32_t* cliques, int max_n,
                              uint8_t* rot_inliers, uint8_t* trans_inliers) {
  cudaSetDevice(ctx->device);
  Batch bt;
  int rc = setup_batch(ctx, B, n, true, &bt, params->rotation_tim_graph == 1);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  const size_t per = (size_t)n * 3 * sizeof(double);
  rc = ensure_pinned(ctx, 2 * per * B + (size_t)B * sizeof(tzr_solution) + (size_t)B * n * sizeof(int32_t));
  if (rc) return rc;
  char* hp = (char*)ctx->h_pin;
  double* h_src = (double*)hp;
  double* h_dst = (double*)(hp + per * B);
  tzr_solution* h_sol = (tzr_solution*)(hp + 2 * per * B);
  int32_t* h_clq = (int32_t*)(hp + 2 * per * B + (size_t)B * sizeof(tzr_solution));
  // Fast path: the caller's buffers are one contiguous, page-locked block (e.g. a pinned batch tensor) ->
  // DMA straight from user memory.  Otherwise stage through the context's pinned buffer.
  bool contiguous = true;
  for (int b = 1; b < B; ++b)
    contiguous &= (src[b] == src[0] + (size_t)b * n * 3) && (dst[b] == dst[0] + (size_t)b * n * 3);
  bool pinned = false;
  if (contiguous) {
    cudaPointerAttributes a1, a2;
    if (cudaPointerGetAttributes(&a1, src[0]) == cudaSuccess && cudaPointerGetAttributes(&a2, dst[0]) == cudaSuccess)
      pinned = (a1.type == cudaMemoryTypeHost) && (a2.type == cudaMemoryTypeHost);
    cudaGetLastError();
  }
  const double* hs = src[0];
  const double* hd = dst[0];
  const bool staged = !(contiguous && pinned);  // stage through the context's pinned buffer, chunk by chunk (below)
  if (staged) {
    hs = h_src;
    hd = h_dst;
  }
  // Chunked pipeline: the H2D copy of chunk k+1 (copy stream) overlaps the kernels of chunk k (compute streams).
  const std::vector<int> bounds = chunk_bounds(B, n, *params);
  const int n_chunks = (int)bounds.size() - 1;
  while ((int)ctx->chunk_ev.size() < n_chunks + 1) {
    cudaEvent_t e;
    CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    ctx->chunk_ev.push_back(e);
  }
  cudaStream_t cs = n_chunks > 1 ? ctx->copy_stream : st;
  if (n_chunks > 1) {
    // the copy stream must not overwrite inputs that an earlier call's kernels may still read
    CK(cudaEventRecord(ctx->chunk_ev[n_chunks], st));
    CK(cudaStreamWaitEvent(cs, ctx->chunk_ev[n_chunks], 0));
  }
  // Per chunk, on the host: (staged inputs only) copy the chunk into the pinned area with a few threads, then enqueue its
  // H2D copies; run_chunked enqueues the chunk's kernels right after, so the GPU works on chunk k while the host stages
  // chunk k+1.
  auto feed_chunk = [&](int c) -> int {
    const int b0 = bounds[c], Bc = bounds[c + 1] - b0;
    if (staged) {
      parallel_stage((char*)h_src + per * b0, src, b0, Bc, per);
      parallel_stage((char*)h_dst + per * b0, dst, b0, Bc, per);
    }
    if (cudaMemcpyAsync((void*)(bt.src + (size_t)b0 * n * 3), (const char*)hs + per * b0, per * Bc,
                        cudaMemcpyHostToDevice, cs) != cudaSuccess ||
        cudaMemcpyAsync((void*)(bt.dst + (size_t)b0 * n * 3), (const char*)hd + per * b0, per * Bc,
                        cudaMemcpyHostToDevice, cs) != cudaSuccess)
      return TZR_ERR_CUDA;
    if (n_chunks > 1 && cudaEventRecord(ctx->chunk_ev[c], cs) != cudaSuccess) return TZR_ERR_CUDA;
    return TZR_OK;
  };
  rc = run_chunked(ctx, bt, *params, bounds, n_chunks > 1 ? ctx->chunk_ev.data() : nullptr, feed_chunk);
  if (rc) return rc;
  CK(cudaMemcpyAsync(h_sol, bt.sol, (size_t)B * sizeof(tzr_solution), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (cliques) {  // only the used prefix of every clique row crosses PCIe (rows are n int32 wide, cliques ~5 % of n)
    int max_m = 0;
    for (int b = 0; b < B; ++b) max_m = std::max(max_m, std::min(n, std::max(0, h_sol[b].clique_size)));
    if (max_m > 0) {
      CK(cudaMemcpy2DAsync(h_clq, (size_t)n * sizeof(int32_t), bt.sorted_clq, (size_t)n * sizeof(int32_t),
                           (size_t)max_m * sizeof(int32_t), B, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
    }
  }
  memcpy(solutions, h_sol, (size_t)B * sizeof(tzr_solution));
  for (int b = 0; b < B; ++b)
    if (h_sol[b].clique_proven_optimal == -2) {
      ctx->last_error = "COMPLETE TIM graph of this clique does not fit the rotation workspace";
      return TZR_ERR_TOO_LARGE;
    }
  if (B == 1 && h_sol[0].valid) {  // single-problem masks (getRotationInliersMask / getTranslationInliersMask)
    const long long m = h_sol[0].clique_size;
    const long long n_rot = params->rotation_tim_graph == 1 ? m * (m - 1) / 2 : m;
    if (rot_inliers && n_rot > 0) CK(cudaMemcpy(rot_inliers, bt.rot_mask, (size_t)n_rot, cudaMemcpyDeviceToHost));
    if (trans_inliers && m > 0) CK(cudaMemcpy(trans_inliers, bt.trans_mask, (size_t)m, cudaMemcpyDeviceToHost));
  }
  if (cliques)
    for (int b = 0; b < B; ++b) {
      const int m = std::max(0, std::min(n, h_sol[b].clique_size));
      memcpy(cliques + (size_t)b * max_n, h_clq + (size_t)b * n, (size_t)m * sizeof(int32_t));
    }
  return TZR_OK;
}

int tzr_solve(tzr_ctx* ctx, const tzr_params* params, const double* src, const double* dst, int n,
              tzr_solution* solution, int32_t* clique, uint8_t* rot_inliers, uint8_t* trans_inliers) {
  if (!ctx || !params || !src || !dst || !solution || n <= 0) return TZR_ERR_INVALID_ARG;
  const double* s[1] = {src};
  const double* d[1] = {dst};
  int rc = solve_uniform_host(ctx, params, 1, n, s, d, solution, clique, n, rot_inliers, trans_inliers);
  if (rc) return rc;
  double st4[4] = {0, 0, 0, 0};
  if (tzr_last_stage_ms(ctx, &st4[0], &st4[1], &st4[2], &st4[3]) == TZR_OK) {
    for (int i = 0; i < 4; ++i) solution->stage_ms[i] = st4[i];  // prep | graph | clique | rot+trans
    solution->stage_ms[6] = st4[0] + st4[1] + st4[2] + st4[3];
  }
  return TZR_OK;
}

int tzr_solve_batch(tzr_ctx* ctx, const tzr_params* params, int B, const int32_t* n, const double* const* src,
                    const double* const* dst, tzr_solution* solutions, int32_t* cliques, int max_n) {
  if (!ctx || !params || !n || !src || !dst || !solutions || B <= 0) return TZR_ERR_INVALID_ARG;
  bool uniform = true;
  for (int b = 1; b < B; ++b) uniform &= (n[b] == n[0]);
  if (cliques && max_n < *std::max_element(n, n + B)) return TZR_ERR_INVALID_ARG;
  if (uniform) return solve_uniform_host(ctx, params, B, n[0], src, dst, solutions, cliques, max_n, nullptr, nullptr);
  // ragged batch: size classes (solve_ragged_dev) over the problems staged back to back, one read-back at the end
  long long N = 0;
  for (int b = 0; b < B; ++b) {
    if (n[b] <= 0 || !src[b] || !dst[b]) return TZR_ERR_INVALID_ARG;
    N += n[b];
  }
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t pts = (size_t)N * 3 * sizeof(double), o_clq = al256((size_t)B * sizeof(tzr_solution));
  const size_t out_bytes = o_clq + (size_t)N * sizeof(int32_t);
  int rc;
  if ((rc = ensure(ctx, ctx->m_in, 2 * al256(pts))) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->m_out, out_bytes)) != TZR_OK) return rc;
  if ((rc = ensure_pinned(ctx, std::max(2 * al256(pts), out_bytes))) != TZR_OK) return rc;
  char* h = (char*)ctx->h_pin;
  std::vector<CopySpan> spans;
  size_t at = 0;
  for (int b = 0; b < B; ++b) {
    const size_t bytes = (size_t)n[b] * 3 * sizeof(double);
    spans.push_back(CopySpan{h + at, src[b], bytes});
    spans.push_back(CopySpan{h + al256(pts) + at, dst[b], bytes});
    at += bytes;
  }
  parallel_copy(spans);
  char* d_in = (char*)ctx->m_in.p;
  char* d_out = (char*)ctx->m_out.p;
  CK(cudaMemcpyAsync(d_in, h, 2 * al256(pts), cudaMemcpyHostToDevice, st));
  rc = solve_ragged_dev(ctx, *params, B, n, (const double*)d_in, (const double*)(d_in + al256(pts)),
                        (tzr_solution*)d_out, cliques ? (int32_t*)(d_out + o_clq) : nullptr);
  if (rc) return rc;
  CK(cudaMemcpyAsync(h, d_out, cliques ? out_bytes : (size_t)B * sizeof(tzr_solution), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const tzr_solution* h_sol = (const tzr_solution*)h;
  memcpy(solutions, h_sol, (size_t)B * sizeof(tzr_solution));
  if (cliques) {
    spans.clear();
    const int32_t* h_clq = (const int32_t*)(h + o_clq);
    size_t row = 0;
    for (int b = 0; b < B; ++b) {
      const int m = std::max(0, std::min(n[b], h_sol[b].clique_size));
      spans.push_back(CopySpan{cliques + (size_t)b * max_n, h_clq + row, (size_t)m * sizeof(int32_t)});
      row += (size_t)n[b];
    }
    parallel_copy(spans);
  }
  for (int b = 0; b < B; ++b)
    if (h_sol[b].clique_proven_optimal == -2) {
      ctx->last_error = "COMPLETE TIM graph of this clique does not fit the rotation workspace";
      return TZR_ERR_TOO_LARGE;
    }
  return TZR_OK;
}

int tzr_solve_batch_ragged_dev(tzr_ctx* ctx, const tzr_params* params, int B, const int32_t* n, const double* src_dev,
                               const double* dst_dev, tzr_solution* solutions_dev, int32_t* cliques_dev) {
  if (!ctx || !params || !n || !src_dev || !dst_dev || !solutions_dev || B <= 0) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  return solve_ragged_dev(ctx, *params, B, n, src_dev, dst_dev, solutions_dev, cliques_dev);
}

int tzr_last_graph(tzr_ctx* ctx, int b, uint64_t* adj_bits, int32_t* degree) {
  if (!ctx || b < 0 || b >= (int)ctx->last.at.size()) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  // problem b's own n rows of its slot (padded to its class's n after a ragged solve)
  const int n = ctx->last.at[b].n;
  const Batch v = retained_problem(ctx, b);
  if (!ctx->last.has_graph) {  // inlier selection NONE: the reference never populates the graph -> no edges
    if (adj_bits) memset(adj_bits, 0, (size_t)n * words64(n) * 8);
    if (degree) memset(degree, 0, (size_t)n * 4);
    return TZR_OK;
  }
  cudaStream_t st = ctx->stream;
  if (adj_bits)
    CK(cudaMemcpy2DAsync(adj_bits, (size_t)words64(n) * 8, v.adj, (size_t)pitch64(v.n) * 8, (size_t)words64(n) * 8, n,
                         cudaMemcpyDeviceToHost, st));
  if (degree) CK(cudaMemcpyAsync(degree, v.deg, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return TZR_OK;
}

int tzr_last_graph_info(const tzr_ctx* ctx, int32_t* B, int32_t* n, int32_t* has_graph, uint64_t* generation) {
  if (!ctx) return TZR_ERR_INVALID_ARG;
  const Retained& r = ctx->last;
  if (B) *B = (int32_t)r.at.size();
  if (n) *n = r.cls.empty() ? 0 : r.cls[0].n;  // the largest n: the classes run largest first
  if (has_graph) *has_graph = (!r.at.empty() && r.has_graph) ? 1 : 0;
  if (generation) *generation = ctx->generation;
  return TZR_OK;
}

// rotation TIMs (and rotation mask bytes) of a retained solution record: 0 when it is not valid
static long long last_rot_count(const tzr_ctx* ctx, const tzr_solution& s) {
  if (!s.valid) return 0;
  const long long m = std::max(0, s.clique_size);
  return ctx->last.complete ? m * (m - 1) / 2 : m;
}

int tzr_last_inliers(tzr_ctx* ctx, int b, uint8_t* rot_inliers, uint8_t* trans_inliers, int64_t* n_rot,
                     int32_t* n_trans) {
  if (!ctx || !ctx->last.is_solve || b < 0 || b >= (int)ctx->last.at.size()) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  // every stream of the solve joins ctx->stream before its call returns: work queued here runs after all of it
  cudaStream_t st = ctx->stream;
  const Batch v = retained_problem(ctx, b);
  tzr_solution rec;
  CK(cudaMemcpyAsync(&rec, v.sol, sizeof(rec), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const long long nr = last_rot_count(ctx, rec);
  const int nt = rec.valid ? std::max(0, rec.clique_size) : 0;
  if (rot_inliers && nr > 0) CK(cudaMemcpyAsync(rot_inliers, v.rot_mask, (size_t)nr, cudaMemcpyDeviceToHost, st));
  if (trans_inliers && nt > 0) CK(cudaMemcpyAsync(trans_inliers, v.trans_mask, (size_t)nt, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (n_rot) *n_rot = nr;
  if (n_trans) *n_trans = nt;
  return TZR_OK;
}

int tzr_certify_last_solve(tzr_ctx* ctx, const tzr_certifier_params* params, int count, const int32_t* problems,
                           tzr_certification_result* results, int32_t* status, double* const* traj,
                           const int32_t* traj_capacity) {
  if (!ctx || !params || !results || count <= 0 || (traj && !traj_capacity)) return TZR_ERR_INVALID_ARG;
  if (!ctx->last.is_solve) {
    ctx->last_error = "no solve is retained on this context";
    return TZR_ERR_INVALID_ARG;
  }
  const int B = (int)ctx->last.at.size();
  if (!problems && count != B) return TZR_ERR_INVALID_ARG;
  for (int j = 0; j < count; ++j) {
    const int b = problems ? problems[j] : j;
    if (b < 0 || b >= B || (traj_capacity && traj_capacity[j] < 0)) return TZR_ERR_INVALID_ARG;
  }
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  // the B solution records: one read-back of the span of the workspace that holds them (the size classes of a ragged
  // solve lie back to back in one buffer)
  std::vector<const tzr_solution*> at((size_t)B);
  const char *lo = nullptr, *hi = nullptr;
  for (int b = 0; b < B; ++b) {
    at[b] = retained_problem(ctx, b).sol;
    const char* p = (const char*)at[b];
    if (!lo || p < lo) lo = p;
    if (!hi || p + sizeof(tzr_solution) > hi) hi = p + sizeof(tzr_solution);
  }
  std::vector<char> span((size_t)(hi - lo));
  CK(cudaMemcpyAsync(span.data(), lo, span.size(), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  // the certifiable entries: a valid record and 4N + 4 <= 32768 (non-finite measurements: flagged by the gather)
  std::vector<int32_t> N;
  std::vector<double> R;
  std::vector<CertGatherProb> gin;
  std::vector<int> which;
  std::vector<double*> tr;
  std::vector<int32_t> tc;
  bool too_large = false;
  for (int j = 0; j < count; ++j) {
    const int b = problems ? problems[j] : j;
    tzr_solution s;
    memcpy(&s, span.data() + ((const char*)at[b] - lo), sizeof(s));
    results[j].is_optimal = 0;
    results[j].n_iterations = 0;
    results[j].best_suboptimality = INFINITY;
    int stj = TZR_OK;
    const long long nr = last_rot_count(ctx, s);
    if (nr <= 0) {
      stj = TZR_ERR_INVALID_ARG;
    } else if (4 * nr + 4 > 32768) {
      stj = TZR_ERR_TOO_LARGE;
      too_large = true;
    } else {
      const Batch v = retained_problem(ctx, b);
      const double nb = params->noise_bound / s.scale;
      CertGatherProb g;
      g.src = v.src;
      g.dst = v.dst;
      g.clq = v.sorted_clq;
      g.rmask = v.rot_mask;
      g.scale = s.scale;
      g.nbs = params->cbar2 * nb * nb;
      g.m = s.clique_size;
      g.complete = ctx->last.complete ? 1 : 0;
      g.k_off = g.v_off = 0;
      gin.push_back(g);
      N.push_back((int32_t)nr);
      R.insert(R.end(), s.rotation, s.rotation + 9);
      which.push_back(j);
      tr.push_back(traj ? traj[j] : nullptr);
      tc.push_back(traj ? traj_capacity[j] : 0);
    }
    if (status) status[j] = stj;
  }
  if (!gin.empty()) {
    const int K = (int)gin.size();
    std::vector<tzr_certification_result> res((size_t)K);
    std::vector<int32_t> ok((size_t)K, 0);
    const int rc = certify_batch_device(CertMode::kCertify, *params, K, N.data(), R.data(), nullptr, nullptr, nullptr,
                                        gin.data(), ok.data(), res.data(), traj ? tr.data() : nullptr,
                                        traj ? tc.data() : nullptr, nullptr, nullptr, nullptr, nullptr,
                                        (ctx->flags & 2097152u) != 0, &ctx->certb.p, &ctx->certb.cap,
                                        &ctx->solver_handle, &ctx->launches, st, &ctx->last_error);
    if (rc != TZR_OK) return rc;
    for (int i = 0; i < K; ++i) {
      const int j = which[i];
      if (!ok[i]) {  // a non-finite gathered measurement: never certified
        if (status) status[j] = TZR_ERR_INVALID_ARG;
        continue;
      }
      results[j] = res[i];
    }
  }
  if (too_large) {
    ctx->last_error = "a problem's certifier matrix exceeds 32768 rows (4N + 4)";
    return TZR_ERR_TOO_LARGE;
  }
  return TZR_OK;
}

int tzr_match_correspondences(tzr_ctx* ctx, const float* src_pts, int ns, const float* dst_pts, int nd,
                              const float* src_feat, const float* dst_feat, int dim, int use_absolute_scale,
                              int use_crosscheck, int use_tuple_test, float tuple_scale, uint64_t tuple_seed,
                              int32_t* pairs, int64_t capacity, int64_t* n_pairs, float* global_scale) {
  const int32_t ns1 = ns, nd1 = nd;
  return match_run(ctx, 1, &ns1, &src_pts, &nd1, &dst_pts, &src_feat, &dst_feat, dim, use_absolute_scale,
                   use_crosscheck, use_tuple_test, tuple_scale, &tuple_seed, &pairs, &capacity, n_pairs, global_scale);
}

int tzr_match_correspondences_batch(tzr_ctx* ctx, int B, const int32_t* ns, const float* const* src_pts,
                                    const int32_t* nd, const float* const* dst_pts, const float* const* src_feat,
                                    const float* const* dst_feat, int dim, int use_absolute_scale, int use_crosscheck,
                                    int use_tuple_test, float tuple_scale, const uint64_t* tuple_seeds,
                                    int32_t* const* pairs, const int64_t* capacity, int64_t* n_pairs,
                                    float* global_scale) {
  return match_run(ctx, B, ns, src_pts, nd, dst_pts, src_feat, dst_feat, dim, use_absolute_scale, use_crosscheck,
                   use_tuple_test, tuple_scale, tuple_seeds, pairs, capacity, n_pairs, global_scale);
}

void tzr_certifier_params_default(tzr_certifier_params* p) {
  if (!p) return;
  p->noise_bound = 0.01;      // certification.h:74
  p->cbar2 = 1;               // :80
  p->sub_optimality = 1e-3;   // :87
  p->max_iterations = 2e2;    // :92
  p->gamma_tau = 1.999999;    // :98
  p->eig_decomposition_solver = 0;
  p->reserved = 0;
}

int tzr_certify(tzr_ctx* ctx, const tzr_certifier_params* params, const double* R_colmajor9, const double* src_3xN,
                const double* dst_3xN, const double* theta, int n, tzr_certification_result* result, double* traj,
                int traj_capacity) {
  if (!ctx || !params || !R_colmajor9 || !src_3xN || !dst_3xN || !theta || !result || n <= 0 || traj_capacity < 0)
    return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  const int32_t N = n, cap = traj_capacity;
  return certify_batch_device(CertMode::kCertify, *params, 1, &N, R_colmajor9, &src_3xN, &dst_3xN, &theta, nullptr,
                              nullptr, result, traj ? &traj : nullptr, &cap, nullptr, nullptr, nullptr, nullptr, false,
                              &ctx->certb.p, &ctx->certb.cap, &ctx->solver_handle, &ctx->launches, ctx->stream,
                              &ctx->last_error);
}

int tzr_certify_batch(tzr_ctx* ctx, const tzr_certifier_params* params, int B, const int32_t* N,
                      const double* R_colmajor9xB, const double* const* src_3xN, const double* const* dst_3xN,
                      const double* const* theta, tzr_certification_result* results, double* const* traj,
                      const int32_t* traj_capacity) {
  if (!ctx || !params || B <= 0 || !N || !R_colmajor9xB || !src_3xN || !dst_3xN || !theta || !results ||
      (traj && !traj_capacity))
    return TZR_ERR_INVALID_ARG;
  for (int b = 0; b < B; ++b)
    if (N[b] <= 0 || !src_3xN[b] || !dst_3xN[b] || !theta[b] || (traj_capacity && traj_capacity[b] < 0))
      return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  return certify_batch_device(CertMode::kCertify, *params, B, N, R_colmajor9xB, src_3xN, dst_3xN, theta, nullptr,
                              nullptr, results, traj, traj_capacity, nullptr, nullptr, nullptr, nullptr,
                              (ctx->flags & 2097152u) != 0, &ctx->certb.p, &ctx->certb.cap, &ctx->solver_handle,
                              &ctx->launches, ctx->stream, &ctx->last_error);
}

int tzr_certifier_initial_matrix(tzr_ctx* ctx, const tzr_certifier_params* params, const double* R_colmajor9,
                                 const double* src_3xN, const double* dst_3xN, const double* theta, int n,
                                 double* M_init, double* mu) {
  if (!ctx || !params || !R_colmajor9 || !src_3xN || !dst_3xN || !theta || !M_init || !mu || n <= 0)
    return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  const int32_t N = n;
  return certify_batch_device(CertMode::kSetup, *params, 1, &N, R_colmajor9, &src_3xN, &dst_3xN, &theta, nullptr,
                              nullptr, nullptr, nullptr, nullptr, nullptr, &M_init, nullptr, mu, false, &ctx->certb.p,
                              &ctx->certb.cap, &ctx->solver_handle, &ctx->launches, ctx->stream, &ctx->last_error);
}

// the building blocks (certify_batch_device's kPsd and kDual): B problems of N[b] >= 1 measurements; w (kPsd, may be
// NULL) as certify_batch_device's w_out
static int certifier_block(tzr_ctx* ctx, CertMode mode, int B, const int32_t* N, const double* const* X,
                           const double* const* theta, double* const* Y, double* const* w) {
  const bool dual = mode == CertMode::kDual;
  if (!ctx || B <= 0 || !N || !X || !Y || (dual && !theta)) return TZR_ERR_INVALID_ARG;
  for (int b = 0; b < B; ++b)
    if (N[b] <= 0 || !X[b] || !Y[b] || (dual && !theta[b])) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  tzr_certifier_params prm;
  tzr_certifier_params_default(&prm);
  return certify_batch_device(mode, prm, B, N, nullptr, nullptr, nullptr, theta, nullptr, nullptr, nullptr, nullptr,
                              nullptr, X, Y, w, nullptr, (ctx->flags & 2097152u) != 0, &ctx->certb.p, &ctx->certb.cap,
                              &ctx->solver_handle, &ctx->launches, ctx->stream, &ctx->last_error);
}

int tzr_certifier_dual_projection(tzr_ctx* ctx, const double* W, const double* theta, int n, double* W_dual) {
  const int32_t N = n;
  return certifier_block(ctx, CertMode::kDual, 1, &N, &W, &theta, &W_dual, nullptr);
}

int tzr_certifier_psd_projection(tzr_ctx* ctx, const double* M, int n, double* M_psd, double* w) {
  if (!w) return TZR_ERR_INVALID_ARG;
  const int32_t N = n;
  return certifier_block(ctx, CertMode::kPsd, 1, &N, &M, nullptr, &M_psd, &w);
}

int tzr_certifier_batch_psd_projection(tzr_ctx* ctx, int B, const int32_t* N, const double* const* M,
                                       double* const* M_psd) {
  return certifier_block(ctx, CertMode::kPsd, B, N, M, nullptr, M_psd, nullptr);
}

int tzr_certifier_batch_dual_projection(tzr_ctx* ctx, int B, const int32_t* N, const double* const* W,
                                        const double* const* theta, double* const* W_dual) {
  return certifier_block(ctx, CertMode::kDual, B, N, W, theta, W_dual, nullptr);
}

int tzr_compute_fpfh(tzr_ctx* ctx, const float* pts, int n, double normal_search_radius, double fpfh_search_radius,
                     float* fpfh_out, float* normals_out) {
  const int32_t n1 = n;
  return fpfh_run(ctx, 1, &n1, &pts, normal_search_radius, fpfh_search_radius, &fpfh_out, &normals_out, nullptr);
}

int tzr_compute_fpfh_batch(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts,
                           double normal_search_radius, double fpfh_search_radius, float* const* fpfh_out,
                           float* const* normals_out, int32_t* status) {
  return fpfh_run(ctx, B, n, pts, normal_search_radius, fpfh_search_radius, fpfh_out, normals_out, status);
}

int tzr_estimate_normals(tzr_ctx* ctx, const float* pts, int n, double normal_search_radius, float* normals_out) {
  const int32_t n1 = n;
  return fpfh_run(ctx, 1, &n1, &pts, normal_search_radius, 0.0, nullptr, &normals_out, nullptr, true);
}

int tzr_estimate_normals_batch(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts,
                               double normal_search_radius, float* const* normals_out, int32_t* status) {
  return fpfh_run(ctx, B, n, pts, normal_search_radius, 0.0, nullptr, normals_out, status, true);
}

int tzr_estimate_color_gradients(tzr_ctx* ctx, const float* pts, int n, const float* normals, const float* colors,
                                 double radius, double* grad_out) {
  const int32_t n1 = n;
  return gradients_run(ctx, 1, &n1, &pts, &normals, &colors, radius, &grad_out, nullptr);
}

int tzr_estimate_color_gradients_batch(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts,
                                       const float* const* normals, const float* const* colors, double radius,
                                       double* const* grad_out, int32_t* status) {
  return gradients_run(ctx, B, n, pts, normals, colors, radius, grad_out, status);
}

void tzr_frontend_params_default(tzr_frontend_params* p) {
  if (!p) return;
  p->normal_search_radius = 0.03;  // fpfh.h:39-41
  p->fpfh_search_radius = 0.05;
  p->use_absolute_scale = 1;       // matcher.h:39-43
  p->use_crosscheck = 1;
  p->use_tuple_test = 1;
  p->tuple_scale = 0.f;
}

static bool icp_params_ok(const tzr_icp_params* p) {
  return p && p->max_correspondence_distance > 0 && std::isfinite(p->max_correspondence_distance) &&
         p->max_iteration >= 0 && !std::isnan(p->relative_fitness) && !std::isnan(p->relative_rmse);
}

// generalized ICP's epsilon: finite and > 0
static bool icp_epsilon_ok(double epsilon) { return std::isfinite(epsilon) && epsilon > 0; }

// a transform that ICP or the information matrices start from: scale finite and > 0, R and t finite
static bool similarity_ok(const tzr_similarity& s) {
  bool ok = std::isfinite(s.scale) && s.scale > 0;
  for (int k = 0; k < 9; ++k) ok &= std::isfinite(s.rotation[k]) != 0;
  for (int k = 0; k < 3; ++k) ok &= std::isfinite(s.translation[k]) != 0;
  return ok;
}

// launch_icp's iteration settings (kernel: the robust kernel of the point-to-plane and generalized modes, NULL = L2)
static void icp_iteration_settings(IcpPlan* plan, const tzr_icp_params& p, int mode, double epsilon,
                                   const tzr_robust_kernel* kernel) {
  plan->max_iteration = p.max_iteration;
  plan->mode = mode;
  plan->epsilon = epsilon;
  if (kernel) {
    plan->loss = kernel->type;
    plan->loss_k = kernel->k;
  }
  plan->relative_fitness = p.relative_fitness;
  plan->relative_rmse = p.relative_rmse;
}

// a robust kernel (DESIGN.md §3.15): a known type, and k finite and > 0 where the weight reads it
static bool robust_kernel_ok(const tzr_robust_kernel* k) {
  if (!k) return false;
  switch (k->type) {
    case TZR_LOSS_L2:
    case TZR_LOSS_L1:
      return true;
    case TZR_LOSS_HUBER:
    case TZR_LOSS_CAUCHY:
    case TZR_LOSS_GM:
    case TZR_LOSS_TUKEY:
      return std::isfinite(k->k) && k->k > 0;
    default:
      return false;
  }
}

// ---- multiway registration: the robust pose graph (DESIGN.md §3.16) ----------------------------------------------------
static bool pg_params_ok(const tzr_pose_graph_params* p) {
  return p && std::isfinite(p->max_correspondence_distance) && p->max_correspondence_distance > 0 &&
         std::isfinite(p->gnc_factor) && p->gnc_factor > 1 && !std::isnan(p->cost_threshold) &&
         p->max_iterations >= 1 && p->max_inner_iterations >= 1;
}

// a rigid transform: finite, R^T R = I to 1e-6 in every entry, det R > 0 (the scale is not read)
static bool rigid_ok(const tzr_similarity& T) {
  const double* R = T.rotation;
  for (int k = 0; k < 9; ++k)
    if (!std::isfinite(R[k])) return false;
  for (int k = 0; k < 3; ++k)
    if (!std::isfinite(T.translation[k])) return false;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      const double d = (R[3 * a] * R[3 * b] + R[3 * a + 1] * R[3 * b + 1]) + R[3 * a + 2] * R[3 * b + 2];
      if (std::fabs(d - (a == b ? 1.0 : 0.0)) > 1e-6) return false;
    }
  const double det = R[0] * (R[4] * R[8] - R[7] * R[5]) - R[3] * (R[1] * R[8] - R[7] * R[2]) +
                     R[6] * (R[1] * R[5] - R[4] * R[2]);
  return det > 0;
}

// c = a b (column-major 3 x 3), entry (r, k) = (a(r,0) b(0,k) + a(r,1) b(1,k)) + a(r,2) b(2,k); y = a x likewise
static void h_m33(const double* a, const double* b, double* c) {
  for (int k = 0; k < 3; ++k)
    for (int r = 0; r < 3; ++r) c[3 * k + r] = (a[r] * b[3 * k] + a[3 + r] * b[3 * k + 1]) + a[6 + r] * b[3 * k + 2];
}
static void h_mv3(const double* a, const double* x, double* y) {
  for (int r = 0; r < 3; ++r) y[r] = (a[r] * x[0] + a[3 + r] * x[1]) + a[6 + r] * x[2];
}

// The breadth-first initial poses and the connectivity check (include/teaser_b200.h): false when some node is not
// reached from the reference node.  pose: K x 12 (R column-major, t); with `given` the poses are kept, only reached.
static bool pg_bfs(int K, int E, const int32_t* ends, const tzr_similarity* T, const std::vector<char>& live,
                   const int32_t* uncertain, int ref, bool given, std::vector<double>* pose) {
  std::vector<std::vector<int>> adj((size_t)K);
  for (int e = 0; e < E; ++e)
    if (live[e]) {
      adj[ends[2 * e]].push_back(e);
      adj[ends[2 * e + 1]].push_back(e);
    }
  std::vector<char> seen((size_t)K, 0);
  std::vector<int> order{ref};
  seen[ref] = 1;
  if (!given) {
    double* P = pose->data() + 12 * (size_t)ref;
    for (int k = 0; k < 12; ++k) P[k] = (k == 0 || k == 4 || k == 8) ? 1.0 : 0.0;
  }
  for (int phase = 0; phase < 2; ++phase) {
    std::vector<int> queue = order;
    for (size_t head = 0; head < queue.size(); ++head) {
      const int u = queue[head];
      for (int e : adj[u]) {
        if (phase == 0 && uncertain && uncertain[e]) continue;
        const int s = ends[2 * e], d = ends[2 * e + 1], v = u == s ? d : s;
        if (seen[v]) continue;
        seen[v] = 1;
        queue.push_back(v);
        order.push_back(v);
        if (given) continue;
        const double* Ru = pose->data() + 12 * (size_t)u;
        double* Pv = pose->data() + 12 * (size_t)v;
        const double* Rsd = T[e].rotation;
        const double* tsd = T[e].translation;
        if (u == d) {  // T_s = T_d T_sd
          double x[3];
          h_m33(Ru, Rsd, Pv);
          h_mv3(Ru, tsd, x);
          for (int r = 0; r < 3; ++r) Pv[9 + r] = x[r] + Ru[9 + r];
        } else {  // T_d = T_s T_sd^-1: R_d = R_s R_sd^T, t_d = t_s - R_d t_sd
          double Rt[9], x[3];
          for (int k = 0; k < 3; ++k)
            for (int r = 0; r < 3; ++r) Rt[3 * k + r] = Rsd[3 * r + k];
          h_m33(Ru, Rt, Pv);
          h_mv3(Pv, tsd, x);
          for (int r = 0; r < 3; ++r) Pv[9 + r] = Ru[9 + r] - x[r];
        }
      }
    }
  }
  return (int)order.size() == K;
}

static int pose_graph_run(tzr_ctx* ctx, const tzr_pose_graph_params* prm, int K, int E, const int32_t* ends,
                          const tzr_similarity* T, const double* info, const int32_t* uncertain,
                          const tzr_similarity* init, tzr_similarity* poses, double* weights, uint8_t* inlier_mask,
                          double* residuals, tzr_pose_graph_summary* summary) {
  if (!ctx || !pg_params_ok(prm) || K < 2 || E < 1 || !ends || !T || !info || !poses) {
    if (ctx) ctx->last_error = "pose graph: invalid arguments (K >= 2, E >= 1 and the parameters' ranges)";
    return TZR_ERR_INVALID_ARG;
  }
  if (K > 1024) {
    ctx->last_error = "pose graph: more than 1024 nodes";
    return TZR_ERR_TOO_LARGE;
  }
  const int ref = prm->reference_node;
  if (ref < 0 || ref >= K) {
    ctx->last_error = "pose graph: reference_node " + std::to_string(ref) + " is not a node";
    return TZR_ERR_INVALID_ARG;
  }
  std::vector<char> live((size_t)E);
  double info_sum = 0.0;
  for (int e = 0; e < E; ++e) {
    const int s = ends[2 * e], d = ends[2 * e + 1];
    if (s < 0 || s >= K || d < 0 || d >= K || !rigid_ok(T[e])) {
      ctx->last_error = "pose graph: edge " + std::to_string(e) + " has a node out of range or is not rigid";
      return TZR_ERR_INVALID_ARG;
    }
    for (int k = 0; k < 36; ++k)
      if (!std::isfinite(info[36 * (size_t)e + k])) {
        ctx->last_error = "pose graph: edge " + std::to_string(e) + " has a non-finite information entry";
        return TZR_ERR_INVALID_ARG;
      }
    const double l55 = info[36 * (size_t)e + 35];
    if (l55 < 0) {
      ctx->last_error = "pose graph: edge " + std::to_string(e) + " has Lambda(5,5) < 0";
      return TZR_ERR_INVALID_ARG;
    }
    live[e] = s != d && l55 > 0;
    info_sum += l55;
  }
  if (init)
    for (int k = 0; k < K; ++k)
      if (!rigid_ok(init[k])) {
        ctx->last_error = "pose graph: initial pose " + std::to_string(k) + " is not rigid and finite";
        return TZR_ERR_INVALID_ARG;
      }
  std::vector<double> pose((size_t)K * 12);
  if (init)
    for (int k = 0; k < K; ++k) {
      memcpy(&pose[12 * (size_t)k], init[k].rotation, 72);
      memcpy(&pose[12 * (size_t)k + 9], init[k].translation, 24);
    }
  if (!pg_bfs(K, E, ends, T, live, uncertain, ref, init != nullptr, &pose)) {
    ctx->last_error = "pose graph: the edges do not connect every node to the reference node";
    return TZR_ERR_INVALID_ARG;
  }
  const double c = prm->max_correspondence_distance;
  // edge table; the plan of H's lower blocks and of the right-hand side, each block's terms in ascending edge index
  std::vector<PgEdge> ed((size_t)E);
  std::map<std::pair<int, int>, std::vector<PgTerm>> plan_map;
  for (int e = 0; e < E; ++e) {
    PgEdge& x = ed[e];
    x = PgEdge{};
    x.s = ends[2 * e];
    x.d = ends[2 * e + 1];
    x.fs = x.s == ref ? -1 : x.s < ref ? x.s : x.s - 1;
    x.fd = x.d == ref ? -1 : x.d < ref ? x.d : x.d - 1;
    x.uncertain = uncertain && uncertain[e] ? 1 : 0;
    memcpy(x.R, T[e].rotation, 72);
    memcpy(x.t, T[e].translation, 24);
    const double l55 = info[36 * (size_t)e + 35];
    if (l55 > 0) {
      memcpy(x.L, info + 36 * (size_t)e, 36 * 8);
      x.inv_norm = 1.0 / ((c * c) * l55);
    }
    if (!live[e]) continue;
    if (x.fs >= 0) {
      plan_map[{x.fs, x.fs}].push_back(PgTerm{e, 1});
      plan_map[{x.fs, -1}].push_back(PgTerm{e, 1});
    }
    if (x.fd >= 0) {
      plan_map[{x.fd, x.fd}].push_back(PgTerm{e, 1});
      plan_map[{x.fd, -1}].push_back(PgTerm{e, -1});
    }
    if (x.fs >= 0 && x.fd >= 0) plan_map[{std::max(x.fs, x.fd), std::min(x.fs, x.fd)}].push_back(PgTerm{e, -1});
  }
  std::vector<PgBlock> blocks;
  std::vector<PgTerm> terms;
  for (const auto& kv : plan_map) {
    blocks.push_back(PgBlock{kv.first.first, kv.first.second, (int)terms.size(), 0});
    terms.insert(terms.end(), kv.second.begin(), kv.second.end());
    blocks.back().hi = (int)terms.size();
  }
  PgPlan plan;
  plan.K = K;
  plan.E = E;
  plan.n = 6 * (K - 1);
  plan.blocks = (int)blocks.size();
  plan.max_inner = prm->max_inner_iterations;
  plan.gnc_factor = prm->gnc_factor;
  plan.cost_threshold = prm->cost_threshold;
  const double cost_floor = 1e-24 * (c * c) * info_sum;
  const size_t n = (size_t)plan.n;
  // workspace: [edges | blocks | terms | poses (2 buffers) | weights | state] staged in one copy, then the edge terms,
  // H, g and the factorisation's workspace
  const size_t o_blk = al256((size_t)E * sizeof(PgEdge)), o_trm = o_blk + al256(blocks.size() * sizeof(PgBlock)),
               o_pose = o_trm + al256(terms.size() * sizeof(PgTerm)), o_w = o_pose + al256((size_t)K * 24 * 8),
               o_st = o_w + al256((size_t)E * 8), in_bytes = o_st + sizeof(PgState),
               o_term = al256(in_bytes), o_H = o_term + al256((size_t)E * 2 * kPgTermStride * 8),
               o_g = o_H + al256(n * n * 8), o_work = o_g + al256(n * 8);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  int rc;
  if ((rc = ensure(ctx, ctx->pg, o_work + 256)) != TZR_OK) return rc;
  int lwork = 0;
  if ((rc = dense_cholesky_setup(&ctx->solver_handle, (int)n, (double*)((char*)ctx->pg.p + o_H), &lwork, st,
                                 &ctx->last_error)) != TZR_OK)
    return rc;
  if ((rc = ensure(ctx, ctx->pg, o_work + (size_t)std::max(lwork, 1) * 8)) != TZR_OK) return rc;
  char* d = (char*)ctx->pg.p;
  std::vector<char> h(in_bytes, 0);
  memcpy(h.data(), ed.data(), (size_t)E * sizeof(PgEdge));
  memcpy(h.data() + o_blk, blocks.data(), blocks.size() * sizeof(PgBlock));
  memcpy(h.data() + o_trm, terms.data(), terms.size() * sizeof(PgTerm));
  memcpy(h.data() + o_pose, pose.data(), (size_t)K * 12 * 8);
  for (int e = 0; e < E; ++e) ((double*)(h.data() + o_w))[e] = 1.0;
  PgState s0{};
  s0.gnc_cost = INFINITY;
  memcpy(h.data() + o_st, &s0, sizeof(s0));
  CK(cudaMemcpyAsync(d, h.data(), in_bytes, cudaMemcpyHostToDevice, st));
  PgDev dv{(const PgEdge*)d, (const PgBlock*)(d + o_blk), (const PgTerm*)(d + o_trm), (double*)(d + o_pose),
           (double*)(d + o_term), (double*)(d + o_w), (double*)(d + o_H), (double*)(d + o_g), (PgState*)(d + o_st)};
  PgState hs{};
  int outer = 0;
  long long inner_total = 0;
  for (int it = 0; it < prm->max_iterations; ++it) {
    ctx->launches += launch_pose_graph_begin(plan, dv, cost_floor, st);
    for (int j = 0; j < plan.max_inner; ++j) {
      CK(cudaMemsetAsync(dv.H, 0, n * n * 8, st));
      ctx->launches += launch_pose_graph_assemble(plan, dv, st);
      if ((rc = dense_cholesky_solve(ctx->solver_handle, (int)n, dv.H, dv.g, (double*)(d + o_work), lwork,
                                     dv.state->info, &ctx->last_error)) != TZR_OK)
        return rc;
      ctx->launches += launch_pose_graph_step(plan, dv, ref, cost_floor, st);
    }
    ctx->launches += launch_pose_graph_gnc(plan, dv, it, st);
    if ((rc = check_launch(ctx, "pose graph launch")) != TZR_OK) return rc;
    // the one read-back of a GNC iteration
    CK(cudaMemcpyAsync(&hs, dv.state, sizeof(hs), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    outer = it + 1;
    inner_total += hs.inner;
    if (hs.stop) break;
  }
  std::vector<double> w((size_t)E), terms_out((size_t)E * kPgTermStride);
  CK(cudaMemcpyAsync(pose.data(), dv.poses + (size_t)hs.cur * K * 12, (size_t)K * 12 * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(w.data(), dv.weight, (size_t)E * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(terms_out.data(), dv.eterm + (size_t)hs.cur * E * kPgTermStride, (size_t)E * kPgTermStride * 8,
                     cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  for (int k = 0; k < K; ++k) {
    memset(&poses[k], 0, sizeof(tzr_similarity));
    poses[k].scale = 1.0;
    memcpy(poses[k].rotation, &pose[12 * (size_t)k], 72);
    memcpy(poses[k].translation, &pose[12 * (size_t)k + 9], 24);
  }
  for (int e = 0; e < E; ++e) {
    if (weights) weights[e] = w[e];
    if (inlier_mask) inlier_mask[e] = w[e] >= 0.5 ? 1 : 0;
    if (residuals) residuals[e] = terms_out[(size_t)e * kPgTermStride + 43];
  }
  if (summary) {
    summary->iterations = outer;
    summary->inner_iterations = (int32_t)inner_total;
    summary->cost = hs.cost;
  }
  return TZR_OK;
}

// what tzr_register_cloud_pairs_multiway adds to register_pairs_run (include/teaser_b200.h)
struct MultiwayOut {
  const int32_t* uncertain;
  const tzr_pose_graph_params* pg;
  double* information;
  int32_t* info_counts;
  double* edge_weights;
  uint8_t* edge_mask;
  tzr_similarity* poses;
  tzr_pose_graph_summary* summary;
  int32_t* pg_status;
};

static void icp_result_of(const IcpProb& pr, tzr_icp_result* out) {
  memset(out, 0, sizeof(*out));
  if (!pr.seeded) return;
  out->transform.scale = pr.s;
  for (int k = 0; k < 9; ++k) out->transform.rotation[k] = pr.R[k];
  for (int k = 0; k < 3; ++k) out->transform.translation[k] = pr.t[k];
  out->fitness = pr.fitness;
  out->inlier_rmse = pr.rmse;
  out->iterations = pr.iterations;
  out->n_correspondences = pr.count;
  out->converged = pr.converged;
}

// FPFH over the clouds, matching over the pairs, the ragged solve over the pairs that can be solved (DESIGN.md §3.10).
// Workspace: m_in holds the clouds and every table, m_scratch the FPFH scratch and then the matcher's, m_out the stages'
// outputs (descriptors alive while matching runs) and the solve's inputs and outputs.  All of it is sized before any work.
// icp (may be NULL): after the solve, ICP of every solved pair on its two clouds (already in m_in), seeded on the device
// from its record (ctx->icp holds the ICP workspace); icp_results (P entries) then receives the refinements, zeroed for a
// pair that was not refined.  Without icp the launches, synchronisations and outputs are tzr_register_cloud_pairs'.
// icp_kernel: the robust kernel of the point-to-plane, generalized and coloured modes (checked by the caller; NULL = L2).
// colors, lambda_geometric: the coloured mode's (n_clouds entries aligned with pts; lambda already checked and mapped
// into [0, 1] by the caller).
static int register_pairs_run(tzr_ctx* ctx, const tzr_frontend_params* fp, const tzr_params* params, int n_clouds,
                              const int32_t* n, const float* const* pts, int P, const int32_t* pair_clouds,
                              const uint64_t* tuple_seeds, tzr_solution* solutions, int32_t* status,
                              int32_t* problem_index, int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques,
                              float* global_scale, const tzr_icp_params* icp, tzr_icp_result* icp_results,
                              int icp_mode = kIcpPointToPoint, double icp_epsilon = 0,
                              const tzr_robust_kernel* icp_kernel = nullptr, const MultiwayOut* mw = nullptr,
                              const float* const* colors = nullptr, double lambda_geometric = 0) {
  const bool colored = icp && icp_mode == kIcpColored;
  if (!ctx || !fp || !params || n_clouds < 1 || !n || !pts || P < 1 || !pair_clouds || !solutions || !status ||
      !n_corr || !(fp->normal_search_radius > 0) || !(fp->fpfh_search_radius > 0))
    return TZR_ERR_INVALID_ARG;
  if (icp && (!icp_params_ok(icp) || !icp_results)) return TZR_ERR_INVALID_ARG;
  if (mw && (!icp || params->estimate_scaling || !mw->uncertain || !pg_params_ok(mw->pg) || !mw->information ||
             !mw->info_counts || !mw->edge_weights || !mw->edge_mask || !mw->poses || !mw->pg_status))
    return TZR_ERR_INVALID_ARG;
  if (icp && icp_mode == kIcpGeneralized && !icp_epsilon_ok(icp_epsilon)) return TZR_ERR_INVALID_ARG;
  if (colored && !colors) return TZR_ERR_INVALID_ARG;
  for (int c = 0; c < n_clouds; ++c)
    if (n[c] <= 0 || !pts[c] || (colored && !colors[c])) return TZR_ERR_INVALID_ARG;
  std::vector<int32_t> ns(P), nd(P);
  std::vector<uint64_t> seeds(P, 0);
  std::vector<int2> cloud_lo(P);
  for (int p = 0; p < P; ++p) {
    const int a = pair_clouds[2 * p], b = pair_clouds[2 * p + 1];
    if (a < 0 || a >= n_clouds || b < 0 || b >= n_clouds) return TZR_ERR_INVALID_ARG;
    ns[p] = n[a];
    nd[p] = n[b];
    if (tuple_seeds) seeds[p] = tuple_seeds[p];
  }
  std::vector<FpfhCloud> clouds((size_t)n_clouds);
  FpfhPlan fplan;
  std::vector<MatchPair> MP;
  std::vector<NnWork> W;
  MatchPlan mplan;
  const int route = search_route(ctx->flags, kFlagFpfhBrute, kFlagFpfhGrid);
  if (fpfh_plan(n_clouds, n, fp->normal_search_radius, fp->fpfh_search_radius, route, clouds.data(), &fplan) != TZR_OK ||
      match_plan(P, ns.data(), nd.data(), seeds.data(), ctx->num_sms, &MP, &W, &mplan) != TZR_OK) {
    ctx->last_error = "the batch's points do not fit 32-bit indices";
    return TZR_ERR_TOO_LARGE;
  }
  for (int p = 0; p < P; ++p) cloud_lo[p] = make_int2(clouds[pair_clouds[2 * p]].lo, clouds[pair_clouds[2 * p + 1]].lo);
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)fplan.N, NS = (size_t)mplan.NS, ND = (size_t)mplan.ND, C = NS + ND;
  // m_in: cloud points | FPFH cloud table | pair table | NN work list | cloud offsets per pair | (coloured mode: cloud
  // colours | gradient cloud table) | gather table; without colours the two regions are empty
  const size_t o_ct = al256(N * 12), o_mp = o_ct + al256((size_t)n_clouds * sizeof(FpfhCloud)),
               o_w = o_mp + al256((size_t)P * sizeof(MatchPair)), o_lo = o_w + al256(W.size() * sizeof(NnWork)),
               o_col = o_lo + al256((size_t)P * sizeof(int2)), o_gct = o_col + al256(colored ? N * 12 : 0),
               o_g = o_gct + al256(colored ? (size_t)n_clouds * sizeof(FpfhCloud) : 0),
               in_bytes = o_g + (size_t)P * sizeof(PairGather);
  // m_out: [overflow | counts | global scales] | descriptors | normals | matcher points and descriptors | matcher rows |
  // solve src | solve dst | records | compacted index pairs | cliques
  const size_t o_cnt = al256((size_t)n_clouds * 4), o_gs = o_cnt + (size_t)P * 4, head = o_gs + (size_t)P * 4;
  const size_t o_desc = al256(head), o_nrm = o_desc + al256(N * 33 * 4), o_msp = o_nrm + al256(N * 16),
               o_mdp = o_msp + al256(NS * 12), o_msf = o_mdp + al256(ND * 12), o_mdf = o_msf + al256(NS * 33 * 4),
               o_pairs = o_mdf + al256(ND * 33 * 4), o_src = o_pairs + al256(C * 8), o_dst = o_src + al256(C * 24),
               o_sol = o_dst + al256(C * 24), o_corr = o_sol + al256((size_t)P * sizeof(tzr_solution)),
               o_clq = o_corr + al256(C * 8), out_bytes = o_clq + C * 4;
  const size_t scratch_bytes = std::max(al256(N * 33 * 4) + fplan.grid_bytes, match_scratch_bytes(mplan));
  // pinned: staged inputs | read-back head | gather table | records | index pairs | cliques
  const size_t h_head = al256(o_g), h_g = h_head + al256(head), h_sol = h_g + al256((size_t)P * sizeof(PairGather)),
               h_corr = h_sol + al256((size_t)P * sizeof(tzr_solution)), h_clq = h_corr + al256(C * 8),
               pin_base = h_clq + C * 4;
  // with ICP: the refinement of every pair planned here, which sizes its tables and checks them before any work, and
  // planned again over the solved pairs once they are known (plan_icp: sources from a pair's first cloud, targets its
  // second).  Its workspace ctx->icp is laid out from 0 (icp_layout); the pinned area mirrors the layout's tables
  // ([problems | target clouds | chunks], staged in and the problem table read back) and, with the multiway step, holds
  // the [information | counts] of the refined pairs read back.
  // Coloured mode: the gradient pass (tzr_estimate_color_gradients_batch at 2 max_correspondence_distance, the FPFH
  // stage's route) spans every cloud, so it writes each cloud's gradients at its cloud-table rows, where the coloured
  // system reads them through buf.dst, and computes them once however many pairs target the cloud.  Its table does not
  // depend on which pairs are solved, so it is planned once, here, and staged with the clouds and their colours; the
  // layout's own slot for it in ctx->icp stays unused.
  IcpPlan iplan;
  std::vector<FpfhCloud> iclouds, gclouds;
  std::vector<IcpProb> iprobs;
  std::vector<int> ichunks;
  auto plan_icp = [&](const std::vector<int>& pairs) {
    std::vector<int32_t> i_ns, i_slo, i_tc;
    for (int p : pairs) {
      i_ns.push_back(n[pair_clouds[2 * p]]);
      i_slo.push_back(clouds[pair_clouds[2 * p]].lo);
      i_tc.push_back(pair_clouds[2 * p + 1]);
    }
    return icp_plan((int)pairs.size(), i_ns.data(), i_slo.data(), i_tc.data(), n_clouds, n,
                    icp->max_correspondence_distance, search_route(ctx->flags, kFlagIcpBrute, kFlagIcpGrid), nullptr,
                    &iplan, &iclouds, &iprobs, &ichunks);
  };
  IcpLayout il{};
  if (icp) {
    std::vector<int> every(P);
    for (int p = 0; p < P; ++p) every[p] = p;
    icp_iteration_settings(&iplan, *icp, icp_mode, icp_epsilon, icp_kernel);
    iplan.lambda_geometric = lambda_geometric;
    if (colored) {
      iplan.grad_r = 2.0 * icp->max_correspondence_distance;
      gclouds.resize((size_t)n_clouds);
      if (fpfh_plan(n_clouds, n, iplan.grad_r, iplan.grad_r, route, gclouds.data(), &iplan.ggrid) != TZR_OK) {
        ctx->last_error = "the clouds' gradient grid does not fit 32-bit indices";
        return TZR_ERR_TOO_LARGE;
      }
    }
    if (plan_icp(every) != TZR_OK) {
      ctx->last_error = "the refinement's points or target grid do not fit 32-bit indices";
      return TZR_ERR_TOO_LARGE;
    }
    il = icp_layout(iplan, 0, mw != nullptr);
  }
  const size_t hi_tab = al256(pin_base), hi_info = al256(hi_tab + il.match),
               hi_icnt = hi_info + al256((size_t)P * 36 * 8),
               pin_bytes = mw ? hi_icnt + (size_t)P * 4 : icp ? hi_tab + il.match : pin_base;
  int rc;
  if ((rc = ensure(ctx, ctx->m_in, in_bytes)) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->m_scratch, scratch_bytes)) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->m_out, out_bytes)) != TZR_OK) return rc;
  if ((rc = ensure_pinned(ctx, pin_bytes)) != TZR_OK) return rc;
  char* h = (char*)ctx->h_pin;
  char* d_in = (char*)ctx->m_in.p;
  char* d_out = (char*)ctx->m_out.p;
  std::vector<CopySpan> spans;
  for (int c = 0; c < n_clouds; ++c) spans.push_back(CopySpan{h + (size_t)clouds[c].lo * 12, pts[c], (size_t)n[c] * 12});
  spans.push_back(CopySpan{h + o_ct, clouds.data(), (size_t)n_clouds * sizeof(FpfhCloud)});
  spans.push_back(CopySpan{h + o_mp, MP.data(), (size_t)P * sizeof(MatchPair)});
  spans.push_back(CopySpan{h + o_w, W.data(), W.size() * sizeof(NnWork)});
  spans.push_back(CopySpan{h + o_lo, cloud_lo.data(), (size_t)P * sizeof(int2)});
  if (colored) {
    for (int c = 0; c < n_clouds; ++c)
      spans.push_back(CopySpan{h + o_col + (size_t)clouds[c].lo * 12, colors[c], (size_t)n[c] * 12});
    spans.push_back(CopySpan{h + o_gct, gclouds.data(), (size_t)n_clouds * sizeof(FpfhCloud)});
  }
  CK(stage_in(spans, h, d_in, o_ct, o_g, false, st));
  const float* d_pts = (const float*)d_in;
  const MatchPair* d_mp = (const MatchPair*)(d_in + o_mp);
  float* d_desc = (float*)(d_out + o_desc);
  ctx->launches += launch_fpfh(fplan, d_pts, (FpfhCloud*)(d_in + o_ct), fp->normal_search_radius,
                               fp->fpfh_search_radius, (float4*)(d_out + o_nrm), (float*)ctx->m_scratch.p, d_desc,
                               (int*)d_out, fplan.grid_bytes ? (char*)ctx->m_scratch.p + al256(N * 33 * 4) : nullptr, st);
  float* d_msp = (float*)(d_out + o_msp);
  float* d_mdp = (float*)(d_out + o_mdp);
  float* d_msf = (float*)(d_out + o_msf);
  float* d_mdf = (float*)(d_out + o_mdf);
  ctx->launches += launch_pair_rows(mplan, d_mp, (const int2*)(d_in + o_lo), d_pts, d_desc, d_msp, d_mdp, d_msf, d_mdf,
                                    ctx->num_sms, st);
  const int32_t* d_pairs = (const int32_t*)(d_out + o_pairs);
  ctx->launches += launch_match(mplan, d_mp, (const NnWork*)(d_in + o_w), (int)W.size(), d_msp, d_mdp, d_msf, d_mdf,
                                33, fp->use_absolute_scale, fp->use_crosscheck, fp->use_tuple_test, fp->tuple_scale,
                                ctx->m_scratch.p, (int32_t*)d_pairs, (int*)(d_out + o_cnt), (float*)(d_out + o_gs),
                                ctx->num_sms, st);
  if ((rc = check_launch(ctx, "front-end launch")) != TZR_OK) return rc;
  // synchronisation 1: which pairs go on, and their sizes (the solve's size classes are planned on the host)
  CK(cudaMemcpyAsync(h + h_head, d_out, head, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const int* overflow = (const int*)(h + h_head);
  const int* counts = (const int*)(h + h_head + o_cnt);
  const float* gs = (const float*)(h + h_head + o_gs);
  PairGather* table = (PairGather*)(h + h_g);
  std::vector<int32_t> solved_n;
  std::vector<int> solved;  // pair of every retained problem
  std::vector<long long> corr_row(P, -1);
  int n_table = 0, max_count = 0;
  long long corr_rows = 0, solve_rows = 0;
  bool too_large = false;
  for (int p = 0; p < P; ++p) {
    if (global_scale) global_scale[p] = gs[p];
    if (problem_index) problem_index[p] = -1;
    memset(&solutions[p], 0, sizeof(tzr_solution));
    if (overflow[pair_clouds[2 * p]] || overflow[pair_clouds[2 * p + 1]]) {
      status[p] = TZR_ERR_TOO_LARGE;
      n_corr[p] = 0;
      too_large = true;
      continue;
    }
    const int cnt = counts[p];
    n_corr[p] = cnt;
    if (cnt == 0) {
      status[p] = TZR_ERR_INVALID_ARG;
      continue;
    }
    const bool solve = cnt <= ctx->max_n && !(params->estimate_scaling && !scale_scratch_bytes(1, cnt, ctx->flags));
    status[p] = solve ? TZR_OK : TZR_ERR_TOO_LARGE;
    too_large |= !solve;
    const bool want_corr = corr && corr[p];
    if (!solve && !want_corr) continue;
    PairGather& g = table[n_table++];
    g.src_lo = cloud_lo[p].x;
    g.dst_lo = cloud_lo[p].y;
    g.slot = MP[p].s_off + MP[p].d_off;
    g.count = cnt;
    g.corr_row = want_corr ? corr_rows : -1;
    g.solve_row = solve ? solve_rows : -1;
    max_count = std::max(max_count, cnt);
    if (want_corr) {
      corr_row[p] = corr_rows;
      corr_rows += cnt;
    }
    if (solve) {
      if (problem_index) problem_index[p] = (int32_t)solved.size();
      solved.push_back(p);
      solved_n.push_back(cnt);
      solve_rows += cnt;
    }
  }
  double* d_src = (double*)(d_out + o_src);
  double* d_dst = (double*)(d_out + o_dst);
  int2* d_corr = (int2*)(d_out + o_corr);
  if (n_table > 0) {
    CK(cudaMemcpyAsync(d_in + o_g, table, (size_t)n_table * sizeof(PairGather), cudaMemcpyHostToDevice, st));
    ctx->launches += launch_corr_gather((const PairGather*)(d_in + o_g), n_table, max_count, d_pairs, d_pts, d_corr,
                                        d_src, d_dst, st);
    if ((rc = check_launch(ctx, "correspondence gather")) != TZR_OK) return rc;
  }
  const int S = (int)solved.size();
  bool want_clq = false;
  for (int k = 0; k < S && cliques; ++k) want_clq |= cliques[solved[k]] != nullptr;
  tzr_solution* d_sol = (tzr_solution*)(d_out + o_sol);
  int32_t* d_clq = (int32_t*)(d_out + o_clq);
  if (S > 0) {
    rc = solve_ragged_dev(ctx, *params, S, solved_n.data(), d_src, d_dst, d_sol, want_clq ? d_clq : nullptr);
    if (rc) return rc;
  } else {  // nothing solved: no solve is retained
    forget_retained(ctx);
  }
  // the refinement of the solved pairs, seeded on the device from their records (no synchronisation, no upload of points)
  char* hi = h + hi_tab;
  const IcpProb* hi_probs = (const IcpProb*)(hi + il.probs);
  if (icp && S > 0) {
    plan_icp(solved);  // a subset of the pairs planned above: it fits
    il = icp_layout(iplan, 0, mw != nullptr);
    if ((rc = ensure(ctx, ctx->icp, il.end)) != TZR_OK) return rc;
    memcpy(hi + il.probs, iprobs.data(), (size_t)S * sizeof(IcpProb));
    memcpy(hi + il.clouds, iclouds.data(), (size_t)n_clouds * sizeof(FpfhCloud));
    memcpy(hi + il.chunks, ichunks.data(), ichunks.size() * 4);
    char* di = (char*)ctx->icp.p;
    CK(cudaMemcpyAsync(di, hi, il.match, cudaMemcpyHostToDevice, st));
    IcpBuffers buf = icp_buffers(di, il);
    ctx->launches += launch_icp_seed(buf.probs, S, d_sol, st);
    // point-to-plane and generalized: the target (and source) normals are the FPFH stage's (normal_search_radius,
    // viewpoint at the origin), still in m_out: nothing after the FPFH stage writes that region, and they share the
    // cloud table's indexing
    buf.src = buf.dst = d_pts;
    buf.src_normals = buf.dst_normals = (const float4*)(d_out + o_nrm);
    if (colored) {  // the colours and the gradient table share the cloud table's indexing; launch_icp runs the pass
      buf.src_colors = buf.dst_colors = (const float*)(d_in + o_col);
      buf.gclouds = (FpfhCloud*)(d_in + o_gct);
    }
    IcpGrid grid{nullptr, nullptr, nullptr};
    ctx->launches += launch_icp(iplan, buf, st, &grid);
    if ((rc = check_launch(ctx, "icp launch")) != TZR_OK) return rc;
    CK(cudaMemcpyAsync(hi + il.probs, buf.probs, (size_t)S * sizeof(IcpProb), cudaMemcpyDeviceToHost, st));
    if (mw) {  // the information matrices at the refined transforms, from the clouds and the problem table in place
      ctx->launches += launch_icp_information(iplan, buf, true, st, &grid);
      if ((rc = check_launch(ctx, "information launch")) != TZR_OK) return rc;
      CK(cudaMemcpyAsync(h + hi_info, buf.info, (size_t)S * 36 * 8, cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(h + hi_icnt, buf.counts, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
    }
  }
  // synchronisation 2: the records, and the index pairs and cliques that were asked for
  if (S > 0) CK(cudaMemcpyAsync(h + h_sol, d_sol, (size_t)S * sizeof(tzr_solution), cudaMemcpyDeviceToHost, st));
  if (corr_rows > 0) CK(cudaMemcpyAsync(h + h_corr, d_corr, (size_t)corr_rows * 8, cudaMemcpyDeviceToHost, st));
  if (want_clq) CK(cudaMemcpyAsync(h + h_clq, d_clq, (size_t)solve_rows * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const tzr_solution* sol = (const tzr_solution*)(h + h_sol);
  spans.clear();
  for (int p = 0; p < P; ++p)
    if (corr_row[p] >= 0) spans.push_back(CopySpan{corr[p], h + h_corr + (size_t)corr_row[p] * 8, (size_t)n_corr[p] * 8});
  bool no_room = false;
  long long row = 0;
  for (int k = 0; k < S; ++k) {
    const int p = solved[k];
    solutions[p] = sol[k];
    no_room |= sol[k].clique_proven_optimal == -2;
    const int m = std::max(0, std::min(solved_n[k], sol[k].clique_size));
    if (want_clq && cliques[p]) spans.push_back(CopySpan{cliques[p], h + h_clq + (size_t)row * 4, (size_t)m * 4});
    row += solved_n[k];
  }
  parallel_copy(spans);
  if (icp) {
    for (int p = 0; p < P; ++p) memset(&icp_results[p], 0, sizeof(tzr_icp_result));
    for (int k = 0; k < S; ++k) icp_result_of(hi_probs[k], &icp_results[solved[k]]);
  }
  if (mw) {  // the pose graph over the refined pairs, in pair order
    memset(mw->information, 0, (size_t)P * 36 * 8);
    memset(mw->info_counts, 0, (size_t)P * 4);
    memset(mw->edge_weights, 0, (size_t)P * 8);
    memset(mw->edge_mask, 0, (size_t)P);
    memset(mw->poses, 0, (size_t)n_clouds * sizeof(tzr_similarity));
    std::vector<int> edge_pair;
    std::vector<int32_t> ends, unc;
    std::vector<tzr_similarity> Tsd;
    for (int k = 0; k < S; ++k) {
      if (!hi_probs[k].seeded) continue;
      const int p = solved[k];
      memcpy(mw->information + (size_t)p * 36, h + hi_info + (size_t)k * 36 * 8, 36 * 8);
      mw->info_counts[p] = ((const int*)(h + hi_icnt))[k];
      edge_pair.push_back(p);
      ends.push_back(pair_clouds[2 * p]);
      ends.push_back(pair_clouds[2 * p + 1]);
      unc.push_back(mw->uncertain[p]);
      Tsd.push_back(icp_results[p].transform);
    }
    const int E = (int)edge_pair.size();
    std::vector<double> L((size_t)std::max(E, 1) * 36), w(std::max(E, 1));
    std::vector<uint8_t> m(std::max(E, 1));
    for (int e = 0; e < E; ++e) memcpy(&L[(size_t)e * 36], mw->information + (size_t)edge_pair[e] * 36, 36 * 8);
    const std::string reg_error = ctx->last_error;
    *mw->pg_status = pose_graph_run(ctx, mw->pg, n_clouds, E, ends.data(), Tsd.data(), L.data(), unc.data(), nullptr,
                                    mw->poses, w.data(), m.data(), nullptr, mw->summary);
    if (*mw->pg_status == TZR_OK) {
      for (int e = 0; e < E; ++e) {
        mw->edge_weights[edge_pair[e]] = w[e];
        mw->edge_mask[edge_pair[e]] = m[e];
      }
    } else {
      memset(mw->poses, 0, (size_t)n_clouds * sizeof(tzr_similarity));
      if (mw->summary) memset(mw->summary, 0, sizeof(*mw->summary));
      if (*mw->pg_status == TZR_ERR_CUDA) return TZR_ERR_CUDA;
    }
    if (no_room || too_large) ctx->last_error = reg_error;
  }
  if (no_room) {
    ctx->last_error = "COMPLETE TIM graph of this clique does not fit the rotation workspace";
    return TZR_ERR_TOO_LARGE;
  }
  if (too_large) {
    ctx->last_error = "a pair's cloud has a point with more than 4096 neighbours inside a radius, or its correspondences "
                      "exceed the solve's size limit";
    return TZR_ERR_TOO_LARGE;
  }
  return TZR_OK;
}

int tzr_register_cloud_pairs(tzr_ctx* ctx, const tzr_frontend_params* fp, const tzr_params* params, int n_clouds,
                             const int32_t* n, const float* const* pts, int P, const int32_t* pair_clouds,
                             const uint64_t* tuple_seeds, tzr_solution* solutions, int32_t* status,
                             int32_t* problem_index, int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques,
                             float* global_scale) {
  return register_pairs_run(ctx, fp, params, n_clouds, n, pts, P, pair_clouds, tuple_seeds, solutions, status,
                            problem_index, n_corr, corr, cliques, global_scale, nullptr, nullptr);
}

int tzr_register_cloud_pairs_icp(tzr_ctx* ctx, const tzr_frontend_params* fp, const tzr_params* params, int n_clouds,
                                 const int32_t* n, const float* const* pts, int P, const int32_t* pair_clouds,
                                 const uint64_t* tuple_seeds, tzr_solution* solutions, int32_t* status,
                                 int32_t* problem_index, int64_t* n_corr, int32_t* const* corr,
                                 int32_t* const* cliques, float* global_scale, const tzr_icp_params* icp,
                                 tzr_icp_result* icp_results) {
  if (!icp) return TZR_ERR_INVALID_ARG;
  return register_pairs_run(ctx, fp, params, n_clouds, n, pts, P, pair_clouds, tuple_seeds, solutions, status,
                            problem_index, n_corr, corr, cliques, global_scale, icp, icp_results);
}

int tzr_register_cloud_pairs_icp_point_to_plane(tzr_ctx* ctx, const tzr_frontend_params* fp, const tzr_params* params,
                                                int n_clouds, const int32_t* n, const float* const* pts, int P,
                                                const int32_t* pair_clouds, const uint64_t* tuple_seeds,
                                                tzr_solution* solutions, int32_t* status, int32_t* problem_index,
                                                int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques,
                                                float* global_scale, const tzr_icp_params* icp,
                                                tzr_icp_result* icp_results) {
  if (!icp) return TZR_ERR_INVALID_ARG;
  return register_pairs_run(ctx, fp, params, n_clouds, n, pts, P, pair_clouds, tuple_seeds, solutions, status,
                            problem_index, n_corr, corr, cliques, global_scale, icp, icp_results, kIcpPointToPlane);
}

int tzr_register_cloud_pairs_icp_generalized(tzr_ctx* ctx, const tzr_frontend_params* fp, const tzr_params* params,
                                             int n_clouds, const int32_t* n, const float* const* pts, int P,
                                             const int32_t* pair_clouds, const uint64_t* tuple_seeds,
                                             tzr_solution* solutions, int32_t* status, int32_t* problem_index,
                                             int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques,
                                             float* global_scale, const tzr_icp_params* icp, double epsilon,
                                             tzr_icp_result* icp_results) {
  if (!icp) return TZR_ERR_INVALID_ARG;
  return register_pairs_run(ctx, fp, params, n_clouds, n, pts, P, pair_clouds, tuple_seeds, solutions, status,
                            problem_index, n_corr, corr, cliques, global_scale, icp, icp_results, kIcpGeneralized,
                            epsilon);
}

int tzr_register_cloud_pairs_icp_robust(tzr_ctx* ctx, const tzr_frontend_params* fp, const tzr_params* params,
                                        int n_clouds, const int32_t* n, const float* const* pts, int P,
                                        const int32_t* pair_clouds, const uint64_t* tuple_seeds,
                                        tzr_solution* solutions, int32_t* status, int32_t* problem_index,
                                        int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques,
                                        float* global_scale, const tzr_icp_params* icp, int32_t method,
                                        double epsilon, const tzr_robust_kernel* kernel,
                                        tzr_icp_result* icp_results) {
  if (!icp || (method != 1 && method != 2) || !robust_kernel_ok(kernel)) return TZR_ERR_INVALID_ARG;
  return register_pairs_run(ctx, fp, params, n_clouds, n, pts, P, pair_clouds, tuple_seeds, solutions, status,
                            problem_index, n_corr, corr, cliques, global_scale, icp, icp_results,
                            method == 1 ? kIcpPointToPlane : kIcpGeneralized, epsilon, kernel);
}

// every coloured entry's lambda and kernel, checked before any device work: TZR_OK when they pass, lambda then mapped
// into [0, 1] (outside it: 0.968, Open3D's TransformationEstimationForColoredICP)
static int colored_args(double* lambda_geometric, const tzr_robust_kernel* kernel) {
  if (!std::isfinite(*lambda_geometric) || (kernel && !robust_kernel_ok(kernel))) return TZR_ERR_INVALID_ARG;
  if (*lambda_geometric < 0.0 || *lambda_geometric > 1.0) *lambda_geometric = 0.968;
  return TZR_OK;
}

int tzr_register_cloud_pairs_icp_colored(tzr_ctx* ctx, const tzr_frontend_params* fp, const tzr_params* params,
                                         int n_clouds, const int32_t* n, const float* const* pts, int P,
                                         const int32_t* pair_clouds, const uint64_t* tuple_seeds,
                                         tzr_solution* solutions, int32_t* status, int32_t* problem_index,
                                         int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques,
                                         float* global_scale, const tzr_icp_params* icp, const float* const* colors,
                                         double lambda_geometric, const tzr_robust_kernel* kernel,
                                         tzr_icp_result* icp_results) {
  if (!icp || !colors || colored_args(&lambda_geometric, kernel) != TZR_OK) return TZR_ERR_INVALID_ARG;
  return register_pairs_run(ctx, fp, params, n_clouds, n, pts, P, pair_clouds, tuple_seeds, solutions, status,
                            problem_index, n_corr, corr, cliques, global_scale, icp, icp_results, kIcpColored, 0,
                            kernel, nullptr, colors, lambda_geometric);
}

void tzr_icp_params_default(tzr_icp_params* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->max_correspondence_distance = 0;  // no default (Open3D takes it as an argument)
  p->relative_fitness = 1e-6;
  p->relative_rmse = 1e-6;
  p->max_iteration = 30;
}

// Validation, planning and staging of tzr_icp*(_batch) and tzr_information_matrix(_batch): the problems planned by
// icp_plan and seeded from init, then [sources | targets | (target normals | (source normals))] and the layout's
// tables after them ([problems | target clouds | chunks], icp_layout) staged in one H2D copy into ctx->icp.  plan->mode
// (set by the caller) decides which normals are required and staged; information: room for the information matrices.
// On success *probs holds the staged problem table and *buf the workspace's device buffers.
static int icp_batch_stage(tzr_ctx* ctx, IcpPlan* plan, int B, const int32_t* ns, const float* const* src,
                           const float* const* src_normals, const int32_t* nd, const float* const* dst,
                           const float* const* dst_normals, const tzr_similarity* init, double r, bool information,
                           std::vector<IcpProb>* probs, IcpBuffers* buf, const float* const* src_colors = nullptr,
                           const float* const* dst_colors = nullptr) {
  const bool plane = plan->mode != kIcpPointToPoint, gicp = plan->mode == kIcpGeneralized;
  const bool colored = plan->mode == kIcpColored;
  if (!ctx || B < 1 || !ns || !src || !nd || !dst || (plane && !dst_normals) || (gicp && !src_normals) || !init ||
      (colored && (!src_colors || !dst_colors)))
    return TZR_ERR_INVALID_ARG;
  for (int b = 0; b < B; ++b)
    if (ns[b] < 1 || nd[b] < 1 || !src[b] || !dst[b] || (plane && !dst_normals[b]) || (gicp && !src_normals[b]) ||
        (colored && (!src_colors[b] || !dst_colors[b])) || !similarity_ok(init[b]))
      return TZR_ERR_INVALID_ARG;
  std::vector<FpfhCloud> clouds, gclouds;
  std::vector<int> chunk_prob;
  if (icp_plan(B, ns, nullptr, nullptr, B, nd, r, search_route(ctx->flags, kFlagIcpBrute, kFlagIcpGrid), init, plan,
               &clouds, probs, &chunk_prob) != TZR_OK) {
    ctx->last_error = "the batch's points or target grid do not fit 32-bit indices";
    return TZR_ERR_TOO_LARGE;
  }
  if (colored) {  // the gradient pass: tzr_estimate_color_gradients_batch's plan over the same targets at 2 r
    plan->grad_r = 2.0 * r;
    gclouds.resize((size_t)B);
    if (fpfh_plan(B, nd, plan->grad_r, plan->grad_r, search_route(ctx->flags, kFlagFpfhBrute, kFlagFpfhGrid),
                  gclouds.data(), &plan->ggrid) != TZR_OK) {
      ctx->last_error = "the batch's targets do not fit 32-bit indices";
      return TZR_ERR_TOO_LARGE;
    }
  }
  cudaSetDevice(ctx->device);
  const size_t NS = (size_t)plan->NS, ND = (size_t)plan->ND;
  const size_t o_dst = al256(NS * 12), o_nrm = o_dst + al256(ND * 12), o_snrm = o_nrm + al256(plane ? ND * 16 : 0);
  const size_t o_scol = o_snrm + al256(gicp ? NS * 16 : 0), o_dcol = o_scol + al256(colored ? NS * 12 : 0);
  const IcpLayout L = icp_layout(*plan, al256(o_dcol + (colored ? ND * 12 : 0)), information);
  int rc;
  if ((rc = ensure(ctx, ctx->icp, L.end)) != TZR_OK) return rc;
  std::vector<char> h(L.match);
  for (int b = 0; b < B; ++b) {
    const IcpProb& pr = (*probs)[b];
    memcpy(h.data() + (size_t)pr.s_lo * 12, src[b], (size_t)ns[b] * 12);
    memcpy(h.data() + o_dst + (size_t)pr.d_lo * 12, dst[b], (size_t)nd[b] * 12);
    if (plane) memcpy(h.data() + o_nrm + (size_t)pr.n_lo * 16, dst_normals[b], (size_t)nd[b] * 16);
    if (gicp) memcpy(h.data() + o_snrm + (size_t)pr.sn_lo * 16, src_normals[b], (size_t)ns[b] * 16);
    if (colored) {
      memcpy(h.data() + o_scol + (size_t)pr.s_lo * 12, src_colors[b], (size_t)ns[b] * 12);
      memcpy(h.data() + o_dcol + (size_t)pr.d_lo * 12, dst_colors[b], (size_t)nd[b] * 12);
    }
  }
  memcpy(h.data() + L.probs, probs->data(), (size_t)B * sizeof(IcpProb));
  memcpy(h.data() + L.clouds, clouds.data(), (size_t)B * sizeof(FpfhCloud));
  memcpy(h.data() + L.chunks, chunk_prob.data(), chunk_prob.size() * 4);
  char* d = (char*)ctx->icp.p;
  CK(cudaMemcpyAsync(d, h.data(), L.match, cudaMemcpyHostToDevice, ctx->stream));
  if (colored)
    CK(cudaMemcpyAsync(d + L.gclouds, gclouds.data(), (size_t)B * sizeof(FpfhCloud), cudaMemcpyHostToDevice,
                       ctx->stream));
  *buf = icp_buffers(d, L);
  buf->src = (const float*)d;
  buf->dst = (const float*)(d + o_dst);
  buf->dst_normals = plane ? (const float4*)(d + o_nrm) : nullptr;
  buf->src_normals = gicp ? (const float4*)(d + o_snrm) : nullptr;
  if (colored) {
    buf->src_colors = (const float*)(d + o_scol);
    buf->dst_colors = (const float*)(d + o_dcol);
  }
  return TZR_OK;
}

// tzr_icp(_batch), tzr_icp_point_to_plane(_batch) and tzr_icp_generalized(_batch): icp_batch_stage, every iteration
// enqueued (launch_icp), one D2H copy of the problem table (and of the per-point matches when correspondences are asked
// for).  dst_normals: required for kIcpPointToPlane and kIcpGeneralized, src_normals and epsilon for kIcpGeneralized;
// unused otherwise.  kernel: the robust kernel of the point-to-plane and generalized modes (checked by the caller;
// NULL = L2).
static int icp_batch_run(tzr_ctx* ctx, const tzr_icp_params* params, int mode, int B, const int32_t* ns,
                         const float* const* src, const float* const* src_normals, const int32_t* nd,
                         const float* const* dst, const float* const* dst_normals, double epsilon,
                         const tzr_similarity* init, tzr_icp_result* results, int32_t* const* corr,
                         const tzr_robust_kernel* kernel = nullptr, double lambda_geometric = 0.0,
                         const float* const* src_colors = nullptr, const float* const* dst_colors = nullptr) {
  if (!icp_params_ok(params) || (mode == kIcpGeneralized && !icp_epsilon_ok(epsilon)) || !results)
    return TZR_ERR_INVALID_ARG;
  IcpPlan plan;
  icp_iteration_settings(&plan, *params, mode, epsilon, kernel);
  plan.lambda_geometric = lambda_geometric;
  std::vector<IcpProb> probs;
  IcpBuffers buf;
  int rc = icp_batch_stage(ctx, &plan, B, ns, src, src_normals, nd, dst, dst_normals, init,
                           params->max_correspondence_distance, false, &probs, &buf, src_colors, dst_colors);
  if (rc != TZR_OK) return rc;
  cudaStream_t st = ctx->stream;
  ctx->launches += launch_icp(plan, buf, st);
  if ((rc = check_launch(ctx, "icp launch")) != TZR_OK) return rc;
  CK(cudaMemcpyAsync(probs.data(), buf.probs, (size_t)B * sizeof(IcpProb), cudaMemcpyDeviceToHost, st));
  bool want_corr = false;
  for (int b = 0; b < B && corr; ++b) want_corr |= corr[b] != nullptr;
  std::vector<int32_t> match(want_corr ? (size_t)plan.NS : 0);
  if (want_corr) CK(cudaMemcpyAsync(match.data(), buf.match, (size_t)plan.NS * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  for (int b = 0; b < B; ++b) {
    const IcpProb& pr = probs[b];
    icp_result_of(pr, &results[b]);
    if (corr && corr[b]) {
      int32_t* rows = corr[b];
      long long k = 0;
      for (int i = 0; i < pr.ns; ++i) {
        const int j = match[(size_t)pr.m_lo + i];
        if (j < 0) continue;
        rows[2 * k] = i;
        rows[2 * k + 1] = j;
        ++k;
      }
    }
  }
  return TZR_OK;
}

int tzr_icp_batch(tzr_ctx* ctx, const tzr_icp_params* params, int B, const int32_t* ns, const float* const* src,
                  const int32_t* nd, const float* const* dst, const tzr_similarity* init, tzr_icp_result* results,
                  int32_t* const* corr) {
  return icp_batch_run(ctx, params, kIcpPointToPoint, B, ns, src, nullptr, nd, dst, nullptr, 0.0, init, results, corr);
}

int tzr_icp_point_to_plane_batch(tzr_ctx* ctx, const tzr_icp_params* params, int B, const int32_t* ns,
                                 const float* const* src, const int32_t* nd, const float* const* dst,
                                 const float* const* dst_normals, const tzr_similarity* init,
                                 tzr_icp_result* results, int32_t* const* corr) {
  return icp_batch_run(ctx, params, kIcpPointToPlane, B, ns, src, nullptr, nd, dst, dst_normals, 0.0, init, results,
                       corr);
}

int tzr_icp_generalized_batch(tzr_ctx* ctx, const tzr_icp_params* params, double epsilon, int B, const int32_t* ns,
                              const float* const* src, const float* const* src_normals, const int32_t* nd,
                              const float* const* dst, const float* const* dst_normals, const tzr_similarity* init,
                              tzr_icp_result* results, int32_t* const* corr) {
  return icp_batch_run(ctx, params, kIcpGeneralized, B, ns, src, src_normals, nd, dst, dst_normals, epsilon, init,
                       results, corr);
}

int tzr_icp_point_to_plane_robust_batch(tzr_ctx* ctx, const tzr_icp_params* params, int B, const int32_t* ns,
                                        const float* const* src, const int32_t* nd, const float* const* dst,
                                        const float* const* dst_normals, const tzr_similarity* init,
                                        tzr_icp_result* results, int32_t* const* corr,
                                        const tzr_robust_kernel* kernel) {
  if (!robust_kernel_ok(kernel)) return TZR_ERR_INVALID_ARG;
  return icp_batch_run(ctx, params, kIcpPointToPlane, B, ns, src, nullptr, nd, dst, dst_normals, 0.0, init, results,
                       corr, kernel);
}

int tzr_icp_generalized_robust_batch(tzr_ctx* ctx, const tzr_icp_params* params, double epsilon, int B,
                                     const int32_t* ns, const float* const* src, const float* const* src_normals,
                                     const int32_t* nd, const float* const* dst, const float* const* dst_normals,
                                     const tzr_similarity* init, tzr_icp_result* results, int32_t* const* corr,
                                     const tzr_robust_kernel* kernel) {
  if (!robust_kernel_ok(kernel)) return TZR_ERR_INVALID_ARG;
  return icp_batch_run(ctx, params, kIcpGeneralized, B, ns, src, src_normals, nd, dst, dst_normals, epsilon, init,
                       results, corr, kernel);
}

// tzr_icp_colored(_batch): lambda outside [0, 1] becomes 0.968 (Open3D's TransformationEstimationForColoredICP), a
// non-finite one and a bad kernel are refused before any device work; NULL kernel = L2.
int tzr_icp_colored_batch(tzr_ctx* ctx, const tzr_icp_params* params, int B, const int32_t* ns,
                          const float* const* src, const int32_t* nd, const float* const* dst,
                          const float* const* dst_normals, const tzr_similarity* init, tzr_icp_result* results,
                          int32_t* const* corr, const float* const* src_colors, const float* const* dst_colors,
                          double lambda_geometric, const tzr_robust_kernel* kernel) {
  if (colored_args(&lambda_geometric, kernel) != TZR_OK) return TZR_ERR_INVALID_ARG;
  return icp_batch_run(ctx, params, kIcpColored, B, ns, src, nullptr, nd, dst, dst_normals, 0.0, init, results, corr,
                       kernel, lambda_geometric, src_colors, dst_colors);
}

int tzr_icp_colored(tzr_ctx* ctx, const tzr_icp_params* params, const float* src, int ns, const float* dst, int nd,
                    const float* dst_normals, const tzr_similarity* init, tzr_icp_result* result, int32_t* corr,
                    const float* src_colors, const float* dst_colors, double lambda_geometric,
                    const tzr_robust_kernel* kernel) {
  tzr_similarity id;
  if (!init) {
    memset(&id, 0, sizeof(id));
    id.scale = 1.0;
    id.rotation[0] = id.rotation[4] = id.rotation[8] = 1.0;
    init = &id;
  }
  int32_t* const corrs[1] = {corr};
  return tzr_icp_colored_batch(ctx, params, 1, &ns, &src, &nd, &dst, &dst_normals, init, result,
                               corr ? corrs : nullptr, &src_colors, &dst_colors, lambda_geometric, kernel);
}

// the single-problem entries: icp_batch_run with B = 1 and init NULL meaning the identity
static int icp_single(tzr_ctx* ctx, const tzr_icp_params* params, int mode, const float* src, int ns,
                      const float* src_normals, const float* dst, int nd, const float* dst_normals, double epsilon,
                      const tzr_similarity* init, tzr_icp_result* result, int32_t* corr) {
  tzr_similarity id;
  if (!init) {
    memset(&id, 0, sizeof(id));
    id.scale = 1.0;
    id.rotation[0] = id.rotation[4] = id.rotation[8] = 1.0;
    init = &id;
  }
  int32_t* const corrs[1] = {corr};
  return icp_batch_run(ctx, params, mode, 1, &ns, &src, src_normals ? &src_normals : nullptr, &nd, &dst,
                       dst_normals ? &dst_normals : nullptr, epsilon, init, result, corr ? corrs : nullptr);
}

int tzr_icp(tzr_ctx* ctx, const tzr_icp_params* params, const float* src, int ns, const float* dst, int nd,
            const tzr_similarity* init, tzr_icp_result* result, int32_t* corr) {
  return icp_single(ctx, params, kIcpPointToPoint, src, ns, nullptr, dst, nd, nullptr, 0.0, init, result, corr);
}

int tzr_icp_point_to_plane(tzr_ctx* ctx, const tzr_icp_params* params, const float* src, int ns, const float* dst,
                           int nd, const float* dst_normals, const tzr_similarity* init, tzr_icp_result* result,
                           int32_t* corr) {
  return icp_single(ctx, params, kIcpPointToPlane, src, ns, nullptr, dst, nd, dst_normals, 0.0, init, result, corr);
}

int tzr_icp_generalized(tzr_ctx* ctx, const tzr_icp_params* params, double epsilon, const float* src, int ns,
                        const float* src_normals, const float* dst, int nd, const float* dst_normals,
                        const tzr_similarity* init, tzr_icp_result* result, int32_t* corr) {
  return icp_single(ctx, params, kIcpGeneralized, src, ns, src_normals, dst, nd, dst_normals, epsilon, init, result,
                    corr);
}

// tzr_information_matrix(_batch): icp_batch_stage (point-to-point, no normals), the search and the sums
// (launch_icp_information), one read-back
int tzr_information_matrix_batch(tzr_ctx* ctx, int B, const int32_t* ns, const float* const* src, const int32_t* nd,
                                 const float* const* dst, const tzr_similarity* transforms,
                                 double max_correspondence_distance, double* information, int32_t* counts) {
  const double r = max_correspondence_distance;
  if (!information || !(r > 0) || !std::isfinite(r)) return TZR_ERR_INVALID_ARG;
  IcpPlan plan;
  std::vector<IcpProb> probs;
  IcpBuffers buf;
  int rc = icp_batch_stage(ctx, &plan, B, ns, src, nullptr, nd, dst, nullptr, transforms, r, true, &probs, &buf);
  if (rc != TZR_OK) return rc;
  cudaStream_t st = ctx->stream;
  ctx->launches += launch_icp_information(plan, buf, false, st);
  if ((rc = check_launch(ctx, "information launch")) != TZR_OK) return rc;
  std::vector<int32_t> cnt((size_t)B);
  CK(cudaMemcpyAsync(information, buf.info, (size_t)B * 36 * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(cnt.data(), buf.counts, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (counts) memcpy(counts, cnt.data(), (size_t)B * 4);
  return TZR_OK;
}

int tzr_information_matrix(tzr_ctx* ctx, const float* src, int ns, const float* dst, int nd,
                           const tzr_similarity* transform, double max_correspondence_distance, double* information,
                           int32_t* count) {
  return tzr_information_matrix_batch(ctx, 1, &ns, &src, &nd, &dst, transform, max_correspondence_distance,
                                      information, count);
}

// ---- multi-scale ICP (DESIGN.md §3.19) ------------------------------------------------------------------------------
static bool icp_scale_ok(const tzr_icp_scale& sc, bool normals) {
  return std::isfinite(sc.voxel_size) && sc.voxel_size >= 0 && std::isfinite(sc.max_correspondence_distance) &&
         sc.max_correspondence_distance > 0 && sc.max_iteration >= 0 && !std::isnan(sc.relative_fitness) &&
         !std::isnan(sc.relative_rmse) &&
         (!normals || (std::isfinite(sc.normal_search_radius) && sc.normal_search_radius > 0));
}

// One scale of the schedule, planned on the host from its cloud sizes exactly as the public calls plan them
struct IcpScalePlan {
  std::vector<int32_t> nd;     // points of every cloud at this scale
  FpfhPlan nplan;              // the normals pass over every cloud (tzr_estimate_normals_batch's plan)
  std::vector<FpfhCloud> ncl;
  IcpPlan ip;                  // ICP of the refined pairs onto the cloud table (and the gradient pass, coloured)
  std::vector<FpfhCloud> icl, gcl;
  std::vector<IcpProb> probs;
  std::vector<int> chunks, pair_of, prob_of;
};

// Plans scale s over clouds of nd points (prob_of / pair_of: the pairs whose two clouds have points).  TZR_OK, or
// TZR_ERR_TOO_LARGE when a table does not fit 32-bit indices.
static int icp_scale_plan(const tzr_ctx* ctx, const tzr_icp_scale& sc, int method, double epsilon,
                          double lambda_geometric, const tzr_robust_kernel* kernel, int n_clouds,
                          const int32_t* nd, int P, const int32_t* pair_clouds, IcpScalePlan* out) {
  const int froute = search_route(ctx->flags, kFlagFpfhBrute, kFlagFpfhGrid);
  out->nd.assign(nd, nd + n_clouds);
  out->ncl.resize((size_t)n_clouds);
  if (method != kIcpPointToPoint &&
      fpfh_plan(n_clouds, nd, sc.normal_search_radius, sc.normal_search_radius, froute, out->ncl.data(),
                &out->nplan) != TZR_OK)
    return TZR_ERR_TOO_LARGE;
  std::vector<int32_t> lo((size_t)n_clouds), ns, slo, tc;
  for (int c = 0, l = 0; c < n_clouds; l += nd[c], ++c) lo[c] = l;
  out->prob_of.assign((size_t)P, -1);
  out->pair_of.clear();
  for (int p = 0; p < P; ++p) {
    const int a = pair_clouds[2 * p], b = pair_clouds[2 * p + 1];
    if (nd[a] < 1 || nd[b] < 1) continue;
    out->prob_of[p] = (int)out->pair_of.size();
    out->pair_of.push_back(p);
    ns.push_back(nd[a]);
    slo.push_back(lo[a]);
    tc.push_back(b);
  }
  const tzr_icp_params prm{sc.max_correspondence_distance, sc.relative_fitness, sc.relative_rmse, sc.max_iteration, 0};
  out->ip = IcpPlan{};
  icp_iteration_settings(&out->ip, prm, method, epsilon, kernel);
  out->ip.lambda_geometric = lambda_geometric;
  if (out->pair_of.empty()) return TZR_OK;
  if (method == kIcpColored) {  // every cloud's gradients at 2 r, as the chained coloured entries take them
    out->ip.grad_r = 2.0 * sc.max_correspondence_distance;
    out->gcl.resize((size_t)n_clouds);
    if (fpfh_plan(n_clouds, nd, out->ip.grad_r, out->ip.grad_r, froute, out->gcl.data(), &out->ip.ggrid) != TZR_OK)
      return TZR_ERR_TOO_LARGE;
  }
  return icp_plan((int)ns.size(), ns.data(), slo.data(), tc.data(), n_clouds, nd, sc.max_correspondence_distance,
                  search_route(ctx->flags, kFlagIcpBrute, kFlagIcpGrid), nullptr, &out->ip, &out->icl, &out->probs,
                  &out->chunks);
}

// Bytes of scale work in the shared region: [normals | max(normals grid, ICP workspace from its layout)]
static size_t icp_scale_work(const IcpScalePlan& sp, int method, size_t n_points, bool information) {
  const size_t nrm = method != kIcpPointToPoint ? al256(n_points * 16) : 0;
  const size_t icp = sp.pair_of.empty() ? 0 : icp_layout(sp.ip, 0, information).end;
  return nrm + std::max(method != kIcpPointToPoint ? sp.nplan.grid_bytes : 0, icp);
}

// Workspace ctx->icp: [clouds | colours | voxel tables | poses] (one upload) | per voxel scale: voxels | their colours |
// per scale: tables (one upload) | records | normals overflow flags (one read-back) | shared scale work.  Every region
// is sized from the dense clouds before any device work: a scale never has more points than the clouds as given, and
// every table and grid grows with the points.
int tzr_icp_multiscale_batch(tzr_ctx* ctx, int method, int S, const tzr_icp_scale* scales, int n_clouds,
                             const int32_t* n, const float* const* pts, const float* const* colors, int P,
                             const int32_t* pair_clouds, const tzr_similarity* init, double epsilon,
                             double lambda_geometric, const tzr_robust_kernel* kernel, tzr_icp_result* results,
                             int32_t* n_down, int32_t* status, double* information, int32_t* info_counts) {
  const bool normals = method != kIcpPointToPoint, colored = method == kIcpColored;
  if (!ctx || method < kIcpPointToPoint || method > kIcpColored || S < 1 || !scales || n_clouds < 1 || !n || !pts ||
      P < 1 || !pair_clouds || !init || !results || (colored && !colors))
    return TZR_ERR_INVALID_ARG;
  if ((method == kIcpPointToPoint && kernel) || (method == kIcpGeneralized && !icp_epsilon_ok(epsilon)))
    return TZR_ERR_INVALID_ARG;
  if (colored ? colored_args(&lambda_geometric, kernel) != TZR_OK : kernel && !robust_kernel_ok(kernel))
    return TZR_ERR_INVALID_ARG;
  if (!colored) lambda_geometric = 0.0;
  for (int s = 0; s < S; ++s)
    if (!icp_scale_ok(scales[s], normals)) return TZR_ERR_INVALID_ARG;
  for (int c = 0; c < n_clouds; ++c)
    if (n[c] < 1 || !pts[c] || (colored && !colors[c])) return TZR_ERR_INVALID_ARG;
  for (int p = 0; p < P; ++p) {
    const int a = pair_clouds[2 * p], b = pair_clouds[2 * p + 1];
    if (a < 0 || a >= n_clouds || b < 0 || b >= n_clouds || !similarity_ok(init[p])) return TZR_ERR_INVALID_ARG;
  }
  std::vector<VoxCloud> vt0((size_t)n_clouds);
  VoxPlan vplan;
  if (voxel_plan(n_clouds, n, vt0.data(), &vplan) != TZR_OK) {
    ctx->last_error = "the clouds' points do not fit 32-bit indices";
    return TZR_ERR_TOO_LARGE;
  }
  std::vector<int> vox((size_t)S, -1);  // the voxel output slot of every scale, -1: the clouds as given
  int SV = 0;
  for (int s = 0; s < S; ++s)
    if (scales[s].voxel_size > 0) vox[s] = SV++;
  // the bounds: every scale planned at the dense sizes
  const size_t N = (size_t)vplan.N, C = (size_t)n_clouds;
  const bool want_info = information || info_counts;  // either output alone runs the information pass
  size_t work = al256(vplan.scratch_bytes) + N * 4, max_chunks = 0;
  IcpScalePlan sp;
  for (int s = 0; s < S; ++s) {
    if (icp_scale_plan(ctx, scales[s], method, epsilon, lambda_geometric, kernel, n_clouds, n, P, pair_clouds, &sp) !=
        TZR_OK) {
      ctx->last_error = "the clouds' points or grids do not fit 32-bit indices";
      return TZR_ERR_TOO_LARGE;
    }
    work = std::max(work, icp_scale_work(sp, method, N, want_info));
    max_chunks = std::max(max_chunks, sp.chunks.size());
  }
  // one scale's tables: [problems | ICP cloud table | chunks | normals cloud table | gradient cloud table | pair_of |
  // prob_of]
  const size_t t_icl = al256((size_t)P * sizeof(IcpProb)), t_chk = t_icl + al256(C * sizeof(FpfhCloud)),
               t_ncl = t_chk + al256(max_chunks * 4), t_gcl = t_ncl + al256(C * sizeof(FpfhCloud)),
               t_pair = t_gcl + al256(C * sizeof(FpfhCloud)), t_prob = t_pair + al256((size_t)P * 4),
               tab = al256(t_prob + (size_t)P * 4);
  const size_t o_col = al256(N * 12), o_vtab = o_col + al256(colored ? N * 12 : 0),
               o_pose = o_vtab + al256((size_t)SV * C * sizeof(VoxCloud)),
               in_bytes = o_pose + (size_t)P * sizeof(tzr_similarity), o_vout = al256(in_bytes),
               o_vcol = o_vout + al256((size_t)SV * N * 12), o_tab = o_vcol + al256(colored ? (size_t)SV * N * 12 : 0),
               o_rec = o_tab + (size_t)S * tab, o_ovf = o_rec + al256((size_t)P * S * sizeof(tzr_icp_result)),
               out_bytes = o_ovf + (size_t)S * C * 4 - o_rec, o_work = al256(o_rec + out_bytes);
  // pinned: [upload | tables], host writes that may overlap the copies in flight; then [records | overflow flags |
  // information | counts], read back once every copy before them has run
  const size_t h_tab = al256(in_bytes), h_info = al256(out_bytes), h_cnt = h_info + al256((size_t)P * 36 * 8),
               pin = std::max(h_tab + (size_t)S * tab, h_cnt + (size_t)P * 4);
  int rc;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  if ((rc = ensure(ctx, ctx->icp, o_work + work)) != TZR_OK) return rc;
  if ((rc = ensure_pinned(ctx, pin)) != TZR_OK) return rc;
  char* h = (char*)ctx->h_pin;
  char* d = (char*)ctx->icp.p;
  std::vector<CopySpan> spans;
  for (int c = 0; c < n_clouds; ++c) {
    spans.push_back(CopySpan{h + (size_t)vt0[c].lo * 12, pts[c], (size_t)n[c] * 12});
    if (colored) spans.push_back(CopySpan{h + o_col + (size_t)vt0[c].lo * 12, colors[c], (size_t)n[c] * 12});
  }
  for (int v = 0; v < SV; ++v)
    spans.push_back(CopySpan{h + o_vtab + (size_t)v * C * sizeof(VoxCloud), vt0.data(), C * sizeof(VoxCloud)});
  spans.push_back(CopySpan{h + o_pose, init, (size_t)P * sizeof(tzr_similarity)});
  CK(stage_in(spans, h, d, o_vtab, in_bytes, false, st));
  const float* d_pts = (const float*)d;
  const float* d_col = colored ? (const float*)(d + o_col) : nullptr;
  VoxCloud* d_vtab = (VoxCloud*)(d + o_vtab);
  tzr_similarity* d_pose = (tzr_similarity*)(d + o_pose);
  char* d_work = d + o_work;
  for (int s = 0; s < S; ++s)
    if (vox[s] >= 0)
      ctx->launches += launch_voxel(vplan, scales[s].voxel_size, d_pts, d_vtab + (size_t)vox[s] * C, d_work,
                                    (float*)(d + o_vout) + (size_t)vox[s] * N * 3, (int*)(d_work + al256(vplan.scratch_bytes)),
                                    st, d_col, colored ? (float*)(d + o_vcol) + (size_t)vox[s] * N * 3 : nullptr);
  if ((rc = check_launch(ctx, "multi-scale voxel launch")) != TZR_OK) return rc;
  // synchronisation 1 (with a voxel scale): every scale's cloud sizes
  std::vector<VoxCloud> vt((size_t)SV * C);
  if (SV > 0) {
    CK(cudaMemcpyAsync(vt.data(), d_vtab, vt.size() * sizeof(VoxCloud), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  std::vector<int32_t> nd(C * S);  // cloud-major, as n_down
  bool grid_too_large = false;
  for (int c = 0; c < n_clouds; ++c)
    for (int s = 0; s < S; ++s) {
      const VoxCloud* v = vox[s] >= 0 ? &vt[(size_t)vox[s] * C + c] : nullptr;
      nd[(size_t)c * S + s] = v ? v->n_out : n[c];
      if (n_down) n_down[(size_t)c * S + s] = nd[(size_t)c * S + s];
      if (status) status[(size_t)c * S + s] = v ? v->status : TZR_OK;
      grid_too_large |= v && v->status != TZR_OK;
    }
  if (grid_too_large) {
    memset(results, 0, (size_t)P * S * sizeof(tzr_icp_result));
    if (information) memset(information, 0, (size_t)P * 36 * 8);
    if (info_counts) memset(info_counts, 0, (size_t)P * 4);
    ctx->last_error = "a cloud's voxel grid is too large for a scale's voxel size (Open3D's INT_MAX check or 2^62 cells)";
    return TZR_ERR_TOO_LARGE;
  }
  // every scale planned from its sizes, its tables staged in one upload
  std::vector<IcpScalePlan> plans((size_t)S);
  std::vector<int32_t> nds((size_t)n_clouds);
  for (int s = 0; s < S; ++s) {
    for (int c = 0; c < n_clouds; ++c) nds[c] = nd[(size_t)c * S + s];
    IcpScalePlan& q = plans[s];
    if (icp_scale_plan(ctx, scales[s], method, epsilon, lambda_geometric, kernel, n_clouds, nds.data(), P,
                       pair_clouds, &q) != TZR_OK ||
        q.chunks.size() > max_chunks || icp_scale_work(q, method, N, want_info) > work) {
      ctx->last_error = "a scale's plan exceeds the workspace sized from the clouds as given";
      return TZR_ERR_TOO_LARGE;
    }
    char* t = h + h_tab + (size_t)s * tab;
    memcpy(t, q.probs.data(), q.probs.size() * sizeof(IcpProb));
    if (!q.pair_of.empty()) memcpy(t + t_icl, q.icl.data(), C * sizeof(FpfhCloud));
    memcpy(t + t_chk, q.chunks.data(), q.chunks.size() * 4);
    if (normals) memcpy(t + t_ncl, q.ncl.data(), C * sizeof(FpfhCloud));
    if (!q.gcl.empty()) memcpy(t + t_gcl, q.gcl.data(), C * sizeof(FpfhCloud));
    memcpy(t + t_pair, q.pair_of.data(), q.pair_of.size() * 4);
    memcpy(t + t_prob, q.prob_of.data(), (size_t)P * 4);
  }
  CK(cudaMemcpyAsync(d + o_tab, h + h_tab, (size_t)S * tab, cudaMemcpyHostToDevice, st));
  // every scale enqueued: normals, pose load, ICP (with the gradient pass), pose store; the information at the end
  float4* d_nrm = (float4*)d_work;
  char* d_scr = d_work + (normals ? al256(N * 16) : 0);
  tzr_icp_result* d_rec = (tzr_icp_result*)(d + o_rec);
  IcpBuffers last{};
  for (int s = 0; s < S; ++s) {
    const IcpScalePlan& q = plans[s];
    char* t = d + o_tab + (size_t)s * tab;
    const float* sp_pts = vox[s] >= 0 ? (const float*)(d + o_vout) + (size_t)vox[s] * N * 3 : d_pts;
    const float* sp_col = !colored ? nullptr : vox[s] >= 0 ? (const float*)(d + o_vcol) + (size_t)vox[s] * N * 3 : d_col;
    if (normals && q.nplan.N > 0)
      ctx->launches += launch_fpfh(q.nplan, sp_pts, (FpfhCloud*)(t + t_ncl), scales[s].normal_search_radius,
                                   scales[s].normal_search_radius, d_nrm, nullptr, nullptr,
                                   (int*)(d + o_ovf) + (size_t)s * C, q.nplan.grid_bytes ? d_scr : nullptr, st);
    const int B = (int)q.pair_of.size();
    const bool info_here = want_info && s == S - 1 && B > 0;
    IcpBuffers buf{};
    IcpGrid grid{nullptr, nullptr, nullptr};
    if (B > 0) {
      buf = icp_buffers(d_scr, icp_layout(q.ip, 0, info_here));
      buf.probs = (IcpProb*)t;
      buf.clouds = (FpfhCloud*)(t + t_icl);
      buf.chunk_prob = (const int*)(t + t_chk);
      buf.src = buf.dst = sp_pts;
      if (normals) buf.src_normals = buf.dst_normals = d_nrm;
      if (colored) {
        buf.src_colors = buf.dst_colors = sp_col;
        buf.gclouds = (FpfhCloud*)(t + t_gcl);
      }
      ctx->launches += launch_icp_pose_load(buf.probs, B, (const int*)(t + t_pair), d_pose, st);
      ctx->launches += launch_icp(q.ip, buf, st, &grid);
    }
    ctx->launches += launch_icp_pose_store(B > 0 ? buf.probs : nullptr, P, (const int*)(t + t_prob), d_pose, d_rec + s,
                                           S, st);
    if (info_here) {
      ctx->launches += launch_icp_information(q.ip, buf, true, st, &grid);
      last = buf;
    }
    if ((rc = check_launch(ctx, "multi-scale icp launch")) != TZR_OK) return rc;
  }
  // synchronisation 2: the records, the overflow flags and the information matrices
  const IcpScalePlan& ql = plans[S - 1];
  const int BL = (int)ql.pair_of.size();
  CK(cudaMemcpyAsync(h, d + o_rec, out_bytes, cudaMemcpyDeviceToHost, st));
  if (last.info) {
    CK(cudaMemcpyAsync(h + h_info, last.info, (size_t)BL * 36 * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(h + h_cnt, last.counts, (size_t)BL * 4, cudaMemcpyDeviceToHost, st));
  }
  CK(cudaStreamSynchronize(st));
  memcpy(results, h, (size_t)P * S * sizeof(tzr_icp_result));
  const int* ovf = (const int*)(h + (o_ovf - o_rec));
  std::vector<int> first_bad((size_t)n_clouds, S);  // the first scale at which the cloud's normals overflowed
  bool overflow = false;
  for (int s = 0; s < S; ++s) {
    if (!normals || plans[s].nplan.N == 0) continue;
    for (int c = 0; c < n_clouds; ++c)
      if (ovf[(size_t)s * C + c]) {
        if (status) status[(size_t)c * S + s] = TZR_ERR_TOO_LARGE;
        first_bad[c] = std::min(first_bad[c], s);
        overflow = true;
      }
  }
  if (information) memset(information, 0, (size_t)P * 36 * 8);
  if (info_counts) memset(info_counts, 0, (size_t)P * 4);
  for (int p = 0; p < P; ++p) {
    const int s0 = std::min(first_bad[pair_clouds[2 * p]], first_bad[pair_clouds[2 * p + 1]]);
    for (int s = s0; s < S; ++s) memset(&results[(size_t)p * S + s], 0, sizeof(tzr_icp_result));
    const int k = ql.prob_of[p];
    if (!last.info || k < 0 || s0 < S) continue;
    if (information) memcpy(information + (size_t)p * 36, h + h_info + (size_t)k * 36 * 8, 36 * 8);
    if (info_counts) info_counts[p] = ((const int*)(h + h_cnt))[k];
  }
  if (overflow) {
    ctx->last_error = "a cloud has a point with more than 4096 neighbours inside a scale's normal radius";
    return TZR_ERR_TOO_LARGE;
  }
  return TZR_OK;
}

void tzr_pose_graph_params_default(tzr_pose_graph_params* p) {
  if (!p) return;
  memset(p, 0, sizeof(*p));
  p->max_correspondence_distance = 0;  // no default (the caller's ICP distance)
  p->gnc_factor = 1.4;
  p->cost_threshold = 1e-6;
  p->max_iterations = 100;
  p->max_inner_iterations = 10;
  p->reference_node = 0;
}

int tzr_pose_graph_optimize(tzr_ctx* ctx, const tzr_pose_graph_params* params, int K, int E, const int32_t* edges,
                            const tzr_similarity* edge_transforms, const double* information, const int32_t* uncertain,
                            const tzr_similarity* initial_poses, tzr_similarity* poses, double* weights,
                            uint8_t* inlier_mask, double* residuals, tzr_pose_graph_summary* summary) {
  return pose_graph_run(ctx, params, K, E, edges, edge_transforms, information, uncertain, initial_poses, poses,
                        weights, inlier_mask, residuals, summary);
}

int tzr_register_cloud_pairs_multiway(tzr_ctx* ctx, const tzr_frontend_params* fp, const tzr_params* params,
                                      int n_clouds, const int32_t* n, const float* const* pts, int P,
                                      const int32_t* pair_clouds, const uint64_t* tuple_seeds,
                                      tzr_solution* solutions, int32_t* status, int32_t* problem_index,
                                      int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques,
                                      float* global_scale, const tzr_icp_params* icp, tzr_icp_result* icp_results,
                                      const int32_t* uncertain, const tzr_pose_graph_params* pg, double* information,
                                      int32_t* info_counts, double* edge_weights, uint8_t* edge_mask,
                                      tzr_similarity* poses, tzr_pose_graph_summary* pg_summary, int32_t* pg_status) {
  if (!icp) return TZR_ERR_INVALID_ARG;
  const MultiwayOut mw{uncertain, pg, information, info_counts, edge_weights, edge_mask, poses, pg_summary, pg_status};
  return register_pairs_run(ctx, fp, params, n_clouds, n, pts, P, pair_clouds, tuple_seeds, solutions, status,
                            problem_index, n_corr, corr, cliques, global_scale, icp, icp_results, kIcpPointToPlane, 0,
                            nullptr, &mw);
}

int tzr_register_cloud_pairs_multiway_colored(
    tzr_ctx* ctx, const tzr_frontend_params* fp, const tzr_params* params, int n_clouds, const int32_t* n,
    const float* const* pts, int P, const int32_t* pair_clouds, const uint64_t* tuple_seeds, tzr_solution* solutions,
    int32_t* status, int32_t* problem_index, int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques,
    float* global_scale, const tzr_icp_params* icp, const float* const* colors, double lambda_geometric,
    const tzr_robust_kernel* kernel, tzr_icp_result* icp_results, const int32_t* uncertain,
    const tzr_pose_graph_params* pg, double* information, int32_t* info_counts, double* edge_weights,
    uint8_t* edge_mask, tzr_similarity* poses, tzr_pose_graph_summary* pg_summary, int32_t* pg_status) {
  if (!icp || !colors || colored_args(&lambda_geometric, kernel) != TZR_OK) return TZR_ERR_INVALID_ARG;
  const MultiwayOut mw{uncertain, pg, information, info_counts, edge_weights, edge_mask, poses, pg_summary, pg_status};
  return register_pairs_run(ctx, fp, params, n_clouds, n, pts, P, pair_clouds, tuple_seeds, solutions, status,
                            problem_index, n_corr, corr, cliques, global_scale, icp, icp_results, kIcpColored, 0,
                            kernel, &mw, colors, lambda_geometric);
}

// tzr_voxel_downsample(_batch): the clouds staged back to back (one H2D copy), the batch's launches (launch_voxel), a
// read-back of the cloud table, then one D2H copy of the batch's voxels (and of voxel_of when some cloud asks for it).
// Workspace ctx->vox: [points | cloud table | voxels | voxel_of | scratch]; the pinned area mirrors its first four.
// With colours (tzr_voxel_downsample_colors(_batch)): [points | colours | cloud table | voxels | colour means | voxel_of
// | scratch]; without them the colour regions are empty and the layout is the one above.
static int voxel_run(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts, double voxel_size,
                     float* const* pts_out, int32_t* n_out, int32_t* const* voxel_of, int32_t* status,
                     const float* const* colors, float* const* colors_out, bool with_colors) {
  if (!ctx || B < 1 || !n || !pts || !pts_out || !n_out || !(voxel_size > 0) || !std::isfinite(voxel_size) ||
      (with_colors && (!colors || !colors_out)))
    return TZR_ERR_INVALID_ARG;
  bool want_trace = false;
  for (int b = 0; b < B; ++b) {
    if (n[b] < 1 || !pts[b] || !pts_out[b] || (with_colors && (!colors[b] || !colors_out[b])))
      return TZR_ERR_INVALID_ARG;
    want_trace |= voxel_of && voxel_of[b];
  }
  std::vector<VoxCloud> clouds((size_t)B);
  VoxPlan plan;
  if (voxel_plan(B, n, clouds.data(), &plan) != TZR_OK) {
    ctx->last_error = "the batch's points do not fit 32-bit indices";
    return TZR_ERR_TOO_LARGE;
  }
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)plan.N, pb = N * 12, tb = (size_t)B * sizeof(VoxCloud), cb = with_colors ? pb : 0;
  const size_t o_col = al256(pb), o_tab = o_col + al256(cb), in_bytes = o_tab + tb, o_out = al256(in_bytes),
               o_cout = o_out + al256(pb), o_vo = o_cout + al256(cb), o_scr = o_vo + al256(N * 4),
               total = o_scr + plan.scratch_bytes;
  int rc;
  if ((rc = ensure(ctx, ctx->vox, total)) != TZR_OK) return rc;
  if ((rc = ensure_pinned(ctx, o_scr)) != TZR_OK) return rc;
  char* h = (char*)ctx->h_pin;
  char* d = (char*)ctx->vox.p;
  std::vector<CopySpan> spans;
  for (int b = 0; b < B; ++b) spans.push_back(CopySpan{h + (size_t)clouds[b].lo * 12, pts[b], (size_t)n[b] * 12});
  if (with_colors)
    for (int b = 0; b < B; ++b)
      spans.push_back(CopySpan{h + o_col + (size_t)clouds[b].lo * 12, colors[b], (size_t)n[b] * 12});
  spans.push_back(CopySpan{h + o_tab, clouds.data(), tb});
  CK(stage_in(spans, h, d, o_tab, in_bytes, B == 1, st));
  ctx->launches += launch_voxel(plan, voxel_size, (const float*)d, (VoxCloud*)(d + o_tab), d + o_scr,
                                (float*)(d + o_out), (int*)(d + o_vo), st,
                                with_colors ? (const float*)(d + o_col) : nullptr,
                                with_colors ? (float*)(d + o_cout) : nullptr);
  if ((rc = check_launch(ctx, "voxel launch")) != TZR_OK) return rc;
  CK(cudaMemcpyAsync(clouds.data(), d + o_tab, tb, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const size_t rows = (size_t)clouds[B - 1].out_lo + (size_t)clouds[B - 1].n_out;
  spans.clear();
  for (int b = 0; b < B; ++b) {
    const VoxCloud& c = clouds[b];
    spans.push_back(CopySpan{pts_out[b], h + o_out + (size_t)c.out_lo * 12, (size_t)c.n_out * 12});
    if (with_colors)
      spans.push_back(CopySpan{colors_out[b], h + o_cout + (size_t)c.out_lo * 12, (size_t)c.n_out * 12});
    if (voxel_of && voxel_of[b]) spans.push_back(CopySpan{voxel_of[b], h + o_vo + (size_t)c.lo * 4, (size_t)c.n * 4});
  }
  if (B == 1) {  // straight into the caller's buffers
    for (const CopySpan& s : spans)
      if (s.bytes) CK(cudaMemcpyAsync(s.dst, d + ((const char*)s.src - h), s.bytes, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  } else {
    if (rows) CK(cudaMemcpyAsync(h + o_out, d + o_out, rows * 12, cudaMemcpyDeviceToHost, st));
    if (rows && with_colors) CK(cudaMemcpyAsync(h + o_cout, d + o_cout, rows * 12, cudaMemcpyDeviceToHost, st));
    if (want_trace) CK(cudaMemcpyAsync(h + o_vo, d + o_vo, N * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    parallel_copy(spans);
  }
  bool too_large = false;
  for (int b = 0; b < B; ++b) {
    n_out[b] = clouds[b].n_out;
    if (status) status[b] = clouds[b].status;
    too_large |= clouds[b].status != TZR_OK;
  }
  if (too_large) {
    ctx->last_error = "a cloud's voxel grid is too large for the voxel size (Open3D's INT_MAX check or 2^62 cells)";
    return TZR_ERR_TOO_LARGE;
  }
  return TZR_OK;
}

int tzr_voxel_downsample_batch(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts, double voxel_size,
                               float* const* pts_out, int32_t* n_out, int32_t* const* voxel_of, int32_t* status) {
  return voxel_run(ctx, B, n, pts, voxel_size, pts_out, n_out, voxel_of, status, nullptr, nullptr, false);
}

int tzr_voxel_downsample_colors_batch(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts,
                                      double voxel_size, float* const* pts_out, int32_t* n_out,
                                      int32_t* const* voxel_of, int32_t* status, const float* const* colors,
                                      float* const* colors_out) {
  return voxel_run(ctx, B, n, pts, voxel_size, pts_out, n_out, voxel_of, status, colors, colors_out, true);
}

int tzr_voxel_downsample_colors(tzr_ctx* ctx, const float* pts, int n, double voxel_size, float* pts_out,
                                int32_t* n_out, int32_t* voxel_of, const float* colors, float* colors_out) {
  const int32_t n1 = n;
  int32_t* const vo[1] = {voxel_of};
  return tzr_voxel_downsample_colors_batch(ctx, 1, &n1, &pts, voxel_size, &pts_out, n_out, vo, nullptr, &colors,
                                           &colors_out);
}

int tzr_voxel_downsample(tzr_ctx* ctx, const float* pts, int n, double voxel_size, float* pts_out, int32_t* n_out,
                         int32_t* voxel_of) {
  const int32_t n1 = n;
  int32_t* const vo[1] = {voxel_of};
  return tzr_voxel_downsample_batch(ctx, 1, &n1, &pts, voxel_size, &pts_out, n_out, vo, nullptr);
}

int tzr_fpfh_pair_features(tzr_ctx* ctx, int n, const float* p1, const float* n1, const float* p2, const float* n2,
                           float* f_out, int32_t* ok_out) {
  if (!ctx || n <= 0 || !p1 || !n1 || !p2 || !n2 || !f_out || !ok_out) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t vb = (size_t)n * 12;
  int rc;
  if ((rc = ensure(ctx, ctx->m_in, 4 * al256(vb))) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->m_out, al256(vb) + (size_t)n * 4)) != TZR_OK) return rc;
  char* d_in = (char*)ctx->m_in.p;
  const float* h_in[4] = {p1, n1, p2, n2};
  for (int k = 0; k < 4; ++k) CK(cudaMemcpyAsync(d_in + k * al256(vb), h_in[k], vb, cudaMemcpyHostToDevice, st));
  float* d_f = (float*)ctx->m_out.p;
  int32_t* d_ok = (int32_t*)((char*)ctx->m_out.p + al256(vb));
  launch_fpfh_pair_features(n, (const float*)d_in, (const float*)(d_in + al256(vb)),
                            (const float*)(d_in + 2 * al256(vb)), (const float*)(d_in + 3 * al256(vb)), d_f, d_ok, st);
  ctx->launches += 1;
  if ((rc = check_launch(ctx, "pair features launch")) != TZR_OK) return rc;
  CK(cudaMemcpyAsync(f_out, d_f, vb, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(ok_out, d_ok, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return TZR_OK;
}

int tzr_fpfh_smallest_eigenpair(tzr_ctx* ctx, int n, const float* cov, float* ev_out, float* vec_out) {
  if (!ctx || n <= 0 || !cov || !ev_out || !vec_out) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  const size_t cb = (size_t)n * 36, eb = (size_t)n * 4, vb = (size_t)n * 12;
  int rc;
  if ((rc = ensure(ctx, ctx->m_in, cb)) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->m_out, al256(eb) + vb)) != TZR_OK) return rc;
  float* d_cov = (float*)ctx->m_in.p;
  float* d_ev = (float*)ctx->m_out.p;
  float* d_vec = (float*)((char*)ctx->m_out.p + al256(eb));
  CK(cudaMemcpyAsync(d_cov, cov, cb, cudaMemcpyHostToDevice, st));
  launch_fpfh_smallest_eigenpair(n, d_cov, d_ev, d_vec, st);
  ctx->launches += 1;
  if ((rc = check_launch(ctx, "smallest eigenpair launch")) != TZR_OK) return rc;
  CK(cudaMemcpyAsync(ev_out, d_ev, eb, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(vec_out, d_vec, vb, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return TZR_OK;
}

int tzr_feature_nn(tzr_ctx* ctx, const float* query, int nq, const float* db, int ndb, int dim, int32_t* nn_index,
                   float* nn_dist) {
  if (!ctx || !query || !db || !nn_index || nq <= 0 || ndb <= 0 || dim < 1 || dim > kMatchMaxDim)
    return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  cudaStream_t st = ctx->stream;
  auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t qb = (size_t)nq * dim * 4, dbb = (size_t)ndb * dim * 4;
  std::vector<NnWork> work;  // ~4 CTAs per SM
  const long long tile_pairs = (long long)((nq + 63) / 64) * ((ndb + 63) / 64);
  nn_work_append(&work, 0, 0, nq, 0, ndb, nn_tiles_per_seg(tile_pairs, 4 * ctx->num_sms));
  const size_t wb = work.size() * sizeof(NnWork);
  int rc;
  if ((rc = ensure(ctx, ctx->m_in, al(qb) + al(dbb) + wb)) != TZR_OK) return rc;
  if ((rc = ensure(ctx, ctx->m_out, (size_t)nq * 8)) != TZR_OK) return rc;
  float* d_q = (float*)ctx->m_in.p;
  float* d_db = (float*)((char*)ctx->m_in.p + al(qb));
  NnWork* d_work = (NnWork*)((char*)ctx->m_in.p + al(qb) + al(dbb));
  unsigned long long* d_best = (unsigned long long*)ctx->m_out.p;
  CK(cudaMemcpyAsync(d_q, query, qb, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_db, db, dbb, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d_work, work.data(), wb, cudaMemcpyHostToDevice, st));
  ctx->launches += launch_feature_nn(d_work, (int)work.size(), d_q, d_db, dim, d_best, nullptr, nq, st);
  if ((rc = check_launch(ctx, "feature nn launch")) != TZR_OK) return rc;
  std::vector<unsigned long long> h((size_t)nq);
  CK(cudaMemcpyAsync(h.data(), d_best, (size_t)nq * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  for (int q = 0; q < nq; ++q) {
    nn_index[q] = (int32_t)(h[q] & 0xffffffffu);
    if (nn_dist) {
      const uint32_t bits = (uint32_t)(h[q] >> 32);
      memcpy(&nn_dist[q], &bits, 4);
    }
  }
  return TZR_OK;
}

static int sum_stage_events(tzr_ctx* ctx, int c0, int c1, int g0, int g1, double acc[4]) {
  for (int i = 0; i < 4; ++i) acc[i] = 0;
  for (int c = c0; c < c1; ++c)
    for (int i = 0; i < 4; ++i) {
      float ms = 0;
      if (cudaEventElapsedTime(&ms, ctx->stage_ev[5 * c + i], ctx->stage_ev[5 * c + i + 1]) != cudaSuccess)
        return TZR_ERR_CUDA;
      acc[i] += ms;
    }
  // graph = the graph kernel launches alone (operand tiles + tensor-core kernel + strip kernel); the interleaved degree
  // launches are booked under "clique"
  double g = 0;
  for (int k = g0; k + 1 < g1; k += 2) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, ctx->graph_ev[k], ctx->graph_ev[k + 1]) != cudaSuccess) return TZR_ERR_CUDA;
    g += ms;
  }
  if (g1 > g0) {
    acc[2] += acc[1] - g;
    acc[1] = g;
  }
  return TZR_OK;
}

int tzr_last_stage_ms(tzr_ctx* ctx, double* prep_ms, double* graph_ms, double* clique_ms, double* rot_trans_ms) {
  if (!ctx || ctx->last.at.empty()) return TZR_ERR_INVALID_ARG;
  double acc[4];
  const int rc = sum_stage_events(ctx, ctx->stage_first, ctx->stage_chunks, ctx->graph_first, ctx->graph_ev_used, acc);
  if (rc) return rc;
  double* outs[4] = {prep_ms, graph_ms, clique_ms, rot_trans_ms};
  for (int i = 0; i < 4; ++i)
    if (outs[i]) *outs[i] = acc[i];
  return TZR_OK;
}

int tzr_ctx_stage_log(tzr_ctx* ctx, int enable) {
  if (!ctx) return TZR_ERR_INVALID_ARG;
  ctx->stage_log = enable != 0;
  ctx->stage_chunks = ctx->stage_first = 0;
  ctx->graph_ev_used = ctx->graph_first = 0;
  ctx->stage_log_calls = 0;
  return TZR_OK;
}

int tzr_ctx_stage_log_read(tzr_ctx* ctx, double* sums_ms4, int32_t* n_calls) {
  if (!ctx || !sums_ms4) return TZR_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  CK(cudaStreamSynchronize(ctx->stream));
  const int rc = sum_stage_events(ctx, 0, ctx->stage_chunks, 0, ctx->graph_ev_used, sums_ms4);
  if (rc) return rc;
  if (n_calls) *n_calls = ctx->stage_log_calls;
  ctx->stage_chunks = ctx->stage_first = 0;
  ctx->graph_ev_used = ctx->graph_first = 0;
  ctx->stage_log_calls = 0;
  return TZR_OK;
}

// ------------------------------------------------------------------------------------------------
// multi-GPU fan-out inside the library: one context + one host thread per device, contiguous shards balanced by
// sum n_b^2 (the graph stage dominates), no collective (SURVEY §8e).
// ------------------------------------------------------------------------------------------------
namespace {
struct DevicePool {
  std::mutex mu;
  std::map<int, tzr_ctx*> ctxs;
  ~DevicePool() {
    for (auto& kv : ctxs) tzr_ctx_destroy(kv.second);
  }
};
DevicePool& device_pool() {
  static DevicePool pool;
  return pool;
}
}  // namespace

int tzr_solve_batch_multi(const int32_t* devices, int n_devices, const tzr_params* params, int B, const int32_t* n,
                          const double* const* src, const double* const* dst, tzr_solution* solutions,
                          int32_t* cliques, int max_n) {
  if (!params || !n || !src || !dst || !solutions || B <= 0) return TZR_ERR_INVALID_ARG;
  std::vector<int> devs;
  if (!devices || n_devices <= 0) {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) return TZR_ERR_NO_DEVICE;
    for (int d = 0; d < count; ++d) devs.push_back(d);
  } else {
    devs.assign(devices, devices + n_devices);
  }
  DevicePool& pool = device_pool();
  std::lock_guard<std::mutex> lock(pool.mu);
  for (int d : devs)
    if (!pool.ctxs.count(d)) {
      tzr_ctx* c = nullptr;
      const int rc = tzr_ctx_create(d, &c);
      if (rc) return rc;
      pool.ctxs[d] = c;
    }
  const int G = std::min<int>((int)devs.size(), B);
  // contiguous shards with balanced sum n^2
  std::vector<double> cum(B + 1, 0.0);
  for (int b = 0; b < B; ++b) cum[b + 1] = cum[b] + (double)n[b] * (double)n[b];
  std::vector<int> cut(G + 1, 0);
  cut[G] = B;
  for (int g = 1; g < G; ++g) {
    const double target = cum[B] * g / G;
    int b = cut[g - 1] + 1;  // at least one problem per shard
    while (b < B - (G - g) && cum[b] < target) ++b;
    cut[g] = b;
  }
  std::vector<int> rcs(G, TZR_OK);
  std::vector<std::thread> threads;
  for (int g = 0; g < G; ++g) {
    threads.emplace_back([&, g] {
      const int b0 = cut[g], Bg = cut[g + 1] - cut[g];
      if (Bg <= 0) return;
      rcs[g] = tzr_solve_batch(pool.ctxs[devs[g]], params, Bg, n + b0, src + b0, dst + b0, solutions + b0,
                               cliques ? cliques + (size_t)b0 * max_n : nullptr, max_n);
    });
  }
  for (auto& t : threads) t.join();
  for (int g = 0; g < G; ++g)
    if (rcs[g]) return rcs[g];
  return TZR_OK;
}

}  // extern "C"

// dpgo_capi.cu -- implementation of the C ABI in include/dpgo_b200.h, part 1 of 4: error state, devices, the handle's
// lifecycle, Q and G (CSR -> block-CSR conversion, the launch tables), evaluation, the optimiser, X transfer and the
// diagnostics.  The exact preconditioners are in dpgo_capi_precond.cu, the edge records and robust re-weighting in
// dpgo_capi_edges.cu, the per-agent and batched multi-agent calls in dpgo_capi_agents.cu; dpgo_handle.cuh is what they
// share.  No CPU compute fallback exists here: every numeric entry point runs the sm_90a kernels.
#include <cuda_runtime.h>
#include <algorithm>
#include <chrono>
#include <cstring>
#include <numeric>
#include <string>
#include <vector>

#include "dpgo_handle.cuh"

namespace dpgo::capi {
namespace {

thread_local std::string g_last_error;

void fill_kparams(const dpgo_problem *p, dpgo::KParams &kp, int op, const dpgo_opt_params_t &prm) {
  kp.n = p->n;
  kp.N = p->N;
  kp.grid = p->grid;
  kp.op = op;
  kp.rowptr = p->bsr.rowptr.get();
  kp.bcol = p->bsr.bcol.get();
  kp.bval = p->bsr.bval.get();
  kp.dinv = p->bsr.dinv.get();
  kp.cta_rows = p->bsr.cta_rows.get();
  kp.G = p->G.get();
  for (int i = 0; i < dpgo::V_COUNT; ++i) kp.v[i] = p->vec[i].get();
  for (int i = 0; i < 2; ++i) kp.S[i] = p->S[i].get();
  kp.partials = p->bsr.partials.get();
  kp.bar_counter = p->bar.get();
  kp.bar_epoch = p->bar.get() + 1;
  const dpgo_problem::Nd &F = p->nd[nd_slot(prm.precond)];
  kp.nd = F.k;
  if (!F.ready) kp.nd.nphases = 0;
  kp.cluster = p->cluster ? 1 : 0;
  kp.smem_doubles = 0;
  kp.phase_ns = p->phase_ns.get();
  kp.opt_record = p->status.opt_record.get();
  kp.gate = p->gate;
  kp.prm = prm;
  kp.result = p->result.get();
}

cudaError_t run_spmv(const dpgo_problem *p, const double *X, const double *G, double *out) {
  if (p->bsr.ngroups > 0)
    return dpgo::launch_spmv_tma(p->r, p->dh, p->bsr.ngroups, p->bsr.groups.get(), p->bsr.rowptr.get(), p->bsr.bcol.get(),
                                 p->bsr.bval.get(), X, G, out, p->sms, p->stream);
  return dpgo::launch_spmv(p->r, p->dh, p->n, p->bsr.rowptr.get(), p->bsr.bcol.get(), p->bsr.bval.get(), X, G, out, p->stream);
}

int check_precond(dpgo_problem *p, int precond) {
  if (precond < 0 || precond > 3) return fail(DPGO_ERR_INVALID_ARG, "unknown preconditioner id");
  if (precond == DPGO_PRECOND_SPARSE_EXACT || precond == DPGO_PRECOND_DENSE_EXACT) return ensure_nd(p, nd_slot(precond));
  if (precond == DPGO_PRECOND_BLOCK_JACOBI && !p->bsr.dinv)
    return fail(DPGO_ERR_STATE, "block-Jacobi preconditioner was not prepared by set_Q (precond_mask)");
  return DPGO_OK;
}

int run_op(dpgo_problem *p, int op, const dpgo_opt_params_t &prm) {
  DPGO_REQUIRE(p->bsr.have, DPGO_ERR_STATE, "set_Q has not been called");
  dpgo::KParams kp;
  fill_kparams(p, kp, op, prm);
  DPGO_CUDA(dpgo::launch_optimize(p->r, p->dh, kp, p->stream));
  return DPGO_OK;
}

int fetch_result(dpgo_problem *p) {
  DPGO_CUDA(cudaMemcpyAsync(p->h_result.get(), p->result.get(), sizeof(dpgo_opt_result_t), cudaMemcpyDeviceToHost, p->stream));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return check_refactor_fail(p);
}

// The parameters of the single-operation entry points: the defaults, without a preconditioner.
dpgo_opt_params_t plain_params() {
  dpgo_opt_params_t prm;
  dpgo_opt_params_default(&prm);
  prm.precond = DPGO_PRECOND_NONE;
  return prm;
}

int eval_at(dpgo_problem_t *p, const double *X_host) {
  DPGO_REQUIRE(X_host, DPGO_ERR_INVALID_ARG, "null X");
  DPGO_TRY(upload_vec(p, dpgo::V_X0, X_host));
  DPGO_TRY(run_op(p, dpgo::OP_EVAL, plain_params()));
  return DPGO_OK;
}

}  // namespace

int fail(int code, const std::string &msg) {
  g_last_error = msg;
  return code;
}

int require_device(int device) {
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
    cudaGetLastError();
    return fail(DPGO_ERR_NO_DEVICE, "no CUDA device available: the GPU path has no CPU fallback");
  }
  DPGO_REQUIRE(device >= 0 && device < count, DPGO_ERR_NO_DEVICE, "device index out of range");
  return DPGO_OK;
}

// ---- host-side block assembly ---------------------------------------------------------------
// block triplets -> block-CSR (rows = output tiles, duplicates summed in a fixed order)
void assemble_bsr(int n, const std::vector<BlockTriplet> &trip, std::vector<int> &rowptr, std::vector<int> &bcol,
                  std::vector<double> &bval) {
  // sort by (output tile = bcol, neighbour tile = brow); stable so duplicate summation order is fixed
  std::vector<int64_t> order(trip.size());
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int64_t x, int64_t y) {
    if (trip[x].bcol != trip[y].bcol) return trip[x].bcol < trip[y].bcol;
    return trip[x].brow < trip[y].brow;
  });
  rowptr.assign((size_t)n + 1, 0);
  bcol.clear();
  bval.clear();
  bcol.reserve(trip.size());
  bval.reserve(trip.size() * 16);
  int last_j = -1, last_i = -1;
  for (int64_t o : order) {
    const BlockTriplet &t = trip[o];
    if (t.bcol == last_j && t.brow == last_i) {
      double *dst = &bval[bval.size() - 16];
      for (int e = 0; e < 16; ++e) dst[e] += t.v[e];
    } else {
      bcol.push_back(t.brow);
      bval.insert(bval.end(), t.v, t.v + 16);
      rowptr[t.bcol + 1]++;
      last_j = t.bcol;
      last_i = t.brow;
    }
  }
  for (int j = 0; j < n; ++j) rowptr[j + 1] += rowptr[j];
}

int blocks_to_triplets(int n, int dh, int64_t nb, const int32_t *brow, const int32_t *bcol, const double *blocks,
                       std::vector<BlockTriplet> &trip) {
  trip.assign((size_t)nb, BlockTriplet{});
  for (int64_t q = 0; q < nb; ++q) {
    if (brow[q] < 0 || brow[q] >= n || bcol[q] < 0 || bcol[q] >= n)
      return fail(DPGO_ERR_INVALID_ARG, "block index out of range");
    trip[(size_t)q].brow = brow[q];
    trip[(size_t)q].bcol = bcol[q];
    for (int k = 0; k < dh; ++k)
      for (int c = 0; c < dh; ++c) trip[(size_t)q].v[k * 4 + c] = blocks[(size_t)q * dh * dh + k * dh + c];
  }
  return DPGO_OK;
}

int build_from_triplets(dpgo_problem *p, std::vector<BlockTriplet> &trip, unsigned precond_mask) {
  const int n = p->n, dh = p->dh;
  std::vector<int> rowptr, bcol;
  std::vector<double> bval;
  assemble_bsr(n, trip, rowptr, bcol, bval);
  const int64_t nb = (int64_t)bcol.size();

  std::vector<double> dinv;
  if (precond_mask & (1u << DPGO_PRECOND_BLOCK_JACOBI)) jacobi_blocks(n, dh, rowptr, bcol, bval, dinv);

  // persistent-kernel grid and balanced row partition
  const int sg = (p->r > 4) ? 32 : ((p->r > 2) ? 16 : 8);
  const int rows_per_pass = (dpgo::OPT_THREADS / 32) * (32 / sg);
  int grid = p->max_grid;
  const bool dense = (precond_mask & ((1u << DPGO_PRECOND_DENSE_EXACT) | (1u << DPGO_PRECOND_SPARSE_EXACT))) != 0;
  if (!dense) grid = std::max(1, std::min(grid, (n + rows_per_pass - 1) / rows_per_pass));
  // Launch mode 1 (dpgo_problem_set_launch_mode): the step kernel runs as ONE thread-block cluster (<= 16 CTAs) whose
  // phase ends are hardware cluster barriers instead of the atomic-counter grid barrier.  For one agent alone this is
  // SLOWER than the full grid (10-16 SMs stream the preconditioner blocks more slowly than all of them;
  // scripts/phase_times.py --agents 8 / 16 compares the two); its point is that a cluster launch is not cooperative, so
  // the agents of a colour class run side by side on one GPU and the round captures into a CUDA graph
  // (dpgo_agents_round_async).
  p->cluster = false;
  if (p->max_cluster >= 8 && p->launch_mode == 1) {
    // (one CTA per 16 poses is enough: always taking 16 CTAs makes small agents slower)
    grid = std::max(1, std::min(p->max_cluster, (n + rows_per_pass - 1) / rows_per_pass));
    p->cluster = true;
  }
  std::vector<int> cta_rows(grid + 1, 0);
  {
    // cost model: blocks + constant epilogue weight per row
    const double wrow = 4.0;
    double total = 0.0;
    for (int j = 0; j < n; ++j) total += (rowptr[j + 1] - rowptr[j]) + wrow;
    double accw = 0.0;
    int ci = 1;
    for (int j = 0; j < n; ++j) {
      accw += (rowptr[j + 1] - rowptr[j]) + wrow;
      while (ci < grid && accw >= total * ci / grid) cta_rows[ci++] = j + 1;
    }
    while (ci <= grid) cta_rows[ci++] = n;
  }

  // upload
  cudaSetDevice(p->device);
  p->bsr = {};
  free_nd(p);
  dpgo_problem::BlockQ &B = p->bsr;
  B.h_rowptr = rowptr;
  B.h_bcol = bcol;
  B.h_bval = bval;
  // +8 ints of slack: the bulk-TMA windows are rounded out to 16 bytes
  DPGO_CUDA(B.rowptr.alloc((size_t)n + 1 + 8));
  DPGO_CUDA(B.bcol.alloc((size_t)std::max<int64_t>(nb, 1) + 8));
  DPGO_CUDA(cudaMemsetAsync(B.rowptr.get(), 0, sizeof(int) * (n + 1 + 8), p->stream));
  DPGO_CUDA(cudaMemsetAsync(B.bcol.get(), 0, sizeof(int) * (std::max<int64_t>(nb, 1) + 8), p->stream));
  DPGO_CUDA(B.bval.alloc(16 * (size_t)std::max<int64_t>(nb, 1)));
  DPGO_CUDA(B.cta_rows.assign(cta_rows.data(), cta_rows.size(), p->stream));
  DPGO_CUDA(B.partials.alloc((size_t)2 * grid * dpgo::NRED));
  DPGO_CUDA(B.rowptr.upload(rowptr.data(), (size_t)n + 1, p->stream));
  DPGO_CUDA(B.bcol.upload(bcol.data(), (size_t)nb, p->stream));
  DPGO_CUDA(B.bval.upload(bval.data(), 16 * (size_t)nb, p->stream));
  DPGO_CUDA(cudaMemsetAsync(B.partials.get(), 0, sizeof(double) * 2 * grid * dpgo::NRED, p->stream));
  if (!dinv.empty()) DPGO_CUDA(B.dinv.assign(dinv.data(), dinv.size(), p->stream));
  // row groups for the TMA-fed SpMV: consecutive rows, <= SPMV_GROUP_BLOCKS blocks and rows each
  {
    const int BT = dpgo::spmv_group_blocks();
    std::vector<int2> groups;
    bool ok = true;
    int rr = 0;
    while (rr < n) {
      const int start = rr;
      int blocks = 0;
      while (rr < n && (rr - start) < BT && blocks + (rowptr[rr + 1] - rowptr[rr]) <= BT) {
        blocks += rowptr[rr + 1] - rowptr[rr];
        ++rr;
      }
      if (rr == start) { ok = false; break; }        // a single row exceeds the stage: fall back to the gather kernel
      groups.push_back(make_int2(start, rowptr[start]));
    }
    if (ok && nb > 0) {
      groups.push_back(make_int2(n, (int)nb));
      DPGO_CUDA(B.groups.assign(groups.data(), groups.size(), p->stream));
      B.ngroups = (int)groups.size() - 1;
    }
  }
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  B.nb = nb;
  p->grid = grid;
  B.precond_mask = precond_mask;

  B.have = true;
  return DPGO_OK;
}

int upload_vec(dpgo_problem *p, int id, const double *host) {
  DPGO_CUDA(cudaMemcpyAsync(p->vec[id].get(), host, p->vec_bytes(), cudaMemcpyHostToDevice, p->stream));
  return DPGO_OK;
}
int download_vec(dpgo_problem *p, int id, double *host) {
  DPGO_CUDA(cudaMemcpyAsync(host, p->vec[id].get(), p->vec_bytes(), cudaMemcpyDeviceToHost, p->stream));
  return DPGO_OK;
}

// After the stream has been synchronised: report (once) a device refactorisation that met a matrix that was not positive
// definite.  Only read when an asynchronous re-weight ran since the last read.
int check_refactor_fail(dpgo_problem *p) {
  dpgo_problem::Edges &E = p->edges;
  if (!E.fail_armed) return DPGO_OK;
  E.fail_armed = false;
  int flag = 0;
  DPGO_CUDA(cudaMemcpy(&flag, E.fail.get(), sizeof(int), cudaMemcpyDeviceToHost));
  if (!flag) return DPGO_OK;
  DPGO_CUDA(cudaMemset(E.fail.get(), 0, sizeof(int)));
  return fail(DPGO_ERR_CUDA, "device refactorisation: Q + 0.1 I is not positive definite (negative edge weight?)");
}

int check_params(dpgo_problem *p, const dpgo_opt_params_t *prm) {
  DPGO_REQUIRE(prm, DPGO_ERR_INVALID_ARG, "null params");
  DPGO_REQUIRE(prm->algorithm == DPGO_ALG_RTR || prm->algorithm == DPGO_ALG_RGD, DPGO_ERR_INVALID_ARG, "unknown algorithm");
  DPGO_REQUIRE(prm->tr_iterations >= 1 && prm->tr_max_inner >= 1, DPGO_ERR_INVALID_ARG, "iteration counts must be >= 1");
  DPGO_REQUIRE(prm->tr_initial_radius > 0 && prm->tr_tolerance >= 0, DPGO_ERR_INVALID_ARG, "bad radius / tolerance");
  if (prm->algorithm == DPGO_ALG_RTR) DPGO_TRY(check_precond(p, prm->precond));
  return DPGO_OK;
}

}  // namespace dpgo::capi

using namespace dpgo::capi;

extern "C" {

int dpgo_abi_version(void) { return DPGO_B200_ABI_VERSION; }
const char *dpgo_last_error(void) { return g_last_error.c_str(); }

int dpgo_device_count(int *count) {
  DPGO_REQUIRE(count, DPGO_ERR_INVALID_ARG, "null count");
  int c = 0;
  cudaError_t e = cudaGetDeviceCount(&c);
  if (e != cudaSuccess) {
    *count = 0;
    return fail(DPGO_ERR_NO_DEVICE, std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e));
  }
  *count = c;
  return DPGO_OK;
}

void dpgo_opt_params_default(dpgo_opt_params_t *p) {
  if (!p) return;
  p->algorithm = DPGO_ALG_RTR;        // ref: src/QuadraticOptimizer.cpp:22-28
  p->tr_iterations = 1;
  p->tr_max_inner = 50;
  p->precond = DPGO_PRECOND_SPARSE_EXACT;
  p->rgd_stepsize = 1e-3;
  p->tr_tolerance = 1e-2;
  p->tr_initial_radius = 1e1;
}

int dpgo_problem_create(int n, int d, int r, int device, dpgo_problem_t **out) {
  DPGO_REQUIRE(out, DPGO_ERR_INVALID_ARG, "null output handle");
  *out = nullptr;
  DPGO_REQUIRE(n >= 1, DPGO_ERR_INVALID_ARG, "n must be >= 1");
  DPGO_REQUIRE(n <= 100000000, DPGO_ERR_UNSUPPORTED, "n above 1e8 poses: element offsets are 32-bit in the kernels");
  DPGO_REQUIRE(d == 2 || d == 3, DPGO_ERR_UNSUPPORTED, "d must be 2 or 3");
  DPGO_REQUIRE(r >= d, DPGO_ERR_INVALID_ARG, "r must be >= d (ref: assert(r >= d), src/QuadraticProblem.cpp:19)");
  DPGO_REQUIRE(r <= DPGO_MAX_RANK, DPGO_ERR_UNSUPPORTED,
               "r must be <= 8 (DPGO_MAX_RANK: the lifted rows of a pose tile are the 8 rows of an fp64 MMA fragment)");
  DPGO_TRY(require_device(device));
  DPGO_CUDA(cudaSetDevice(device));
  dpgo_problem *p = new (std::nothrow) dpgo_problem();
  if (!p) return fail(DPGO_ERR_ALLOC, "host allocation failed");
  p->n = n; p->d = d; p->r = r; p->dh = d + 1; p->N = (d + 1) * n; p->ts = r * (d + 1);
  {
    static uint64_t serial = 0;             // handles are created from one thread at a time (as the rest of this API)
    p->generation = (++serial) << 24;       // a recycled address never matches the key of a captured round
  }
  p->device = device;
  auto bail = [&](int code, const std::string &m) { dpgo_problem_destroy(p); return fail(code, m); };
  if (cudaDeviceGetAttribute(&p->sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess)
    return bail(DPGO_ERR_CUDA, "cudaDeviceGetAttribute failed");
  cudaStream_t own = nullptr;
  const cudaError_t se = cudaStreamCreateWithFlags(&own, cudaStreamNonBlocking);
  p->own_stream.reset(own);
  if (se != cudaSuccess) return bail(DPGO_ERR_CUDA, "cudaStreamCreate failed");
  p->stream = own;
  p->max_grid = dpgo::optimize_max_grid(r, d + 1, device);
  p->max_cluster = dpgo::optimize_max_cluster(r, d + 1, device);
  if (p->max_grid <= 0) return bail(DPGO_ERR_CUDA, "persistent kernel cannot be made resident on this device");
  const size_t vb = p->vec_bytes();
  for (int i = 0; i < dpgo::V_COUNT; ++i) {
    if (p->vec[i].alloc((size_t)r * p->N) != cudaSuccess) return bail(DPGO_ERR_ALLOC, "device allocation failed (vectors)");
    cudaMemsetAsync(p->vec[i].get(), 0, vb, p->stream);
  }
  if (p->G.alloc((size_t)r * p->N) != cudaSuccess) return bail(DPGO_ERR_ALLOC, "device allocation failed (G)");
  cudaMemsetAsync(p->G.get(), 0, vb, p->stream);
  for (int i = 0; i < 2; ++i) {
    if (p->S[i].alloc(9 * (size_t)n) != cudaSuccess) return bail(DPGO_ERR_ALLOC, "device allocation failed (S)");
    cudaMemsetAsync(p->S[i].get(), 0, sizeof(double) * 9 * (size_t)n, p->stream);
  }
  if (p->bar.alloc(2) != cudaSuccess) return bail(DPGO_ERR_ALLOC, "device allocation failed");
  cudaMemsetAsync(p->bar.get(), 0, 2 * sizeof(unsigned), p->stream);
  if (p->result.alloc(1) != cudaSuccess) return bail(DPGO_ERR_ALLOC, "device allocation failed");
  if (p->status.opt_record.alloc(2) != cudaSuccess || p->status.part.alloc(3 * (size_t)dpgo::status_ctas(n)) != cudaSuccess ||
      p->status.ticket.alloc(1) != cudaSuccess)
    return bail(DPGO_ERR_ALLOC, "device allocation failed (status)");
  cudaMemsetAsync(p->status.opt_record.get(), 0, 2 * sizeof(double), p->stream);
  cudaMemsetAsync(p->status.ticket.get(), 0, sizeof(unsigned), p->stream);
  dpgo_opt_result_t *pinned = nullptr;
  const cudaError_t he = cudaMallocHost(&pinned, sizeof(dpgo_opt_result_t));
  p->h_result.reset(pinned);
  if (he != cudaSuccess) return bail(DPGO_ERR_ALLOC, "pinned allocation failed");
  if (cudaStreamSynchronize(p->stream) != cudaSuccess) return bail(DPGO_ERR_CUDA, "device initialisation failed");
  // empty Q (ref: ctor calls setQ(SparseMatrix(N,N)), src/QuadraticProblem.cpp:23)
  std::vector<BlockTriplet> none;
  int s = build_from_triplets(p, none, 1u << DPGO_PRECOND_BLOCK_JACOBI);
  if (s != DPGO_OK) { std::string m = g_last_error; dpgo_problem_destroy(p); return fail(s, m); }
  *out = p;
  return DPGO_OK;
}

int dpgo_problem_destroy(dpgo_problem_t *p) {
  if (!p) return DPGO_OK;
  cudaSetDevice(p->device);
  if (p->stream) cudaStreamSynchronize(p->stream);
  delete p;
  return DPGO_OK;
}

int dpgo_problem_set_stream(dpgo_problem_t *p, void *cuda_stream) {
  DPGO_CHECK_HANDLE(p);
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  p->stream = cuda_stream ? (cudaStream_t)cuda_stream : p->own_stream.get();
  return DPGO_OK;
}

int dpgo_problem_sync(dpgo_problem_t *p) {
  DPGO_CHECK_HANDLE(p);
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return check_refactor_fail(p);
}

int dpgo_problem_set_launch_mode(dpgo_problem_t *p, int mode) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(mode >= -1 && mode <= 1, DPGO_ERR_INVALID_ARG, "launch mode must be -1 (default), 0 (grid) or 1 (cluster)");
  DPGO_REQUIRE(mode != 1 || p->max_cluster >= 8, DPGO_ERR_UNSUPPORTED, "this device cannot co-schedule a cluster of >= 8 CTAs of the step kernel");
  p->launch_mode = mode;
  return DPGO_OK;
}

int dpgo_problem_launch_info(const dpgo_problem_t *p, int *grid, int *cluster) {
  DPGO_REQUIRE(p, DPGO_ERR_INVALID_ARG, "null problem handle");
  if (grid) *grid = p->grid;
  if (cluster) *cluster = p->cluster ? 1 : 0;
  return DPGO_OK;
}

int dpgo_problem_dims(const dpgo_problem_t *p, int *n, int *d, int *r, int64_t *num_blocks) {
  DPGO_REQUIRE(p, DPGO_ERR_INVALID_ARG, "null problem handle");
  if (n) *n = p->n;
  if (d) *d = p->d;
  if (r) *r = p->r;
  if (num_blocks) *num_blocks = p->bsr.nb;
  return DPGO_OK;
}

int dpgo_problem_set_Q_csr(dpgo_problem_t *p, int nrows, const int32_t *rowptr, const int32_t *colind,
                           const double *values, unsigned precond_mask) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(nrows == p->N, DPGO_ERR_INVALID_ARG, "Q must be (d+1)n x (d+1)n");
  DPGO_REQUIRE(rowptr, DPGO_ERR_INVALID_ARG, "null CSR row pointer");
  DPGO_REQUIRE(rowptr[0] == 0, DPGO_ERR_INVALID_ARG, "CSR row pointer must start at 0");
  for (int i = 0; i < nrows; ++i)
    if (rowptr[i + 1] < rowptr[i]) return fail(DPGO_ERR_INVALID_ARG, "CSR row pointer is not non-decreasing");
  DPGO_REQUIRE(rowptr[nrows] == 0 || (colind && values), DPGO_ERR_INVALID_ARG, "null CSR arrays");
  const int dh = p->dh;
  std::vector<BlockTriplet> trip;
  trip.reserve((size_t)rowptr[nrows] / (dh * dh) + 16);
  for (int ib = 0; ib < p->n; ++ib) {
    const size_t first = trip.size();
    for (int k = 0; k < dh; ++k) {
      const int rr = ib * dh + k;
      for (int q = rowptr[rr]; q < rowptr[rr + 1]; ++q) {
        const int cc = colind[q];
        if (cc < 0 || cc >= p->N) return fail(DPGO_ERR_INVALID_ARG, "column index out of range");
        const int jb = cc / dh, c = cc - jb * dh;
        size_t t = first;
        for (; t < trip.size(); ++t)
          if (trip[t].bcol == jb) break;
        if (t == trip.size()) {
          BlockTriplet bt;
          bt.brow = ib;
          bt.bcol = jb;
          std::memset(bt.v, 0, sizeof(bt.v));
          trip.push_back(bt);
        }
        trip[t].v[k * 4 + c] += values[q];
      }
    }
  }
  return build_from_triplets(p, trip, precond_mask);
}

int dpgo_problem_set_Q_blocks(dpgo_problem_t *p, int64_t nb, const int32_t *brow, const int32_t *bcol,
                              const double *blocks, unsigned precond_mask) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(nb >= 0 && (nb == 0 || (brow && bcol && blocks)), DPGO_ERR_INVALID_ARG, "null block arrays");
  std::vector<BlockTriplet> trip;
  DPGO_TRY(blocks_to_triplets(p->n, p->dh, nb, brow, bcol, blocks, trip));
  return build_from_triplets(p, trip, precond_mask);
}

int dpgo_problem_set_G_dense(dpgo_problem_t *p, const double *G_host) {
  DPGO_CHECK_HANDLE(p);
  p->G_dirty = true;
  if (!G_host) {
    DPGO_CUDA(cudaMemsetAsync(p->G.get(), 0, p->vec_bytes(), p->stream));
  } else {
    DPGO_CUDA(cudaMemcpyAsync(p->G.get(), G_host, p->vec_bytes(), cudaMemcpyHostToDevice, p->stream));
  }
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_problem_set_G_csr(dpgo_problem_t *p, const int32_t *rowptr, const int32_t *colind, const double *values) {
  DPGO_CHECK_HANDLE(p);
  if (!rowptr) return dpgo_problem_set_G_dense(p, nullptr);
  std::vector<double> G((size_t)p->r * p->N, 0.0);
  for (int a = 0; a < p->r; ++a)
    for (int q = rowptr[a]; q < rowptr[a + 1]; ++q) {
      if (colind[q] < 0 || colind[q] >= p->N) return fail(DPGO_ERR_INVALID_ARG, "G column index out of range");
      G[(size_t)colind[q] * p->r + a] += values[q];
    }
  return dpgo_problem_set_G_dense(p, G.data());
}

// ---- evaluation ---------------------------------------------------------------------------------
int dpgo_problem_f(dpgo_problem_t *p, const double *X_host, double *f_out) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(f_out, DPGO_ERR_INVALID_ARG, "null output");
  DPGO_TRY(eval_at(p, X_host));
  DPGO_TRY(fetch_result(p));
  *f_out = p->h_result->f_init;
  return DPGO_OK;
}

int dpgo_problem_egrad(dpgo_problem_t *p, const double *X_host, double *out_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(out_host, DPGO_ERR_INVALID_ARG, "null output");
  DPGO_TRY(eval_at(p, X_host));
  DPGO_TRY(download_vec(p, dpgo::V_EG0, out_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_problem_ehess(dpgo_problem_t *p, const double *V_host, double *out_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(V_host && out_host, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_REQUIRE(p->bsr.have, DPGO_ERR_STATE, "set_Q has not been called");
  DPGO_TRY(upload_vec(p, dpgo::V_AUX, V_host));
  DPGO_CUDA(run_spmv(p, p->vec[dpgo::V_AUX].get(), nullptr, p->vec[dpgo::V_HD].get()));
  DPGO_TRY(download_vec(p, dpgo::V_HD, out_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_problem_rgrad(dpgo_problem_t *p, const double *X_host, double *out_host, double *norm_out) {
  DPGO_CHECK_HANDLE(p);
  DPGO_TRY(eval_at(p, X_host));
  if (out_host) DPGO_TRY(download_vec(p, dpgo::V_RG0, out_host));
  DPGO_TRY(fetch_result(p));
  if (norm_out) *norm_out = p->h_result->gradnorm_init;
  return DPGO_OK;
}

int dpgo_problem_f_rgradnorm(dpgo_problem_t *p, const double *X_host, double *f_out, double *norm_out) {
  DPGO_CHECK_HANDLE(p);
  DPGO_TRY(eval_at(p, X_host));
  DPGO_TRY(fetch_result(p));
  if (f_out) *f_out = p->h_result->f_init;
  if (norm_out) *norm_out = p->h_result->gradnorm_init;
  return DPGO_OK;
}

int dpgo_agent_f_rgradnorm_resident(dpgo_problem_t *p, double *f_out, double *norm_out) {
  DPGO_CHECK_HANDLE(p);
  DPGO_TRY(run_op(p, dpgo::OP_EVAL, plain_params()));
  DPGO_TRY(fetch_result(p));
  if (f_out) *f_out = p->h_result->f_init;
  if (norm_out) *norm_out = p->h_result->gradnorm_init;
  return DPGO_OK;
}

int dpgo_problem_rhess(dpgo_problem_t *p, const double *X_host, const double *V_host, double *out_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host && V_host && out_host, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_TRY(upload_vec(p, dpgo::V_X0, X_host));
  DPGO_TRY(upload_vec(p, dpgo::V_AUX, V_host));
  DPGO_TRY(run_op(p, dpgo::OP_RHESS, plain_params()));
  DPGO_TRY(download_vec(p, dpgo::V_HD, out_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_problem_precon(dpgo_problem_t *p, int precond, const double *X_host, const double *V_host, double *out_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host && V_host && out_host, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_TRY(check_precond(p, precond));
  DPGO_TRY(upload_vec(p, dpgo::V_X0, X_host));
  DPGO_TRY(upload_vec(p, dpgo::V_AUX, V_host));
  dpgo_opt_params_t prm;
  dpgo_opt_params_default(&prm);
  prm.precond = precond;
  DPGO_TRY(run_op(p, dpgo::OP_PRECON, prm));
  DPGO_TRY(download_vec(p, dpgo::V_Z, out_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_manifold_tangent_project(dpgo_problem_t *p, const double *X_host, const double *Z_host, double *out_host) {
  return dpgo_problem_precon(p, DPGO_PRECOND_NONE, X_host, Z_host, out_host);
}

int dpgo_manifold_retract(dpgo_problem_t *p, const double *X_host, const double *eta_host, double *out_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host && eta_host && out_host, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_TRY(upload_vec(p, dpgo::V_X0, X_host));
  DPGO_TRY(upload_vec(p, dpgo::V_AUX, eta_host));
  DPGO_TRY(run_op(p, dpgo::OP_RETRACT, plain_params()));
  DPGO_TRY(download_vec(p, dpgo::V_X1, out_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_manifold_project(dpgo_problem_t *p, const double *M_host, double *out_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(M_host && out_host, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_TRY(upload_vec(p, dpgo::V_AUX, M_host));
  DPGO_CUDA(dpgo::launch_stiefel_project(p->r, p->dh, p->n, p->vec[dpgo::V_AUX].get(), p->vec[dpgo::V_T].get(), p->stream));
  DPGO_TRY(download_vec(p, dpgo::V_T, out_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

// ---- optimiser -----------------------------------------------------------------------------------
int dpgo_optimize(dpgo_problem_t *p, const dpgo_opt_params_t *params, const double *X_in_host, double *X_out_host,
                  dpgo_opt_result_t *result) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_in_host && X_out_host, DPGO_ERR_INVALID_ARG, "null X");
  DPGO_TRY(check_params(p, params));
  const auto t0 = std::chrono::high_resolution_clock::now();
  DPGO_TRY(upload_vec(p, dpgo::V_X0, X_in_host));
  DPGO_TRY(run_op(p, dpgo::OP_OPTIMIZE, *params));
  DPGO_TRY(download_vec(p, dpgo::V_X0, X_out_host));
  DPGO_TRY(fetch_result(p));
  const auto t1 = std::chrono::high_resolution_clock::now();
  p->h_result->elapsed_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
  if (result) *result = *p->h_result;
  return DPGO_OK;
}

int dpgo_problem_upload_X(dpgo_problem_t *p, const double *X_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host, DPGO_ERR_INVALID_ARG, "null X");
  DPGO_TRY(upload_vec(p, dpgo::V_X0, X_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_problem_download_X(dpgo_problem_t *p, double *X_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host, DPGO_ERR_INVALID_ARG, "null X");
  DPGO_TRY(download_vec(p, dpgo::V_X0, X_host));
  DPGO_CUDA(cudaStreamSynchronize(p->stream));
  return DPGO_OK;
}

int dpgo_problem_upload_X_async(dpgo_problem_t *p, const double *X_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host, DPGO_ERR_INVALID_ARG, "null X");
  return upload_vec(p, dpgo::V_X0, X_host);
}

int dpgo_problem_download_X_async(dpgo_problem_t *p, double *X_host) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_host, DPGO_ERR_INVALID_ARG, "null X");
  return download_vec(p, dpgo::V_X0, X_host);
}

int dpgo_problem_copy_X_from_device(dpgo_problem_t *p, const double *X_dev) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_dev, DPGO_ERR_INVALID_ARG, "null X");
  DPGO_CUDA(cudaMemcpyAsync(p->vec[dpgo::V_X0].get(), X_dev, p->vec_bytes(), cudaMemcpyDeviceToDevice, p->stream));
  return DPGO_OK;
}

int dpgo_problem_device_X(dpgo_problem_t *p, double **X_dev) {
  DPGO_REQUIRE(p && X_dev, DPGO_ERR_INVALID_ARG, "null argument");
  *X_dev = p->vec[dpgo::V_X0].get();
  return DPGO_OK;
}

int dpgo_problem_device_G(dpgo_problem_t *p, double **G_dev) {
  DPGO_REQUIRE(p && G_dev, DPGO_ERR_INVALID_ARG, "null argument");
  *G_dev = p->G.get();
  p->G_dirty = true;             // the caller may write G directly
  return DPGO_OK;
}

int dpgo_optimize_resident_async(dpgo_problem_t *p, const dpgo_opt_params_t *params) {
  DPGO_CHECK_HANDLE(p);
  DPGO_TRY(check_params(p, params));
  p->async_t0 = std::chrono::high_resolution_clock::now();
  DPGO_TRY(run_op(p, dpgo::OP_OPTIMIZE, *params));
  p->async_pending = true;
  return DPGO_OK;
}

int dpgo_optimize_result(dpgo_problem_t *p, dpgo_opt_result_t *result) {
  DPGO_CHECK_HANDLE(p);
  DPGO_TRY(fetch_result(p));
  if (p->async_pending) {
    const auto t1 = std::chrono::high_resolution_clock::now();
    p->h_result->elapsed_ms = std::chrono::duration<double, std::milli>(t1 - p->async_t0).count();
    p->async_pending = false;
  }
  if (result) *result = *p->h_result;
  return DPGO_OK;
}

int dpgo_debug_phase_latency(dpgo_problem_t *p, int phases, double *us_per_phase, double *us_launch) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(phases >= 1 && us_per_phase, DPGO_ERR_INVALID_ARG, "bad arguments");
  dpgo_opt_params_t prm = plain_params();
  dpgo::Event e0, e1;
  DPGO_CUDA(dpgo::create_event(e0, cudaEventDefault));
  DPGO_CUDA(dpgo::create_event(e1, cudaEventDefault));
  float ms[2] = {0, 0};
  const int counts[2] = {1, phases + 1};
  for (int rep = 0; rep < 2; ++rep) {
    prm.tr_max_inner = counts[rep];
    for (int w = 0; w < 3; ++w) DPGO_TRY(run_op(p, dpgo::OP_PHASE_BENCH, prm));
    DPGO_CUDA(cudaEventRecord(e0.get(), p->stream));
    for (int w = 0; w < 10; ++w) DPGO_TRY(run_op(p, dpgo::OP_PHASE_BENCH, prm));
    DPGO_CUDA(cudaEventRecord(e1.get(), p->stream));
    DPGO_CUDA(cudaEventSynchronize(e1.get()));
    DPGO_CUDA(cudaEventElapsedTime(&ms[rep], e0.get(), e1.get()));
  }
  *us_per_phase = 1e3 * (ms[1] - ms[0]) / 10.0 / phases;
  if (us_launch) *us_launch = 1e3 * ms[0] / 10.0 - *us_per_phase;
  return DPGO_OK;
}

int dpgo_debug_phase_times64(dpgo_problem_t *p, int enable, double *ms_by_kind) {
  DPGO_CHECK_HANDLE(p);
  if (enable && !p->phase_ns) {
    DPGO_CUDA(p->phase_ns.alloc(64));
    DPGO_CUDA(cudaMemsetAsync(p->phase_ns.get(), 0, 64 * sizeof(unsigned long long), p->stream));
  }
  if (p->phase_ns) {
    unsigned long long ns[64];
    DPGO_CUDA(cudaStreamSynchronize(p->stream));
    DPGO_CUDA(cudaMemcpy(ns, p->phase_ns.get(), sizeof(ns), cudaMemcpyDeviceToHost));
    if (ms_by_kind)
      for (int i = 0; i < 64; ++i) ms_by_kind[i] = 1e-6 * (double)ns[i];
    DPGO_CUDA(cudaMemset(p->phase_ns.get(), 0, sizeof(ns)));
    if (!enable) p->phase_ns = {};
  } else if (ms_by_kind) {
    for (int i = 0; i < 64; ++i) ms_by_kind[i] = 0.0;
  }
  return DPGO_OK;
}

int dpgo_spmv_device(dpgo_problem_t *p, const double *X_dev, double *out_dev, int add_G) {
  DPGO_CHECK_HANDLE(p);
  DPGO_REQUIRE(X_dev && out_dev, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_REQUIRE(p->bsr.have, DPGO_ERR_STATE, "set_Q has not been called");
  DPGO_CUDA(run_spmv(p, X_dev, add_G ? p->G.get() : nullptr, out_dev));
  return DPGO_OK;
}

int64_t dpgo_spmv_algorithmic_bytes(const dpgo_problem_t *p, int add_G) {
  if (!p) return 0;
  // SURVEY 8(d): nb*((d+1)^2*8 + 4) + (n+1)*4 + 2*r*(d+1)*n*8 (+ r*(d+1)*n*8 if G is read)
  const int64_t dh = p->dh;
  int64_t b = p->bsr.nb * (dh * dh * 8 + 4) + ((int64_t)p->n + 1) * 4 + 2 * (int64_t)p->r * dh * p->n * 8;
  if (add_G) b += (int64_t)p->r * dh * p->n * 8;
  return b;
}

int64_t dpgo_precond_algorithmic_bytes(const dpgo_problem_t *p, int preconditioner) {
  if (!p) return 0;
  const int64_t N = (int64_t)p->dh * p->n, vec = (int64_t)p->r * N * 8;
  if (preconditioner == DPGO_PRECOND_BLOCK_JACOBI) return (int64_t)p->n * 16 * 8 + 2 * vec;
  if (preconditioner != DPGO_PRECOND_SPARSE_EXACT && preconditioner != DPGO_PRECOND_DENSE_EXACT) return 0;
  const dpgo_problem::Nd &F = p->nd[nd_slot(preconditioner)];
  return F.ready ? F.info[4] + 2 * vec : 0;
}

// ---- plain device helpers ----------------------------------------------------------------------
int dpgo_device_set(int device) {
  DPGO_CUDA(cudaSetDevice(device));
  return DPGO_OK;
}
int dpgo_device_malloc(int device, size_t bytes, void **ptr) {
  DPGO_REQUIRE(ptr, DPGO_ERR_INVALID_ARG, "null argument");
  *ptr = nullptr;
  DPGO_CUDA(cudaSetDevice(device));
  DPGO_CUDA(cudaMalloc(ptr, std::max<size_t>(bytes, 8)));
  DPGO_CUDA(cudaMemset(*ptr, 0, std::max<size_t>(bytes, 8)));
  return DPGO_OK;
}
int dpgo_device_free(int device, void *ptr) {
  DPGO_CUDA(cudaSetDevice(device));
  if (ptr) DPGO_CUDA(cudaFree(ptr));
  return DPGO_OK;
}
int dpgo_stream_create(int device, void **cuda_stream) {
  DPGO_REQUIRE(cuda_stream, DPGO_ERR_INVALID_ARG, "null argument");
  DPGO_CUDA(cudaSetDevice(device));
  cudaStream_t s;
  DPGO_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  *cuda_stream = (void *)s;
  return DPGO_OK;
}
int dpgo_stream_destroy(int device, void *cuda_stream) {
  DPGO_CUDA(cudaSetDevice(device));
  if (cuda_stream) DPGO_CUDA(cudaStreamDestroy((cudaStream_t)cuda_stream));
  return DPGO_OK;
}
int dpgo_stream_synchronize(int device, void *cuda_stream) {
  DPGO_CUDA(cudaSetDevice(device));
  DPGO_CUDA(cudaStreamSynchronize((cudaStream_t)cuda_stream));
  return DPGO_OK;
}

int dpgo_host_alloc_pinned(size_t bytes, void **ptr) {
  DPGO_TRY(require_device());
  DPGO_REQUIRE(ptr && bytes > 0, DPGO_ERR_INVALID_ARG, "null output or zero size");
  DPGO_CUDA(cudaMallocHost(ptr, bytes));
  return DPGO_OK;
}

int dpgo_host_free_pinned(void *ptr) {
  if (ptr) DPGO_CUDA(cudaFreeHost(ptr));
  return DPGO_OK;
}

int dpgo_copy_to_host_async(int device, void *dst_host, const void *src_dev, size_t bytes, void *stream) {
  DPGO_TRY(require_device());
  DPGO_REQUIRE(dst_host && src_dev, DPGO_ERR_INVALID_ARG, "null buffer");
  DPGO_CUDA(cudaSetDevice(device));
  DPGO_CUDA(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return DPGO_OK;
}

}  // extern "C"

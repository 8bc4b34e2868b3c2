// dpgo_select.cu -- greedy independent-set selection of the device RBCD runners (schedule "greedy_set").
//
//  k_select_independent   one CTA per GPU and round.  Thread a reads agent a's |rgrad|^2 (field 2 of its status record,
//                         dpgo_status.cu) into shared memory and counts the agents ahead of it: larger norm, or the same
//                         norm and a lower id (std::max_element's tie rule).  That rank is a permutation, so the sort is
//                         deterministic.  Thread 0 then walks the agents in rank order and takes an agent unless one of
//                         its neighbours (CSR agent graph) is already taken: a maximal independent set whose first member
//                         is the reference's greedy choice (ref examples/MultiRobotExample.cpp:308-325).  Agents of the
//                         set share no edge, so stepping them side by side is one exact block update, as for a colour
//                         class.  The k-byte mask gates the round's kernels and is appended to the selection log.
// Every rank runs it on the same all-gathered records, so every rank takes the same set.
#include <cuda_runtime.h>

#include "dpgo_kernels.cuh"

namespace dpgo {

namespace {

__global__ void __launch_bounds__(SELECT_MAX_AGENTS) k_select_independent(int k, const double *__restrict__ records,
                                                                          const int *__restrict__ adj_ptr,
                                                                          const int *__restrict__ adj,
                                                                          unsigned char *__restrict__ mask,
                                                                          unsigned char *__restrict__ log,
                                                                          unsigned long long *__restrict__ log_count) {
  __shared__ double key[SELECT_MAX_AGENTS];
  __shared__ short order[SELECT_MAX_AGENTS];
  __shared__ unsigned char taken[SELECT_MAX_AGENTS];
  __shared__ unsigned long long row;
  const int a = threadIdx.x;
  if (a < k) {
    const double g = records[(size_t)a * DPGO_STATUS_DOUBLES + 2];
    key[a] = (g == g) ? g : -1.0;                        // a NaN norm ranks last (norms are >= 0)
    taken[a] = 0;
  }
  __syncthreads();
  if (a < k) {
    const double ga = key[a];
    int rank = 0;
    for (int b = 0; b < k; ++b) {
      const double gb = key[b];
      rank += (gb > ga) || (gb == ga && b < a);
    }
    order[rank] = (short)a;
  }
  __syncthreads();
  if (a == 0) {
    for (int i = 0; i < k; ++i) {
      const int c = order[i];
      bool free = true;
      for (int e = adj_ptr[c]; e < adj_ptr[c + 1] && free; ++e) free = !taken[adj[e]];
      taken[c] = free ? 1 : 0;
    }
    row = *log_count;
    *log_count = row + 1;
  }
  __syncthreads();
  if (a < k) {
    mask[a] = taken[a];
    log[row * (unsigned long long)k + a] = taken[a];
  }
}

}  // namespace

cudaError_t launch_select_independent(int k, const double *records, const int *adj_ptr, const int *adj, unsigned char *mask,
                                      unsigned char *log, unsigned long long *log_count, cudaStream_t stream) {
  if (k < 1 || k > SELECT_MAX_AGENTS) return cudaErrorInvalidValue;
  k_select_independent<<<1, (k + 31) / 32 * 32, 0, stream>>>(k, records, adj_ptr, adj, mask, log, log_count);
  return cudaGetLastError();
}

}  // namespace dpgo

// dpgo_spmv_tma.cu -- the Q.X product (Out = X Q [+ G]) as a persistent, TMA-fed streaming kernel.
//
// Why: the measurement-block stream (128 B per block, contiguous for a contiguous range of pose tiles)
// is >75 % of the algorithmic bytes; a per-row gather kernel serialises 5-8 dependent DRAM latencies per
// row (rowptr -> indices -> blocks, batch after batch) and stays far below HBM peak.
// Here the row structure and the DRAM stream are decoupled:
//   * the host cuts the pose tiles into "row groups" of <= BT blocks (consecutive rows);
//   * each CTA walks its groups with an NSTAGE-deep ring of shared-memory stages; one elected thread
//     issues three 1-D bulk TMA copies per group (cp.async.bulk ... mbarrier::complete_tx): the 4x4 blocks,
//     their column indices, and the row-pointer slice -- 100+ KB in flight per SM, L2 evict-first policy
//     so the stream does not push the pose tiles (X) out of L2;
//   * the warps consume a group from shared memory: indices and blocks come from smem (no dependent global
//     round trips), only the X gathers go to L2, issued for a whole batch of 8 blocks at once.
// Lane mapping and reduce-scatter are those of dpgo_device.cuh (lane (a,k) holds P_i[a,k] and row k of
// the block; result element (a,c) ends in lane (a,c)).
#include "dpgo_device.cuh"
#include "dpgo_kernels.cuh"

namespace dpgo {

namespace {

constexpr int TMA_THREADS = 512;
constexpr int TMA_NSTAGE = 4;
constexpr int SPMV_BATCH = 12;   // blocks whose loads are issued together (predicated); rows <= 12 blocks take one round

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// 1-D bulk copy global -> shared, completion reported on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void *dst_smem, const void *src_gmem, unsigned bytes, uint64_t *bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
      : "memory");
}

// Shared-memory loads through 32-bit shared-window addresses: the consumer loop keeps three such addresses per group in
// registers; with generic pointers the compiler re-derives the window base (S2R SR_CgaCtaId, ...) inside the row loop.
__device__ __forceinline__ int lds_i32(uint32_t addr) {
  int v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ double lds_f64(uint32_t addr) {
  double v;
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr));
  return v;
}

}  // namespace

__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// group g covers rows [gi[g].x, gi[g+1].x) and blocks [gi[g].y, gi[g+1].y)
//
// Warp roles: warp NCONS is the producer (one lane issues the bulk TMA copies of a group as soon as its
// stage has been released by all consumer warps -- "empty" mbarrier, count NCONS); warps 0..NCONS-1 are
// consumers that wait on the stage's "full" mbarrier (transaction bytes), process their share of the
// group's rows and release the stage.  No CTA-wide barrier in the steady state: fast warps run up to
// NSTAGE-1 groups ahead.
//
// With 30 warps per SM the consumer loop is as much instruction- as latency-bound, so it is written predicate-light:
// rows >= R of the A fragment and columns >= 4 of the B fragment only reach accumulator entries that are never stored,
// hence those lanes load any in-bounds address instead of a predicated zero; batches of 4 blocks run without per-block
// predicates, only a row's last 1-3 blocks are predicated.  Two CTAs of 105 KB shared memory each fit an H100 SM.
template <int R, int DH, int BT, bool HAS_G>
__global__ void __launch_bounds__(TMA_THREADS, 2)
    k_spmv_tma(int ngroups, const int2 *__restrict__ gi, const int *__restrict__ rowptr, const int *__restrict__ bcol,
               const double *__restrict__ bval, const double *__restrict__ X, const double *__restrict__ G,
               double *__restrict__ out) {
  constexpr int TS = R * DH;
  constexpr int IDX_CAP = BT + 8;        // ints per stage for indices (alignment slack)
  constexpr int RP_CAP = BT + 12;        // ints per stage for the row-pointer slice (a group has <= BT rows)
  constexpr int NCONS = TMA_THREADS / 32 - 1;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  double *sq = reinterpret_cast<double *>(smem_raw);                                     // NSTAGE * BT * 16
  int *sidx = reinterpret_cast<int *>(smem_raw + (size_t)TMA_NSTAGE * BT * 128);        // NSTAGE * IDX_CAP
  int *srp = sidx + TMA_NSTAGE * IDX_CAP;                                                // NSTAGE * RP_CAP
  uint64_t *full = reinterpret_cast<uint64_t *>(srp + TMA_NSTAGE * RP_CAP);              // NSTAGE
  uint64_t *empty = full + TMA_NSTAGE;                                                    // NSTAGE

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int s = 0; s < TMA_NSTAGE; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], NCONS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == NCONS) {
    // ---------------- producer ----------------
    if (lane == 0) {
      const uint64_t pol = policy_evict_first();
      int it = 0;
      for (int g = blockIdx.x; g < ngroups; g += gridDim.x, ++it) {
        const int s = it % TMA_NSTAGE;
        if (it >= TMA_NSTAGE) mbar_wait(&empty[s], (unsigned)(((it / TMA_NSTAGE) - 1) & 1));
        const int2 g0 = __ldg(gi + g), g1 = __ldg(gi + g + 1);
        const int b0 = g0.y, b1 = g1.y, r0 = g0.x, r1 = g1.x;
        const unsigned qbytes = (unsigned)(b1 - b0) * 128u;
        const int ib = b0 & ~3;                                   // 16-byte aligned index window
        const unsigned ibytes = (unsigned)(((b1 - ib) + 3) & ~3) * 4u;
        const int rb = r0 & ~3;                                   // rowptr[r0 .. r1] inclusive
        const unsigned rbytes = (unsigned)(((r1 + 1 - rb) + 3) & ~3) * 4u;
        // a group of empty rows whose first block index is a multiple of 4 has no index window (ibytes = 0).  The PTX ISA
        // asks cp.async.bulk for a size that is a multiple of 16 and does not say what a size of 0 does, so no zero-size
        // copy is issued; expect_tx counts the bytes of the copies that are
        mbar_expect_tx(&full[s], qbytes + ibytes + rbytes);
        if (qbytes) tma_load_1d(sq + (size_t)s * BT * 16, bval + (size_t)b0 * 16, qbytes, &full[s], pol);
        if (ibytes) tma_load_1d(sidx + s * IDX_CAP, bcol + ib, ibytes, &full[s], pol);
        tma_load_1d(srp + s * RP_CAP, rowptr + rb, rbytes, &full[s], pol);
      }
    }
    return;
  }

  // ---------------- consumers ----------------
  // One warp per pose tile.  The 4x4 block product runs on the fp64 tensor pipe (mma.sync m8n8k4, SASS DMMA):
  // the A fragment IS the lane mapping (lane = 4a + k holds P_i[a,k]), the B fragment is one 8-byte shared
  // load per lane (lanes 0..15 cover the 128-byte block exactly once -> a single smem wavefront), and the
  // accumulator fragment leaves Out_j[a, 2k..2k+1] in lane (a,k), k < 2 -- no shuffles, no 128-bit smem
  // broadcasts.  The starting warp rotates with the group so that short groups load all warps evenly.
  const int a = lane >> 2, k = lane & 3;
  constexpr bool KPRED = (DH < 4);                          // k >= DH is summed over: it must contribute zeros
  const bool kok = k < DH;
  const double *Xg = X + (kok ? k * R : 0) + ((a < R) ? a : 0);   // lanes a >= R: row 0 of the tile (result row discarded)
  // B fragment: column n = lane>>2, row k = lane&3; columns >= 4 alias columns 0..3 (same 128 bytes: one wavefront)
  const int boff = k * 4 + ((lane >> 2) & 3);
  const bool st = (a < R) && (k < 2);
  const int ooff = a + 2 * k * R;
  int it = 0;
  for (int g = blockIdx.x; g < ngroups; g += gridDim.x, ++it) {
    const int s = it % TMA_NSTAGE;
    mbar_wait(&full[s], (unsigned)((it / TMA_NSTAGE) & 1));
    const int2 g0 = __ldg(gi + g), g1 = __ldg(gi + g + 1);
    const int r0 = g0.x, r1 = g1.x, b0 = g0.y;
    // shared-window addresses rebased so that they are indexed by the ABSOLUTE row / block number (wrap-around
    // arithmetic), made opaque so that they stay in three registers instead of being re-derived per row
    uint32_t q_a = smem_u32(sq + (size_t)s * BT * 16 + boff) - 128u * (uint32_t)b0;
    uint32_t idx_a = smem_u32(sidx + s * IDX_CAP) - 4u * (uint32_t)(b0 & ~3);
    uint32_t rp_a = smem_u32(srp + s * RP_CAP) - 4u * (uint32_t)(r0 & ~3);
    asm volatile("" : "+r"(q_a), "+r"(idx_a), "+r"(rp_a));
    const int wrot = (warp + it * 7) % NCONS;
    for (int j = r0 + wrot; j < r1; j += NCONS) {
      const uint32_t rpj = rp_a + 4u * (uint32_t)j;
      const int lb0 = lds_i32(rpj), lb1 = lds_i32(rpj + 4);
      double c0 = 0.0, c1 = 0.0, e0 = 0.0, e1 = 0.0;       // two accumulator pairs (shorter DMMA chains)
      for (int bb = lb0; bb < lb1; bb += SPMV_BATCH) {
        const int nb = min(lb1 - bb, SPMV_BATCH);          // warp-uniform
        const int nfull = nb >> 2, rem = nb & 3;
        const uint32_t ib = idx_a + 4u * (uint32_t)bb;
        double x[SPMV_BATCH];
#pragma unroll
        for (int t = 0; t < SPMV_BATCH / 4; ++t) {           // all global gathers of the batch in flight together
          if (t < nfull) {
#pragma unroll
            for (int u = 4 * t; u < 4 * t + 4; ++u) {
              const int col = lds_i32(ib + 4u * u);
              if (KPRED) { x[u] = 0.0; if (kok) x[u] = __ldg(Xg + (size_t)col * TS); }
              else x[u] = __ldg(Xg + (size_t)col * TS);
            }
          } else if (t == nfull && rem != 0) {
#pragma unroll
            for (int u = 4 * t; u < 4 * t + 4; ++u) {
              x[u] = 0.0;
              if (u - 4 * t < rem && (!KPRED || kok)) x[u] = __ldg(Xg + (size_t)lds_i32(ib + 4u * u) * TS);
            }
          }
        }
#pragma unroll
        for (int t = 0; t < SPMV_BATCH / 4; ++t) {
          const uint32_t qb = q_a + 128u * (uint32_t)(bb + 4 * t);
          if (t < nfull) {
            const double q0 = lds_f64(qb), q1 = lds_f64(qb + 128), q2 = lds_f64(qb + 256), q3 = lds_f64(qb + 384);
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(c0), "+d"(c1) : "d"(x[4 * t]), "d"(q0));
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(e0), "+d"(e1) : "d"(x[4 * t + 1]), "d"(q1));
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(c0), "+d"(c1) : "d"(x[4 * t + 2]), "d"(q2));
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(e0), "+d"(e1) : "d"(x[4 * t + 3]), "d"(q3));
          } else if (t == nfull && rem != 0) {
            // the B operand past the row's last block belongs to another row: it must not meet a non-zero A
            const double q0 = lds_f64(qb);
            double q1 = 0.0, q2 = 0.0;
            if (rem > 1) q1 = lds_f64(qb + 128);
            if (rem > 2) q2 = lds_f64(qb + 256);
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(c0), "+d"(c1) : "d"(x[4 * t]), "d"(q0));
            if (rem > 1)
              asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                           : "+d"(e0), "+d"(e1) : "d"(x[4 * t + 1]), "d"(q1));
            if (rem > 2)
              asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                           : "+d"(c0), "+d"(c1) : "d"(x[4 * t + 2]), "d"(q2));
          }
        }
      }
      c0 += e0;
      c1 += e1;
      // lane (a, k): c0 = Out_j[a, 2k], c1 = Out_j[a, 2k+1]
      if (st) {
        const int oi = j * TS + ooff;                        // n * TS < 2^31 (checked by the host)
        if (HAS_G) {
          c0 += __ldg(G + oi);
          if (2 * k + 1 < DH) c1 += __ldg(G + oi + R);
        }
        out[oi] = c0;
        if (2 * k + 1 < DH) out[oi + R] = c1;
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);                 // this warp is done with stage s
  }
}

template <int R, int DH, bool HAS_G>
static cudaError_t launch_tma_g(int ngroups, const int2 *gi, const int *rowptr, const int *bcol, const double *bval,
                                const double *X, const double *G, double *out, int sms, cudaStream_t stream) {
  constexpr int BT = SPMV_GROUP_BLOCKS;
  const size_t smem = (size_t)TMA_NSTAGE * BT * 128 + (size_t)TMA_NSTAGE * (BT + 8) * 4 + (size_t)TMA_NSTAGE * (BT + 12) * 4 +
                      2 * TMA_NSTAGE * 8 + 128;
  static bool attr_set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(k_spmv_tma<R, DH, BT, HAS_G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  int grid = 2 * sms;
  if (grid > ngroups) grid = ngroups;
  if (grid < 1) grid = 1;
  k_spmv_tma<R, DH, BT, HAS_G><<<grid, TMA_THREADS, smem, stream>>>(ngroups, gi, rowptr, bcol, bval, X, G, out);
  return cudaGetLastError();
}

template <int R, int DH>
static cudaError_t launch_tma_t(int ngroups, const int2 *gi, const int *rowptr, const int *bcol, const double *bval,
                                const double *X, const double *G, double *out, int sms, cudaStream_t stream) {
  return G ? launch_tma_g<R, DH, true>(ngroups, gi, rowptr, bcol, bval, X, G, out, sms, stream)
           : launch_tma_g<R, DH, false>(ngroups, gi, rowptr, bcol, bval, X, G, out, sms, stream);
}

int spmv_group_blocks() { return SPMV_GROUP_BLOCKS; }

cudaError_t launch_spmv_tma(int r, int dh, int ngroups, const int2 *gi, const int *rowptr, const int *bcol,
                            const double *bval, const double *X, const double *G, double *out, int sms,
                            cudaStream_t stream) {
  cudaError_t e = cudaErrorInvalidValue;
  DPGO_DISPATCH(r, dh, e = (launch_tma_t<R, DH>(ngroups, gi, rowptr, bcol, bval, X, G, out, sms, stream)));
  return e;
}

}  // namespace dpgo

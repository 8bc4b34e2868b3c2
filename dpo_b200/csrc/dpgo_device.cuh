// dpgo_device.cuh -- device-side building blocks of the pose-graph hot path (H100, sm_90a).
//
// Data layout in HBM (see DESIGN.md):
//   * vectors (X, gradients, tCG work vectors): column-major r x (d+1)n fp64, pose i = one
//     contiguous r x (d+1) tile (TS = r*(d+1) doubles; 160 B at r=5,d=3; 96 B at r=3).
//   * Q: block-CSR over pose pairs, every block padded to 4x4 fp64 = 128 B = one cache line,
//     bval[b*16 + k*4 + c] = Q[(d+1)i + k, (d+1)j + c] for the block b of output tile j whose
//     neighbour tile is i = bcol[b]  (so Out_j[a,c] = sum_b sum_k P_i[a,k] * bval[b][k][c]).
//
// Lane mapping ("element per lane") of the persistent kernel: a sub-group of SG lanes owns one pose
// tile; lane l holds element (a = l>>2, c = l&3) of every vector's tile, valid iff a < R and c < DH.
// The same mapping is the (a,k) operand position of the gather: lane (a,k) loads P_i[a,k] once (the
// sub-group covers the neighbour tile exactly once, coalesced) and row k of the 4x4 block
// (2 x 128-bit loads, broadcast across a), accumulates 4 partial outputs, and a reduce-scatter
// over k (warp shuffles) leaves Out_j[a,c] in lane (a,c).  (The stand-alone SpMV in
// dpgo_spmv_tma.cu feeds the same operands to the fp64 tensor pipe instead.)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dpgo {

constexpr unsigned FULL = 0xffffffffu;

template <int R> struct SubGroup { static constexpr int SG = (R > 4) ? 32 : ((R > 2) ? 16 : 8); };

// ---- loads -----------------------------------------------------------------------------
// Constant data (Q blocks, indices, Jacobi blocks): read-only path, L1-allocating.
__device__ __forceinline__ double ld_const(const double *p) { return __ldg(p); }
__device__ __forceinline__ int ld_const(const int *p) { return __ldg(p); }
__device__ __forceinline__ double2 ld_const2(const double *p) {
  return __ldg(reinterpret_cast<const double2 *>(p));
}
// Read-once streams (the dense preconditioner): no L1 allocation
__device__ __forceinline__ double ld_stream(const double *p) {
  double v;
  asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}
// Vectors that other SMs rewrite between phases of the persistent kernel: L2-only (ld.global.cg)
// so no stale L1 line can be observed after a grid barrier.
template <bool COHERENT> __device__ __forceinline__ double ld_vec(const double *p) {
  if (COHERENT) return __ldcg(p);
  return __ldg(p);
}

// ---- shuffles ----------------------------------------------------------------------------
__device__ __forceinline__ double shfl_xor(double v, int m) { return __shfl_xor_sync(FULL, v, m); }
__device__ __forceinline__ double shfl_idx(double v, int src) { return __shfl_sync(FULL, v, src); }
// element (a, c1) of the same tile row a (lanes of one quad share a)
__device__ __forceinline__ double quad_get(double v, int c1) {
  return __shfl_sync(FULL, v, (threadIdx.x & 28) | c1, 32);
}
// sum over a (lane bits 2..log2(SG)-1); every lane of the sub-group gets the column total
template <int SG> __device__ __forceinline__ double sum_over_a(double v) {
#pragma unroll
  for (int m = 4; m < SG; m <<= 1) v += shfl_xor(v, m);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) v += shfl_xor(v, m);
  return v;
}
__device__ __forceinline__ double pick3(double p0, double p1, double p2, int idx) {
  return idx == 0 ? p0 : (idx == 1 ? p1 : (idx == 2 ? p2 : 0.0));
}

// ---- gather: one output tile of P * Q ------------------------------------------------------
// Returns Out_j[a,c] in lane (a,c) (garbage-free zero in invalid lanes).  If ONFLY, the operand
// is formed on the fly as P_i = -Zs_i + beta * Dold_i (the tCG direction update fused into the
// Hessian-vector product so no separate pass / grid barrier is needed for it).
// rowptr / bcol are read with plain (generic) loads: the persistent kernel passes its shared-memory copy of the CTA's
// row range (local block offsets, bval rebased accordingly), the stand-alone kernel the global arrays.
template <int R, int DH, bool COHERENT, bool ONFLY>
__device__ __forceinline__ double gather_tile(const int *rowptr, const int *bcol,
                                              const double *__restrict__ bval, const double *P,
                                              const double *Dold, double beta, int j, int a, int k) {
  constexpr int TS = R * DH;
  const bool valid = (a < R) && (k < DH);
  const int off = k * R + a;
  double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0, acc3 = 0.0;
  const int b0 = rowptr[j], b1 = rowptr[j + 1];
  int b = b0;
  // 4-deep batches: all loads of a batch are issued before the first FMA (memory-level parallelism)
  for (; b + 4 <= b1; b += 4) {
    int i0 = bcol[b], i1 = bcol[b + 1], i2 = bcol[b + 2], i3 = bcol[b + 3];
    double x0 = 0, x1 = 0, x2 = 0, x3 = 0;
    if (valid) {
      x0 = ld_vec<COHERENT>(P + (size_t)i0 * TS + off);
      x1 = ld_vec<COHERENT>(P + (size_t)i1 * TS + off);
      x2 = ld_vec<COHERENT>(P + (size_t)i2 * TS + off);
      x3 = ld_vec<COHERENT>(P + (size_t)i3 * TS + off);
      if (ONFLY) {
        x0 = -x0; x1 = -x1; x2 = -x2; x3 = -x3;
        if (beta != 0.0) {
          x0 = fma(beta, ld_vec<COHERENT>(Dold + (size_t)i0 * TS + off), x0);
          x1 = fma(beta, ld_vec<COHERENT>(Dold + (size_t)i1 * TS + off), x1);
          x2 = fma(beta, ld_vec<COHERENT>(Dold + (size_t)i2 * TS + off), x2);
          x3 = fma(beta, ld_vec<COHERENT>(Dold + (size_t)i3 * TS + off), x3);
        }
      }
    }
    const double *q = bval + (size_t)b * 16 + k * 4;
    double2 q0a = ld_const2(q), q0b = ld_const2(q + 2);
    double2 q1a = ld_const2(q + 16), q1b = ld_const2(q + 18);
    double2 q2a = ld_const2(q + 32), q2b = ld_const2(q + 34);
    double2 q3a = ld_const2(q + 48), q3b = ld_const2(q + 50);
    acc0 = fma(x0, q0a.x, acc0); acc1 = fma(x0, q0a.y, acc1); acc2 = fma(x0, q0b.x, acc2); acc3 = fma(x0, q0b.y, acc3);
    acc0 = fma(x1, q1a.x, acc0); acc1 = fma(x1, q1a.y, acc1); acc2 = fma(x1, q1b.x, acc2); acc3 = fma(x1, q1b.y, acc3);
    acc0 = fma(x2, q2a.x, acc0); acc1 = fma(x2, q2a.y, acc1); acc2 = fma(x2, q2b.x, acc2); acc3 = fma(x2, q2b.y, acc3);
    acc0 = fma(x3, q3a.x, acc0); acc1 = fma(x3, q3a.y, acc1); acc2 = fma(x3, q3b.x, acc2); acc3 = fma(x3, q3b.y, acc3);
  }
  for (; b < b1; ++b) {
    int i0 = bcol[b];
    double x0 = 0;
    if (valid) {
      x0 = ld_vec<COHERENT>(P + (size_t)i0 * TS + off);
      if (ONFLY) {
        x0 = -x0;
        if (beta != 0.0) x0 = fma(beta, ld_vec<COHERENT>(Dold + (size_t)i0 * TS + off), x0);
      }
    }
    const double *q = bval + (size_t)b * 16 + k * 4;
    double2 qa = ld_const2(q), qb = ld_const2(q + 2);
    acc0 = fma(x0, qa.x, acc0); acc1 = fma(x0, qa.y, acc1); acc2 = fma(x0, qb.x, acc2); acc3 = fma(x0, qb.y, acc3);
  }
  // reduce-scatter over k (lane bits 0,1): 3 fp64 shuffles instead of 8
  {
    const bool hi = (k & 2) != 0;                     // hi lanes keep c in {2,3}
    double s0 = hi ? acc0 : acc2, s1 = hi ? acc1 : acc3;   // what I send to partner k^2
    double k0 = hi ? acc2 : acc0, k1 = hi ? acc3 : acc1;   // what I keep
    k0 += shfl_xor(s0, 2);
    k1 += shfl_xor(s1, 2);
    const bool odd = (k & 1) != 0;                    // odd lanes keep the upper of the pair
    double s = odd ? k0 : k1, kk = odd ? k1 : k0;
    kk += shfl_xor(s, 1);
    return kk;                                        // = Out_j[a, c = k]
  }
}

// ---- per-pose primitives in element-per-lane layout ------------------------------------------
// Tangent projection at Y of z: lane (a,c) gets z - sum_c1 Y[a,c1] sym(Y^T Z)[c1][c] for c < D,
// z unchanged for the translation column.  ya[] returns Y[a, 0..2]; symcol[] the column c of
// sym(Y^T Z) (rows c1 = 0..2) -- cached by the caller as S for Riemannian Hessian products.
// ref: ROPTLIB ProductManifold::Projection -> Stiefel::ExtrProjection (call sites
// src/QuadraticProblem.cpp:82,95; src/QuadraticOptimizer.cpp:139).
template <int R, int DH>
__device__ __forceinline__ double tangent_project_elem(double y, double z, int a, int c, double ya[3],
                                                       double symcol[3]) {
  constexpr int D = DH - 1;
  constexpr int SG = SubGroup<R>::SG;
  const bool rot = (a < R) && (c < D);
  const double yy = rot ? y : 0.0, zz = rot ? z : 0.0;
  double p[3];
#pragma unroll
  for (int c1 = 0; c1 < 3; ++c1) {
    ya[c1] = (c1 < D) ? quad_get(yy, c1) : 0.0;
    p[c1] = sum_over_a<SG>(ya[c1] * zz);              // S[c1][c]
  }
  symcol[0] = p[0]; symcol[1] = p[1]; symcol[2] = p[2];
#pragma unroll
  for (int rho = 1; rho < 4; ++rho) {
    const int s = (c + rho) & 3;                       // partner column
    const double sel = pick3(p[0], p[1], p[2], (c - rho) & 3);   // my S[(c-rho)&3][c]
    const double got = quad_get(sel, s);               // = S[c][s]
    if (s < 3) {
      const double sym = 0.5 * (pick3(p[0], p[1], p[2], s) + got);
      if (s == 0) symcol[0] = sym; else if (s == 1) symcol[1] = sym; else symcol[2] = sym;
    }
  }
  double out = z;
  if (rot) out = z - (ya[0] * symcol[0] + ya[1] * symcol[1] + ya[2] * symcol[2]);
  return out;
}

// Projection with an already known Y row (ya) -- used when Y was exchanged before.
// QF retraction of one tile: w = x + eta -> qf(w) (diag(R) > 0) on the rotation columns,
// translation column passes through.  Modified Gram-Schmidt run twice (second sweep restores
// orthogonality to machine precision; R2 ~ I so the sign convention diag(R) > 0 is kept).
// ref: ROPTLIB Stiefel::qfRetraction (call site src/QuadraticOptimizer.cpp:146).
template <int R, int DH> __device__ __forceinline__ double qf_retract_elem(double w, int a, int c) {
  constexpr int D = DH - 1;
  constexpr int SG = SubGroup<R>::SG;
  const bool rot = (a < R) && (c < D);
  double v = rot ? w : 0.0;
#pragma unroll
  for (int sweep = 0; sweep < 2; ++sweep) {
#pragma unroll
    for (int t = 0; t < D; ++t) {
      double wt = quad_get(v, t);                       // column t, row a
      double nrm2 = sum_over_a<SG>(wt * wt);
      double qt = wt * (1.0 / sqrt(nrm2));
      double proj = sum_over_a<SG>(qt * v);             // <q_t, w_c> for my column c
      if (c == t) v = qt;
      else if (c > t && c < D) v = fma(-proj, qt, v);
    }
  }
  return rot ? v : w;
}

// Block-Jacobi solve for one tile: out[a,c] = sum_k v[a,k] Dinv_j[k][c]
template <int R, int DH>
__device__ __forceinline__ double jacobi_elem(const double *__restrict__ dinv, int j, double v, int a, int c) {
  const double vv = (a < R && c < DH) ? v : 0.0;
  double out = 0.0;
  const double *D = dinv + (size_t)j * 16 + c;
#pragma unroll
  for (int k = 0; k < DH; ++k) out = fma(quad_get(vv, k), ld_const(D + 4 * k), out);
  return out;
}

// ---- grid-wide barrier for the persistent kernel ------------------------------------------------
// Monotonic arrival counter (wrap-safe signed comparison); every CTA is resident (cooperative launch).
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned *p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// Grid-wide phase end of the persistent kernel (phase_end in dpgo_kernels.cu).
// Release side: red.release (MEMBAR.GPU + RED) publishes every write of the CTA (ordered before it by a bar.sync).
// Acquire side: by default the poll is a RELAXED gpu-scope load.  An acquire load would add CCTL.IVALL, i.e. drop the
// SM's whole L1 at every phase end -- and with it the constant data the phases re-read all the time (block-CSR
// indices and blocks, plan records).  That invalidation protects weak loads of data other SMs rewrite; this kernel
// has none: every vector / workspace another CTA may have written is read with ld.global.cg (L2) or ld.relaxed.gpu,
// never through L1, and read-only data is never rewritten during a launch.  Ordering of those L2 reads after the
// poll: the poll loop's exit branch depends on the loaded value and the other threads wait at the bar.sync behind it.

}  // namespace dpgo

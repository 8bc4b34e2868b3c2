// nd_precond.h -- host side of the sparse EXACT preconditioner  Z = (Q + shift I)^-1 V  (r right-hand sides at once).
//
// ref: QuadraticProblem::setQ (src/QuadraticProblem.cpp:31-42: CHOLMOD factorisation of Q + 0.1 I) and
//      QuadraticProblem::PreConditioner (:75-87: solve, then tangent projection).
//
// Design: a GPU triangular solve along an elimination tree is a chain of ~2 log2(n) dependent grid-wide steps, and a
// grid-wide step costs 1.7 us on an H100 SXM at a 400 W power limit (an empty phase of the step kernel over its 132
// CTAs, dpgo_debug_phase_latency).  So the tree is
// flattened: a nested-dissection tree of the pose graph is cut into a FEW macro levels (usually 2-3); every macro node v
// (a fragment of the dissection tree: its separators / leaf interiors) keeps
//     W_v = S_v^-1        dense inverse of its Schur complement (own x own),
//     F_v = W_v E_v       coupling to the ancestors' variables it touches (own x bnd),
// so that the solve is  2 * levels - 1  phases of small dense panel products:
//     forward  (leaves -> root):  y_v = b_v - sum_children c_child ;  t_v = W_v y_v ;  c_v = F_v^T y_v + pass-through
//     root:                       x_root = W_root y_root
//     backward (root -> leaves):  x_v = t_v - F_v x_bnd(v)
// All blocks together are ~10x the sparse factor but ~15-30x smaller than the dense inverse, and L2-resident for
// sphere2500-sized agents.  Matrices are stored as 8-row panels, column-major inside a panel (a warp reads 256
// contiguous bytes per step); the work of every phase is a host-built static plan (per CTA: steps of gathers into
// shared memory / warp jobs = panel x column piece / epilogues per pose), interpreted by phase_nd in dpgo_kernels.cu.
// Everything is deterministic (fixed summation orders).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace dpgo {
namespace nd {

// ---- device-facing plan records (plain ints, uploaded as they are) ------------------------------------------
// Records are sized in whole 16-byte words and carry what the kernel needs WITHOUT a second dependent load: the first
// step of a CTA sits in its (phase, CTA) record, the first four contribution tiles sit in the gather / epilogue record.
struct Step { int g0, g1, j0, j1, e0, e1, pad0, pad1; };              // ranges into gathers / jobs / epis
struct CtaPhase { int s0, s1; int g0, g1, j0, j1, e0, e1; };          // steps [s0, s1) of one CTA in one phase + step s0 inline
constexpr int INLINE_CONTRIB = 4;
struct Gather { int ytile; int src; int nc; int cext; int ci[INLINE_CONTRIB]; };   // smem tile <- source tile - sum of nc contribution tiles
// one warp: panel piece x y.  The first nres columns (0, a multiple of RES_ROUND, or all ncols) are resident: the first
// application of a launch copies them to the CTA's shared-memory region at double offset soff, later ones read them there
// (groups of 4 columns x 8 rows, 32 doubles each, in lane order: lane 4 row + k holds column 4 g + k)
struct Job { long long mat; int ncols; int ycol; int slot; int accum; int soff, nres; };
struct Epi { int kind; int slot0; int nslots; int half; int out; int aux; int nc; int cext; int ci[INLINE_CONTRIB]; };   // one pose (dh rows of a panel)
enum EpiKind { EPI_F_OWN = 0, EPI_F_BND = 1, EPI_B_OWN = 2, EPI_ROOT = 3 };
struct Phase { int dir; int stage; int cta0; int pad; };              // dir 0 forward (source = V, pose ids), 1 backward (source = TX); cta0 = first CtaPhase record
constexpr int MAX_PHASES = 16;

constexpr int PANEL_ROWS = 8;
constexpr int RES_ROUND = 32;     // columns per round of the job loop (8 independent loads of 4 columns)
// shared-memory doubles of a job's resident columns
inline int resident_doubles(int nres) { return (nres + 3) / 4 * 32; }

struct Options {
  int grid = 132;            // CTAs of the persistent kernel (one per SM of an H100 SXM)
  int r = 5;                 // right-hand sides (rows of the residual)
  int warps = 16;            // warps per CTA
  int leaf_size = 12;        // dissection stops below this many poses
  int max_cuts = 3;          // macro levels <= max_cuts + 1
  int ycap_tiles = 600;      // shared-memory capacity for gathered tiles per step
  int slot_cap = 240;        // shared-memory partial-sum slots (8 x r doubles each) per step
  double t_phase_us = 3.5;   // cost model: fixed part of one phase (grid barrier + the stages' dependent L2 round trips)
  double t_tile_us = 0.012;  // cost model: staging one tile of a phase's largest input vector (per CTA, redundant over CTAs)
  double bw_gbs = 3000.0;    // cost model: effective streaming bandwidth of the panel products
  int force_ncuts = -1;      // >= 0: use exactly this many cuts (tests)
  double shift = 0.1;
};

struct MacroNode {
  int stage = 0;             // 0 = deepest macro level ... nstages-1 = root level
  int parent = -1;
  std::vector<int> own;      // pose ids, elimination order
  std::vector<int> bnd;      // pose ids owned by ancestors that the Schur complement touches
  std::vector<int> children;
  int perm0 = 0;             // first permuted tile index of own
  int cbuf0 = 0;             // first contribution tile of this node
  int64_t gf_off = 0, gb_off = 0;   // panel blobs (doubles): forward [W ; F^T] (rows own+bnd, cols own), backward F (rows own, cols bnd)
};

struct Hierarchy {
  int n = 0, dh = 4;
  std::vector<MacroNode> nodes;
  int nstages = 0;
  std::vector<int> perm;       // permuted tile index -> pose id
  std::vector<int> iperm;      // pose id -> permuted tile index
  std::vector<int> node_of;    // pose id -> macro node
  int cbuf_tiles = 0;
  int64_t blob_doubles = 0;
  std::vector<int> cuts;       // dissection levels where macro levels start (diagnostic)
  int nd_depth = 0;
};

struct Plan {
  std::vector<Phase> phases;       // 2 * nstages - 1
  std::vector<CtaPhase> cta_phase; // phases * grid
  std::vector<Step> steps;
  std::vector<Gather> gathers;
  std::vector<Job> jobs;
  std::vector<Epi> epis;
  std::vector<int> csrc;           // contribution tile ids beyond the INLINE_CONTRIB kept in the records
  int grid = 0, r = 0;
  int max_ytiles = 0, max_slots = 0;
  int64_t bytes_per_apply = 0;     // matrix bytes streamed by one application (all phases)
  std::vector<int> resident_doubles;   // per CTA: shared-memory region of its resident columns (assign_residency)
  int max_resident_doubles = 0;
  int64_t resident_bytes = 0;      // matrix bytes of one application read from shared memory after the first
};

// block-CSR input: rowptr[n+1], bcol[nb], bval[nb*16] with bval[b][k][c] = Q[dh*bcol[b]+k, dh*j+c] for b in row j
struct BsrView { int n; int dh; const int *rowptr; const int *bcol; const double *bval; };

// 1. ordering + macro levels (symbolic).  Throws std::runtime_error on impossible input.
void build_hierarchy(const BsrView &Q, const Options &opt, Hierarchy &H);
// 2. numeric: fills the panel blob (host, OpenMP over columns)
void build_numeric(const BsrView &Q, const Options &opt, Hierarchy &H, std::vector<double> &blob);
// 3. static work plan of every phase
void build_plan(const Hierarchy &H, const Options &opt, Plan &P);
// 4. residency: annotates the jobs (soff, nres) so that every CTA keeps at most budget_bytes of its panels in shared
//    memory for the whole launch.  Only an annotation: the jobs, their order and their arithmetic stay as they are.
//    Within a (CTA, phase) every warp streams the same number of rounds per step (or all of its own, if fewer).
void assign_residency(Plan &P, int warps, int64_t budget_bytes);
// host emulation of the plan exactly as the kernel interprets it (verification only; never on a product path):
// V, Z are r x (dh n) column-major (pose tiles), Z = (Q + shift I)^-1 V   (no tangent projection).  With resident
// columns, a first pass fills a simulated per-CTA region and the result is that of a second pass reading from it.
void emulate_apply(const Hierarchy &H, const Plan &P, const std::vector<double> &blob, int r, const double *V, double *Z);

std::string describe(const Hierarchy &H, const Plan &P);

// ---- numeric refactorisation on the device (nd_refactor.cu): the algorithm of build_numeric over the fronts of the macro
// nodes, stage by stage, for a Q whose block pattern is unchanged.  The front of node v is the dense symmetric matrix
// [Foo Fob; Fob^T Fbb] over its front poses (own, then bnd), column-major, leading dimension M = dh (own + bnd); a
// Gauss-Jordan sweep over its first s = dh own pivots leaves W = Foo^-1, Fm = W Fob and U = Fbb - Fob^T Fm in place, and
// U stays there until the parent's stage has added it.  Fronts of stage st live in the arena at base (st even: 0, odd:
// arena_even), so a child's U (stage st - 1) is never overwritten while its parent (stage st) is assembled.
constexpr int REFACTOR_PIVOT_BLOCK = 32;   // pivots per Gauss-Jordan step (dense_inverse.cu GJB)
struct RefactorNode {
  long long front;           // arena offset (doubles) of the front
  long long ws;              // workspace offset (doubles): pivot block, row panel, column panel of the sweep
  long long gf, gb;          // panel blob offsets (MacroNode::gf_off / gb_off)
  int no, nb;                // own / boundary poses
  int pose0;                 // first front pose in Refactor::poses
  int ch0, nch;              // children in Refactor::child (mn.children order)
  int pad;
};
struct RefactorChild { int node; int map0; };   // refactor-node index of the child; map0: Refactor::cmap offset (one entry per parent front pose)
struct Refactor {
  std::vector<RefactorNode> nodes;   // stage by stage, deepest first (the order build_numeric visits)
  std::vector<int> stage0;           // nstages + 1: node range of every stage
  std::vector<int> poses;            // front poses of every node, own then bnd
  std::vector<RefactorChild> child;
  std::vector<int> cmap;             // position of a parent front pose in the child's bnd list, -1 when absent
  std::vector<int> max_nfr, max_s;   // per stage: largest front (poses), largest pivot count (scalars)
  std::vector<int64_t> max_blob;     // per stage: largest panel region of one node (doubles)
  int64_t arena_even = 0, arena_doubles = 0, ws_doubles = 0;
};
// Throws std::runtime_error when a child is not exactly one stage below its parent (the arena parity relies on it).
void build_refactor(const Hierarchy &H, Refactor &R);

// ---- selected inversion over the same fronts (dpgo_covariance.cu): with W = Foo^-1 and Fm = W Fob of every node (the
// panels a factorisation with shift 0 leaves), the front inverse  Sigma_front = (A^-1) restricted to the node's front poses
// follows from the parent's, root to leaves:
//     Sigma_bb = parent's Sigma_front at the node's boundary poses,   Sigma_ob = -Fm Sigma_bb,   Sigma_oo = W - Sigma_ob Fm^T.
// Fronts are M x M column-major (M = dh (own + bnd), own then bnd) and only their upper triangle (row <= col) is read.
// pmap: per refactor node (R's order), the position of each of its boundary poses in its parent's front; pmap0 / parent.
struct Selinv {
  std::vector<int> parent;    // refactor index of the parent, -1 at a root
  std::vector<int> pmap0;     // offset into pmap (nb entries per node)
  std::vector<int> pmap;
  std::vector<int> macro;     // refactor index -> macro node (H.nodes index)
  std::vector<int> max_b;     // per stage: largest boundary (scalars)
};
void build_selinv(const Hierarchy &H, const Refactor &R, Selinv &S);
// HOST ONLY, verification: the sweep of the device selected inversion, with the same recurrence and the same summation
// order, over the panels of build_numeric (Options::shift = 0).  front[q] (refactor order) receives node q's front inverse.
void emulate_selinv(const Hierarchy &H, const Refactor &R, const Selinv &S, const std::vector<double> &blob,
                    std::vector<std::vector<double>> &front);

}  // namespace nd
}  // namespace dpgo

// hb2_kernels_fp64.cuh -- fp64 CUDA kernels of the likelihood hot path (sm_90a).
//
//   expm64_dmma_kernel / expm_small_kernel  P = exp(Q t) per (branch, rate class)
//                                           (replaces _Matrix::Exponentiate, reference matrix.cpp:5537-5951)
//   prune_small_walk_kernel<Dp, PP>         Felsenstein pruning pass for 4 / 8 padded states, PP patterns per thread:
//                                           all children folded (leaf column gather, ambiguity mat-vec, internal
//                                           contraction), per-pattern renormalisation, root pi-dot
//                                           (replaces ComputeTreeBlockByBranch, reference tree_evaluator.cpp:3556-4171)
//   combine_kernel / final_sum_kernel       rate-class mixture, log, pattern-frequency weighting, deterministic sum
//                                           (replaces likefunc2.cpp:828-859,1446-1506 and tree_evaluator.cpp:4093-4149)
//
// Device data layout (Dp = padded state count, Sp = pattern count padded to 64):
//   PT    [C][B][Dp][Dp]   TRANSPOSED transition matrices: PT[j][k] = P(parent k -> child j); padding = 0
//   cond  [C][I][Sp][Dp]   conditionals of internal nodes, renormalised per (node, pattern) so max_k = [0.5,1)
//   scal  [C][I][Sp]       int32 binary exponent: true conditional = cond * 2^scal
//   leaf  [L][Sp]          int32 state code (>=0) or -(ambiguity row + 1)
//   ambig [nAmb][Dp]       0/1 rows
// Underflow handling is the engine's own (exact power-of-two renormalisation at every node) and is converted to the
// reference's 2^64-count convention only at the boundary (SURVEY.md Appendix C, last bullet).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include <cooperative_groups.h>

namespace hb2 {

constexpr int LD64 = 66;            // smem leading dimension (doubles) for 64x64 operands: conflict-free row pairs

// Tensor-path operands of one 64-state transition matrix (written by the expm stage, read by hb2_kernels_tc.cuh).
constexpr int TC_PB_FLOATS = 2 * 4096;         // per (class, branch): Ph tile + Pl tile in canonical layout
constexpr int TC_PTF_ROW = 68;                 // floats per row of the fp32 P^T table (64 + 4 padding: 272-byte rows)
constexpr int TC_PTF_FLOATS = 64 * TC_PTF_ROW; // per (class, branch)

// Two different roundings to tf32 (round to nearest, ties away from zero); call sites keep the one they use.
// tf32_rn: integer add-and-mask, two full-rate instructions; a NaN with bits above 0x7fffe000 comes out as -0.0.
__device__ __forceinline__ float tf32_rn(float x) {
    return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}
// tf32_rn_cvt: the conversion instruction cvt.rna.tf32.f32 (a quarter of the ALU rate); NaN stays NaN.
__device__ __forceinline__ float tf32_rn_cvt(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

// Device-side waits are bounded by TIME (globaltimer), not by an iteration count: a slow producer (another partition or
// process sharing the GPU, fewer co-resident CTAs than planned) only makes the pass slower; a protocol bug still surfaces
// as an error code in the partition's error flag (the host returns an error, see wait_timeout), never as a hung GPU.
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
constexpr unsigned long long HB2_WAIT_LIMIT_NS = 4000000000ull;         // waits within one device
constexpr unsigned long long HB2_PEER_WAIT_LIMIT_NS = 20000000000ull;   // waits for another rank: longer, a rank is gone
// What a timed-out wait was waiting for: the value it leaves in the error flag.
enum WaitCode : int {
    WAIT_TC_STAGING = 1,      // operand staging / the tensor pipe (mbarrier)
    WAIT_LANE = 2,            // another lane's conditionals
    WAIT_PEER = 3,            // a peer rank's partials
    WAIT_EXPM_POWERS = 4,     // a coefficient matrix of the shared-powers exponential
};

struct TreeDev {
    const int *child_start;         // [I+1]
    const int *child_ids;           // flat node ids of the children of each internal node
};

struct PruneArgs {
    const double *PT;               // [C][B][Dp*Dp]
    double *cond;                   // [C][I][Sp][Dp]
    int *scal;                      // [C][I][Sp]
    const int *leaf;                // [L][Sp]
    const double *ambig;            // [nAmb][Dp]
    const double *pi;               // [Dp] root frequencies (padding 0)
    double *rootL;                  // [C][Sp]
    int *rootE;                     // [C][Sp]
    TreeDev tree;
    int L, I, B, D, Sp, cat0;
    // forced states (reference setBranch / setBranchTo, tree_evaluator.cpp:3624,173-181,4059): flat id of ONE node whose
    // state is pinned per pattern to forced[s] (a leaf: its observed state is replaced; an internal node or the root: its
    // conditional vector is masked to that state), or -1
    const int *forced;
    int forced_node;
};

__device__ __forceinline__ double exp2i(int e) {   // exact 2^e for |e| < 1022
    return __longlong_as_double((long long)(e + 1023) << 52);
}

// Rescaling inside a node.  The pruning kernels multiply all children of a node together and renormalise once, at the end
// of the node.  For a node with many children (a polytomy, a star tree) the running product can fall below the smallest
// normal double before that: 400 codon leaves on branches of mean length 2 reach about 2^-1300.  So from the third child on,
// a running product whose maximum has fallen below RESCALE_BELOW is brought back to [0.5, 1) by an exact power of two and
// the exponent is carried, as the reference rescales after every child (tree.cpp:161-205).  The rescaling is exact, so a
// product that does not underflow gives the same bits with or without it; binary nodes never take it.
constexpr double RESCALE_BELOW = 0x1p-256;

template <int N>
__device__ __forceinline__ void rescale_running(double (&v)[N], int &ex) {      // one thread holds the pattern's N values
    double m = 0.0;
#pragma unroll
    for (int k = 0; k < N; k++) m = fmax(m, v[k]);
    if (m > 0.0 && m < RESCALE_BELOW) {
        const int e = ilogb(m) + 1;
        const double s1 = exp2i(-(e / 2)), s2 = exp2i(-(e - e / 2));
#pragma unroll
        for (int k = 0; k < N; k++) v[k] = v[k] * s1 * s2;
        ex += e;
    }
}

// The same for a pattern whose values are spread over the 4 lanes q4 = 0..3 of a quad (FP64 tensor-pipe kernels).  Called
// by the whole warp.
template <int NT>
__device__ __forceinline__ void rescale_running_quad(double (&v)[NT][2], int &ex) {
    double m = 0.0;
#pragma unroll
    for (int t = 0; t < NT; t++) m = fmax(m, fmax(v[t][0], v[t][1]));
    m = fmax(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmax(m, __shfl_xor_sync(0xffffffffu, m, 2));
    if (m > 0.0 && m < RESCALE_BELOW) {
        const int e = ilogb(m) + 1;
        const double s1 = exp2i(-(e / 2)), s2 = exp2i(-(e - e / 2));
#pragma unroll
        for (int t = 0; t < NT; t++) { v[t][0] = v[t][0] * s1 * s2; v[t][1] = v[t][1] * s1 * s2; }
        ex += e;
    }
}

// ------------------------------------------------------------------------------------------------
// Matrix exponential.  One wave of CTAs over the batch (expm64_dmma_kernel), one CTA per matrix (expm_small_kernel), or
// the shared-powers path below.
//   in : Q [n][D*D] row-major rate matrices (Q*t, diagonal = -rowsum), dst[n] = slot index into PT
//   out: PT[slot] = exp(Q)^T with padding rows/cols zeroed, negatives clamped, columns repaired to sum to 1
// Algorithm (engine's own, same result as the reference's Taylor+squaring to ~1e-15): scale by 2^-s, Taylor polynomial
// by Paterson-Stockmeyer, s squarings.
// ------------------------------------------------------------------------------------------------
struct ExpmArgs {
    const double *Q;        // [n][D*D]
    const int *dst;         // [n] destination slot; < 0: retired entry (the slot was handed over again), skipped
    double *PT;
    double *Qres;           // nullable [slots][D*D]: resident copy of the rate matrices, written while loading
    int D;
    int is_trans;           // 1: input already a transition matrix -> just transpose/pad
    // compiled-template input (replaces dense Q when tmpl_nnz > 0): Q[row][col] = V[blk][formula[e]] * colfreq[col],
    // diagonal = -(off-diagonal row sum); mirrors _CompiledMatrixData + MultByFreqs (reference matrix.h:69, matrix.cpp:1546)
    const double *V;        // [n][nF] formula values per matrix
    const int *tmpl_index;  // [nnz] row*D + col
    const int *tmpl_formula;// [nnz]
    const double *tmpl_colfreq;  // nullable [D]
    int tmpl_nnz, nF;
    // shared-powers path (64-state kernels, see expm_classify_kernel): per-entry group, proportionality flag and L1 weight
    const int *group;       // nullable [n]: power-table group of the entry (rate class; mixture component), < 0 none
    const int *flag;        // nullable [n]: 1 = the entry is a scalar multiple of its group's reference direction
    const double *weight;   // [n]: sum of |input values| of the entry (formula values or matrix entries)
    const struct ExpmGroup *groups;   // [G] reference info of every group
    const double *pow;      // [G][EXPM_POW_TERMS][4096] Taylor coefficient matrices of the groups (PT layout)
};

// Shared powers.  In the models the optimiser spends its time in, all branches of a rate class share ONE rate matrix up
// to the branch length: A_b = rho_b * R with ||R||_inf = 1 (SURVEY §7, VERDICT r1 "what's weak" 4).  Then
//     exp(A_b) = sum_m (R^m / m!) * rho_b^m
// is, element by element, a scalar polynomial in rho_b whose coefficient matrices S_m = R^m/m! are the same for every
// branch of the group: they are built ONCE per group and evaluation (expm_powers_kernel: 23 products of 64^3 arranged as
// a 5-level tree S_{a+b} = S_a S_b / C(a+b,a), one CTA per product, dependencies resolved through generation flags),
// after which a branch costs 24 FMAs per matrix element (expm_poly_kernel) instead of ~5 matrix products; only matrices
// with rho_b > 2.3 still need squarings (s of them, x = rho_b / 2^s <= 2.3; degree 24 truncates below 1e-16 there).  Proportionality is CHECKED on the device for every matrix
// (expm_classify_kernel), never assumed: anything that is not a multiple of its group's reference direction to 1e-13
// takes the general scaling-and-squaring path inside the same launch.
constexpr int EXPM_POW_TERMS = 25;        // S_0 = I (not stored, slot unused) .. S_24
constexpr double EXPM_POLY_THETA = 2.3;   // x^25/25! < 1e-16 for x <= 2.33: degree 24 needs no squaring up to here
struct ExpmGroup {
    double nu;        // ||A_ref||_inf of the reference matrix the powers were built from
    double weight;    // its L1 weight (same measure as ExpmArgs::weight)
    int kind;         // 0 invalid, 1 reference direction held as formula values (compiled input), 2 as dense matrix entries
    int pad;
};

// Builds A1[j][i] = Q[i][j] (transposed, zero padded, leading dimension LD) from dense or compiled input and leaves a
// dense resident copy in Qres when asked.  All threads of the CTA call it; ends with a barrier.
template <int DP, int LD, int NT>
__device__ __forceinline__ void load_rate_matrix(const ExpmArgs &a, double *A1, int tid, int entry = -1) {
    const int D = a.D;
    if (entry < 0) entry = blockIdx.x;
    const size_t slot = a.dst[entry];
    if (a.tmpl_nnz > 0) {
        for (int idx = tid; idx < DP * LD; idx += NT) A1[idx] = 0.0;
        __syncthreads();
        const double *V = a.V + (size_t)entry * a.nF;
        for (int e = tid; e < a.tmpl_nnz; e += NT) {
            const int rc = a.tmpl_index[e], r = rc / D, c = rc - r * D;
            double v = V[a.tmpl_formula[e]];
            if (a.tmpl_colfreq) v *= a.tmpl_colfreq[c];
            if (r != c) A1[c * LD + r] = v;
        }
        __syncthreads();
        if (tid < D) {
            double s = 0.0;
            for (int c = 0; c < D; c++) if (c != tid) s += A1[c * LD + tid];
            A1[tid * LD + tid] = -s;
        }
        __syncthreads();
        if (a.Qres)
            for (int idx = tid; idx < D * D; idx += NT) { const int i = idx / D, j = idx - i * D; a.Qres[slot * D * D + idx] = A1[j * LD + i]; }
    } else {
        const double *Q = a.Q + (size_t)entry * D * D;
#pragma unroll                                    // every load of the thread in flight at once
        for (int it = 0; it < (DP * DP + NT - 1) / NT; it++) {
            const int idx = tid + it * NT, i = idx / DP, j = idx - i * DP;
            if (idx >= DP * DP) break;
            const double v = (i < D && j < D) ? Q[(size_t)i * D + j] : 0.0;
            A1[j * LD + i] = v;
            if (a.Qres && i < D && j < D) a.Qres[slot * D * D + (size_t)i * D + j] = v;
        }
    }
    __syncthreads();
}

// Taylor coefficients 1/k!, k = 0..17: the small-state polynomial uses 16 of them, expm64_dmma_kernel's up to 18.
__constant__ double c_taylor[18] = {1.0, 1.0, 0.5, 1.0 / 6, 1.0 / 24, 1.0 / 120, 1.0 / 720, 1.0 / 5040, 1.0 / 40320,
                                    1.0 / 362880, 1.0 / 3628800, 1.0 / 39916800, 1.0 / 479001600, 1.0 / 6227020800.0,
                                    1.0 / 87178291200.0, 1.0 / 1307674368000.0, 1.0 / 20922789888000.0,
                                    1.0 / 355687428096000.0};

// ------------------------------------------------------------------------------------------------
// expm64_dmma_kernel: 64 padded states, products on the FP64 tensor pipe (mma.sync.m8n8k4.f64, DMMA)
// and a Paterson-Stockmeyer polynomial whose degree follows the norm:
//   p(A) = sum_{q=0..Q} A3^q * (c_{3q} I + c_{3q+1} A + c_{3q+2} A2),   A3 = A^3,   degree 3Q+2,   2+Q products,
//   Q chosen so that theta^(3Q+3)/(3Q+3)! <= 1e-16 with theta = ||A||/2^s <= 0.975; s squarings follow.
// 8 warps; warp (wr,wc) owns rows 16wr..16wr+15 and columns 32wc..32wc+31 of the product as 2x4 m8n8 tiles; lane
// (g = lane/4, q = lane%4) holds element (row 16wr+8i+g, col 32wc+8j+2q+e) in acc[i][j][e].
// Optional fused epilogue for the tensor-core pruning path: PB (hi/lo canonical tiles of P) and PTf (fp32 PT).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void dmma884(double (&c)[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}

__device__ __forceinline__ void tile_mm64_dmma(const double *__restrict__ A, const double *__restrict__ Bm, int wr, int wc,
                                               int g, int q, double (&acc)[2][4][2]) {
    const double *a0 = A + (16 * wr + g) * LD64 + q;
    const double *b0 = Bm + q * LD64 + 32 * wc + g;
#pragma unroll 4
    for (int k0 = 0; k0 < 64; k0 += 4) {
        const double x0 = a0[k0], x1 = a0[8 * LD64 + k0];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const double b = b0[k0 * LD64 + 8 * j];
            dmma884(acc[0][j], x0, b);
            dmma884(acc[1][j], x1, b);
        }
    }
}

struct ExpmTcOut {
    float *PB;      // nullable: [slots][2][4096] canonical hi/lo tiles (see hb2_kernels_tc.cuh)
    float *PTf;     // [slots][64 rows][68 floats] (rows padded: conflict-free shared-memory gathers after a flat bulk copy)
};

// ---- Finishing rules of a 64-state matrix (expm64_dmma_kernel, expm_powers_kernel, expm_poly_kernel, mix_reduce_kernel)
// A NaN or infinite input or absurd rates: the whole slot is NaN, tensor-path operands included (the host sees NaN lnL).
__device__ __forceinline__ void expm64_poison(double *out, const ExpmTcOut &tc, size_t slot, int tid) {
    for (int idx = tid; idx < 4096; idx += 256) out[idx] = __longlong_as_double(0x7ff8000000000000LL);
    if (tc.PB) {
        for (int idx = tid; idx < TC_PB_FLOATS; idx += 256) tc.PB[slot * TC_PB_FLOATS + idx] = __int_as_float(0x7fc00000);
        for (int idx = tid; idx < TC_PTF_FLOATS; idx += 256) tc.PTf[slot * TC_PTF_FLOATS + idx] = __int_as_float(0x7fc00000);
    }
}

// Index maps of the tensor-path operands for element (r, c) of PT (r = child state, c = parent state): row r of the
// padded fp32 table, and chunk r/4, offset 4c + r%4 of the canonical tiles (hb2_kernels_tc.cuh).
__device__ __forceinline__ int tc_ptf_index(int r, int c) { return r * TC_PTF_ROW + c; }
__device__ __forceinline__ int tc_pb_index(int r, int c) { return (r >> 2) * 256 + c * 4 + (r & 3); }

// The hi/lo split of P element p into position o of the slot's tiles pb (Ph, then Pl): CVT rounds with tf32_rn_cvt, else
// with tf32_rn.
template <bool CVT>
__device__ __forceinline__ void tc_split_store(float *pb, int o, double p) {
    const float hi = CVT ? tf32_rn_cvt((float)p) : tf32_rn((float)p);
    const float lo = (float)(p - (double)hi);
    pb[o] = hi;
    pb[TC_PB_FLOATS / 2 + o] = CVT ? tf32_rn_cvt(lo) : tf32_rn(lo);
}

// Both tensor-path operands of a finished PT (leading dimension ld) in the tiles' order, 256 threads.
template <bool CVT>
__device__ __forceinline__ void tc_store_operands(const double *PT, int ld, float *pb, float *pf, int tid) {
    for (int o = tid; o < 4096; o += 256) {
        const int r = (o >> 8) * 4 + (o & 3), c = (o >> 2) & 63;       // tc_pb_index(r, c) == o
        tc_split_store<CVT>(pb, o, PT[r * ld + c]);
        pf[tc_ptf_index(o >> 6, o & 63)] = (float)PT[(o >> 6) * ld + (o & 63)];
    }
}

// Row-sum norm of a 64x64 matrix A held transposed in X (leading dimension LD64): the 64 sums by threads 0..63 into red,
// then their maximum and a NaN / inf scan by warp 0 (fmax is exact).  Called by every thread of the CTA; the result and
// `bad` are valid in warp 0.
__device__ __forceinline__ double expm64_norm(const double *X, double *red, int tid, bool &bad) {
    if (tid < 64) {
        double s = 0.0;
        for (int j = 0; j < 64; j++) s += fabs(X[j * LD64 + tid]);
        red[tid] = s;
    }
    __syncthreads();
    double m = 0.0;
    bad = false;
    if (tid < 32) {
        m = fmax(red[tid], red[tid + 32]);
        bad = !(red[tid] == red[tid]) || !(red[tid + 32] == red[tid + 32]) || isinf(red[tid]) || isinf(red[tid + 32]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
        bad = __any_sync(0xffffffffu, bad);
    }
    return m;
}


// ------------------------------------------------------------------------------------------------
// Shared-powers path, stage 1: one small CTA per batch entry.  Measures the entry (weight = sum of |values|: formula
// values of a compiled hand-over, matrix entries of a dense one), keeps the resident copy of the input (Vres / Qres:
// hb2_time_resident replays from it) and decides whether the entry is a scalar multiple of its group's reference
// direction:  |v_k[f] * w_ref - v_ref[f] * w_k| <= 1e-13 * |v_ref[f]| * w_k  for every value f, so every value matches
// its scaled reference value to 1e-13 of itself and a zero matches only a zero (a bound by the value's share of the weight,
// 1e-13 * w_k * w_ref, would let a value with a small share drift by far more than 1e-13 of itself).  The reference is either
// entry ref[k] of this batch (its powers are (re)built by expm_powers_kernel in this launch sequence) or, for small
// batches, the direction the group's power table was last built from (refvec, kept on the device).
// ------------------------------------------------------------------------------------------------
struct ExpmClassifyArgs {
    const double *V;          // compiled input [n][nV] or dense input [n][D*D] (nV = D*D)
    int nV;
    int kind;                 // 1 compiled, 2 dense
    const int *dst;           // [n]
    const int *group;         // [n]
    const int *ref;           // [n] batch index of the group's reference entry, or -1: use the cached direction
    ExpmGroup *groups;        // [G]; the weight of a group whose reference entry is in the batch is written here
    const double *refvec;     // [G][nVmax] cached reference directions
    int refvec_stride;
    double *weight;           // out [n]
    int *flag;                // out [n]
    double *res;              // nullable: resident copy [slots][nV]
};

// What both classification kernels do once an entry's sums and flag are known.  The weight of a group's reference entry
// (k == ref[k]) goes to the group's record here rather than in expm_powers_kernel, which runs at the same time on the
// partition's side stream and writes only the other fields (nu, kind).
__device__ __forceinline__ void expm_classify_result(const ExpmClassifyArgs &a, int k, int g, int r, int ok, double wk) {
    a.flag[k] = ok;
    a.weight[k] = wk;
    if (g >= 0 && r == k) a.groups[g].weight = wk;
}

// The reference of an entry of group g (g < 0: none): entry r of this batch, or for r < 0 the direction the group's
// table was last built from, if it holds this kind of input; then wr_cached is that table's weight, otherwise -1.
__device__ __forceinline__ const double *expm_classify_ref(const ExpmClassifyArgs &a, int g, int r, double &wr_cached) {
    wr_cached = -1.0;
    if (g < 0) return nullptr;
    if (r >= 0) return a.V + (size_t)r * a.nV;
    if (a.groups[g].kind != a.kind) return nullptr;
    wr_cached = a.groups[g].weight;
    return a.refvec + (size_t)g * a.refvec_stride;
}

// The acceptance test: a reference and two finite weights, the reference's positive (NaN fails every comparison) ...
__device__ __forceinline__ bool expm_classify_usable(const double *vr, double wk, double wr) {
    return (vr != nullptr) && (wr > 0.0) && (wk >= 0.0) && (wk < INFINITY) && (wr < INFINITY);
}
// ... and every value x matching its reference value xr scaled by wk / wr to tol = 1e-13 * wk of |xr|.
__device__ __forceinline__ bool expm_classify_match(double x, double xr, double wk, double wr, double tol) {
    return fabs(x * wr - xr * wk) <= tol * fabs(xr);
}

// Inputs of more than 256 values (dense: nV = D*D <= 4096): each thread holds its up to EXPM_CLASSIFY_REGS values of the
// entry and of the reference in registers, all loads issued before any sum, so the entry is read from memory once and the
// proportionality check runs from registers.  Values f = tid + 128 i are summed in increasing i, as a plain strided loop
// would; the loop past the register tile only serves longer compiled inputs.
constexpr int EXPM_CLASSIFY_REGS = 32;
__global__ void __launch_bounds__(128) expm_classify_kernel(ExpmClassifyArgs a) {
    __shared__ double red[2][4];
    __shared__ int bad[4];
    const int k = blockIdx.x, tid = threadIdx.x, nV = a.nV;
    const int slot = a.dst[k];
    if (slot < 0) { if (tid == 0) expm_classify_result(a, k, -1, -1, 0, 0.0); return; }
    const double *v = a.V + (size_t)k * nV;
    const int g = a.group[k], r = a.ref[k];
    double wr_cached;
    const double *vr = expm_classify_ref(a, g, r, wr_cached);
    double xv[EXPM_CLASSIFY_REGS], xr[EXPM_CLASSIFY_REGS];
#pragma unroll
    for (int i = 0; i < EXPM_CLASSIFY_REGS; i++) {
        const int f = tid + 128 * i;
        xv[i] = f < nV ? v[f] : 0.0;
        xr[i] = vr && f < nV ? vr[f] : 0.0;
    }
    double wk = 0.0, wr = 0.0;
#pragma unroll
    for (int i = 0; i < EXPM_CLASSIFY_REGS; i++) {       // the zeros past nV leave the (non-negative) sums unchanged
        wk += fabs(xv[i]);
        wr += fabs(xr[i]);
    }
    for (int f = tid + 128 * EXPM_CLASSIFY_REGS; f < nV; f += 128) {
        wk += fabs(v[f]);
        if (vr) wr += fabs(vr[f]);
    }
    if (a.res) {
        double *res = a.res + (size_t)slot * nV;
#pragma unroll
        for (int i = 0; i < EXPM_CLASSIFY_REGS; i++) if (tid + 128 * i < nV) res[tid + 128 * i] = xv[i];
        for (int f = tid + 128 * EXPM_CLASSIFY_REGS; f < nV; f += 128) res[f] = v[f];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { wk += __shfl_xor_sync(0xffffffffu, wk, o); wr += __shfl_xor_sync(0xffffffffu, wr, o); }
    if ((tid & 31) == 0) { red[0][tid >> 5] = wk; red[1][tid >> 5] = wr; }
    __syncthreads();
    wk = red[0][0] + red[0][1] + red[0][2] + red[0][3];
    wr = red[1][0] + red[1][1] + red[1][2] + red[1][3];
    if (wr_cached >= 0.0) wr = wr_cached;
    int ok = expm_classify_usable(vr, wk, wr);
    if (ok) {
        const double tol = 1e-13 * wk;
#pragma unroll
        for (int i = 0; i < EXPM_CLASSIFY_REGS; i++)
            if (tid + 128 * i < nV && !expm_classify_match(xv[i], xr[i], wk, wr, tol)) ok = 0;
        for (int f = tid + 128 * EXPM_CLASSIFY_REGS; f < nV; f += 128)
            if (!expm_classify_match(v[f], vr[f], wk, wr, tol)) ok = 0;
    }
    ok = __all_sync(0xffffffffu, ok);
    if ((tid & 31) == 0) bad[tid >> 5] = !ok;
    __syncthreads();
    if (tid == 0) expm_classify_result(a, k, g, r, !(bad[0] | bad[1] | bad[2] | bad[3]), wk);
}

// The same classification with one WARP per entry, eight entries per CTA, for short inputs (compiled hand-overs: ~50 formula
// values): 1588 CTAs of 128 threads that each touch 47 doubles cost 17 us of launch and drain; n/8 CTAs are one wave.
// (Sums are taken lane-strided, then by xor-shuffle: a fixed order, different from the 128-thread kernel's.)
__global__ void __launch_bounds__(256) expm_classify_warp_kernel(ExpmClassifyArgs a, int n) {
    const int lane = threadIdx.x & 31, k = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (k >= n) return;
    const int slot = a.dst[k];
    if (slot < 0) { if (lane == 0) expm_classify_result(a, k, -1, -1, 0, 0.0); return; }
    const double *v = a.V + (size_t)k * a.nV;
    const int g = a.group[k], r = a.ref[k];
    double wr_cached;
    const double *vr = expm_classify_ref(a, g, r, wr_cached);
    double wk = 0.0, wr = 0.0;
    for (int f = lane; f < a.nV; f += 32) {
        const double x = v[f];
        wk += fabs(x);
        if (vr) wr += fabs(vr[f]);
        if (a.res) a.res[(size_t)slot * a.nV + f] = x;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { wk += __shfl_xor_sync(0xffffffffu, wk, o); wr += __shfl_xor_sync(0xffffffffu, wr, o); }
    if (wr_cached >= 0.0) wr = wr_cached;
    int ok = expm_classify_usable(vr, wk, wr);
    if (ok) {
        const double tol = 1e-13 * wk;
        for (int f = lane; f < a.nV; f += 32)
            if (!expm_classify_match(v[f], vr[f], wk, wr, tol)) ok = 0;
    }
    ok = __all_sync(0xffffffffu, ok);
    if (lane == 0) expm_classify_result(a, k, g, r, ok, wk);
}

// Shared-powers entry: rho = ||A||_inf estimated from the entry's weight w and its group's reference (nu, wref), and the
// squarings that bring it to rho / 2^shift <= EXPM_POLY_THETA.  expm_poly_kernel evaluates the polynomial there;
// expm64_dmma_kernel squares it, or writes NaN (expm_poly_nan).
__device__ __forceinline__ int expm_poly_shift(double nu, double wref, double w, double &rho) {
    rho = nu * (w / wref);
    int shift = 0;
    if (rho > EXPM_POLY_THETA) { int e = 0; frexp(rho / EXPM_POLY_THETA, &e); shift = max(e, 0); }
    return shift;
}
__device__ __forceinline__ int expm_poly_shift(const ExpmArgs &a, int k, double &rho) {
    const ExpmGroup gi = a.groups[a.group[k]];
    return expm_poly_shift(gi.nu, gi.weight, a.weight[k], rho);
}
// NaN input or absurd rates: the entry's matrix is NaN.
__device__ __forceinline__ bool expm_poly_nan(int shift, double rho) { return !(rho == rho) || shift > 900; }
// Live entry k has been finished by expm_poly_kernel: shared powers, no squaring and a usable rate.
__device__ __forceinline__ bool expm_poly_finished(const ExpmArgs &a, int k) {
    double rho;
    return a.flag && a.flag[k] && expm_poly_shift(a, k, rho) == 0 && rho == rho;
}

// One entry of expm64_dmma_kernel, listed by it as live and not finished by expm_poly_kernel.  Three shared 64x64 fp64
// buffers (101 KB) so that TWO CTAs share an SM and one CTA's load/norm/epilogue phases overlap the other's DMMA
// products:  X0 = A -> later R,  X1 = A^2,  X2 = A^3.  The polynomial blocks need A at the thread's own output positions
// after X0 has become R: those values are parked in the (not yet written) output slot PT[slot] in global memory (L2
// resident, same [row][col] layout) and re-read per Horner step.  Every exit is CTA-uniform; the caller separates entries
// with a barrier.  Kept out of line: inlined into the kernel's entry loop, the body no longer fits the 128 registers of two
// CTAs per SM and spills.
__device__ __noinline__ void expm64_dmma_entry(const ExpmArgs a, const ExpmTcOut tc, int entry, double *sm) {
    double *X0 = sm, *X1 = X0 + 64 * LD64, *X2 = X1 + 64 * LD64;
    __shared__ double red[64];
    __shared__ int s_shift, s_Q;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wr = warp >> 1, wc = warp & 1, g = lane >> 2, q4 = lane & 3;
    const int D = a.D;
    const size_t slot = a.dst[entry];
    double *out = a.PT + slot * 4096;
    double *park = out;
    double *R = X0;

    const bool shared_powers = a.flag && a.flag[entry];
    if (shared_powers) {
        // expm_poly_kernel has left the Taylor polynomial of A / 2^shift in the output slot; squarings and the epilogue
        // (clamp, row repair, tensor-path operands) remain.  shift is recomputed exactly as the polynomial stage chose it.
        double rho;
        const int shift = expm_poly_shift(a, entry, rho);
        if (expm_poly_nan(shift, rho)) { expm64_poison(out, tc, slot, tid); return; }
        for (int idx = tid; idx < 4096; idx += 256) R[(idx >> 6) * LD64 + (idx & 63)] = __ldcg(out + idx);
        if (tid == 0) s_shift = shift;
        __syncthreads();
    } else
    load_rate_matrix<64, LD64, 256>(a, X0, tid, entry);
    if (shared_powers || !a.is_trans) {
      double acc[2][4][2];
      auto zero = [&]() {
#pragma unroll
          for (int i = 0; i < 2; i++)
#pragma unroll
              for (int j = 0; j < 4; j++) { acc[i][j][0] = 0.0; acc[i][j][1] = 0.0; }
      };
      auto off = [&](int i, int j) { return (16 * wr + 8 * i + g) * LD64 + 32 * wc + 8 * j + 2 * q4; };
      auto goff = [&](int i, int j) { return (16 * wr + 8 * i + g) * 64 + 32 * wc + 8 * j + 2 * q4; };
      auto store = [&](double *M) {
#pragma unroll
          for (int i = 0; i < 2; i++)
#pragma unroll
              for (int j = 0; j < 4; j++) *reinterpret_cast<double2 *>(M + off(i, j)) = make_double2(acc[i][j][0], acc[i][j][1]);
      };
      if (!shared_powers) {
        bool bad;
        const double m = expm64_norm(X0, red, tid, bad);
        if (tid == 0) {
            int shift = 0;
            if (!bad && m > 0.975) {
                int e = 0;
                frexp(m / 0.975, &e);          // m/0.975 = f*2^e, f in [0.5,1)  ->  m/2^e <= 0.975
                shift = max(e, 0);
            }
            const double theta = bad ? 0.0 : ldexp(m, -shift);
            s_Q = theta <= 0.0064 ? 1 : theta <= 0.069 ? 2 : theta <= 0.245 ? 3 : theta <= 0.55 ? 4 : 5;
            s_shift = bad ? -1 : shift;
        }
        __syncthreads();
        const int shift = s_shift, Q = s_Q;
        if (shift < 0 || shift > 900) { expm64_poison(out, tc, slot, tid); return; }   // NaN/inf or absurd rates
        {   // scale A in place and park a copy in the output slot (coalesced)
            const double sc = exp2i(-shift);
            for (int idx = tid; idx < 64 * 64; idx += 256) {
                const int o = (idx >> 6) * LD64 + (idx & 63);
                const double v = X0[o] * sc;
                X0[o] = v;
                park[idx] = v;
            }
            __syncthreads();
        }
        zero(); tile_mm64_dmma(X0, X0, wr, wc, g, q4, acc); store(X1);
        __syncthreads();
        zero(); tile_mm64_dmma(X1, X0, wr, wc, g, q4, acc); store(X2);
        __syncthreads();                             // every warp is done reading A from X0: it becomes R
        // R = B_Q, then R = R*A3 + B_q for q = Q-1..0, with B_q = c_{3q} I + c_{3q+1} A + c_{3q+2} A^2 at own positions
        auto poly2 = [&](int qq, int i, int j) -> double2 {
            const int r = 16 * wr + 8 * i + g, c = 32 * wc + 8 * j + 2 * q4;
            const double2 a1 = __ldcg(reinterpret_cast<const double2 *>(park + goff(i, j)));
            const double2 a2 = *reinterpret_cast<const double2 *>(X1 + off(i, j));
            double2 v = make_double2(c_taylor[3 * qq + 1] * a1.x + c_taylor[3 * qq + 2] * a2.x,
                                     c_taylor[3 * qq + 1] * a1.y + c_taylor[3 * qq + 2] * a2.y);
            if (r == c) v.x += c_taylor[3 * qq];
            if (r == c + 1) v.y += c_taylor[3 * qq];
            return v;
        };
#pragma unroll
        for (int i = 0; i < 2; i++)
#pragma unroll
            for (int j = 0; j < 4; j++) *reinterpret_cast<double2 *>(R + off(i, j)) = poly2(Q, i, j);
        __syncthreads();
        for (int qq = Q - 1; qq >= 0; qq--) {
            zero(); tile_mm64_dmma(R, X2, wr, wc, g, q4, acc);
            __syncthreads();
#pragma unroll
            for (int i = 0; i < 2; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const double2 pv = poly2(qq, i, j);
                    *reinterpret_cast<double2 *>(R + off(i, j)) = make_double2(acc[i][j][0] + pv.x, acc[i][j][1] + pv.y);
                }
            __syncthreads();
        }
      }   // general path: R = Taylor polynomial of A / 2^shift
        const int n_sq = s_shift;
        for (int s = 0; s < n_sq; s++) {
            zero(); tile_mm64_dmma(R, R, wr, wc, g, q4, acc);
            __syncthreads();
            store(R);
            __syncthreads();
        }
        // clamp negatives, zero the padding, repair: column k of PT (= row k of P) must sum to 1
        for (int idx = tid; idx < 64 * 64; idx += 256) {
            int j = idx >> 6, kk = idx & 63;
            double v = R[j * LD64 + kk];
            if (j >= D || kk >= D) v = 0.0; else if (v < 0.0) v = 0.0;
            R[j * LD64 + kk] = v;
        }
        __syncthreads();
        {   // column sums by all 256 threads: 4 threads per column, 16 rows each
            const int col = tid & 63, part = tid >> 6;
            double s = 0.0;
            for (int j = part * 16; j < part * 16 + 16; j++) if (j != col) s += R[j * LD64 + col];
            X1[part * 64 + col] = s;                 // X1 (A^2) is no longer needed
        }
        __syncthreads();
        if (tid < D) R[tid * LD64 + tid] = fmax(1.0 - (X1[tid] + X1[64 + tid] + X1[128 + tid] + X1[192 + tid]), 0.0);
        __syncthreads();
    }
    for (int idx = tid; idx < 4096; idx += 256) out[idx] = R[(idx >> 6) * LD64 + (idx & 63)];
    if (tc.PB) tc_store_operands<true>(R, LD64, tc.PB + slot * TC_PB_FLOATS, tc.PTf + slot * TC_PTF_FLOATS, tid);
}

// One wave of CTAs (gridDim.x <= 2 per SM) striding over the n entries of a batch.  Per round of up to 256 entries of
// its share, the CTA first lists the entries with work left, one thread per entry (on the shared-powers path
// expm_poly_kernel has finished most of them), then processes the listed ones in turn.
__global__ void __launch_bounds__(256, 2) expm64_dmma_kernel(ExpmArgs a, ExpmTcOut tc, int n) {
    extern __shared__ __align__(16) double sm[];
    __shared__ int s_list[256], s_count;
    for (int base = blockIdx.x; base < n; base += 256 * gridDim.x) {
        if (threadIdx.x == 0) s_count = 0;
        __syncthreads();
        const int k = base + threadIdx.x * gridDim.x;
        if (k < n && a.dst[k] >= 0 && !expm_poly_finished(a, k)) s_list[atomicAdd(&s_count, 1)] = k;
        __syncthreads();
        const int count = s_count;
        for (int j = 0; j < count; j++) {
            expm64_dmma_entry(a, tc, s_list[j], sm);
            __syncthreads();                     // the next entry overwrites the shared buffers
        }
        __syncthreads();                         // every thread has read s_count
    }
}

// ------------------------------------------------------------------------------------------------
// Shared-powers path, stage 2: S_m = R^m / m! (PT layout, i.e. powers of the TRANSPOSED reference matrix), m = 1..24, for
// every group whose reference is (re)established in this batch.  grid = (24, number of such groups); CTA (j, g) produces
// S_{j+1}:  j = 0 assembles the reference matrix, normalises it (R = A_ref / ||A_ref||_inf -> S_1) and records the
// group's nu, kind and direction; CTA j >= 1 multiplies two EARLIER coefficient matrices,
//     S_m = S_a S_b / C(m, a),   (a, b) = (1,1) (2,1) (2,2) (4,1..4) (8,1..8) (16,1..8),
// which it awaits on generation flags (flag[group][m] == gen once S_m is complete; the producer fences before it
// publishes).  Blocks are dispatched in index order and only wait for lower indices of their own column, so the scheme
// cannot deadlock even if not all of them are co-resident; waits are time-bounded like every device-side wait here.
// Critical path: 5 products instead of 23.  The kernel runs on the partition's side stream while the classification runs
// (launch_expm), so it reads none of the classification's outputs and writes nothing the classification reads for the
// batch: the groups it rebuilds have no entry classified against their cached direction (plan_shared).
// ------------------------------------------------------------------------------------------------
struct ExpmPowersArgs {
    ExpmArgs a;               // input description (dense or compiled); a.Qres must be null, a.weight / a.flag unused
    const int *refs;          // [gridDim.y] batch indices of the reference entries
    ExpmGroup *groups;        // out
    double *pow;              // out [G][EXPM_POW_TERMS][4096]
    double *refvec;           // out [G][refvec_stride]
    int refvec_stride, nV, kind;
    const double *Vin;        // the raw input vectors [n][nV] (formula values or dense entries)
    unsigned long long *flags;   // [G][EXPM_POW_TERMS] generation of each coefficient matrix
    unsigned long long gen;
    int *err;
};

__device__ __forceinline__ bool expm_await_flag(const unsigned long long *f, unsigned long long gen, int *err) {
    unsigned long long t0 = 0;
    for (int it = 0;; it++) {
        unsigned long long v;
        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(f) : "memory");
        if (v == gen) return true;
        if ((it & 255) == 255) {
            const unsigned long long now = globaltimer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > HB2_WAIT_LIMIT_NS) { atomicExch(err, WAIT_EXPM_POWERS); return false; }
        }
    }
}

__global__ void __launch_bounds__(256, 1) expm_powers_kernel(ExpmPowersArgs pa) {
    extern __shared__ __align__(16) double sm[];
    double *X0 = sm, *X1 = X0 + 64 * LD64;
    __shared__ double red[64];
    __shared__ double s_nu;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wr = warp >> 1, wc = warp & 1, g = lane >> 2, q4 = lane & 3;
    const int entry = pa.refs[blockIdx.y];
    const int grp = pa.a.group[entry];
    if (grp < 0 || pa.a.dst[entry] < 0) return;                       // (cannot happen: the host lists live references only)
    const int m = blockIdx.x + 1;                                      // this CTA produces S_m
    double *pw = pa.pow + (size_t)grp * EXPM_POW_TERMS * 4096;
    unsigned long long *flags = pa.flags + (size_t)grp * EXPM_POW_TERMS;
    if (m == 1) {
        load_rate_matrix<64, LD64, 256>(pa.a, X0, tid, entry);        // X0 = A_ref^T, zero padded
        bool bad;
        const double mx = expm64_norm(X0, red, tid, bad);
        if (tid == 0) s_nu = (bad || !(mx > 0.0)) ? 0.0 : mx;
        __syncthreads();
        const double nu = s_nu;
        if (tid == 0) {                      // the weight is the classification's (expm_classify_result), written beside this
            pa.groups[grp].nu = nu;
            pa.groups[grp].kind = nu > 0.0 ? pa.kind : 0;
        }
        // (no entry can have been flagged against a reference with nu == 0; the other CTAs of the column still need S_1)
        const double inv = nu > 0.0 ? 1.0 / nu : 0.0;
        for (int idx = tid; idx < 4096; idx += 256) pw[4096 + idx] = X0[(idx >> 6) * LD64 + (idx & 63)] * inv;
        __threadfence();
        __syncthreads();
        if (tid == 0) asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(flags + 1), "l"(pa.gen) : "memory");
        // the direction is read by later batches only: off the critical path of the products
        for (int f = tid; f < pa.nV; f += 256) pa.refvec[(size_t)grp * pa.refvec_stride + f] = pa.Vin[(size_t)entry * pa.nV + f];
        return;
    }
    const int a = m <= 2 ? 1 : m <= 4 ? 2 : m <= 8 ? 4 : m <= 16 ? 8 : 16, b = m - a;
    if (tid == 0) expm_await_flag(flags + a, pa.gen, pa.err);
    if (tid == 32) expm_await_flag(flags + b, pa.gen, pa.err);
    __syncthreads();
#pragma unroll
    for (int it = 0; it < 8; it++) {                                  // both operands as double2, coalesced, all loads in flight
        const int idx = tid + 256 * it, r = idx >> 5, c2 = (idx & 31) * 2;
        *reinterpret_cast<double2 *>(X0 + r * LD64 + c2) = __ldcg(reinterpret_cast<const double2 *>(pw + (size_t)a * 4096 + r * 64 + c2));
        *reinterpret_cast<double2 *>(X1 + r * LD64 + c2) = __ldcg(reinterpret_cast<const double2 *>(pw + (size_t)b * 4096 + r * 64 + c2));
    }
    __syncthreads();
    double acc[2][4][2];
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) { acc[i][j][0] = 0.0; acc[i][j][1] = 0.0; }
    tile_mm64_dmma(X0, X1, wr, wc, g, q4, acc);                       // S_a * S_b (powers of one matrix commute)
    double binom = 1.0;                                                // C(m, a), exact in fp64 for m <= 24
    for (int i = 1; i <= a; i++) binom = binom * (double)(m - a + i) / (double)i;
    const double inv = 1.0 / binom;
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int r = 16 * wr + 8 * i + g, c = 32 * wc + 8 * j + 2 * q4;
            __stcg(reinterpret_cast<double2 *>(pw + (size_t)m * 4096 + r * 64 + c), make_double2(acc[i][j][0] * inv, acc[i][j][1] * inv));
        }
    __threadfence();
    __syncthreads();
    if (tid == 0) asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(flags + m), "l"(pa.gen) : "memory");
}

// ------------------------------------------------------------------------------------------------
// Shared-powers path, stage 3: P = sum_m S_m x^m with x = rho / 2^shift <= EXPM_POLY_THETA for every flagged entry, fused
// with the epilogue for the (common) entries that need no squaring.
// grid = (16 row slices, chunks of EXPM_POLY_CHUNK entries); the 16 slices of a chunk form one thread-block cluster
// (EXPM_POLY_CLUSTER, a non-portable size).  Thread t of slice sl owns element (row 4 sl + t%4, column t/4) of the PT
// layout (row = child state, column = parent state) and keeps that element's 24 coefficients in registers while it walks
// its chunk (reloaded only when the group changes: batches are class-major); the chunk's metadata is fetched up front so
// that the loop carries no dependent global loads.
//   shift == 0: the value is final up to the row repair.  It is clamped at 0, padding is zeroed, and PT (fp64), PTf (fp32
//               table) and PB (tf32 hi/lo tiles; chunk sl of the canonical layout is exactly this slice, offset t) are
//               written directly; the partial column sums of the slice (4 rows, diagonal excluded; 4 adjacent lanes) stay
//               in shared memory.  After a cluster barrier the slice that holds diagonal (c, c) adds the 16 slices'
//               partials of column c through distributed shared memory, in slice order, and writes 1 - sum (clamped at 0):
//               rows of P sum to 1.  The entry is then final.
//   shift  > 0: the raw polynomial value goes to PT; expm64_dmma_kernel squares and finishes the entry.
// ------------------------------------------------------------------------------------------------
constexpr int EXPM_POLY_CHUNK = 16;
constexpr int EXPM_POLY_CLUSTER = 16;
__global__ void __launch_bounds__(256, 3) expm_poly_kernel(ExpmArgs a, ExpmTcOut tc, int n) {
    __shared__ int s_slot[EXPM_POLY_CHUNK], s_grp[EXPM_POLY_CHUNK], s_fin[EXPM_POLY_CHUNK];
    __shared__ double s_wgt[EXPM_POLY_CHUNK];
    __shared__ double s_part[EXPM_POLY_CHUNK][64];                  // this slice's column partials of the finished entries
    const int tid = threadIdx.x, sl = blockIdx.x;
    const int row = 4 * sl + (tid & 3), col = tid >> 2;
    const int e = row * 64 + col;                                     // element index in the 64x64 PT layout
    const double unit = (row == col) ? 1.0 : 0.0;
    const bool pad = row >= a.D || col >= a.D;
    const int k0 = blockIdx.y * EXPM_POLY_CHUNK;
    if (tid < EXPM_POLY_CHUNK) {                                      // the chunk's metadata, once per CTA
        const int k = k0 + tid;
        int sv = -1, gv = -1;
        double wv = 0.0;
        if (k < n) {
            sv = a.dst[k];
            if (sv >= 0 && !a.flag[k]) sv = -1;
            gv = a.group[k];
            wv = a.weight[k];
        }
        s_slot[tid] = sv; s_grp[tid] = gv; s_wgt[tid] = wv; s_fin[tid] = 0;
    }
    __syncthreads();
    double c[EXPM_POW_TERMS];
    int cur = -1;
    double nu = 0.0, wref = 1.0;
    const int out_pt = e, out_ptf = tc_ptf_index(row, col), out_pb = tc_pb_index(row, col);   // out_pb = 256 sl + tid
    for (int i = 0; i < EXPM_POLY_CHUNK; i++) {
        const int slot = s_slot[i];
        if (slot < 0) continue;
        if (s_grp[i] != cur) {
            cur = s_grp[i];
            const double *pw = a.pow + (size_t)cur * EXPM_POW_TERMS * 4096 + e;
#pragma unroll
            for (int m = 1; m < EXPM_POW_TERMS; m++) c[m] = __ldcg(pw + (size_t)m * 4096);
            nu = a.groups[cur].nu; wref = a.groups[cur].weight;
        }
        double rho;
        const int shift = expm_poly_shift(nu, wref, s_wgt[i], rho);
        if (expm_poly_nan(shift, rho)) continue;                      // the finishing kernel writes NaN
        const double x = shift > 0 ? ldexp(rho, -shift) : rho;
        // p(x) = 1 + x (c1 + c3 x^2 + .. + c23 x^22) + x^2 (c2 + c4 x^2 + .. + c24 x^22): two interleaved Horner chains in
        // x^2 halve the dependent-FMA depth
        static_assert(EXPM_POW_TERMS == 25, "the even/odd split below assumes degree 24");
        const double x2 = x * x;
        double ve = c[24], vo = c[23];
#pragma unroll
        for (int m = 22; m >= 2; m -= 2) { ve = fma(ve, x2, c[m]); vo = fma(vo, x2, c[m - 1]); }
        double v = fma(vo, x, fma(ve, x2, unit));
        const size_t sidx = (size_t)slot;
        if (shift > 0) { __stcg(a.PT + sidx * 4096 + out_pt, v); continue; }
        v = (pad || v < 0.0) ? 0.0 : v;
        // column sums over this slice's 4 rows (lanes t, t^1, t^2, t^3 share a column), diagonal element excluded
        double part = (row == col) ? 0.0 : v;
        part += __shfl_xor_sync(0xffffffffu, part, 1);
        part += __shfl_xor_sync(0xffffffffu, part, 2);
        if ((tid & 3) == 0) s_part[i][col] = part;
        if (tid == 0) s_fin[i] = 1;
        if (row != col) {                                             // the diagonal is written after the cluster barrier
            __stcg(a.PT + sidx * 4096 + out_pt, v);
            if (tc.PB) {
                tc.PTf[sidx * TC_PTF_FLOATS + out_ptf] = (float)v;
                tc_split_store<true>(tc.PB + sidx * TC_PB_FLOATS, out_pb, v);
            }
        }
    }
    // row repair: thread t handles entry t/4 and diagonal column 4 sl + t%4
    static_assert(4 * EXPM_POLY_CHUNK <= 256, "one thread per (entry, diagonal column) of the slice");
    cooperative_groups::cluster_group cluster = cooperative_groups::this_cluster();
    cluster.sync();                                                   // every slice's partials are in its shared memory
    if (tid < 4 * EXPM_POLY_CHUNK && s_fin[tid >> 2]) {
        const int i = tid >> 2, c = 4 * sl + (tid & 3);
        double s = 0.0;
#pragma unroll
        for (int r = 0; r < EXPM_POLY_CLUSTER; r++) s += cluster.map_shared_rank(&s_part[i][0], r)[c];
        const double d = c < a.D ? fmax(1.0 - s, 0.0) : 0.0;
        const size_t sidx = (size_t)s_slot[i];
        a.PT[sidx * 4096 + c * 64 + c] = d;
        if (tc.PB) {
            tc.PTf[sidx * TC_PTF_FLOATS + tc_ptf_index(c, c)] = (float)d;
            tc_split_store<true>(tc.PB + sidx * TC_PB_FLOATS, tc_pb_index(c, c), d);
        }
    }
    cluster.sync();                                                   // peers may still be reading this slice's partials
}

// Explicit-form mixtures (BS-REL, reference tree.cpp:3047-3089): PT[slot_i] = sum_k w[i][k] * comp[i*K + k], components
// added in order k = 0..K-1 (deterministic); 64-state tensor partitions also get the split tiles and the fp32 table, the
// split rounded by tf32_rn (unlike the exponential's epilogues).
// One CTA per node; comp = scratch matrices [n*K][Dp*Dp] in the PT layout (transposed).
__global__ void __launch_bounds__(256) mix_reduce_kernel(const double *__restrict__ comp, const double *__restrict__ w,
                                                          const int *__restrict__ slots, int K, int Dp, double *__restrict__ PT,
                                                          float *__restrict__ PB, float *__restrict__ PTf) {
    const size_t slot = slots[blockIdx.x];
    const int dpdp = Dp * Dp;
    double *dst = PT + slot * dpdp;
    const double *src = comp + (size_t)blockIdx.x * K * dpdp;
    const double *wk = w + (size_t)blockIdx.x * K;
    for (int o = threadIdx.x; o < dpdp; o += 256) {
        double s = 0.0;
        for (int k = 0; k < K; k++) s += wk[k] * src[(size_t)k * dpdp + o];
        dst[o] = s;
    }
    if (PB && Dp == 64) {
        __syncthreads();                         // this CTA's own global writes are visible to it after the barrier
        tc_store_operands<false>(dst, 64, PB + slot * TC_PB_FLOATS, PTf + slot * TC_PTF_FLOATS, threadIdx.x);
    }
}

// Small state spaces (Dp <= 32): one CTA of 128 threads per matrix, plain shared-memory products.
constexpr size_t expm_small_smem_bytes(int DP) { return (size_t)6 * DP * (DP + 1) * sizeof(double); }

// The per-entry rules of the small-state exponential, shared by expm_small_kernel (one matrix per CTA) and
// expm_rates_kernel (several per CTA).  Matrices sit in shared memory transposed, leading dimension LD: A1[j*LD + i] = A[i][j].
// Row-sum norm of row i of A (column i of A1), in column order.
template <int DP, int LD>
__device__ __forceinline__ double expm_small_norm(const double *A1, int i) {
    double s = 0.0;
    for (int j = 0; j < DP; j++) s += fabs(A1[j * LD + i]);
    return s;
}

// Scaling shift from the DP row norms: the binary exponent of the largest, at least 0; -1 when one is NaN or infinite.
template <int DP>
__device__ __forceinline__ int expm_small_shift(const double *red) {
    double m = 0.0; bool bad = false;
    for (int i = 0; i < DP; i++) { if (!(red[i] == red[i]) || isinf(red[i])) bad = true; m = fmax(m, red[i]); }
    int e = 0;
    if (m > 0.0) frexp(m, &e);
    return bad ? -1 : max(e, 0);
}

// Entry (r, c) of X*Y, fma over k in order.
template <int DP, int LD>
__device__ __forceinline__ double expm_small_dot(const double *X, const double *Y, int r, int c) {
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < DP; k++) s = fma(X[r * LD + k], Y[k * LD + c], s);
    return s;
}

// Entry (r, c) of the q-th Horner block c_{4q} I + c_{4q+1} A + c_{4q+2} A^2 + c_{4q+3} A^3.
template <int LD>
__device__ __forceinline__ double expm_small_poly(const double *A1, const double *A2, const double *A3, int q, int r, int c) {
    int o = r * LD + c;
    double v = c_taylor[4 * q + 1] * A1[o] + c_taylor[4 * q + 2] * A2[o] + c_taylor[4 * q + 3] * A3[o];
    if (r == c) v += c_taylor[4 * q];
    return v;
}

// Padding and negative entries of the result go to 0.
__device__ __forceinline__ double expm_small_clamp(double v, int j, int k, int D) {
    if (j >= D || k >= D) v = 0.0; else if (v < 0.0) v = 0.0;
    return v;
}

// Diagonal repair of column c of the clamped result R (a row of P): 1 minus its other entries, at least 0.
template <int DP, int LD>
__device__ __forceinline__ double expm_small_diag(const double *R, int c) {
    double s = 0.0;
    for (int j = 0; j < DP; j++) if (j != c) s += R[j * LD + c];
    return fmax(1.0 - s, 0.0);
}

// Barrier of one team: the CTA, a pair of warps (named barrier 1 + team), or a half-warp.
template <int T>
__device__ __forceinline__ void team_sync(int team) {
    if constexpr (T == 128) __syncthreads();
    else if constexpr (T == 64) {
        if (team == 0) asm volatile("bar.sync 1, 64;" ::: "memory");
        else asm volatile("bar.sync 2, 64;" ::: "memory");
    }
    else {
        static_assert(T == 16, "teams of 16, 64 or 128 threads");
        __syncwarp(0xffffu << (threadIdx.x & 16));
    }
}

// The small-state exponential of one matrix by a team of T threads (lt = 0..T-1), from the loaded, transposed A1 to the
// stored result: norm, shift (NaN for a NaN or infinite input or absurd rates), scaling, A^2, A^3, A^4, Horner blocks of
// degree 15, squarings, clamp, diagonal repair and the store to out.  A1 is the first of the team's 6 matrices of DP*LD
// doubles; red [DP] and s_shift are the team's shared scratch.  Every exit is team-uniform.
template <int DP, int T>
__device__ __forceinline__ void expm_small_body(double *A1, double *red, int &s_shift, int lt, int team, int D, double *out) {
    constexpr int LD = DP + 1, MS = DP * LD;
    double *A2 = A1 + MS, *A3 = A2 + MS, *A4 = A3 + MS, *R = A4 + MS, *Tm = R + MS;
    if (lt < DP) red[lt] = expm_small_norm<DP, LD>(A1, lt);
    team_sync<T>(team);
    if (lt == 0) s_shift = expm_small_shift<DP>(red);
    team_sync<T>(team);
    const int shift = s_shift;
    if (shift < 0 || shift > 900) {
        for (int idx = lt; idx < DP * DP; idx += T) out[idx] = __longlong_as_double(0x7ff8000000000000LL);
        return;
    }
    if (shift > 0) {
        const double sc = exp2i(-shift);
        for (int idx = lt; idx < DP * DP; idx += T) A1[(idx / DP) * LD + idx % DP] *= sc;
        team_sync<T>(team);
    }
    auto mm = [&](double *Cm, const double *X, const double *Y) {      // Cm = X*Y (Cm distinct from X,Y)
        for (int idx = lt; idx < DP * DP; idx += T) {
            int r = idx / DP, c = idx % DP;
            Cm[r * LD + c] = expm_small_dot<DP, LD>(X, Y, r, c);
        }
        team_sync<T>(team);
    };
    mm(A2, A1, A1); mm(A3, A2, A1); mm(A4, A2, A2);
    for (int idx = lt; idx < DP * DP; idx += T) R[(idx / DP) * LD + idx % DP] = expm_small_poly<LD>(A1, A2, A3, 3, idx / DP, idx % DP);
    team_sync<T>(team);
    for (int q = 2; q >= 0; q--) {
        mm(Tm, R, A4);
        for (int idx = lt; idx < DP * DP; idx += T) { int r = idx / DP, c = idx % DP; R[r * LD + c] = Tm[r * LD + c] + expm_small_poly<LD>(A1, A2, A3, q, r, c); }
        team_sync<T>(team);
    }
    for (int s = 0; s < shift; s++) {
        mm(Tm, R, R);
        for (int idx = lt; idx < DP * DP; idx += T) { int o = (idx / DP) * LD + idx % DP; R[o] = Tm[o]; }
        team_sync<T>(team);
    }
    for (int idx = lt; idx < DP * DP; idx += T) {
        int j = idx / DP, k = idx % DP;
        R[j * LD + k] = expm_small_clamp(R[j * LD + k], j, k, D);
    }
    team_sync<T>(team);
    if (lt < D) R[lt * LD + lt] = expm_small_diag<DP, LD>(R, lt);
    team_sync<T>(team);
    for (int idx = lt; idx < DP * DP; idx += T) out[idx] = R[(idx / DP) * LD + idx % DP];
}

template <int DP>
__global__ void __launch_bounds__(128) expm_small_kernel(ExpmArgs a) {
    constexpr int LD = DP + 1;
    extern __shared__ __align__(16) double sm[];          // 6 matrices of DP*LD doubles (expm_small_smem_bytes)
    __shared__ double red[DP];
    __shared__ int s_shift;
    const int tid = threadIdx.x;
    if (a.dst[blockIdx.x] < 0) return;
    double *out = a.PT + (size_t)a.dst[blockIdx.x] * DP * DP;
    load_rate_matrix<DP, LD, 128>(a, sm, tid);
    if (a.is_trans) {
        for (int idx = tid; idx < DP * DP; idx += 128) out[idx] = sm[(idx / DP) * LD + idx % DP];
        return;
    }
    expm_small_body<DP, 128>(sm, red, s_shift, tid, 0, a.D, out);
}

// ------------------------------------------------------------------------------------------------
// expm_rates_kernel (hb2_batch_site_rates): P = exp(r_s A_b) for every (set s, branch b) of a chunk, A_b the resident rate
// matrix of the call's class (d_Qres, row-major D*D), scaled by the set's rate while it is loaded.  A team of
// expm_rates_team(DP) threads owns one matrix and runs expm_small_body as expm_small_kernel does, so that rate 1 gives
// the resident path's matrices; 4 and 8 states pack 8 and 2 matrices into a CTA, one thread per entry.  Output: PT[s][b][DP*DP], transposed like every P.
// ------------------------------------------------------------------------------------------------
struct ExpmRatesArgs {
    const double *Q;          // [B][D*D] resident rate matrices of the class
    const double *rate;       // [sets]
    double *PT;               // [sets][B][DP*DP]
    int D, B;
    long long n;              // sets * B matrices
};

__host__ __device__ constexpr int expm_rates_team(int DP) { return DP * DP < 128 ? DP * DP : 128; }
constexpr size_t expm_rates_smem_bytes(int DP) { return (size_t)(128 / expm_rates_team(DP)) * expm_small_smem_bytes(DP); }

template <int DP>
__global__ void __launch_bounds__(128) expm_rates_kernel(ExpmRatesArgs a) {
    constexpr int LD = DP + 1, T = expm_rates_team(DP), M = 128 / T;
    extern __shared__ __align__(16) double sm[];          // M teams x 6 matrices of DP*LD doubles (expm_rates_smem_bytes)
    __shared__ double red_all[M][DP];
    __shared__ int shift_all[M];
    const int team = threadIdx.x / T, lt = threadIdx.x % T, D = a.D;
    const long long e = (long long)blockIdx.x * M + team;
    if (e >= a.n) return;
    double *A1 = sm + (size_t)team * 6 * DP * LD;
    const double r = a.rate[e / a.B];
    const double *Q = a.Q + (size_t)(e % a.B) * D * D;
    for (int idx = lt; idx < DP * DP; idx += T) {
        const int i = idx / DP, j = idx - i * DP;
        A1[j * LD + i] = (i < D && j < D) ? r * Q[(size_t)i * D + j] : 0.0;
    }
    team_sync<T>(team);
    expm_small_body<DP, T>(A1, red_all[team], shift_all[team], lt, team, D, a.PT + (size_t)e * DP * DP);
}


// A pinned node (PruneArgs::forced_node) keeps only the pattern's forced state f.
template <int N>
__device__ __forceinline__ void keep_state(double (&v)[N], int f) {
#pragma unroll
    for (int k = 0; k < N; k++) if (k != f) v[k] = 0.0;
}

// ------------------------------------------------------------------------------------------------
// 4 / 8 padded states, whole pruning pass in ONE launch: each thread owns PP patterns and walks the dirty internal nodes in
// post-order.  Every dependency is thread-local (a child's conditionals were written by the same thread earlier in the
// same launch, or are a valid cache from an earlier evaluation), so there is no synchronisation of any kind; P^T of a
// branch is read by all threads at the same address (L1 broadcast).  HBM traffic per evaluation is the algorithmic
// minimum: one coalesced write and (at most) one read of Dp*8+4 bytes per (node, pattern) plus 4 B per leaf state.
// The node computed by the previous job is, in post-order, very often a child of the current one (every node follows its
// last child): its vectors are handed over in registers instead of being re-read from L2 (the thread would wait a full L2
// round trip for data it wrote a moment ago).
// PP = 1 (4 and 8 states) is bound by the latency of each thread's serial node chain, and -- every CTA walking the whole
// tree -- by wave quantisation (256 x 200 k nucleotides: 1563 CTAs on 1332 resident = 1.17 waves, i.e. two passes).  With
// PP = 2 (4 states) the loads and the arithmetic of both patterns are in flight together (the pass gets 1.55x longer, not
// 2x) and half as many CTAs cover the alignment; the host picks the variant with the cheaper (passes x pass cost).
// Thread t of CTA b owns patterns (b*PP + u)*128 + t: coalesced for every u.
// grid = (ceil(Sp / (128*PP)), classes), block = 128.  jobs = dirty internal indices, ascending (= post-order).
// ------------------------------------------------------------------------------------------------
// (Forcing 16 CTAs/SM for 4 states -- 32 registers, spills -- was slower.  PP = 1 takes no minimum: a minimum of 1 CTA/SM
// lets ptxas spend up to 216 registers.)
template <int DP, int PP>
__global__ void __launch_bounds__(128, PP == 1 ? 0 : 6) prune_small_walk_kernel(PruneArgs a, const int *__restrict__ jobs, int njobs) {
    // P^T of a branch (16 / 64 doubles) is read straight through L1; 16..32 states run prune_small_dmma_kernel.
    static_assert(DP <= 8, "patterns in registers are used for 4 and 8 padded states only");
    const int tid = threadIdx.x;
    const int cat = a.cat0 + blockIdx.y;
    const size_t Sp = a.Sp;
    size_t s[PP];
    bool live[PP];
#pragma unroll
    for (int u = 0; u < PP; u++) {
        s[u] = ((size_t)blockIdx.x * PP + u) * 128 + tid;
        live[u] = PP == 1 || s[u] < Sp;       // Sp is a multiple of 128: with one pattern per thread every slot is live
        if (!live[u]) s[u] = Sp - 1;          // loads stay in range; nothing is stored for a dead slot
    }
    double pv[PP][DP];
    int prev = -1, pex[PP];
#pragma unroll
    for (int u = 0; u < PP; u++) pex[u] = 0;
    for (int jb = 0; jb < njobs; jb++) {
        const int par = __ldg(jobs + jb);
        double v[PP][DP];
        int ex[PP];
#pragma unroll
        for (int u = 0; u < PP; u++) {
            ex[u] = 0;
#pragma unroll
            for (int k = 0; k < DP; k++) v[u][k] = 1.0;
        }
        const int c_begin = __ldg(a.tree.child_start + par), c_end = __ldg(a.tree.child_start + par + 1);
        for (int ci = c_begin; ci < c_end; ci++) {
            const int child = __ldg(a.tree.child_ids + ci);
            const double *PT = a.PT + ((size_t)cat * a.B + child) * DP * DP;
            if (child < a.L) {
                int code[PP];
#pragma unroll
                for (int u = 0; u < PP; u++) code[u] = (child == a.forced_node) ? __ldg(a.forced + s[u]) : __ldg(a.leaf + (size_t)child * Sp + s[u]);
#pragma unroll
                for (int u = 0; u < PP; u++) {
                    if (code[u] >= 0) {
                        const double2 *row = reinterpret_cast<const double2 *>(PT + (size_t)code[u] * DP);
#pragma unroll
                        for (int k = 0; k < DP; k += 2) { const double2 r = __ldg(row + k / 2); v[u][k] *= r.x; v[u][k + 1] *= r.y; }
                    } else {
                        const double *amb = a.ambig + (size_t)(-code[u] - 1) * DP;
                        double acc[DP];
#pragma unroll
                        for (int k = 0; k < DP; k++) acc[k] = 0.0;
                        for (int j = 0; j < a.D; j++) {
                            const double wgt = __ldg(amb + j);
                            const double2 *row = reinterpret_cast<const double2 *>(PT + (size_t)j * DP);
#pragma unroll
                            for (int k = 0; k < DP; k += 2) { const double2 r = __ldg(row + k / 2); acc[k] = fma(wgt, r.x, acc[k]); acc[k + 1] = fma(wgt, r.y, acc[k + 1]); }
                        }
#pragma unroll
                        for (int k = 0; k < DP; k++) v[u][k] *= acc[k];
                    }
                }
            } else {
                const int cin = child - a.L;
                double x[PP][DP];
                if (cin == prev) {
#pragma unroll
                    for (int u = 0; u < PP; u++) {
#pragma unroll
                        for (int j = 0; j < DP; j++) x[u][j] = pv[u][j];
                        ex[u] += pex[u];
                    }
                } else {
#pragma unroll
                    for (int u = 0; u < PP; u++) {
                        const double2 *X = reinterpret_cast<const double2 *>(a.cond + (((size_t)cat * a.I + cin) * Sp + s[u]) * DP);
#pragma unroll
                        for (int j = 0; j < DP; j += 2) { const double2 t = X[j / 2]; x[u][j] = t.x; x[u][j + 1] = t.y; }
                    }
#pragma unroll
                    for (int u = 0; u < PP; u++) ex[u] += a.scal[((size_t)cat * a.I + cin) * Sp + s[u]];
                }
                double acc[PP][DP];
#pragma unroll
                for (int u = 0; u < PP; u++)
#pragma unroll
                    for (int k = 0; k < DP; k++) acc[u][k] = 0.0;
#pragma unroll
                for (int j = 0; j < DP; j++) {
                    const double2 *row = reinterpret_cast<const double2 *>(PT + (size_t)j * DP);
#pragma unroll
                    for (int k = 0; k < DP; k += 2) {
                        const double2 r = __ldg(row + k / 2);           // one load serves all PP patterns
#pragma unroll
                        for (int u = 0; u < PP; u++) { acc[u][k] = fma(x[u][j], r.x, acc[u][k]); acc[u][k + 1] = fma(x[u][j], r.y, acc[u][k + 1]); }
                    }
                }
#pragma unroll
                for (int u = 0; u < PP; u++)
#pragma unroll
                    for (int k = 0; k < DP; k++) v[u][k] *= acc[u][k];
            }
            if (ci - c_begin >= 1 && ci + 1 < c_end) {       // wide node: before its third and later children
#pragma unroll
                for (int u = 0; u < PP; u++) {
                    // pinned: rescale by the forced state, the only one that survives
                    if (a.L + par == a.forced_node) keep_state(v[u], __ldg(a.forced + s[u]));
                    rescale_running(v[u], ex[u]);
                }
            }
        }
        const bool pinned = a.L + par == a.forced_node;
#pragma unroll
        for (int u = 0; u < PP; u++) {
            if (pinned) keep_state(v[u], __ldg(a.forced + s[u]));
            double m = 0.0;
#pragma unroll
            for (int k = 0; k < DP; k++) m = fmax(m, v[u][k]);
            if (m > 0.0 && m < INFINITY) {
                const int e = ilogb(m) + 1;
                const double s1 = exp2i(-(e / 2)), s2 = exp2i(-(e - e / 2));
#pragma unroll
                for (int k = 0; k < DP; k++) v[u][k] = v[u][k] * s1 * s2;
                ex[u] += e;
            }
            if (live[u]) {
                double2 *outp = reinterpret_cast<double2 *>(a.cond + (((size_t)cat * a.I + par) * Sp + s[u]) * DP);
#pragma unroll
                for (int k = 0; k < DP; k += 2) outp[k / 2] = make_double2(v[u][k], v[u][k + 1]);
                a.scal[((size_t)cat * a.I + par) * Sp + s[u]] = ex[u];
                if (par == a.I - 1) {
                    double r = 0.0;
#pragma unroll
                    for (int k = 0; k < DP; k++) r = fma(v[u][k], a.pi[k], r);
                    a.rootL[(size_t)cat * Sp + s[u]] = r;
                    a.rootE[(size_t)cat * Sp + s[u]] = ex[u];
                }
            }
#pragma unroll
            for (int k = 0; k < DP; k++) pv[u][k] = v[u][k];
            pex[u] = ex[u];
        }
        prev = par;
    }
}

// ------------------------------------------------------------------------------------------------
// Root reduction: rate-class mixture + log + pattern frequency + block partial sums.
//   L_s = sum_c w_c * rootL[c][s] * 2^(rootE[c][s]);  lnL_s = log(sum_c w_c rootL 2^(e_c-emax)) + emax ln2
// Optional per-pattern outputs in the reference's convention: siteL * 2^(-64*siteScale).
// partial[block] = sum over the block's patterns of freq*lnL_s (tree reduction, deterministic);
// flag[0] |= 1 if any pattern with freq>0 has L <= 0.
// ------------------------------------------------------------------------------------------------
// x = m * 2^k with |m| in [0.5, 1) for finite x != 0, subnormals included (frexp without its out-pointer)
__device__ __forceinline__ double split_pow2(double x, int &k) {
    int adj = 0;
    if (fabs(x) < 0x1p-1022) { x *= 0x1p64; adj = 64; }
    const long long b = __double_as_longlong(x);
    k = (int)((b >> 52) & 0x7ff) - 1022 - adj;
    return __longlong_as_double((b & (long long)0x800fffffffffffffULL) | 0x3fe0000000000000LL);
}

// The rate-class merge of one pattern, shared by every site that forms such a sum (combine_kernel, the class-group partials
// and the merge of those partials, DESIGN §4.5).  term(c, w, l, e) yields weight w, value l and binary exponent e of term c;
// returns sum and sets emax with sum_c w_c l_c 2^(e_c) = sum * 2^emax.  A term of weight 0 takes no part at all (not in the
// exponent, not in the sum, not in the NaN check), as likefunc2.cpp:668 skips such a class.  A NaN value of weight != 0, or
// a NaN weight, gives NaN; no positive term gives sum 0, emax INT_MIN.
// The fast rule aligns on the largest e_c and drops terms more than 1000 bits below it.  It can lose a term that matters
// when the class holding the largest e_c has a tiny weight, so when a term is dropped or the sum falls below 2^-900 the
// pattern is redone aligned on the contributions w_c l_c 2^(e_c) themselves (w and l split into mantissa and exponent, so
// a subnormal weight does not underflow) and the sum goes out normalised to [0.5, 1) with its true exponent.  Unless a
// class of positive weight sits more than 1000 bits below the highest or the sum falls below 2^-900, that path is not
// taken and the arithmetic is the fast rule's, bit for bit.
template <class Term>
__device__ __forceinline__ double merge_classes(int n, Term term, int &emax_out) {
    double w, l;
    int e;
    int emax = INT_MIN;
    bool nan_seen = false;
    for (int c = 0; c < n; c++) {
        term(c, w, l, e);
        if (w == 0.0) continue;
        if (l != l || w != w) nan_seen = true;
        if (l > 0.0) emax = max(emax, e);
    }
    double sum = 0.0;
    bool cut = false;
    for (int c = 0; c < n; c++) {
        term(c, w, l, e);
        if (w == 0.0 || !(l > 0.0)) continue;
        const int de = e - emax;                                   // <= 0
        if (de < -1000) cut = true;
        else sum += w * l * exp2i(de);
    }
    if (nan_seen) {
        sum = __longlong_as_double(0x7ff8000000000000LL);
    } else if (emax != INT_MIN && (cut || sum < 0x1p-900)) {
        int ebest = INT_MIN;
        for (int c = 0; c < n; c++) {
            term(c, w, l, e);
            if (w == 0.0 || !(l > 0.0)) continue;
            int kw, kl;
            split_pow2(w, kw); split_pow2(l, kl);
            ebest = max(ebest, e + kw + kl);
        }
        sum = 0.0;
        for (int c = 0; c < n; c++) {
            term(c, w, l, e);
            if (w == 0.0 || !(l > 0.0)) continue;
            int kw, kl;
            const double m = split_pow2(w, kw) * split_pow2(l, kl);  // |m| in [0.25, 1)
            const int de = e + kw + kl - ebest;
            if (de >= -1000) sum += m * exp2i(de);
        }
        if (sum > 0.0) {
            int k;
            sum = split_pow2(sum, k);                                // [0.5, 1)
            emax = ebest + k;
        }
    }
    emax_out = emax;
    return sum;
}

// log L of a pattern with L = sum * 2^emax: NaN stays NaN, and a sum that is neither positive nor NaN gives -inf after
// impossible() has run (the caller's flag).
template <class Impossible>
__device__ __forceinline__ double pattern_lnl(double sum, int emax, Impossible impossible) {
    if (sum > 0.0) return log(sum) + (double)emax * 0.693147180559945309417232121458;
    if (sum != sum) return sum;
    impossible();
    return -INFINITY;
}

// The reference's per-pattern output convention for L = sum * 2^emax: L = siteL * 2^(-64*siteScale) with siteL = sum * 2^r,
// r in (-64, 0] (DESIGN §4.5).  A sum that is 0 or NaN goes out as it is, with siteScale 0.
struct SiteOut {
    double L;
    long long scale;
};
__device__ __forceinline__ SiteOut site_output(double sum, int emax) {
    long long cnt = 0; double outL = sum;
    if (sum > 0.0) {
        cnt = (emax < 0) ? (long long)((-emax) / 64) : -(long long)((emax + 63) / 64);
        const int rem = emax + (int)(64 * cnt);    // in (-64, 0]
        outL = sum * exp2i(rem);
    }
    return {outL, cnt};
}

// red[0] = the sum of v over the 256 threads of the block, added in a fixed order: the same bits on every run.  Called by
// every thread; ends with a barrier.
__device__ __forceinline__ void block_sum256(double *red, double v) {
    red[threadIdx.x] = v;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
}

struct CombineArgs {
    const double *rootL; const int *rootE; const double *weights; const double *freq;
    double *partial; int *flag; double *siteL; long long *siteScale;
    int Sp, S, c0, nc;
    unsigned *counter;      // nullable: with `out`, the LAST block to finish adds up the partials (final_sum_kernel's arithmetic,
    double *out;            // same order) and re-arms counter and flag -- one launch and one memset less per evaluation
};

__global__ void __launch_bounds__(256) combine_kernel(CombineArgs a) {
    __shared__ double red[256];
    const int s = blockIdx.x * 256 + threadIdx.x;
    double term = 0.0;
    if (s < a.S) {
        int emax;
        double sum = merge_classes(a.nc, [&](int c, double &w, double &l, int &e) {
            w = a.weights ? a.weights[c] : 1.0;
            l = a.rootL[(size_t)(a.c0 + c) * a.Sp + s];
            e = a.rootE[(size_t)(a.c0 + c) * a.Sp + s];
        }, emax);
        if (emax == INT_MIN) emax = 0;
        const double f = a.freq[s];
        const double lnl = pattern_lnl(sum, emax, [&] { if (f > 0.0) atomicOr(a.flag, 1); });
        term = (f > 0.0) ? f * lnl : 0.0;
        if (a.siteL) {
            const SiteOut o = site_output(sum, emax);
            a.siteL[s] = o.L; a.siteScale[s] = o.scale;
        }
    }
    block_sum256(red, term);
    if (threadIdx.x == 0) a.partial[blockIdx.x] = red[0];
    if (a.counter) {
        __shared__ int s_last;
        if (threadIdx.x == 0) {
            __threadfence();                                   // partial[] (and flag) before the ticket
            s_last = atomicAdd(a.counter, 1u) == gridDim.x - 1;
        }
        __syncthreads();
        if (!s_last) return;
        __threadfence();
        double s = 0.0;
        for (int i = threadIdx.x; i < (int)gridDim.x; i += 256) s += __ldcg(a.partial + i);
        block_sum256(red, s);
        if (threadIdx.x == 0) {
            a.out[0] = __ldcg(a.flag) ? -INFINITY : red[0];
            *a.flag = 0;
            *a.counter = 0u;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Group toolkit of the state-per-thread fp64 kernels (bc_path_kernel, prune_batch_kernel, outside_pass, prune_rates_kernel):
// a group of G = 4, 8, 16, 32 or 64 threads owns one pattern and thread k owns state k.  G = 64 is a CTA of two warps and
// exchanges through the kernel's shared scratch xs[64] and red[2]; G <= 32 is the lanes `mask` of one warp and exchanges
// with width-G shuffles.  Every member is called by the whole group.
// Numerical rules of these kernels:
//   - Renormalisation: a vector whose group maximum m is positive and below `below` is multiplied by 2^-e, e = ilogb(m) + 1,
//     which brings m to [0.5, 1), and e is added to its binary exponent.  The multiply is split in two exact halves so that
//     neither factor overflows when m is subnormal.  A pruned node renormalises at its end (below = INFINITY) and, from its
//     third child on, before each child with below = RESCALE_BELOW (the wide-node rescale); the outside passes renormalise
//     after every factor.
//   - Child message m[k] = sum_j P[k][j] x_j = sum_j x_j PT[j][k] over the states j < D in order, one fma per state (dot):
//     x is an internal child's vector staged to the group.  A leaf gives m = PT[code][k] for a state, or for a 0/1
//     ambiguity row the fma of the row's weight over its nonzero states in order (leaf_message; hb2_create refuses any
//     other weight, so this equals the sum of those entries).  The outside product o[k] = sum_p A_p P[p][k] is the same
//     dot over a row of the transposed table, PT[k][p].  Entries are read through the caller's entry(j): plain, mixed by
//     mix_entry (BranchP), or a Dp-strided table.
//   - Padded states (k >= D) stay 0: their table entries are 0, or the kernel masks them (dot's `live`).
//   - The group sum is one fixed-order xor tree of width G; G = 64 adds the totals of its two warps, red[0] + red[1].  A
//     pattern's sum * 2^ex goes out through pattern_lnl: a likelihood of 0 gives -inf and NaN stays NaN.
//   - Joint reconstruction (joint_ancestors_kernel; the reference's RecoverAncestralSequences, tree.cpp:4209-4510):
//     a max-product replaces each sum.  A child's factor at parent state p is max_c P[p][c] x_c over c ascending, by
//     strict > against a running maximum that starts at 0 with argument 0 (max_product; tree.cpp:4357-4377): ties go to
//     the lowest c, a product that is 0 or NaN never wins, and a row with no positive product gives 0 with argument 0.
//     x is an internal child's vector, or a leaf's 0/1 ambiguity row, which gives the max of P[p][c] over its nonzero
//     states (ambig_max); a resolved leaf multiplies by P[p][code] with no max (tree.cpp:4315-4327).  A child is
//     unresolved when it is a leaf whose row is 1 in all D states or an internal node all of whose children are
//     unresolved: it takes no state and does not multiply its parent (tree.cpp:4350-4356, :4390-4394).  The root state
//     is the lowest k of the largest positive pi_k J_root[k], 0 when none is positive (argmax; tree.cpp:4448-4457).
//     Renormalisation by powers of two changes no comparison, so the reference's own rescaling (:4379-4383) is free to
//     differ.
// ------------------------------------------------------------------------------------------------
template <int G>
struct Group {
    static_assert(G == 4 || G == 8 || G == 16 || G == 32 || G == 64, "a group is 4, 8, 16, 32 or 64 threads");
    static constexpr int W = G < 32 ? G : 32;    // shuffle width
    double *xs, *red;                            // G = 64: the kernel's shared xs[64] and red[2]
    unsigned mask;                               // the group's lanes (G >= 32: every lane)
    int k;                                       // this thread's state

    __device__ __forceinline__ double max(double v) const {
#pragma unroll
        for (int o = W / 2; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(mask, v, o, W));
        if constexpr (G == 64) {
            __syncthreads();
            if ((k & 31) == 0) red[k >> 5] = v;
            __syncthreads();
            v = fmax(red[0], red[1]);
        }
        return v;
    }
    __device__ __forceinline__ double sum(double v) const {
#pragma unroll
        for (int o = W / 2; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o, W);
        if constexpr (G == 64) {
            __syncthreads();
            if ((k & 31) == 0) red[k >> 5] = v;
            __syncthreads();
            v = red[0] + red[1];
        }
        return v;
    }
    __device__ __forceinline__ void renorm(double &v, int &ex, double below = INFINITY) const {
        const double m = max(v);
        if (m > 0.0 && m < below) {
            const int e = ilogb(m) + 1;
            v = v * exp2i(-(e / 2)) * exp2i(-(e - e / 2));
            ex += e;
        }
    }
    // Makes this thread's x readable by the group as x_j = at(staged, j).
    __device__ __forceinline__ double stage(double x) const {
        if constexpr (G == 64) {
            __syncthreads();                     // xs free
            xs[k] = x;
            __syncthreads();
        }
        return x;
    }
    __device__ __forceinline__ double at(double staged, int j) const {
        if constexpr (G == 64) return xs[j];
        else return __shfl_sync(mask, staged, j, G);
    }
    // sum_j x_j entry(j) over j < D for a staged x: an internal child's message, or the outside product.  A thread that is
    // not `live` reads no entry and returns 0 (or NaN for a non-finite x when G <= 32: its lanes take part in the shuffles).
    template <typename Entry>
    __device__ __forceinline__ double dot(double staged, int D, bool live, Entry entry) const {
        double m = 0.0;
        if constexpr (G == 64) {
            if (live)
                for (int j = 0; j < D; j++) m = fma(at(staged, j), entry(j), m);
        } else {
            for (int j = 0; j < D; j++) m = fma(at(staged, j), live ? entry(j) : 0.0, m);
        }
        return m;
    }
    // the message of a leaf child with state code `code`: a state (>= 0) or row -code - 1 of ambig[][stride]
    template <typename Entry>
    __device__ __forceinline__ double leaf_message(int code, const double *ambig, int stride, int D, Entry entry) const {
        double m = 0.0;
        if (code >= 0) m = entry(code);
        else {
            const double *amb = ambig + (size_t)(-code - 1) * stride;
            for (int j = 0; j < D; j++) { const double w = amb[j]; if (w != 0.0) m = fma(w, entry(j), m); }
        }
        return m;
    }
    // max_j x_j entry(j) over j < D for a staged x, and its argument, by the joint reconstruction's strict-> scan; `bad` is
    // set by a NaN product.  A thread that is not `live` reads no entry and returns 0 with argument 0.
    template <typename Entry>
    __device__ __forceinline__ double max_product(double staged, int D, bool live, Entry entry, int &arg, bool &bad) const {
        double best = 0.0;
        int c = 0;
        bool nan = false;
        if (G == 64 && !live) { arg = 0; return 0.0; }
        for (int j = 0; j < D; j++) {
            const double t = at(staged, j) * (live ? entry(j) : 0.0);
            if (t > best) { best = t; c = j; }
            nan |= t != t;
        }
        arg = c;
        bad |= live && nan;
        return best;
    }
    // max_j entry(j) over the nonzero states j < D of a 0/1 ambiguity row (0 when none is positive); `all` tells whether
    // every state is nonzero (an unresolved leaf); `bad` is set by a NaN entry read.
    template <typename Entry>
    __device__ __forceinline__ double ambig_max(const double *row, int D, bool live, Entry entry, bool &all, bool &bad) const {
        double best = 0.0;
        bool full = true, nan = false;
        for (int j = 0; j < D; j++) {
            if (row[j] == 0.0) { full = false; continue; }
            if (!live) continue;
            const double t = entry(j);
            if (t > best) best = t;
            nan |= t != t;
        }
        all = full;
        bad |= nan;
        return best;
    }
    // The lowest k whose x_k is the group's largest positive value, and that value in `best`; 0 and 0.0 when no x_k is
    // positive (a NaN never wins).
    __device__ __forceinline__ int argmax(double x, double &best) const {
        const double v = x > 0.0 ? x : 0.0;
        best = max(v);
        return G - (int)max(v == best ? (double)(G - k) : 0.0);
    }
};

// ------------------------------------------------------------------------------------------------
// Single-branch shortcut (reference: ComputeBranchCache tree_evaluator.cpp:4286, ComputeLLWithBranchCache tree.cpp:3383).
// For a branch b with parent u the likelihood factorises as  L_s = sum_a rest_b[s][a] * (P_b * below_b[s])[a]  where
// below_b = conditionals of b's subtree (already resident) and rest_b[s][a] = everything else, seen from state a at u:
//   out_root[a] = pi_a ;  rest_v[a] = out_u[a] * prod_{siblings c of v at u} (P_c L_c)[a] ;  out_v[a'] = sum_a rest_v[a] P_v[a][a'].
// (No reversibility is needed: the outside vectors are propagated with the transposed matrices instead of re-rooting.)
// bc_path_kernel walks the root->u path once; bc_eval_kernel then costs O(S*D^2) per probe of P_b.
// fp64 throughout; the build runs one CTA per (class, pattern), the probe one thread per (class, pattern).  CondView abstracts the two conditional layouts (fp64 [I][Sp][Dp]; the walk kernel's
// tile-wise fp32 with generation tags).
// ------------------------------------------------------------------------------------------------
struct CondView {
    const double *c64;      // fp64 layout or null
    const float *c32;       // tile-wise fp32 layout ([I][Sp/128][16][128][4], sign bit = tag) or null
    const int *scal;        // exponents; tagged = 1 -> (value << 1) | tag
    int I, Sp, Dp, tagged;
};

__device__ __forceinline__ double cond_at(const CondView &v, int cat, int node, int s, int k) {
    if (v.c64) return v.c64[(((size_t)cat * v.I + node) * v.Sp + s) * v.Dp + k];
    const size_t tile = s >> 7, t = s & 127;
    return (double)fabsf(v.c32[(((((size_t)cat * v.I + node) * (v.Sp >> 7) + tile) * 16 + (k >> 2)) * 128 + t) * 4 + (k & 3)]);
}
__device__ __forceinline__ int exp_at(const CondView &v, int cat, int node, int s) {
    const int e = v.scal[((size_t)cat * v.I + node) * v.Sp + s];
    return v.tagged ? (e >> 1) : e;
}

struct BranchCacheArgs {
    CondView cv;
    const double *PT;       // [C][B][Dp*Dp] transposed transition matrices
    const int *leaf;        // [L][Sp]
    const double *ambig;    // [nAmb][Dp]
    const double *pi;       // [Dp]
    double *out;            // [C][Sp][Dp] outside vector of the current path node (in/out)
    int *outE;              // [C][Sp]
    int L, B, D, Dp, Sp, S, cat0, ncls;
};

// message of child `ch` (flat id) towards its parent for one pattern: m[a] = sum_k P_ch[a][k] x[k]  (PT[k][a] = P[a][k])
__device__ __forceinline__ void bc_message(const BranchCacheArgs &a, int cat, int ch, int s, double *m, int &e) {
    const double *PTc = a.PT + ((size_t)cat * a.B + ch) * a.Dp * a.Dp;
    if (ch < a.L) {
        const int code = a.leaf[(size_t)ch * a.Sp + s];
        if (code >= 0) {
            for (int q = 0; q < a.D; q++) m[q] = __ldg(PTc + (size_t)code * a.Dp + q);
        } else {
            const double *amb = a.ambig + (size_t)(-code - 1) * a.Dp;
            for (int q = 0; q < a.D; q++) m[q] = 0.0;
            for (int k = 0; k < a.D; k++)
                if (__ldg(amb + k) != 0.0)
                    for (int q = 0; q < a.D; q++) m[q] += __ldg(PTc + (size_t)k * a.Dp + q);
        }
    } else {
        const int ci = ch - a.L;
        for (int q = 0; q < a.D; q++) m[q] = 0.0;
        for (int k = 0; k < a.D; k++) {
            const double x = cond_at(a.cv, cat, ci, s, k);
            if (x != 0.0)
                for (int q = 0; q < a.D; q++) m[q] = fma(x, __ldg(PTc + (size_t)k * a.Dp + q), m[q]);
        }
        e += exp_at(a.cv, cat, ci, s);
    }
}

// The whole root -> parent(b) path in ONE launch: one CTA of Dp' = 64 (or 32) threads per (class, pattern), a Group of
// thread q = state q; a matrix column / row is read with consecutive threads on consecutive addresses (the transposed table
// serves messages, its rows serve the outside propagation).  The rules are the group toolkit's, every factor
// renormalised.  Replaces one launch of bc_step_kernel per path node with a serial thread per pattern.
//   path[i]      internal index of the i-th path node (root first), npath nodes
//   sib_off[i]   range of its non-path children in sib[]
//   down[i]      flat id of the path child below path[i] (the next path node), -1 for the last (whose child is the branch b)
struct BranchPathArgs {
    const int *sib, *sib_off, *down;
    int npath;
};

template <int NT>
__global__ void __launch_bounds__(NT) bc_path_kernel(BranchCacheArgs a, BranchPathArgs bp) {
    __shared__ double xs[64];
    __shared__ double red[2];
    const int s = blockIdx.x, cat = a.cat0 + blockIdx.y, q = threadIdx.x;
    const Group<NT> grp{xs, red, 0xffffffffu, q};
    const bool live = q < a.D;
    double r = live ? a.pi[q] : 0.0;             // out_root = pi
    int e = 0;
    for (int i = 0; i < bp.npath; i++) {
        for (int ci = bp.sib_off[i]; ci < bp.sib_off[i + 1]; ci++) {          // rest = out_u * prod over siblings (P_c L_c)
            const int ch = bp.sib[ci];
            const double *PTc = a.PT + ((size_t)cat * a.B + ch) * a.Dp * a.Dp;
            auto entry = [&](int k) { return PTc[(size_t)k * a.Dp + q]; };
            double m = 0.0;
            if (ch < a.L) {
                if (live) m = grp.leaf_message(a.leaf[(size_t)ch * a.Sp + s], a.ambig, a.Dp, a.D, entry);
            } else {
                const int cin = ch - a.L;
                m = grp.dot(grp.stage(live ? cond_at(a.cv, cat, cin, s, q) : 0.0), a.D, live, entry);
                e += exp_at(a.cv, cat, cin, s);
            }
            r *= m;
            grp.renorm(r, e);
        }
        if (bp.down[i] >= 0) {                                                  // out'[q] = sum_k rest[k] * P_down[k][q] = sum_k r[k] PT[q][k]
            const double *PTd = a.PT + ((size_t)cat * a.B + bp.down[i]) * a.Dp * a.Dp;
            r = grp.dot(grp.stage(r), a.D, live, [&](int k) { return PTd[(size_t)q * a.Dp + k]; });
            grp.renorm(r, e);
        }
    }
    if (q < a.Dp) a.out[((size_t)cat * a.Sp + s) * a.Dp + q] = r;
    if (q == 0) a.outE[(size_t)cat * a.Sp + s] = e;
}

// Probe: rootL/rootE <- sum_a rest[a] * (P_b * below)[a] with the CURRENT matrix of branch b.
__global__ void __launch_bounds__(128) bc_eval_kernel(BranchCacheArgs a, int b, double *rootL, int *rootE) {
    const int s = blockIdx.x * 128 + threadIdx.x;
    const int cat = a.cat0 + blockIdx.y;
    if (s >= a.S) return;
    double m[64];
    int e = a.outE[(size_t)cat * a.Sp + s];
    bc_message(a, cat, b, s, m, e);
    const double *o = a.out + ((size_t)cat * a.Sp + s) * a.Dp;
    double acc = 0.0;
    for (int q = 0; q < a.D; q++) acc = fma(o[q], m[q], acc);
    rootL[(size_t)cat * a.Sp + s] = acc;
    rootE[(size_t)cat * a.Sp + s] = e;
}

// Class-group sharding (hb2_comm_class_groups): this rank's share of sum_c w_c L_{c,s}, as (value, binary exponent) per
// pattern, written to send[0..xs) | send[xs..2xs) (exponent as a double; NaN value = numerical failure, value 0 = no
// positive class likelihood).
__global__ void __launch_bounds__(256) class_partial_kernel(const double *rootL, const int *rootE, const double *weights,
                                                            int Sp, int S, int c0, int nc, double *send, int xs) {
    const int s = blockIdx.x * 256 + threadIdx.x;
    if (s >= xs) return;
    double sum = 0.0;
    int emax = 0;
    if (s < S) {
        sum = merge_classes(nc, [&](int c, double &w, double &l, int &e) {
            w = weights[c0 + c];
            l = rootL[(size_t)(c0 + c) * Sp + s];
            e = rootE[(size_t)(c0 + c) * Sp + s];
        }, emax);
        if (emax == INT_MIN) emax = 0;
    }
    send[s] = sum;
    send[xs + s] = (double)emax;
}

// Merges the class-group partials of EVERY pattern shard (gath = gathered buffer, rank-major, 2*xs doubles per rank;
// the G ranks [j*G, j*G+G) hold the class groups of shard j; xfreq = pattern frequencies of every rank, gathered once)
// and finishes like combine_kernel.  Every rank therefore ends up with the complete lnL -- bit-identical on all ranks --
// and no second collective is needed; per-pattern outputs are written for the rank's own shard only.
__global__ void __launch_bounds__(256) class_merge_kernel(const double *gath, const double *xfreq, int xs, int nShards, int G,
                                                          int myShard, double *partial, int *flag, double *siteL,
                                                          long long *siteScale, int S) {
    __shared__ double red[256];
    const int idx = blockIdx.x * 256 + threadIdx.x;
    double term = 0.0;
    if (idx < nShards * xs) {
        const int j = idx / xs, s = idx % xs;
        const double f = xfreq[(size_t)j * G * xs + s];
        int emax;
        double sum = merge_classes(G, [&](int r, double &w, double &m, int &e) {
            const double *q = gath + (size_t)(j * G + r) * 2 * xs;
            w = 1.0; m = q[s]; e = (int)q[xs + s];
        }, emax);
        if (emax == INT_MIN) emax = 0;
        const double lnl = pattern_lnl(sum, emax, [&] { if (f > 0.0) atomicOr(flag, 1); });
        term = (f > 0.0) ? f * lnl : 0.0;
        if (siteL && j == myShard && s < S) {
            const SiteOut o = site_output(sum, emax);
            siteL[s] = o.L; siteScale[s] = o.scale;
        }
    }
    block_sum256(red, term);
    if (threadIdx.x == 0) partial[blockIdx.x] = red[0];
}

// ------------------------------------------------------------------------------------------------
// Batched one-pattern likelihoods (SURVEY §8f row 3: the site phases of FEL / MEME fit thousands of one-pattern likelihood
// functions on the same tree, FEL.bf:1180-1233, MEME.bf:699-746).  Set s prunes pattern pat[s] with ITS OWN transition
// matrices PT[s][b] (64-padded, transposed, as the expm kernels write them).  One CTA of 64 threads per set: thread k owns
// parent state k; a child's vector is broadcast from shared memory and column k of P is read from PT[.][j][k] -- 64
// consecutive doubles per j, coalesced.  fp64 throughout, a Group<64> under the group toolkit's rules.
// Internal-node vectors live in global scratch cond[s][I][64] (L1/L2 resident: 512 bytes per node).
// MIX (explicit-form mixtures, MEME's tested branches, MEME.bf:381-386): set s holds R component matrices PT[s][row];
// branch b mixes rows row_off[b] .. row_off[b+1]-1 (at most 4).  The thread of parent state k forms each entry as
// sum_c w_c PT_c[j][k], components in order as mix_reduce_kernel (tree.cpp:3047-3089), before it enters the contraction:
// the mixed matrix never goes to memory.
// ------------------------------------------------------------------------------------------------
// A branch's mixture as a thread forms it (prune_batch_kernel<true>, sim_cdf_kernel<true>): mix_weights loads the weights
// of its nc <= 4 component rows; mix_entry forms an entry of the mixed matrix as w_0 P_0, then fma(w_c, P_c, .) in
// component order -- the order of mix_reduce_kernel -- from P(c), component c's entry.
__device__ __forceinline__ void mix_weights(double (&w)[4], const double *ws, int nc) {
#pragma unroll
    for (int c = 0; c < 4; c++) w[c] = c < nc ? ws[c] : 0.0;
}

template <typename Component>
__device__ __forceinline__ double mix_entry(const double (&w)[4], int nc, Component P) {
    double v = w[0] * P(0);
#pragma unroll
    for (int c = 1; c < 4; c++)
        if (c < nc) v = fma(w[c], P(c), v);
    return v;
}

struct BatchPruneArgs {
    const double *PT;         // [nSets][B][4096]; MIX: [nSets][R][4096]
    double *cond;             // [nSets][I][64]
    int *node_ex;             // [nSets][I] binary exponents of the node vectors
    const int *pat;           // [nSets] pattern of the partition evaluated by each set
    const int *leaf;          // [L][Sp]
    const double *ambig;      // [nAmb][64]
    const double *pi;         // [64]
    TreeDev tree;
    double *out;              // [nSets] log-likelihood of the pattern
    int L, I, B, D, Sp;
    const double *mix_w;      // MIX: [nSets][R] component weights
    const int *row_off;       // MIX: [B+1] first component row of each branch
    int R;                    // MIX: component rows per set
};

// The transition matrix of a child's branch in a set's P area PTs, as prune_batch_kernel and outside_pass read it: P is
// the branch's first row, nc its component rows from row r0 (one without MIX), w their weights once load_weights() ran.
// Entry (j, k), at offset j * 64 + k of the table, is the row's entry, or with MIX the rows' mix_entry.
template <bool MIX>
struct BranchP {
    const double *P;
    int r0, nc;
    double w[4];
    __device__ __forceinline__ BranchP(const BatchPruneArgs &a, const double *PTs, int child) {
        if constexpr (MIX) { r0 = a.row_off[child]; nc = a.row_off[child + 1] - r0; }
        else { r0 = child; nc = 1; }
        P = PTs + (size_t)r0 * 4096;
    }
    // mw: the set's weights; the same address in every thread, a broadcast
    __device__ __forceinline__ void load_weights(const double *mw) {
        if constexpr (MIX) mix_weights(w, mw + r0, nc);
    }
    __device__ __forceinline__ double operator()(int off) const {
        if constexpr (!MIX) return P[off];
        else return mix_entry(w, nc, [&](int c) { return P[off + (size_t)c * 4096]; });
    }
};

// Each node follows the group toolkit's rules; the root sum is Group<64>::sum.
template <bool MIX>
__global__ void __launch_bounds__(64) prune_batch_kernel(BatchPruneArgs a) {
    __shared__ double xs[64];
    __shared__ double red[2];
    const int s = blockIdx.x, k = threadIdx.x;
    const Group<64> grp{xs, red, 0xffffffffu, k};
    const int pattern = a.pat[s];
    const double *PTs = a.PT + (size_t)s * (MIX ? a.R : a.B) * 4096;
    const double *mw = MIX ? a.mix_w + (size_t)s * a.R : nullptr;
    double *cs = a.cond + (size_t)s * a.I * 64;
    int *node_ex = a.node_ex + (size_t)s * a.I;
    for (int par = 0; par < a.I; par++) {
        double v = k < a.D ? 1.0 : 0.0;
        int ex = 0;
        const int c_begin = a.tree.child_start[par], c_end = a.tree.child_start[par + 1];
        for (int ci = c_begin; ci < c_end; ci++) {
            if (ci - c_begin >= 2) grp.renorm(v, ex, RESCALE_BELOW);
            const int child = a.tree.child_ids[ci];
            BranchP<MIX> P(a, PTs, child);
            P.load_weights(mw);
            auto entry = [&](int j) { return P(j * 64 + k); };
            double m;
            if (child < a.L) m = grp.leaf_message(a.leaf[(size_t)child * a.Sp + pattern], a.ambig, 64, a.D, entry);
            else {
                const int cin = child - a.L;
                m = grp.dot(grp.stage(cs[(size_t)cin * 64 + k]), a.D, true, entry);
                ex += node_ex[cin];
            }
            v *= m;
        }
        grp.renorm(v, ex);
        cs[(size_t)par * 64 + k] = v;
        if (k == 0) node_ex[par] = ex;
        if (par == a.I - 1) {
            const double r = grp.sum(v * a.pi[k]);
            if (k == 0) a.out[s] = pattern_lnl(r, ex, [] {});
        } else {
            __syncthreads();                     // node_ex of this node visible to the block before a parent reads it
        }
    }
}

// ------------------------------------------------------------------------------------------------
// The batch outside pass (outside_pass), behind two kernels that run after prune_batch_kernel on the same chunk, one CTA
// of 64 threads per set, thread = state.  For branch b with child node c, in_c is c's subtree vector (the inside pass's
// cond / node_ex) and A_b the vector at the parent end of b of everything outside c's subtree.
//   branch_rows_kernel (hb2_batch_branch_component_likelihoods, MIX layout only): the likelihood of every set with one
//     branch pinned to one of its mixture components, for MEME's branch-level empirical Bayes factors (MEME.bf:886-944):
//     row r of b has L_{b,r} = sum_p A_b[p] (P_r in_c)[p] with P_r the row's own exponential, whatever the branch's weights.
//   leaf_support_kernel<MIX> (hb2_batch_leaf_support, both layouts): for every leaf l, the predictive distribution of its
//     state given every other leaf (ReconstructAncestors(MARGINAL, DOLEAVES), likefunc2.cpp:974-1006 and :1083-1093):
//     u[k] = sum_p A_l[p] P_l[p][k], written as u[k] / sum_j u[j], or NaN in every entry when that total is 0 or not
//     finite.  A_l leaves out l's own message, so the row does not read l's code.
// Internal nodes are visited in reverse flat order (a pre-order); node n with outside vector O_n (the root: pi, exponent 0)
// and children c_1..c_m:
//   1. m_c = P_c in_c for each child, P_c the branch's matrix (MIX: mixed entry by entry as the inside pass mixes it,
//      mix_entry), leaves by their state or ambiguity row as there; stored in msg[c];
//   2. the suffix products m_{c_{i+1}} ... m_{c_m}, stored in side[c_i];
//   3. forward, with the running prefix O_n m_{c_1} ... m_{c_{i-1}}: A_{c_i} = prefix * suffix (no division, so a zero
//      message does not poison its siblings), then what the kernel emits at c_i (every row of c_i, or for a leaf c_i its
//      support row), then for an internal c_i its outside vector O_{c_i}[j] = sum_p A_{c_i}[p] P_{c_i}[p][j], kept in
//      side[c_i] until c_i is visited.  A leaf's u is the same product.
// The transposed table serves the messages and rows with coalesced reads, as in the inside pass; the outside product reads
// its rows, as bc_path_kernel does.
// Numerical rules: the group toolkit's, with every message, suffix, prefix, A and outside vector renormalised after each
// factor (more often than RESCALE_BELOW requires) and each row's sum encoded by pattern_lnl.
// ------------------------------------------------------------------------------------------------
struct OutsideArgs {
    BatchPruneArgs in;        // the chunk's inside pass: PT, cond, node_ex, pat, leaf, ambig, pi, tree (MIX: mix_w, row_off)
    double *msg, *side;       // [nSets][B][64] messages; suffix products, then A, then outside vectors
    int *msg_ex, *side_ex;    // [nSets][B] their binary exponents
    double *rows;             // branch_rows_kernel: [nSets][R] log-likelihood of each row
    double *support;          // leaf_support_kernel: [nSets][L][D] support of each leaf's states
};

enum class OutsideEmit { BranchRows, LeafSupport };

template <OutsideEmit EMIT, bool MIX>
__device__ __forceinline__ void outside_pass(const OutsideArgs &g) {
    __shared__ double xs[64];
    __shared__ double red[2];
    const BatchPruneArgs &a = g.in;
    const int s = blockIdx.x, k = threadIdx.x;
    const Group<64> grp{xs, red, 0xffffffffu, k};
    const bool live = k < a.D;
    const int pattern = a.pat[s];
    const double *PTs = a.PT + (size_t)s * (MIX ? a.R : a.B) * 4096;
    const double *cs = a.cond + (size_t)s * a.I * 64;
    const int *node_ex = a.node_ex + (size_t)s * a.I;
    const double *mw = MIX ? a.mix_w + (size_t)s * a.R : nullptr;
    double *msg = g.msg + (size_t)s * a.B * 64, *side = g.side + (size_t)s * a.B * 64;
    int *msg_ex = g.msg_ex + (size_t)s * a.B, *side_ex = g.side_ex + (size_t)s * a.B;
    double *rows = EMIT == OutsideEmit::BranchRows ? g.rows + (size_t)s * a.R : nullptr;
    for (int n = a.I - 1; n >= 0; n--) {
        const int c_begin = a.tree.child_start[n], c_end = a.tree.child_start[n + 1];
        // 1. messages
        for (int ci = c_begin; ci < c_end; ci++) {
            const int child = a.tree.child_ids[ci];
            BranchP<MIX> P(a, PTs, child);
            P.load_weights(mw);
            const bool leaf = child < a.L;
            int ex = 0;
            double x = 0.0;
            if (!leaf) { x = grp.stage(cs[(size_t)(child - a.L) * 64 + k]); ex = node_ex[child - a.L]; }
            auto entry = [&](int j) { return P(j * 64 + k); };
            double m = 0.0;
            if (!leaf) m = grp.dot(x, a.D, live, entry);
            else if (live) m = grp.leaf_message(a.leaf[(size_t)child * a.Sp + pattern], a.ambig, 64, a.D, entry);
            grp.renorm(m, ex);
            msg[(size_t)child * 64 + k] = m;
            if (k == 0) msg_ex[child] = ex;
        }
        __syncthreads();                         // msg_ex visible to the block
        // 2. suffix products
        double v = live ? 1.0 : 0.0;
        int ve = 0;
        for (int ci = c_end - 1; ci >= c_begin; ci--) {
            const int child = a.tree.child_ids[ci];
            side[(size_t)child * 64 + k] = v;
            if (k == 0) side_ex[child] = ve;
            v *= msg[(size_t)child * 64 + k];
            ve += msg_ex[child];
            grp.renorm(v, ve);
        }
        // 3. prefix, A, what is emitted and outside vectors; O_n is the root vector or what the parent's visit left in side[L+n]
        __syncthreads();                         // side_ex visible to the block
        if (n == a.I - 1) { v = live ? a.pi[k] : 0.0; ve = 0; }
        else { v = side[(size_t)(a.L + n) * 64 + k]; ve = side_ex[a.L + n]; }
        for (int ci = c_begin; ci < c_end; ci++) {
            const int child = a.tree.child_ids[ci];
            BranchP<MIX> P(a, PTs, child);
            const bool leaf = child < a.L;
            double A = v * side[(size_t)child * 64 + k];
            int ae = ve + side_ex[child];
            grp.renorm(A, ae);
            if constexpr (EMIT == OutsideEmit::BranchRows) {
                int ie = 0;
                double x = 0.0;
                if (!leaf) { x = grp.stage(cs[(size_t)(child - a.L) * 64 + k]); ie = node_ex[child - a.L]; }
                for (int c = 0; c < P.nc; c++) {
                    const double *Pr = P.P + (size_t)c * 4096;
                    auto entry = [&](int j) { return Pr[j * 64 + k]; };
                    double m = 0.0;
                    if (!leaf) m = grp.dot(x, a.D, live, entry);
                    else if (live) m = grp.leaf_message(a.leaf[(size_t)child * a.Sp + pattern], a.ambig, 64, a.D, entry);
                    const double sum = grp.sum(A * m);
                    if (k == 0) rows[P.r0 + c] = pattern_lnl(sum, ae + ie, [] {});
                }
            }
            if (!leaf || EMIT == OutsideEmit::LeafSupport) {   // the outside product: O_child, or a leaf child's u
                P.load_weights(mw);
                const double x = grp.stage(A);
                double o = grp.dot(x, a.D, live, [&](int p) { return P(k * 64 + p); });
                if (!leaf) {
                    grp.renorm(o, ae);
                    side[(size_t)child * 64 + k] = o;
                    if (k == 0) side_ex[child] = ae;
                } else {
                    const double total = grp.sum(o);
                    if (live) g.support[((size_t)s * a.L + child) * a.D + k] = total != 0.0 && isfinite(total) ? o / total : nan("");
                }
            }
            v *= msg[(size_t)child * 64 + k];
            ve += msg_ex[child];
            grp.renorm(v, ve);
        }
    }
}

__global__ void __launch_bounds__(64) branch_rows_kernel(OutsideArgs g) { outside_pass<OutsideEmit::BranchRows, true>(g); }

// A minimum of 8 CTAs per SM (a chunk of at most 1024 sets puts no more on any of the 132 SMs) lets ptxas use 78-80
// registers instead of 44-46; on one H100 at 700 W the kernel then took 22 / 60 / 38 ms instead of 29 / 79 / 52 ms on the
// north-star FEL / MEME-all / MEME-third shapes (tools/bench_leaf_support.py, alternating runs, identical output).
template <bool MIX>
__global__ void __launch_bounds__(64, 8) leaf_support_kernel(OutsideArgs g) { outside_pass<OutsideEmit::LeafSupport, MIX>(g); }

// ------------------------------------------------------------------------------------------------
// joint_ancestors_kernel<MIX> (hb2_batch_joint_ancestors, both layouts): the joint maximum-likelihood states of every
// internal node of a set (Pupko's max-product recursion, the reference's RecoverAncestralSequences).  One CTA of 64
// threads per set, thread p = parent state p, under the group toolkit's rules for joint reconstruction.
//   1. Internal nodes in flat (post-) order, exactly as prune_batch_kernel walks them, with the same BranchP reads of the
//      transposed table, the same wide-node rescale and the same renormalisation at each node's end: J_par[p] is the
//      product over its resolved children of P[p][code] (a resolved leaf), ambig_max (an ambiguous leaf) or max_product
//      over the child's staged J (an internal child), whose argument goes to arg[child][p].  An unresolved internal child's
//      row of arg is 0xFF, and an unresolved node's exponent is JOINT_UNRESOLVED.
//   2. The root state r = argmax of pi_k J_root[k].
//   3. Traceback by thread 0 in reverse flat order (a pre-order): an internal child's state is arg[child][state of its
//      parent], or -1 below an unresolved parent or for an unresolved child.
// The chunk's cond / node_ex hold the joint vectors (the inside pass, when it ran, is done with them).  jointLnL is
// pattern_lnl of pi_r J_root[r] 2^ex, 0.0 for an unresolved root, and NaN when any thread of the set multiplied or compared
// a NaN (one flag per thread, combined by the group at the root).
// ------------------------------------------------------------------------------------------------
constexpr int JOINT_UNRESOLVED = INT_MIN;

// A minimum of 8 CTAs per SM, as leaf_support_kernel (a chunk of at most 1024 sets puts no more on any of the 132 SMs),
// lets ptxas use 56 / 80 registers instead of 42 / 32; on one H100 at 700 W the kernel then took 9.7-9.9 / 16.8 / 12.9 ms
// instead of 9.9 / 42.4 / 33.5-34.0 ms on the north-star FEL / MEME-all / MEME-third shapes (tools/bench_joint_ancestors.py,
// alternating runs, identical output).

struct JointArgs {
    BatchPruneArgs in;        // the chunk's sets: PT, pat, leaf, ambig, pi, tree (MIX: mix_w, row_off); cond / node_ex scratch
    unsigned char *arg;       // [nSets][I][64] state of internal node i given its parent's state; 0xFF: i is unresolved
    long long *states;        // [nSets][I] the reconstruction: a state 0..D-1, or -1
    double *lnl;              // [nSets] jointLnL
};

template <bool MIX>
__global__ void __launch_bounds__(64, 8) joint_ancestors_kernel(JointArgs g) {
    __shared__ double xs[64];
    __shared__ double red[2];
    const BatchPruneArgs &a = g.in;
    const int s = blockIdx.x, k = threadIdx.x;
    const Group<64> grp{xs, red, 0xffffffffu, k};
    const bool live = k < a.D;
    const int pattern = a.pat[s];
    const double *PTs = a.PT + (size_t)s * (MIX ? a.R : a.B) * 4096;
    const double *mw = MIX ? a.mix_w + (size_t)s * a.R : nullptr;
    double *cs = a.cond + (size_t)s * a.I * 64;
    int *node_ex = a.node_ex + (size_t)s * a.I;
    unsigned char *arg = g.arg + (size_t)s * a.I * 64;
    bool bad = false, open = true;               // a NaN was met; the node has no resolved child yet
    double v = 0.0;
    int ex = 0;
    for (int par = 0; par < a.I; par++) {
        v = live ? 1.0 : 0.0;
        ex = 0;
        open = true;
        const int c_begin = a.tree.child_start[par], c_end = a.tree.child_start[par + 1];
        for (int ci = c_begin; ci < c_end; ci++) {
            if (ci - c_begin >= 2) grp.renorm(v, ex, RESCALE_BELOW);
            const int child = a.tree.child_ids[ci];
            BranchP<MIX> P(a, PTs, child);
            P.load_weights(mw);
            auto entry = [&](int j) { return P(j * 64 + k); };
            double m;
            if (child < a.L) {
                const int code = a.leaf[(size_t)child * a.Sp + pattern];
                if (code >= 0) {
                    m = live ? entry(code) : 0.0;
                    bad |= m != m;
                } else {
                    bool all;
                    m = grp.ambig_max(a.ambig + (size_t)(-code - 1) * 64, a.D, live, entry, all, bad);
                    if (all) continue;
                }
            } else {
                const int cin = child - a.L;
                if (node_ex[cin] == JOINT_UNRESOLVED) { arg[(size_t)cin * 64 + k] = 0xFF; continue; }
                int c;
                m = grp.max_product(grp.stage(cs[(size_t)cin * 64 + k]), a.D, live, entry, c, bad);
                arg[(size_t)cin * 64 + k] = (unsigned char)c;
                ex += node_ex[cin];
            }
            v *= m;
            open = false;
        }
        grp.renorm(v, ex);
        cs[(size_t)par * 64 + k] = v;
        if (k == 0) node_ex[par] = open ? JOINT_UNRESOLVED : ex;
        __syncthreads();                         // node_ex and arg rows visible to the block
    }
    // the root (par = I - 1): v, ex and open are its own
    const double x = live ? v * a.pi[k] : 0.0;
    bad |= x != x;
    const bool nan = grp.max(bad ? 1.0 : 0.0) > 0.0;
    double best;
    const int r = grp.argmax(x, best);
    if (k == 0) {
        long long *st = g.states + (size_t)s * a.I;
        st[a.I - 1] = open ? -1 : r;
        for (int n = a.I - 1; n >= 0; n--) {
            const long long sn = st[n];
            for (int ci = a.tree.child_start[n]; ci < a.tree.child_start[n + 1]; ci++) {
                const int child = a.tree.child_ids[ci];
                if (child < a.L) continue;
                const int c = sn < 0 ? 0xFF : arg[(size_t)(child - a.L) * 64 + sn];
                st[child - a.L] = c == 0xFF ? -1 : c;
            }
        }
        g.lnl[s] = open ? 0.0 : nan ? (double)NAN : pattern_lnl(best, ex, [] {});
    }
}

// ------------------------------------------------------------------------------------------------
// prune_rates_kernel (hb2_batch_site_rates): prune_batch_kernel<false>'s recursion for 4..32 padded states.  A group of
// G = 4, 8, 16 or 32 lanes owns one set, lane k = parent state k, and 32/G sets share a warp (24 states take G = 32, so
// a quarter of their lanes idle).  A child's vector is broadcast with width-G shuffles, the node maximum is a group
// shuffle-max, and node vectors live in global scratch cond[s][I][DP] (each lane reads back only the entry it wrote).
// Numerical rules: the group toolkit's, as prune_batch_kernel, but its root sum is Group<G>::sum, one xor tree over the G
// lanes.
// PT [sets][B][DP*DP], ambig [nAmb][DP], pi [DP]; n = sets of the launch.
// ------------------------------------------------------------------------------------------------
template <int DP>
__global__ void __launch_bounds__(128) prune_rates_kernel(BatchPruneArgs a, int n) {
    constexpr int G = DP <= 16 ? DP : 32;
    const int lane = threadIdx.x & 31, k = lane % G;
    const unsigned mask = G == 32 ? 0xffffffffu : ((1u << G) - 1) << (lane / G * G);
    const int s = (int)((blockIdx.x * 128u + threadIdx.x) / G);
    if (s >= n) return;                                  // whole groups
    const Group<G> grp{nullptr, nullptr, mask, k};
    const bool live = k < DP;
    const int pattern = a.pat[s];
    const double *PTs = a.PT + (size_t)s * a.B * DP * DP;
    double *cs = a.cond + (size_t)s * a.I * DP;
    int *node_ex = a.node_ex + (size_t)s * a.I;
    int ex = 0;
    double v = 0.0;
    for (int par = 0; par < a.I; par++) {
        v = k < a.D ? 1.0 : 0.0;
        ex = 0;
        const int c_begin = a.tree.child_start[par], c_end = a.tree.child_start[par + 1];
        for (int ci = c_begin; ci < c_end; ci++) {
            if (ci - c_begin >= 2) grp.renorm(v, ex, RESCALE_BELOW);
            const int child = a.tree.child_ids[ci];
            const double *PT = PTs + (size_t)child * DP * DP;
            auto entry = [&](int j) { return live ? PT[j * DP + k] : 0.0; };
            double m;
            if (child < a.L) m = grp.leaf_message(a.leaf[(size_t)child * a.Sp + pattern], a.ambig, DP, a.D, entry);
            else {
                const int cin = child - a.L;
                m = grp.dot(grp.stage(live ? cs[(size_t)cin * DP + k] : 0.0), a.D, live, entry);
                ex += node_ex[cin];
            }
            v *= m;
        }
        grp.renorm(v, ex);
        if (live) cs[(size_t)par * DP + k] = v;
        if (k == 0) node_ex[par] = ex;
        __syncwarp(mask);                                // node_ex visible to the group before a parent reads it
    }
    const double r = grp.sum(live ? v * a.pi[k] : 0.0);
    if (k == 0) a.out[s] = pattern_lnl(r, ex, [] {});
}

// ------------------------------------------------------------------------------------------------
// Simulated alignments (hb2_simulate; SimulateDataSet, likefunc.cpp:12584, discrete-category mode).  Every draw is one
// Philox4x32-10 call on the counter (lo32(g), hi32(g), slot, 0) with key (lo32(seed), hi32(seed)), g = global site,
// turned into u = (x0 * 2^21 + (x1 >> 11)) * 2^-53, and resolved against the sequential fp64 prefix sums c of the
// weights (entries that are not > 0 count as 0): the smallest j with fl(u * c_last) < c_j, else the last positive j.
// sim_cdf_kernel builds the prefix sums of every matrix row of the drawn classes once per call; simulate_kernel walks
// the tree from the root, one thread per site.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int r = 0; r < 10; r++) {
        if (r > 0) { k.x += 0x9E3779B9u; k.y += 0xBB67AE85u; }
        const unsigned lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const unsigned lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    }
    return c;
}

// Uniform in [0, 1) of draw `slot` of global site g; t is the fourth counter word (0 for hb2_simulate, the global set of
// hb2_batch_site_simulate).
__device__ __forceinline__ double sim_uniform(unsigned long long g, unsigned slot, uint2 key, unsigned t = 0u) {
    const uint4 x = philox4x32_10(make_uint4((unsigned)g, (unsigned)(g >> 32), slot, t), key);
    return (double)(((unsigned long long)x.x << 21) + (x.y >> 11)) * 0x1p-53;
}

// The draw rule on prefix sums c[0..m-1]; *last = the last index of positive weight, read only when u * total rounds up
// to the total.
// Vectors of 17..64 entries (matrix rows and root frequencies; the class vector when C <= 64) first load the total and the
// last entry of each 16-entry segment (one 128-byte line of a 64-padded row) together, so that a draw waits for memory
// about once instead of once per probe; the segment they select holds the result (c is non-decreasing), and the search
// inside it reads a line that is already in L1.  Longer vectors (C > 64 classes) take a plain binary search.
__device__ __forceinline__ int sim_draw(const double *__restrict__ c, int m, const int *last, double u) {
    int lo = 0, hi = m;
    double t;
    if (m > 16 && m <= 64) {
        double b[3];
#pragma unroll
        for (int k = 0; k < 3; k++) b[k] = 16 * k + 15 < m ? __ldg(c + 16 * k + 15) : 0.0;
        t = __dmul_rn(u, __ldg(c + m - 1));
        int s = 0;
#pragma unroll
        for (int k = 0; k < 3; k++) s += (16 * k + 15 < m && b[k] <= t) ? 1 : 0;
        lo = 16 * s;
        hi = min(lo + 16, m);
    } else {
        t = __dmul_rn(u, __ldg(c + m - 1));
    }
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (t < c[mid]) hi = mid; else lo = mid + 1;
    }
    return lo < m ? lo : *last;
}

struct SimArgs {
    const double *PT;          // [C][B][Dp*Dp] transposed transition matrices
    double *cdf;               // [C][B][D][Dp] prefix sums of each row (columns 0..D-1)
    int *last;                 // [C][B][D] last column of positive weight of each row
    const int *active;         // [C] 1 = the class has positive weight (its rows are built and checked)
    int *bad;                  // first bad row ((c * B + b) * D + row), INT_MAX when none
    const double *class_cdf;   // [C] prefix sums of the class weights
    const double *root_cdf;    // [D] prefix sums of the root frequencies
    const int *class_last;     // last class of positive weight
    const int *root_last;      // last state of positive root frequency
    TreeDev tree;
    long long *leaf_out;       // [L][chunk]
    long long *node_out;       // [I][chunk] or null
    int *class_out;            // [chunk] or null
    unsigned char *states;     // [I][chunk] internal states, used when they do not fit in shared memory (else null)
    int L, I, B, C, D, Dp, chunk, n;
    unsigned long long g0;     // global site of the chunk's first site (per-set: global replicate of the set's first column)
    uint2 key;
    // per-set mode (hb2_batch_site_simulate): "class" = set of the chunk
    const double *mix_w;       // MIX: [sets][R] component weights
    const int *row_off;        // MIX: [B+1] first component row of each branch (PT is [sets][R][Dp*Dp])
    int R;                     // MIX: component rows per set
    long long reps;            // replicates per set
    long long col0;            // chunk column of the launch's first thread (column = set * reps + replicate)
    unsigned t0;               // global set of the chunk's first set
};

// One CTA of 64 threads per (class, branch) of a drawn class; thread `row` forms the sequential prefix sums of its row
// (PT column `row`: adjacent threads read adjacent doubles) in shared memory, padded to 65 doubles per row against bank
// conflicts, and the CTA then stores the matrix's D x Dp block of the table with consecutive threads on consecutive
// doubles.  A row whose total is not finite and > 0 is reported through atomicMin.
// MIX (per-set mode, explicit-form mixtures): branch b of set c mixes its component rows row_off[b] .. row_off[b+1]-1 entry
// by entry, w_0 P_0 then fma(w_k, P_k, .) in component order, exactly as prune_batch_kernel<true> forms them.
constexpr int SIM_CDF_LD = 65;
template <bool MIX>
__global__ void __launch_bounds__(64) sim_cdf_kernel(SimArgs a) {
    __shared__ double rows[64 * SIM_CDF_LD];
    const long long cb = blockIdx.x;                       // class * B + branch
    if (!a.active[cb / a.B]) return;                       // uniform over the CTA
    const int row = threadIdx.x;
    if (row < a.D) {
        const double *P = a.PT + (size_t)cb * a.Dp * a.Dp + row;
        double wc[4];
        int nc = 1;
        if constexpr (MIX) {
            const long long set = cb / a.B;
            const int b = (int)(cb - set * a.B), r0 = a.row_off[b];
            nc = a.row_off[b + 1] - r0;
            P = a.PT + ((size_t)set * a.R + r0) * a.Dp * a.Dp + row;
            mix_weights(wc, a.mix_w + (size_t)set * a.R + r0, nc);
        }
        double *c = rows + row * SIM_CDF_LD;
        double s = 0.0;
        int last = -1;
#pragma unroll 4
        for (int j = 0; j < a.D; j++) {
            double v;
            if constexpr (!MIX) v = P[(size_t)j * a.Dp];
            else v = mix_entry(wc, nc, [&](int k) { return P[(size_t)k * a.Dp * a.Dp + (size_t)j * a.Dp]; });
            if (v > 0.0) { s = __dadd_rn(s, v); last = j; }
            c[j] = s;
        }
        const long long r = cb * a.D + row;
        a.last[r] = last;
        if (!(s > 0.0 && s <= 1.7976931348623157e308)) atomicMin(a.bad, (int)r);
    }
    __syncthreads();
    double *out = a.cdf + (size_t)cb * a.D * a.Dp;
    for (int k = threadIdx.x; k < a.D * a.Dp; k += blockDim.x) {
        const int rr = k / a.Dp, j = k - rr * a.Dp;
        if (j < a.D) out[k] = rows[rr * SIM_CDF_LD + j];   // padded columns are never read
    }
}

// The walk of simulate_kernel and batch_simulate_kernel, one thread per column: the block of the table (a rate class, or
// a set), the root state, then every internal node from the root down (flat post-order puts a parent after its children),
// each child's state drawn from the row of its parent's state.  Internal states are bytes in shared memory
// ([I][blockDim]) or, for trees with too many internal nodes, in global scratch ([I][chunk]).
// hb2_simulate (PER_SET false): thread i is site g0 + i; it draws its class, the fourth counter word is 0, and outputs
// are site-minor: leaf_out [L][chunk], node_out [I][chunk], class_out [chunk].
// Per-set mode (hb2_batch_site_simulate): thread i is column col0 + i = set * reps + replicate, consecutive threads on
// consecutive replicates of one set.  The set is the block and t0 + set the fourth counter word; there is no class draw.
// Outputs are column-major: leaf_out [n][L], node_out [n][I].
template <bool PER_SET>
__device__ __forceinline__ void sim_walk(const SimArgs &a) {
    extern __shared__ unsigned char sim_smem[];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    size_t blk = 0;
    unsigned long long g = a.g0 + (unsigned long long)i;
    unsigned t = 0u;
    if constexpr (PER_SET) {
        const long long col = a.col0 + i, set = col / a.reps;
        g = a.g0 + (unsigned long long)(col - set * a.reps);
        t = a.t0 + (unsigned)set;
        blk = (size_t)set;
    }
    const int L = a.L, I = a.I;
    unsigned char *st = a.states ? a.states + i : sim_smem + threadIdx.x;
    const size_t stride = a.states ? (size_t)a.chunk : (size_t)blockDim.x;
    // output index of node n (leaves: len = L, internal nodes: len = I)
    auto out = [&](int n, int len) { return PER_SET ? (size_t)i * len + n : (size_t)n * a.chunk + i; };
    if constexpr (!PER_SET) {
        const int cls = a.C == 1 ? 0 : sim_draw(a.class_cdf, a.C, a.class_last, sim_uniform(g, (unsigned)(L + I), a.key));
        if (a.class_out) a.class_out[i] = cls;
        blk = (size_t)cls;
    }
    int s = sim_draw(a.root_cdf, a.D, a.root_last, sim_uniform(g, (unsigned)(L + I - 1), a.key, t));
    if (a.node_out) a.node_out[out(I - 1, I)] = s;
    const size_t blk_rows = blk * a.B;
    for (int n = I - 1; n >= 0; n--) {
        if (n < I - 1) s = st[(size_t)n * stride];
        const int c_end = a.tree.child_start[n + 1];
        for (int ci = a.tree.child_start[n]; ci < c_end; ci++) {
            const int ch = a.tree.child_ids[ci];
            const size_t r = (blk_rows + ch) * a.D + s;
            const int x = sim_draw(a.cdf + r * a.Dp, a.D, a.last + r, sim_uniform(g, (unsigned)ch, a.key, t));
            if (ch < L) {
                a.leaf_out[out(ch, L)] = x;
            } else {
                st[(size_t)(ch - L) * stride] = (unsigned char)x;
                if (a.node_out) a.node_out[out(ch - L, I)] = x;
            }
        }
    }
}

__global__ void __launch_bounds__(128) simulate_kernel(SimArgs a) { sim_walk<false>(a); }
__global__ void __launch_bounds__(128) batch_simulate_kernel(SimArgs a) { sim_walk<true>(a); }

// ------------------------------------------------------------------------------------------------
// Peer exchange over NVLink (one process per GPU; every rank maps every other rank's exchange buffer through CUDA IPC).
// Buffer of a rank:  data[2 parities][R source ranks][payload doubles]  followed by  flags[2][R] (uint64 generation).
// A writer stores its payload into slot `rank` of EVERY rank's buffer (its own included), fences system-wide and then
// publishes the generation number in the matching flag; a reader spins (time-bounded) on its LOCAL flags.  Two
// parities suffice: a rank can run at most one evaluation ahead of the slowest one (it needs that rank's flag to finish).
// ------------------------------------------------------------------------------------------------
struct PeerBuf {
    double *const *peer;        // [R] device pointers to the ranks' buffers (entry `rank` = the local one)
    int R, rank, payload;
    unsigned long long gen;     // generation of THIS exchange (1, 2, 3, ...)
    int *err;
};
__device__ __forceinline__ double *peer_data(const PeerBuf &b, int dst_rank, int src_rank) {
    return b.peer[dst_rank] + ((size_t)(b.gen & 1ull) * b.R + src_rank) * b.payload;
}
__device__ __forceinline__ unsigned long long *peer_flag(const PeerBuf &b, int dst_rank, int src_rank) {
    return reinterpret_cast<unsigned long long *>(b.peer[dst_rank] + (size_t)2 * b.R * b.payload) + (b.gen & 1ull) * b.R + src_rank;
}
__device__ __forceinline__ void peer_publish(const PeerBuf &b, int dst_rank) {       // after __threadfence_system()
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(peer_flag(b, dst_rank, b.rank)), "l"(b.gen) : "memory");
}
__device__ __forceinline__ bool peer_await(const PeerBuf &b, int src_rank) {
    const unsigned long long *f = peer_flag(b, b.rank, src_rank);
    unsigned long long t0 = 0;
    for (int it = 0;; it++) {
        unsigned long long v;
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(f) : "memory");
        if (v == b.gen) return true;
        if ((it & 255) == 255) {
            const unsigned long long now = globaltimer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > HB2_PEER_WAIT_LIMIT_NS) { atomicExch(b.err, WAIT_PEER); return false; }
        }
    }
}

// Pattern shards only: every rank contributes its partial lnL; all ranks add the R partials in rank order, so the
// result is bit-identical everywhere.  One block, launched after final_sum_kernel.  payload >= 1.
__global__ void __launch_bounds__(64) peer_sum_kernel(PeerBuf b, double *lnL) {
    const int t = threadIdx.x;
    if (t < b.R) *peer_data(b, t, b.rank) = *lnL;
    __threadfence_system();
    __syncthreads();
    if (t < b.R) peer_publish(b, t);
    if (t < b.R) peer_await(b, t);
    __syncthreads();
    if (t == 0) {
        double s = 0.0;
        for (int r = 0; r < b.R; r++) s += __ldcg(peer_data(b, b.rank, r));
        *lnL = s;
    }
}

// Class groups: fused class-partial computation + exchange + merge + final sum (replaces class_partial_kernel, the
// zero-padded all-reduce used as a gather, class_merge_kernel and final_sum_kernel).  payload = 2*xs doubles per rank:
// [0,xs) partial values, [xs,2xs) binary exponents.  The block that finishes its stores LAST publishes the flags, waits
// for the other ranks' and merges every shard (fixed order: bit-identical lnL on all ranks).
struct ClassXchgArgs {
    const double *rootL; const int *rootE; const double *weights;
    int Sp, S, c0, nc, xs;
    PeerBuf pb;
    const double *xfreq;        // [nShards*G][xs] pattern frequencies of every rank (gathered once)
    int nShards, G, myShard;
    double *lnL; double *siteL; long long *siteScale;
    unsigned int *counter;
};

__global__ void __launch_bounds__(256) class_exchange_kernel(ClassXchgArgs a) {
    __shared__ double red[256];
    __shared__ int s_last, s_bad;
    const int tid = threadIdx.x;
    const PeerBuf &b = a.pb;
    const int xs = a.xs;
    for (int s = blockIdx.x * 256 + tid; s < xs; s += gridDim.x * 256) {
        double sum = 0.0;
        int emax = 0;
        if (s < a.S) {
            sum = merge_classes(a.nc, [&](int c, double &w, double &l, int &e) {
                w = a.weights[a.c0 + c];
                l = a.rootL[(size_t)(a.c0 + c) * a.Sp + s];
                e = a.rootE[(size_t)(a.c0 + c) * a.Sp + s];
            }, emax);
            if (emax == INT_MIN) emax = 0;
        }
        for (int r = 0; r < b.R; r++) {
            double *d = peer_data(b, r, b.rank);
            d[s] = sum;
            d[xs + s] = (double)emax;
        }
    }
    __threadfence_system();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(a.counter, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    if (tid == 0) { *a.counter = 0u; s_bad = 0; }
    __threadfence_system();
    if (tid < b.R) peer_publish(b, tid);
    if (tid < b.R) peer_await(b, tid);
    __syncthreads();
    double term = 0.0;
    for (int idx = tid; idx < a.nShards * xs; idx += 256) {
        const int j = idx / xs, s = idx - j * xs;
        const double f = a.xfreq[(size_t)j * a.G * xs + s];
        int emax;
        double sum = merge_classes(a.G, [&](int r, double &w, double &m, int &e) {
            const double *q = peer_data(b, b.rank, j * a.G + r);
            w = 1.0; m = __ldcg(q + s); e = (int)__ldcg(q + xs + s);
        }, emax);
        if (emax == INT_MIN) emax = 0;
        const double lnl = pattern_lnl(sum, emax, [&] { if (f > 0.0) s_bad = 1; });
        if (f > 0.0) term += f * lnl;
        if (a.siteL && j == a.myShard && s < a.S) {
            const SiteOut o = site_output(sum, emax);
            a.siteL[s] = o.L; a.siteScale[s] = o.scale;
        }
    }
    red[tid] = term;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (tid < o) red[tid] += red[tid + o];
        __syncthreads();
    }
    if (tid == 0) *a.lnL = s_bad ? -INFINITY : red[0];
}

__global__ void __launch_bounds__(256) final_sum_kernel(const double *partial, int n, const int *flag, double *out) {
    __shared__ double red[256];
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) s += partial[i];
    block_sum256(red, s);
    if (threadIdx.x == 0) out[0] = (*flag) ? -INFINITY : red[0];
}

}  // namespace hb2

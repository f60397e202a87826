// hb2_kernels_lanes.cuh -- fp64 pruning pass for 33..64 states in ONE launch with K in-order lanes per (class, tile).
//
// Same decomposition as the tensor walk kernel (hb2_kernels_tc.cuh): the host planner (hb2_engine.cu
// plan_walk) list-schedules the dirty jobs -- nodes and side products of nodes with two internal children -- on K lanes;
// CTA (class c, 32-pattern tile t, lane r) executes its lane's steps back to back.  Reference semantics:
// ComputeTreeBlockByBranch (tree_evaluator.cpp:3556-4171) restricted to the nodes DetermineNodesForUpdate marked.
//   * CTA = 4 warps x 8 patterns; the contraction C[pattern][parent] = sum_j X[pattern][j] * PT[j][parent] runs on the FP64
//     tensor pipe (mma.sync.m8n8k4.f64): warp tile 8 x 64, 128 DMMA + 144 shared-memory loads per warp and contraction.
//     A register-blocked DFMA product was slower; splitting the parent states over two warps per 8 patterns (8 warps per
//     CTA) shortened the product but cost more than that in the cross-warp row maximum and in barrier time: not kept;
//   * a thread owns ONE pattern (row 8*warp + lane/4) and 16 of its states (8j + 2*(lane%4) + {0,1}): renormalisation and
//     the root dot product reduce over 4 lanes (two shuffles);
//   * one P buffer + one X buffer = 53 KB, 128 threads: four CTAs per SM, so that the load / renormalise / publish
//     phases of one CTA run under the products of the others;
//   * hand-over between lanes: a flag per (class, job, tile) holding the id of the pass that produced the tile
//     (st.release.gpu by the producer after its stores, ld.acquire.gpu poll by the consumer, time-bounded);
//   * a child produced by THIS CTA in its previous job goes straight from registers to the shared-memory operand;
//   * the transition matrix of the NEXT contraction (its branch id travels in the step descriptor) is staged with
//     cp.async as soon as the current product has released the buffer, i.e. under the epilogue and the leaf steps in
//     between; step descriptors run two steps ahead, leaf state codes one.
// The children of a node are multiplied in plan order; with two children the product is exact-commutative and
// power-of-two rescalings are exact, and nodes with more children are planned in tree order (plan_walk,
// canonical_multi), so conditionals do not depend on the plan: a partial re-evaluation reproduces the full one bit for
// bit.
#pragma once
#include "hb2_kernels_fp64.cuh"
#include "hb2_kernels_tc.cuh"      // step encoding (WALK_*, STEP_*)

namespace hb2 {

struct LaneArgs {
    PruneArgs a;
    double *cond_side;          // [C][I][Sp][64] side products (job I + n)
    int *scal_side;             // [C][I][Sp]
    const int *lane_start;      // [K+1]
    const int4 *steps;          // x: child | WALK_*, y: job | STEP_*, z: branch id of the next contraction of the lane (-1: none),
                                // w: 1 if another lane waits for this job (STEP_LAST publishes its flag)
    int *flags;                 // [C][2I][T] id of the pass that last produced (class, job, tile)
    int *err;
    int K, T, ncls, nslots, pass;
    long long *trace;           // nullable bring-up aid (HB2_WALK_TRACE): 12 clock64 stamps per step of CTA `trace_cta`
    int trace_cta;
};

// CTA shape: 4 warps x 8 patterns (32 patterns, 128 threads, four CTAs per SM).
constexpr int LANES_WARPS = 4, LANES_TILE_P = 8 * LANES_WARPS, LANES_THREADS = 32 * LANES_WARPS, LANES_CTAS_PER_SM = 4;
constexpr int LANES_LDX = 68;                    // leading dimensions (doubles): both fragment loads are 2 wavefronts, the
constexpr int LANES_LDP = 72;                    // minimum for 256 bytes per warp
constexpr int LANES_SMEM_BYTES = (LANES_TILE_P * LANES_LDX + 64 * LANES_LDP) * (int)sizeof(double);

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// warp tile 8 patterns x 64 parent states, K = 64: acc[j] = C[row][8j + 2*q4 + {0,1}]
__device__ __forceinline__ void lanes_mm(const double *__restrict__ Xs, const double *__restrict__ Ps, int row, int g, int q4,
                                         double (&acc)[8][2]) {
    const double *a0 = Xs + row * LANES_LDX + q4;
    const double *b0 = Ps + q4 * LANES_LDP + g;
#pragma unroll 4
    for (int k0 = 0; k0 < 64; k0 += 4) {
        const double x = a0[k0];
#pragma unroll
        for (int j = 0; j < 8; j++) dmma884(acc[j], x, b0[k0 * LANES_LDP + 8 * j]);
    }
}

__global__ void __launch_bounds__(LANES_THREADS, LANES_CTAS_PER_SM) prune64_lanes_kernel(LaneArgs w) {
    extern __shared__ __align__(16) double sm[];
    double *Xs = sm;                              // [LANES_TILE_P][LDX] child conditionals (pattern-major)
    double *Ps = sm + LANES_TILE_P * LANES_LDX;   // [64][LDP] transition matrix (transposed) of the current / next contraction
    const PruneArgs &a = w.a;
    const int tid = threadIdx.x, warp = tid >> 5, g = (tid & 31) >> 2, q4 = tid & 3;
    const int row = 8 * warp + g;                 // this thread's pattern within the tile
    const int c0s = 2 * q4;                       // this thread's states: c0s + 8j + {0,1}, j = 0..7
    const size_t Sp = a.Sp;
    const int r = blockIdx.x % w.K;
    const int i_begin = w.lane_start[r], i_end = w.lane_start[r + 1];
    if (i_begin == i_end) return;

    // ROWS x 64 doubles, contiguous in global memory -> padded rows in shared memory, 16 bytes per copy
    auto stage_rows = [&](double *dst, const int ld, const double *src, const int rows) {
#pragma unroll 8
        for (int idx = tid; idx < rows * 32; idx += LANES_THREADS) {
            const int rr = idx >> 5, c2 = (idx & 31) * 2;
            cp_async16(dst + rr * ld + c2, src + rr * 64 + c2);
        }
    };
    auto stage_P = [&](int cat, int branch) {
        stage_rows(Ps, LANES_LDP, a.PT + ((size_t)cat * a.B + branch) * 4096, 64);
        cp_async_commit();
    };
    // wait until (class, job, tile) has been produced by this pass.  Uniform call (contains a barrier).
    auto wait_flag = [&](int cat, int job, int tile) {
        if (tid == 0) {
            const int *f = w.flags + ((size_t)cat * 2 * a.I + job) * w.T + tile;
            unsigned long long t0 = 0;
            for (int it = 0;; it++) {
                int got;
                asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(got) : "l"(f) : "memory");
                if (got == w.pass) break;
                if ((it & 63) == 63) {                                          // never hang the GPU: time-bounded
                    const unsigned long long now = globaltimer_ns();
                    if (t0 == 0) t0 = now;
                    else if (now - t0 > HB2_WAIT_LIMIT_NS) { atomicExch(w.err, WAIT_LANE); break; }
                }
            }
        }
        __syncthreads();
    };

    for (int ct = blockIdx.x / w.K; ct < w.ncls * w.T; ct += w.nslots) {
        const int cat = a.cat0 + ct / w.T;
        const int tile = ct % w.T;
        const int s0 = tile * LANES_TILE_P;
        const size_t s = (size_t)s0 + row;        // this thread's pattern
        double v[8][2];
        int ex = 0;
        int nmul = 0;                             // factors multiplied into v since the job's first step
        __syncthreads();                          // previous (class, tile): the buffers are free
        int4 st_a = __ldg(w.steps + i_begin);
        int4 st_b = (i_begin + 1 < i_end) ? __ldg(w.steps + i_begin + 1) : make_int4(0, 0, -1, 0);
        {   // the lane's first contraction
            const int c0 = st_a.x & WALK_ID_MASK;
            const int b0 = (c0 >= a.L && !(st_a.x & WALK_MUL)) ? c0 : st_a.z;
            if (b0 >= 0) stage_P(cat, b0);
        }
        auto leaf_code = [&](int4 q) -> int {
            const int ch = q.x & WALK_ID_MASK;
            if (ch >= a.L) return 0;
            return (ch == a.forced_node) ? __ldg(a.forced + s) : __ldg(a.leaf + (size_t)ch * Sp + s);
        };
        int code_next = leaf_code(st_a);
        for (int i = i_begin; i < i_end; i++) {
            const int4 st = st_a;
            const int code = code_next;
            st_a = st_b;
            if (i + 2 < i_end) st_b = __ldg(w.steps + i + 2);       // descriptors two steps ahead ...
            if (i + 1 < i_end) code_next = leaf_code(st_a);          // ... so that this address is ready: codes one step ahead
            const int enc = st.x, flags = st.y;
            const int child = enc & WALK_ID_MASK;
            const int job = flags & WALK_ID_MASK;            // node (< I) or side product (I + node)
            const bool tr = w.trace && tid == 0 && (int)blockIdx.x == w.trace_cta;
            long long *trp = tr ? w.trace + (size_t)(i - i_begin) * 12 : nullptr;
            if (tr) { trp[0] = ((long long)st.x << 32) | (unsigned)st.y; trp[1] = clock64(); }
            if ((flags & STEP_FIRST) && !(enc & WALK_CHAIN)) {
                ex = 0;
#pragma unroll
                for (int j = 0; j < 8; j++) { v[j][0] = 1.0; v[j][1] = 1.0; }
            }
            if (flags & STEP_FIRST) nmul = 0;
            if (nmul++ >= 2) {                    // wide node (hb2_kernels_fp64.cuh); uniform over the CTA
                if (a.L + (job >= a.I ? job - a.I : job) == a.forced_node) {   // pinned: rescale by the forced state alone
                    const int f = __ldg(a.forced + s);
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        if (c0s + 8 * j != f) v[j][0] = 0.0;
                        if (c0s + 8 * j + 1 != f) v[j][1] = 0.0;
                    }
                }
                rescale_running_quad(v, ex);
            }
            if (child < a.L) {
                // leaf: column gather PT[state][k]; ambiguous: sum_j amb[j] PT[j][k]
                const double *PT = a.PT + ((size_t)cat * a.B + child) * 4096 + c0s;
                if (code >= 0) {
                    const double2 *p = reinterpret_cast<const double2 *>(PT + (size_t)code * 64);
                    double2 m[8];
#pragma unroll
                    for (int j = 0; j < 8; j++) m[j] = __ldg(p + 4 * j);
#pragma unroll
                    for (int j = 0; j < 8; j++) { v[j][0] *= m[j].x; v[j][1] *= m[j].y; }
                } else {
                    const double *amb = a.ambig + (size_t)(-code - 1) * 64;
                    double2 m[8];
#pragma unroll
                    for (int j = 0; j < 8; j++) m[j] = make_double2(0.0, 0.0);
                    for (int jj = 0; jj < a.D; jj++) {
                        const double wj = __ldg(amb + jj);
                        if (wj != 0.0) {
                            const double2 *p = reinterpret_cast<const double2 *>(PT + (size_t)jj * 64);
#pragma unroll
                            for (int j = 0; j < 8; j++) {
                                const double2 q = __ldg(p + 4 * j);
                                m[j].x = fma(wj, q.x, m[j].x); m[j].y = fma(wj, q.y, m[j].y);
                            }
                        }
                    }
#pragma unroll
                    for (int j = 0; j < 8; j++) { v[j][0] *= m[j].x; v[j][1] *= m[j].y; }
                }
            } else if (enc & WALK_MUL) {
                // side product of this node (its other children, contracted by another lane or earlier in this one)
                const int n = child - a.L - a.I;
                if (enc & WALK_WAIT) wait_flag(cat, child - a.L, tile);
                const double2 *X = reinterpret_cast<const double2 *>(w.cond_side + (((size_t)cat * a.I + n) * Sp + s) * 64 + c0s);
                double2 m[8];
#pragma unroll
                for (int j = 0; j < 8; j++) m[j] = __ldcg(X + 4 * j);
                ex += __ldcg(w.scal_side + ((size_t)cat * a.I + n) * Sp + s);
#pragma unroll
                for (int j = 0; j < 8; j++) { v[j][0] *= m[j].x; v[j][1] *= m[j].y; }
            } else {
                const int cin = child - a.L;
                int sc = 0;
                if (enc & WALK_CHAIN) {
                    // the child is this lane's previous job: its renormalised values are still in v, its exponent in ex
                    // (Xs is free: every product ends with a barrier)
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        *reinterpret_cast<double2 *>(Xs + row * LANES_LDX + c0s + 8 * j) = make_double2(v[j][0], v[j][1]);
                        v[j][0] = 1.0; v[j][1] = 1.0;
                    }
                } else {
                    if (enc & WALK_WAIT) wait_flag(cat, cin, tile);
                    stage_rows(Xs, LANES_LDX, a.cond + (((size_t)cat * a.I + cin) * Sp + s0) * 64, LANES_TILE_P);
                    cp_async_commit();
                    sc = __ldcg(a.scal + ((size_t)cat * a.I + cin) * Sp + s);
                }
                if (tr) trp[2] = clock64();
                cp_async_wait<0>();               // this step's P (staged after the previous product) and X have landed
                if (tr) trp[3] = clock64();
                __syncthreads();
                if (tr) trp[4] = clock64();
                double acc[8][2];
#pragma unroll
                for (int j = 0; j < 8; j++) { acc[j][0] = 0.0; acc[j][1] = 0.0; }
                lanes_mm(Xs, Ps, row, g, q4, acc);
                if (tr) trp[5] = clock64();
                __syncthreads();                  // every thread is done with Xs and Ps
                if (tr) trp[6] = clock64();
                if (st.z >= 0) stage_P(cat, st.z);    // lands under the epilogue, the leaf steps and the next X load
                ex += sc;
#pragma unroll
                for (int j = 0; j < 8; j++) { v[j][0] *= acc[j][0]; v[j][1] *= acc[j][1]; }
            }
            if (tr) trp[7] = clock64();
            if (flags & STEP_LAST) {
                const bool side = job >= a.I;
                const int node = side ? job - a.I : job;
                if (!side && a.L + node == a.forced_node) {            // pinned internal node: only the forced state survives
                    const int f = __ldg(a.forced + s);
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        if (c0s + 8 * j != f) v[j][0] = 0.0;
                        if (c0s + 8 * j + 1 != f) v[j][1] = 0.0;
                    }
                }
                // per-pattern renormalisation: exact power of two so that max_k lands in [0.5, 1).  The values are
                // non-negative, so the row maximum is the maximum of the bit patterns; its exponent needs the high words only.
                int mh = 0;
#pragma unroll
                for (int j = 0; j < 8; j++) mh = max(mh, max(__double2hiint(v[j][0]), __double2hiint(v[j][1])));
                mh = max(mh, __shfl_xor_sync(0xffffffffu, mh, 1));
                mh = max(mh, __shfl_xor_sync(0xffffffffu, mh, 2));
                int e = 0;
                if (mh >= 0x00100000 && mh < 0x7ff00000) {             // normal, finite, positive maximum
                    e = (mh >> 20) - 1022;                             // m = f * 2^e, f in [0.5, 1); |e| <= 1022: one exact step
                    if (e != 0) {
                        const double sc1 = exp2i(-e);
#pragma unroll
                        for (int j = 0; j < 8; j++) { v[j][0] *= sc1; v[j][1] *= sc1; }
                    }
                } else if (mh < 0x7ff00000) {
                    // zero or subnormal high word (uniform over the four lanes of the pattern): the slow exact path
                    const unsigned gmask = 0xFu << (tid & 28);          // the four lanes of this pattern take this branch together
                    double m = 0.0;
#pragma unroll
                    for (int j = 0; j < 8; j++) m = fmax(m, fmax(v[j][0], v[j][1]));
                    m = fmax(m, __shfl_xor_sync(gmask, m, 1));
                    m = fmax(m, __shfl_xor_sync(gmask, m, 2));
                    if (m > 0.0) {
                        e = ilogb(m) + 1;
                        const double s1 = exp2i(-(e / 2)), s2 = exp2i(-(e - e / 2));
#pragma unroll
                        for (int j = 0; j < 8; j++) { v[j][0] = v[j][0] * s1 * s2; v[j][1] = v[j][1] * s1 * s2; }
                    }
                }                                                     // inf / NaN: left alone
                ex += e;
                const bool is_root = !side && node == a.I - 1;
                double2 *outp = reinterpret_cast<double2 *>((side ? w.cond_side : a.cond) + (((size_t)cat * a.I + node) * Sp + s) * 64 + c0s);
#pragma unroll
                for (int j = 0; j < 8; j++) __stcg(outp + 4 * j, make_double2(v[j][0], v[j][1]));
                if (q4 == 0) __stcg((side ? w.scal_side : a.scal) + ((size_t)cat * a.I + node) * Sp + s, ex);
                if (is_root) {
                    double rr = 0.0;
#pragma unroll
                    for (int j = 0; j < 8; j++) rr += v[j][0] * a.pi[c0s + 8 * j] + v[j][1] * a.pi[c0s + 8 * j + 1];
                    rr += __shfl_xor_sync(0xffffffffu, rr, 1);
                    rr += __shfl_xor_sync(0xffffffffu, rr, 2);
                    if (q4 == 0) {
                        a.rootL[(size_t)cat * Sp + s] = rr;
                        a.rootE[(size_t)cat * Sp + s] = ex;
                    }
                }
                if (tr) trp[8] = clock64();
                __syncthreads();                  // the whole tile is written (and visible to this CTA's later reads)
                if (tr) trp[9] = clock64();
                if (tid == 0 && st.w) {           // publish: another lane of this (class, tile) waits for this job.  The release
                    // is cumulative over the stores this thread observed through the barrier.
                    int *f = w.flags + ((size_t)cat * 2 * a.I + job) * w.T + tile;
                    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(f), "r"(w.pass) : "memory");
                }
                if (tr) trp[10] = clock64();
            }
        }
    }
}

}  // namespace hb2

namespace hb2 {

// ------------------------------------------------------------------------------------------------------------------
// prune_small_dmma_kernel<DP>: 16 / 24 / 32 padded states (proteins: 20 -> 24) on the FP64 tensor pipe, whole pass in one
// launch.  CTA = 8 warps x 8 patterns; every CTA walks the dirty nodes in post-order (jobs ascending), so all dependencies
// are thread-local, like prune_small_walk_kernel -- but a warp contracts 8 patterns with DP/4 x DP/8 DMMA (m8n8k4) instead
// of DP*DP DFMA per thread, a thread carries 2*DP/8 values of ONE pattern instead of four DP-vectors (the one-thread-per-
// pattern kernel needs ~230 registers at DP = 24: two CTAs per SM, 12.5 -> 20 % of the HBM roofline), and
//   * the child's vector is read from global memory directly in A-fragment order (lanes q4 = 0..3 of a pattern read 32
//     contiguous bytes per k-step: whole sectors, no shared-memory round trip);
//   * P^T of the NEXT child is staged with cp.async under the current product (two buffers, one barrier per child);
//   * a child that is the previous job's node is rebuilt from the accumulator fragments with shuffles.
// Layouts, scaling convention and results' meaning are those of prune_small_walk_kernel (reference
// tree_evaluator.cpp:3556-4171, generic-D branch :3704-4043); summation order inside a product differs (rounding).
// ------------------------------------------------------------------------------------------------------------------
// NW warps per CTA.  Every CTA walks the whole tree, so the launch is a few long waves; the host picks the shape (8 warps at
// 4 CTAs per SM, or 4 warps at 9 per SM for DP <= 24) whose resident capacity leaves the smaller tail wave.
template <int DP, int NW>
__global__ void __launch_bounds__(32 * NW, NW == 4 ? 9 : (DP == 32 ? 3 : 4)) prune_small_dmma_kernel(PruneArgs a, const int *__restrict__ jobs, int njobs) {
    constexpr int NT = DP / 8, KS = DP / 4;
    constexpr int LD = (DP == 24) ? 24 : DP + 8;          // 2*LD mod 32 == 16: the 4 rows of a B fragment hit disjoint banks
    __shared__ __align__(16) double Pbuf[2][DP * LD];
    const int tid = threadIdx.x, warp = tid >> 5, g = (tid & 31) >> 2, q4 = tid & 3;
    const int cat = a.cat0 + blockIdx.y;
    const size_t Sp = a.Sp;
    const size_t s = (size_t)blockIdx.x * (8 * NW) + 8 * warp + g;   // this thread's pattern
    if (njobs <= 0) return;

    auto stage_P = [&](int child, int buf) {
        const double *src = a.PT + ((size_t)cat * a.B + child) * DP * DP;
        for (int idx = tid; idx < DP * DP / 2; idx += 32 * NW) {
            const int rr = idx / (DP / 2), c2 = (idx % (DP / 2)) * 2;
            cp_async16(&Pbuf[buf][rr * LD + c2], src + rr * DP + c2);
        }
        cp_async_commit();
    };
    double pv[NT][2];                    // previous job's node (accumulator-fragment order) for the register hand-over
    int prev = -1, pex = 0;
    int step = 0;                        // children processed so far: buffer = step & 1
    stage_P(__ldg(a.tree.child_ids + __ldg(a.tree.child_start + __ldg(jobs))), 0);
    for (int jb = 0; jb < njobs; jb++) {
        const int par = __ldg(jobs + jb);
        double v[NT][2];
#pragma unroll
        for (int t = 0; t < NT; t++) { v[t][0] = 1.0; v[t][1] = 1.0; }
        int ex = 0;
        const int c_begin = __ldg(a.tree.child_start + par), c_end = __ldg(a.tree.child_start + par + 1);
        for (int ci = c_begin; ci < c_end; ci++, step++) {
            const int child = __ldg(a.tree.child_ids + ci);
            // the child after this one (next child of this node, or the first child of the next job)
            int nchild = -1;
            if (ci + 1 < c_end) nchild = __ldg(a.tree.child_ids + ci + 1);
            else if (jb + 1 < njobs) nchild = __ldg(a.tree.child_ids + __ldg(a.tree.child_start + __ldg(jobs + jb + 1)));
            // operands of an internal child: issued before the barrier, consumed after it
            double x[KS];
            int sc = 0;
            const bool internal = child >= a.L;
            const bool chained = internal && (child - a.L == prev);
            int code = 0;
            if (!internal) {
                code = (child == a.forced_node) ? __ldg(a.forced + s) : __ldg(a.leaf + (size_t)child * Sp + s);
            } else if (!chained) {
                const double *X = a.cond + (((size_t)cat * a.I + (child - a.L)) * Sp + s) * DP + q4;
#pragma unroll
                for (int ks = 0; ks < KS; ks++) x[ks] = __ldcg(X + 4 * ks);
                sc = __ldcg(a.scal + ((size_t)cat * a.I + (child - a.L)) * Sp + s);
            } else {
                // rebuild the A fragments from the previous node's accumulator fragments: k = 4 ks + q4 lives in n-tile
                // ks/2, column (ks odd ? 4 : 0) + q4 -> lane (ks odd ? 2 : 0) + q4/2 of this pattern, element q4 & 1
                const int base = (tid & 31) & ~3;
#pragma unroll
                for (int ks = 0; ks < KS; ks++) {
                    const int src = base + ((ks & 1) ? 2 : 0) + (q4 >> 1);
                    const double t0 = __shfl_sync(0xffffffffu, pv[ks >> 1][0], src);
                    const double t1 = __shfl_sync(0xffffffffu, pv[ks >> 1][1], src);
                    x[ks] = (q4 & 1) ? t1 : t0;
                }
                sc = pex;
            }
            cp_async_wait<0>();              // this child's P has landed (this thread's copies) ...
            __syncthreads();                 // ... everyone's; and every warp is past the previous product: the other buffer is free
            if (nchild >= 0) stage_P(nchild, (step + 1) & 1);
            const double *Ps = Pbuf[step & 1];
            if (!internal) {
                if (code >= 0) {
                    const double *row = Ps + code * LD + 2 * q4;
#pragma unroll
                    for (int t = 0; t < NT; t++) { const double2 r = *reinterpret_cast<const double2 *>(row + 8 * t); v[t][0] *= r.x; v[t][1] *= r.y; }
                } else {
                    const double *amb = a.ambig + (size_t)(-code - 1) * DP;
                    double acc[NT][2];
#pragma unroll
                    for (int t = 0; t < NT; t++) { acc[t][0] = 0.0; acc[t][1] = 0.0; }
                    for (int j = 0; j < a.D; j++) {
                        const double wgt = __ldg(amb + j);
                        if (wgt != 0.0) {
                            const double *row = Ps + j * LD + 2 * q4;
#pragma unroll
                            for (int t = 0; t < NT; t++) { const double2 r = *reinterpret_cast<const double2 *>(row + 8 * t); acc[t][0] = fma(wgt, r.x, acc[t][0]); acc[t][1] = fma(wgt, r.y, acc[t][1]); }
                        }
                    }
#pragma unroll
                    for (int t = 0; t < NT; t++) { v[t][0] *= acc[t][0]; v[t][1] *= acc[t][1]; }
                }
            } else {
                double acc[NT][2];
#pragma unroll
                for (int t = 0; t < NT; t++) { acc[t][0] = 0.0; acc[t][1] = 0.0; }
                const double *b0 = Ps + q4 * LD + g;
#pragma unroll
                for (int ks = 0; ks < KS; ks++)
#pragma unroll
                    for (int t = 0; t < NT; t++) dmma884(acc[t], x[ks], b0[4 * ks * LD + 8 * t]);
                ex += sc;
#pragma unroll
                for (int t = 0; t < NT; t++) { v[t][0] *= acc[t][0]; v[t][1] *= acc[t][1]; }
            }
            if (ci - c_begin >= 1 && ci + 1 < c_end) {   // wide node (hb2_kernels_fp64.cuh): before its third and later children
                if (a.L + par == a.forced_node) {          // pinned: rescale by the forced state alone
                    const int f = __ldg(a.forced + s);
#pragma unroll
                    for (int t = 0; t < NT; t++) {
                        if (8 * t + 2 * q4 != f) v[t][0] = 0.0;
                        if (8 * t + 2 * q4 + 1 != f) v[t][1] = 0.0;
                    }
                }
                rescale_running_quad(v, ex);
            }
        }
        if (a.L + par == a.forced_node) {
            const int f = __ldg(a.forced + s);
#pragma unroll
            for (int t = 0; t < NT; t++) {
                if (8 * t + 2 * q4 != f) v[t][0] = 0.0;
                if (8 * t + 2 * q4 + 1 != f) v[t][1] = 0.0;
            }
        }
        // per-pattern renormalisation (max in [0.5, 1)): own values, then the 4 lanes of the pattern
        double m = 0.0;
#pragma unroll
        for (int t = 0; t < NT; t++) m = fmax(m, fmax(v[t][0], v[t][1]));
        m = fmax(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmax(m, __shfl_xor_sync(0xffffffffu, m, 2));
        if (m > 0.0 && m < INFINITY) {
            const int mh = __double2hiint(m);
            int e;
            if (mh >= 0x00100000) {
                e = (mh >> 20) - 1022;
                if (e != 0) {
                    const double sc1 = exp2i(-e);
#pragma unroll
                    for (int t = 0; t < NT; t++) { v[t][0] *= sc1; v[t][1] *= sc1; }
                }
            } else {
                e = ilogb(m) + 1;
                const double s1 = exp2i(-(e / 2)), s2 = exp2i(-(e - e / 2));
#pragma unroll
                for (int t = 0; t < NT; t++) { v[t][0] = v[t][0] * s1 * s2; v[t][1] = v[t][1] * s1 * s2; }
            }
            ex += e;
        }
        double *outp = a.cond + (((size_t)cat * a.I + par) * Sp + s) * DP + 2 * q4;
#pragma unroll
        for (int t = 0; t < NT; t++) *reinterpret_cast<double2 *>(outp + 8 * t) = make_double2(v[t][0], v[t][1]);
        if (q4 == 0) a.scal[((size_t)cat * a.I + par) * Sp + s] = ex;
#pragma unroll
        for (int t = 0; t < NT; t++) { pv[t][0] = v[t][0]; pv[t][1] = v[t][1]; }
        prev = par; pex = ex;
        if (par == a.I - 1) {
            double r = 0.0;
#pragma unroll
            for (int t = 0; t < NT; t++) r += v[t][0] * a.pi[8 * t + 2 * q4] + v[t][1] * a.pi[8 * t + 2 * q4 + 1];
            r += __shfl_xor_sync(0xffffffffu, r, 1);
            r += __shfl_xor_sync(0xffffffffu, r, 2);
            if (q4 == 0) {
                a.rootL[(size_t)cat * Sp + s] = r;
                a.rootE[(size_t)cat * Sp + s] = ex;
            }
        }
    }
}

}  // namespace hb2

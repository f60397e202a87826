// hb2_kernels_tc.cuh -- tensor-core (Hopper wgmma) pruning path for 33..64-state models (sm_90a).
//
// The 61-state codon update  parent[s][n] *= sum_k P[n][k] * child[s][k]  is a dense contraction batched over
// patterns:  D[128 patterns][64 parent states] = X[128][64 child states] * P^T.  The tensor core has no fp64 tf32-class
// kind, so the contraction runs as an error-compensated split in tf32 with fp32 accumulation:
//        X = Xh + Xl,  P = Ph + Pl   (each part exactly representable in tf32, round-to-nearest splits)
//        D = Xl*Ph + Xh*Pl + Xh*Ph   (the dropped Xl*Pl term is ~2^-22 relative)
// All operands are non-negative, so there is no cancellation and the relative error of D is bounded by the
// representation error of the splits (~2^-22) plus fp32 accumulation.  Conditionals are stored in fp32, renormalised
// per (node, pattern) to max in [0.5,1) with an int32 binary exponent, so fp32 range is never an issue.
//
// Anchors.  The tensor core accumulates in fp32 without round-to-nearest, which would bias lnL by ~1e-7*|lnL| over a
// codon tree.  Conditional vectors are sharply peaked (1-3 codons carry almost all the mass), so each thread pulls the
// entries >= 2^-6 of its row ("anchors") out of the tensor operand and multiplies them on the CUDA cores with
// round-to-nearest fp32 FMAs against fp32 rows of P^T while the MMAs run; the tensor core only contracts the diffuse
// remainder, whose rounding bias is scaled down by its share.
//
// Operand staging (wgmma.mma_async m64n128k8, one warpgroup = 128 threads = one 128-pattern tile).  The contraction
// runs transposed, D^T[64 parents][128 patterns] = P * X^T, so that one instruction covers the whole tile: per FMA it
// reads 3/4 of the shared-memory operand bytes of the m64n64k8 shape with X as A, and it needs half the instructions.
//   A (= P, 64 x 64, K-major) comes from SHARED MEMORY in the canonical no-swizzle layout (8x16-byte core matrices;
//     LBO = 1024 B between K chunks, SBO = 128 B between 8-row groups).  The expm stage writes P already split and tiled
//     that way (the ExpmTcOut epilogues of hb2_kernels_fp64.cuh, mix_reduce_kernel), so one 32 KB cp.async.bulk (TMA
//     engine, mbarrier completion) per child stages Ph and Pl.
//   B (= X, 128 x 64, K-major) comes from SHARED MEMORY in the same layout (LBO = 2048 B, SBO = 128 B): each of the 128
//     threads owns one pattern, loads its fp32 row from HBM, splits it in registers and writes Xh / Xl -- the same
//     [chunk][pattern][4] order the conditionals have in HBM, so a thread's stores are 16-byte and conflict-free.
//   D^T (64 x 128 fp32) is accumulated in registers (one 64-register fragment per thread), written to a shared buffer of
//     one row per pattern and read back one row per thread, multiplied into the running product of the parent held in
//     registers.
//
// Replaces (for D in 33..64) reference tree_evaluator.cpp:3875-4008 (_hy_mvp_blocked<61> + _hy_vvmult_sum<61>).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "hb2_kernels_fp64.cuh"

namespace hb2 {

constexpr int TC_TILE_P = 128;                 // patterns per warpgroup (the wgmma N)
constexpr int TC_X_BYTES = 2 * 16 * 128 * 16;  // B operand: Xh | Xl, [16 chunks][128 patterns][4] fp32 each
constexpr int TC_D_ROW = 68;                   // floats per pattern row of the shared accumulator read-back buffer
constexpr int TC_D_BYTES = 128 * TC_D_ROW * 4;
constexpr int WALK_FAST_ANCHORS = 4;           // anchors handled by the unrolled fast path of the walk kernel; more go to a loop
constexpr float TC_ANCHOR_THR = 0.015625f;     // 2^-6 (rows are normalised to max in [0.5,1))

struct PruneTcArgs {
    const float *PB;                // [C][B][2][16][64][4] canonical K-major tiles of P (hi, lo)
    const float *PTf;               // [C][B][64][68] fp32 copy of PT, padded rows (leaf column gather, anchors)
    float *cond;                    // [C][I][Sp/128][16 chunks][128 patterns][4] fp32 conditionals (tile-wise K-major chunks)
    int *scal;                      // [C][I][Sp]
    const int *leaf;                // [L][Sp]
    const double *ambig;            // [nAmb][64]
    const double *pi;               // [64]
    double *rootL;                  // [C][Sp]
    int *rootE;                     // [C][Sp]
    TreeDev tree;
    int *err;                       // device error flag (mbarrier timeout)
    int L, I, B, D, Sp, cat0;
    const int *forced;              // forced states of ONE node (see PruneArgs), or unused when forced_node < 0
    int forced_node;
};

// ---- PTX wrappers ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_wait(uint64_t *bar, uint32_t parity, int *err_flag) {
    const uint32_t addr = smem_u32(bar);
    unsigned long long t0 = 0;
    for (int it = 0;; it++) {
        uint32_t ok;
        asm volatile(
            "{\n\t"
            ".reg .pred P1;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, P1;\n\t"
            "}" : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
        if (ok) return true;
        if ((it & 1023) == 1023) {
            const unsigned long long now = globaltimer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > HB2_WAIT_LIMIT_NS) break;
        }
    }
    atomicExch(err_flag, WAIT_TC_STAGING);
    return false;
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// One lane of a converged warp (used to issue the bulk copies from a warp-uniform branch).
__device__ __forceinline__ uint32_t elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred;
}
// ---- warpgroup MMA (sm_90a) ----------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, no swizzle, K-major: start>>4 @0, LBO>>4 @16 (next 16-byte core-matrix column along
// K), SBO>>4 @32 (next 8-row group along M or N).
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// generic-proxy stores to shared memory -> visible to the async proxy (the wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// keeps the compiler from moving accumulator registers across the asynchronous MMA
__device__ __forceinline__ void wg_pin(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; i++) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 128] (+)= A[64 x 8] * B[128 x 8]^T, tf32 operands from shared memory, fp32 accumulator fragment d
__device__ __forceinline__ void wg_mma_tf32_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
}
// Issues the 24 MMAs of one step, D^T[64 parents][128 patterns] = P * X^T (small terms first: Ph*Xl^T, Pl*Xh^T, then
// Ph*Xh^T; 8 K-steps each) into ONE accumulator.  pb: Ph then Pl (16 KB each, the A operand), xs: the warpgroup's X
// buffer (TC_X_BYTES, Xh then Xl, the B operand).  The caller brackets the issue with wg_fence() / wg_commit() and waits
// with wg_wait_all().
__device__ __forceinline__ void wg_issue_tf32x3(float (&d)[64], uint32_t pb, uint32_t xs) {
    const uint32_t ph = pb, pl = pb + 16384u, xh = xs, xl = xs + TC_X_BYTES / 2;
#pragma unroll
    for (int kk = 0; kk < 8; kk++) wg_mma_tf32_n128(d, wg_desc(ph + kk * 2048u, 1024u, 128u), wg_desc(xl + kk * 4096u, 2048u, 128u), kk > 0);
#pragma unroll
    for (int kk = 0; kk < 8; kk++) wg_mma_tf32_n128(d, wg_desc(pl + kk * 2048u, 1024u, 128u), wg_desc(xh + kk * 4096u, 2048u, 128u), 1u);
#pragma unroll
    for (int kk = 0; kk < 8; kk++) wg_mma_tf32_n128(d, wg_desc(ph + kk * 2048u, 1024u, 128u), wg_desc(xh + kk * 4096u, 2048u, 128u), 1u);
}
// Read-back buffer: one row of TC_D_ROW floats per pattern; within the 16-float group g of a row, position 2a + h holds
// parent 16g + a + 8h.  Accumulator fragment of warp q (of its warpgroup), lane l holds parents 16q + l/4 (+8) x
// patterns 8j + 2(l%4) (+1), j < 16: its two parents of one pattern are adjacent in that order, so each pattern takes
// one 8-byte store, and with 68-float rows a warp's stores hit every bank once per half-warp.  The reading thread
// undoes the permutation in its (compile-time) register indices: see wg_parent.
__device__ __forceinline__ void wg_store_d(float *Ds, const float (&d)[64], int q, int lane) {
    float *r0 = Ds + (size_t)(2 * (lane & 3)) * TC_D_ROW + 16 * q + 2 * (lane >> 2);
#pragma unroll
    for (int j = 0; j < 16; j++) {
        *reinterpret_cast<float2 *>(r0 + 8 * j * TC_D_ROW) = make_float2(d[4 * j], d[4 * j + 2]);
        *reinterpret_cast<float2 *>(r0 + (8 * j + 1) * TC_D_ROW) = make_float2(d[4 * j + 1], d[4 * j + 3]);
    }
}
// parent state at position x of a read-back row
__host__ __device__ constexpr int wg_parent(int x) { return (x & ~15) + ((x & 15) >> 1) + 8 * (x & 1); }
// One pattern's split row (16 chunks of hi and lo, chunk q = states 4q..4q+3) into the X buffer.
__device__ __forceinline__ void store_x_chunk(uint8_t *xs, int q, int pattern, const uint32_t *hi, const uint32_t *lo) {
    *reinterpret_cast<uint4 *>(xs + (size_t)q * 2048 + pattern * 16) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4 *>(xs + TC_X_BYTES / 2 + (size_t)q * 2048 + pattern * 16) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

// Power-of-two renormalisation of a pattern's 64 conditionals: max -> [0.5,1).  `force` = false only rescales when the
// maximum has drifted below 2^-32 (cheap guard between the children of one node); true at the end of a node.
__device__ __forceinline__ void renorm_f32(float (&v)[64], int &ex, bool force) {
    float m0 = v[0], m1 = v[1], m2 = v[2], m3 = v[3];          // four independent chains instead of one of length 64
#pragma unroll
    for (int k = 4; k < 64; k += 4) { m0 = fmaxf(m0, v[k]); m1 = fmaxf(m1, v[k + 1]); m2 = fmaxf(m2, v[k + 2]); m3 = fmaxf(m3, v[k + 3]); }
    const float m = fmaxf(fmaxf(m0, m1), fmaxf(m2, m3));
    if (m > 0.f && m < INFINITY && (force || m < 2.3283064e-10f)) {
        const int e = max((int)((__float_as_uint(m) >> 23) & 0xffu) - 126, -125);   // m = f * 2^e, f in [0.5,1) (normal m)
        if (e != 0) {
            const float sc = __uint_as_float((uint32_t)(127 - e) << 23);           // 2^-e, exact
#pragma unroll
            for (int k = 0; k < 64; k++) v[k] *= sc;
            ex += e;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Persistent "walk" kernel: the whole pruning pass of one evaluation in ONE launch.
//
// Patterns are independent, so all dependencies are tile-local: tile t of node p needs tile t of p's children only.
// CTA (c, u, r) owns rate class c, pattern UNIT u and "lane" r (one of K in-order queues of JOBS the host planner
// fills, hb2_engine.cu run_walk: a job is an internal node or the side product of a node -- all its children but the
// deepest -- kept in node slot I + n); it executes its lane's STEPS (one per child of every job) back to back.
//   * A unit is two tiles (t, t+1) or one.  The CTA has two warpgroups, one per tile of its unit; each runs the
//     per-pattern code below for its own tile, synchronised only with itself (named barriers).  Every tile of a class
//     executes the same step list, so both warpgroups need the same branch operands at every step: they share one
//     staging ring.  One CTA per SM holds 255 registers x 256 threads; while one warpgroup splits, loads or
//     renormalises, the other's MMAs (or loads) run.  In a single-tile unit warpgroup 1 idles.
//   * A child computed by another lane of the same (c, t) is awaited on the DATA ITSELF ("tags"): every job has a
//     generation bit that the host flips each time the job is re-pruned; the producer writes it into the sign bit of
//     every conditional (they are non-negative) and into bit 0 of the exponent word, and the consumer thread -- which
//     needs exactly the 17 words the producer thread of the same pattern wrote -- re-reads them until all carry the new
//     bit.  No flag, no fence, no barrier on either side; a tile is consumed one L2 round trip after it was written.
//   * A child computed by THIS CTA in the previous job (the spine of deep trees) is taken straight from registers.
//   * All K lanes of a (c,t) must be co-resident (the host guarantees grid <= resident capacity); with K == 1 there are
//     no cross-CTA waits at all and a CTA may loop over several (c,t) pairs.
//
// The pass is bound by (tree depth x per-step latency), so every operand of step i+1 is staged while step i runs:
//   * per step, the branch's fp32 P^T table (64 rows x 256 B, padded to 272 B rows) and -- for a contraction -- its
//     Ph|Pl operand tiles are bulk-copied (TMA engine, mbarrier tx completion) into a 2-stage shared-memory ring;
//     leaf column gathers and anchor rows are then shared-memory reads.  Ring slot s is released once per use by each
//     warpgroup of the unit (at its step-begin barrier, a shared-memory counter; the one warpgroup of a single-tile
//     unit counts twice) and the LAST warpgroup to release it issues the copy of the step after next into it, so the
//     staging stays a step ahead of whichever warpgroup runs behind;
//   * the unit's 32 or 64 KB conditional block of the next contraction is prefetched into L2
//     (cp.async.bulk.prefetch.L2) and the next leaf's state codes (or the awaited child's generation bit) into a register;
//   * conditionals are stored tile-wise as [16 chunks][128 patterns][4 floats] (the K-major core-matrix order), so
//     thread t's 16-byte accesses are perfectly coalesced for both the producer and the consumer of a tile.
// Step encoding: x = child id | WALK_WAIT | WALK_CHAIN | WALK_MUL ; y = job's node slot | STEP_FIRST | STEP_LAST.
// ------------------------------------------------------------------------------------------------------------------
constexpr int WALK_WAIT = 1 << 30;
constexpr int WALK_CHAIN = 1 << 29;
constexpr int WALK_MUL = 1 << 28;         // child is a side-product node (index >= I): multiply it in, no contraction
constexpr int WALK_ID_MASK = (1 << 27) - 1;
constexpr int STEP_FIRST = 1 << 28;
constexpr int STEP_LAST = 1 << 29;
constexpr int WALK_PT_ROW = TC_PTF_ROW;        // same padded rows in shared memory: one flat bulk copy stages the table
constexpr int WALK_STAGE_FLOATS = 64 * WALK_PT_ROW + 8192;     // P^T table + Ph|Pl tiles
// ring (shared), then per warpgroup an X buffer whose first TC_D_BYTES double as the accumulator read-back buffer (X is
// dead between a warpgroup's wgmma wait and its next split), then the ring's barriers and release counters
constexpr int WALK_SMEM_BYTES = 2 * WALK_STAGE_FLOATS * 4 + 2 * TC_X_BYTES + 64;
static_assert(TC_D_BYTES <= TC_X_BYTES, "the accumulator read-back buffer aliases the X (B) operand");
static_assert(WALK_SMEM_BYTES <= 232448, "one CTA per SM: the sm_90 opt-in limit per block");

struct WalkArgs {
    PruneTcArgs a;
    const int *lane_start;      // [K+1] offsets into steps
    const int2 *steps;
    const int *gen;             // [C][NI] generation bit of every job's conditionals AFTER this pass (see "tags" above)
    int K, T, ncls, nslots;
    int pairs;                  // two-tile units per class (tiles 0..2*pairs-1); the remaining T - 2*pairs tiles are units of one
    int NI;                     // node slots per class in cond/scal/gen: I real nodes + I side products
    long long *trace;           // nullable debug buffer: 12 clock64 stamps per step of CTA `trace_cta` (HB2_WALK_TRACE)
    long long *trace_cta_times; // nullable: per CTA {smid, clock64 at entry, clock64 at exit, globaltimer at entry}
    int trace_cta;
    float anchor_thr;           // entries >= this (rows are normalised to max in [0.5,1)) bypass the tensor core; default 2^-6
};

// Tagged hand-over between CTAs: relaxed gpu-scope accesses, every 32-bit word carries its own validity bit, so no
// ordering between the words (and no fence) is needed.
__device__ __forceinline__ uint4 ld_relaxed_u4(const void *p) {
    uint4 v;
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_u32(const void *p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void prefetch_l2_bulk(const void *p, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
// float4 index of chunk q of pattern t in the conditional block of (cat, node, tile)
__device__ __forceinline__ size_t cond_f4(int cat, int node, int tile, int q, int t, int I, int T) {
    return ((((size_t)cat * I + node) * T + tile) * 16 + q) * 128 + t;
}
// barrier of the 128 threads of this thread's warpgroup (named barrier 1 + tid/128; 0 is __syncthreads).  The id is
// re-read from %tid.x: the walk kernel has no register to spare for it.
__device__ __forceinline__ void wg_bar() {
    asm volatile("{\n\t.reg .u32 t;\n\tmov.u32 t, %%tid.x;\n\tshr.u32 t, t, 7;\n\tadd.u32 t, t, 1;\n\tbar.sync t, 128;\n\t}" ::"n"(0) : "memory");
}
// warp index within the warpgroup, re-read from %tid.x at the use: held in a register across a step it is spilled
__device__ __forceinline__ int warp_in_wg() {
    uint32_t q;
    asm volatile("{\n\t.reg .u32 t;\n\tmov.u32 t, %%tid.x;\n\tbfe.u32 %0, t, 5, 2;\n\t}" : "=r"(q));
    return (int)q;
}
// One warpgroup releases a ring slot (weight 1, or 2 when it is alone in its unit); true for the release that completes
// the slot's count, i.e. for the last of the two warpgroups.  The counter only grows: it is even between uses.
__device__ __forceinline__ bool ring_release(uint32_t *cnt, uint32_t weight) {
    uint32_t old;
    asm volatile("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(smem_u32(cnt)), "r"(weight) : "memory");
    return ((old + weight) & 1u) == 0u;
}

__global__ void __launch_bounds__(256, 1) prune64_tc_walk_kernel(WalkArgs w) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const PruneTcArgs &a = w.a;
    const int wg = threadIdx.x >> 7;                                                // warpgroup = tile of the unit
    float *stage_base = reinterpret_cast<float *>(smem);                           // 2 x [P^T table | Ph | Pl]
    uint8_t *Xs = smem + 2 * WALK_STAGE_FLOATS * 4 + wg * TC_X_BYTES;               // B operand: Xh | Xl
    float *Ds = reinterpret_cast<float *>(Xs);                                      // [128][TC_D_ROW] accumulator read-back
    uint64_t *bar_full = reinterpret_cast<uint64_t *>(smem + 2 * WALK_STAGE_FLOATS * 4 + 2 * TC_X_BYTES); // [2]
    uint32_t *ring_rel = reinterpret_cast<uint32_t *>(bar_full + 2);                // [2] release counters
    int *unit_info = reinterpret_cast<int *>(ring_rel + 2);   // class, first tile, tiles of the unit: read by the stager
    const int tid = threadIdx.x & 127, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
    const size_t Sp = a.Sp;
    float4 *cond4 = reinterpret_cast<float4 *>(a.cond);

    if (threadIdx.x == 0) {
        mbar_init(bar_full, 1);
        mbar_init(bar_full + 1, 1);
        ring_rel[0] = 0u;
        ring_rel[1] = 0u;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t xs_addr = smem_u32(Xs);
    uint32_t n_step = 0;                     // running counter: selects the ring stage and its barrier parity
    bool bailed = false;                     // a dependency wait timed out: stop waiting, the host reports the error

    const int r = blockIdx.x % w.K;
    const int i_begin = w.lane_start[r], i_end = w.lane_start[r + 1];
    if (w.trace_cta_times && threadIdx.x == 0) {
        uint32_t smid; unsigned long long gt;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
        long long *q = w.trace_cta_times + (size_t)blockIdx.x * 4;
        q[0] = smid; q[1] = clock64(); q[3] = (long long)gt;
    }

    // one lane of warp 3: stage the operands of one step into ring slot (m & 1): two flat bulk copies + one L2 prefetch
    // of the unit's tiles (adjacent in memory)
    auto stage_step = [&](int cat, int tile0, int ntiles, int2 st, uint32_t m) {
        const int child = st.x & WALK_ID_MASK;
        const bool internal = child >= a.L;
        float *dst = stage_base + (m & 1u) * WALK_STAGE_FLOATS;
        uint64_t *bar = bar_full + (m & 1u);
        if (st.x & WALK_MUL) {               // side product: no matrix involved; the slot's phase still has to complete
            mbar_expect_tx(bar, 0u);
            prefetch_l2_bulk(cond4 + cond_f4(cat, child - a.L, tile0, 0, 0, w.NI, w.T), 32768u * ntiles);
            return;
        }
        const size_t slot = (size_t)cat * a.B + child;
        mbar_expect_tx(bar, (uint32_t)(TC_PTF_FLOATS * 4) + (internal ? 32768u : 0u));
        bulk_g2s(dst, a.PTf + slot * TC_PTF_FLOATS, (uint32_t)(TC_PTF_FLOATS * 4), bar);
        if (internal) {
            bulk_g2s(dst + 64 * WALK_PT_ROW, a.PB + slot * TC_PB_FLOATS, 32768u, bar);
            if (!(st.x & WALK_CHAIN))      // pull the child's conditional blocks towards L2 (they may still be in DRAM)
                prefetch_l2_bulk(cond4 + cond_f4(cat, child - a.L, tile0, 0, 0, w.NI, w.T), 32768u * ntiles);
        }
    };

    // This thread's 17 words of another node's tile: 16 x 4 conditionals + the exponent word.  With `await` they are
    // re-read until every word carries generation bit `want` (sign bit / bit 0), i.e. until the producer lane of THIS
    // launch has written them; otherwise the tile is resident and its bits are whatever pass produced it.
    auto load_tile_row = [&](const float4 *xrow, const int *scp, bool await, uint32_t want, uint4 (&x4)[16], uint32_t &sc) {
#pragma unroll
        for (int q = 0; q < 16; q++) x4[q] = __ldcg(reinterpret_cast<const uint4 *>(xrow + (size_t)q * 128));
        sc = (uint32_t)__ldcg(scp);
        if (await) {
            unsigned long long t0 = 0;
            for (int it = 0; !bailed; it++) {
                uint32_t bad = (sc << 31) ^ want;
#pragma unroll
                for (int q = 0; q < 16; q++) bad |= (x4[q].x ^ want) | (x4[q].y ^ want) | (x4[q].z ^ want) | (x4[q].w ^ want);
                if (!(bad >> 31)) break;
                if ((it & 255) == 255) {                                       // never hang the GPU: time-bounded
                    const unsigned long long now = globaltimer_ns();
                    if (t0 == 0) t0 = now;
                    else if (now - t0 > HB2_WAIT_LIMIT_NS) { atomicExch(a.err, WAIT_LANE); bailed = true; }
                }
#pragma unroll
                for (int q = 0; q < 16; q++) x4[q] = ld_relaxed_u4(xrow + (size_t)q * 128);
                sc = ld_relaxed_u32(scp);
            }
        }
    };

    const int units = w.T - w.pairs;         // units per class: `pairs` of two tiles, then single tiles
    for (int ct = blockIdx.x / w.K; ct < w.ncls * units; ct += w.nslots) {
        const int cat = a.cat0 + ct / units;
        const int u = ct % units;
        const int tile0 = u < w.pairs ? 2 * u : w.pairs + u;
        const int ntiles = u < w.pairs ? 2 : 1;
        const int tile = tile0 + wg;
        const size_t s = (size_t)tile * TC_TILE_P + tid;
        float v[64];
        int ex = 0;
        if (i_begin == i_end) continue;
        int2 st = __ldg(w.steps + i_begin);
        int2 nx = (i_begin + 1 < i_end) ? __ldg(w.steps + i_begin + 1) : make_int2(0, 0);
        __syncthreads();                      // previous unit: every read of the ring and of unit_info is complete
        if (threadIdx.x == 0) { unit_info[0] = cat; unit_info[1] = tile0; unit_info[2] = ntiles; }
        __syncthreads();                      // (kept in shared memory: held in registers, they cost a spill)
        if (wg == 0 && warp == 3 && elect_one()) stage_step(cat, tile0, ntiles, st, n_step);   // an elected lane of warp 3 stages
        if (wg >= ntiles) {                   // single-tile unit: warpgroup 1 idles; its ring phases advance all the same
            n_step += (uint32_t)(i_end - i_begin);
            continue;
        }
        // fetched one step ahead: a leaf's state code, or (contractions) the generation bit the child's words must carry
        auto step_aux = [&](int2 q) -> int {
            const int ch = q.x & WALK_ID_MASK;
            if (ch < a.L) return (ch == a.forced_node) ? __ldg(a.forced + s) : __ldg(a.leaf + (size_t)ch * Sp + s);
            return (q.x & WALK_WAIT) ? __ldg(w.gen + (size_t)cat * w.NI + (ch - a.L)) : 0;
        };
        int next_code = step_aux(st);
        for (int i = i_begin; i < i_end; i++) {
            const int enc = st.x;
            const int child = enc & WALK_ID_MASK;
            const int par = st.y & WALK_ID_MASK;
            const int flags = st.y;
            const int code = next_code;
            const uint32_t tagbit = (flags & STEP_LAST) ? ((uint32_t)__ldg(w.gen + (size_t)cat * w.NI + par) << 31) : 0u;   // used at the end
            const bool has_next = (i + 1 < i_end);
            const int2 nx2 = (i + 2 < i_end) ? __ldg(w.steps + i + 2) : make_int2(0, 0);   // descriptors run two steps ahead
            const bool tr = w.trace && threadIdx.x == 0 && (int)blockIdx.x == w.trace_cta;      // warpgroup 0
            long long *trp = tr ? w.trace + (size_t)(i - i_begin) * 12 : nullptr;
            if (tr) { trp[0] = ((long long)st.x << 32) | (unsigned)st.y; trp[1] = clock64(); }
            wg_bar();                       // (1) the warpgroup is done with step i-1 (ring slot (n_step+1)&1, D rows)
            if (has_next) {
                if (warp == 3 && elect_one() && ring_release(ring_rel + ((n_step + 1) & 1u), 3u - (uint32_t)unit_info[2]))
                    stage_step(unit_info[0], unit_info[1], unit_info[2], nx, n_step + 1);
                next_code = step_aux(nx);
            }
            if ((flags & STEP_FIRST) && !(enc & WALK_CHAIN)) {
#pragma unroll
                for (int k = 0; k < 64; k++) v[k] = 1.f;
                ex = 0;
            }
            const float *tab = stage_base + (n_step & 1u) * WALK_STAGE_FLOATS;     // P^T table of this branch
            if (tr) trp[2] = clock64();
            if (child < a.L) {
                mbar_wait(bar_full + (n_step & 1u), (n_step >> 1) & 1u, a.err);
                if (tr) trp[3] = clock64();
                if (code >= 0) {
                    const float4 *row = reinterpret_cast<const float4 *>(tab + code * WALK_PT_ROW);
#pragma unroll
                    for (int q = 0; q < 16; q++) {
                        const float4 rr = row[q];
                        v[4 * q] *= rr.x; v[4 * q + 1] *= rr.y; v[4 * q + 2] *= rr.z; v[4 * q + 3] *= rr.w;
                    }
                } else {
                    float acc[64];
#pragma unroll
                    for (int k = 0; k < 64; k++) acc[k] = 0.f;
                    const double *amb = a.ambig + (size_t)(-code - 1) * 64;
                    for (int jj = 0; jj < a.D; jj++) {
                        if (__ldg(amb + jj) != 0.0) {
                            const float4 *row = reinterpret_cast<const float4 *>(tab + jj * WALK_PT_ROW);
#pragma unroll
                            for (int q = 0; q < 16; q++) {
                                const float4 rr = row[q];
                                acc[4 * q] += rr.x; acc[4 * q + 1] += rr.y; acc[4 * q + 2] += rr.z; acc[4 * q + 3] += rr.w;
                            }
                        }
                    }
#pragma unroll
                    for (int k = 0; k < 64; k++) v[k] *= acc[k];
                }
            } else if (enc & WALK_MUL) {
                // side product of this node (its other children, multiplied up by another lane or earlier in this one):
                // no matrix, just the element-wise product and the exponent.  The step's (empty) ring phase is still
                // awaited: it completes only once both warpgroups released the slot a step earlier, and that keeps this
                // warpgroup within one step of the other.  Without it a warpgroup ran through side products ahead, its
                // ring releases completed the other's count and restaged a slot the other was still reading, and its
                // parity waits two phases ahead returned at once (two-tile units whose tiles run at different speeds).
                mbar_wait(bar_full + (n_step & 1u), (n_step >> 1) & 1u, a.err);
                const int cin = child - a.L;
                const bool await = (enc & WALK_WAIT) != 0;
                uint4 x4[16];
                uint32_t sc;
                load_tile_row(cond4 + cond_f4(cat, cin, tile, 0, tid, w.NI, w.T), a.scal + ((size_t)cat * w.NI + cin) * Sp + s, await,
                              await ? ((uint32_t)code << 31) : 0u, x4, sc);
#pragma unroll
                for (int q = 0; q < 16; q++) {
                    v[4 * q] *= __uint_as_float(x4[q].x & 0x7fffffffu); v[4 * q + 1] *= __uint_as_float(x4[q].y & 0x7fffffffu);
                    v[4 * q + 2] *= __uint_as_float(x4[q].z & 0x7fffffffu); v[4 * q + 3] *= __uint_as_float(x4[q].w & 0x7fffffffu);
                }
                ex += (int)sc >> 1;
                if (tr) trp[3] = clock64();
            } else {
                const int cin = child - a.L;
                // Anchors without a serial dependency: one independent compare per element builds a 64-bit mask and
                // zeroes the element in the tensor operand; the (few) set bits are then enumerated with ffs and their
                // values re-read from the child's conditional block in L2 (the row this thread itself loaded or, on a
                // chain, stored a moment ago), eight loads in flight.
                uint32_t am0 = 0, am1 = 0, am2 = 0, am3 = 0;
                const float4 *xrow = cond4 + cond_f4(cat, cin, tile, 0, tid, w.NI, w.T);
                {
                    uint32_t hi[64], lo[64];
                    if (enc & WALK_CHAIN) {
#pragma unroll
                        for (int k = 0; k < 64; k++) {
                            float x = v[k];
                            v[k] = 1.f;
                            const bool big = x >= w.anchor_thr;
                            if (big) { if (k < 16) am0 |= 1u << k; else if (k < 32) am1 |= 1u << (k - 16); else if (k < 48) am2 |= 1u << (k - 32); else am3 |= 1u << (k - 48); }
                            x = big ? 0.f : x;
                            const float h = tf32_rn(x);
                            hi[k] = __float_as_uint(h);
                            lo[k] = __float_as_uint(x - h);
                        }
                    } else {
                        // A child produced by another lane during THIS launch is awaited on the data itself: every word
                        // must carry the generation bit of this pass (sign bit of a conditional, bit 0 of the exponent
                        // word).  Other children are resident; their bits are whatever pass produced them and are ignored.
                        const bool await = (enc & WALK_WAIT) != 0;
                        const uint32_t want = await ? ((uint32_t)code << 31) : 0u;
                        const int *scp = a.scal + ((size_t)cat * w.NI + cin) * Sp + s;
                        uint4 x4[16];
                        uint32_t sc;
                        load_tile_row(xrow, scp, await, want, x4, sc);
#pragma unroll
                        for (int q = 0; q < 16; q++) {
                            const uint32_t xs[4] = {x4[q].x, x4[q].y, x4[q].z, x4[q].w};
#pragma unroll
                            for (int u = 0; u < 4; u++) {
                                const int kq = 4 * q + u;
                                const float xv = __uint_as_float(xs[u] & 0x7fffffffu);
                                const bool big = xv >= w.anchor_thr;
                                if (big) { if (kq < 16) am0 |= 1u << kq; else if (kq < 32) am1 |= 1u << (kq - 16); else if (kq < 48) am2 |= 1u << (kq - 32); else am3 |= 1u << (kq - 48); }
                                const float x = big ? 0.f : xv;
                                const float h = tf32_rn(x);
                                hi[kq] = __float_as_uint(h);
                                lo[kq] = __float_as_uint(x - h);
                            }
                        }
                        ex += (int)sc >> 1;
                    }
                    if (tr) trp[8] = clock64();
#pragma unroll
                    for (int q = 0; q < 16; q++) store_x_chunk(Xs, q, tid, hi + 4 * q, lo + 4 * q);
                    if (tr) trp[9] = clock64();
                    fence_proxy_async();
                    if (tr) trp[10] = clock64();
                }
                unsigned long long amask = (unsigned long long)(am0 | (am1 << 16)) | ((unsigned long long)(am2 | (am3 << 16)) << 32);
                int ak[WALK_FAST_ANCHORS];
                float av[WALK_FAST_ANCHORS];
                const float *xrow_f = reinterpret_cast<const float *>(xrow);
#pragma unroll
                for (int ai = 0; ai < WALK_FAST_ANCHORS; ai++) {
                    ak[ai] = -1; av[ai] = 0.f;
                    if (amask) {
                        const int kk = __ffsll((long long)amask) - 1;
                        amask &= amask - 1;
                        ak[ai] = kk;
                        av[ai] = __ldcg(xrow_f + ((size_t)(kk >> 2) * 128) * 4 + (kk & 3));   // sign bit = tag: stripped at the use, so the load stays in flight
                    }
                }
                if (tr) trp[3] = clock64();
                wg_bar();                  // (2) X operand complete in shared memory
                if (tr) trp[4] = clock64();
                // 24 wgmma (Ph*Xl^T, Pl*Xh^T, Ph*Xh^T; 8 K-steps of 8 each) into one accumulator, issued by the whole
                // warpgroup once the branch's operands have landed
                mbar_wait(bar_full + (n_step & 1u), (n_step >> 1) & 1u, a.err);
                if (tr) trp[5] = clock64();
                float d[64];
                wg_fence();
                wg_issue_tf32x3(d, smem_u32(tab + 64 * WALK_PT_ROW), xs_addr);
                wg_commit();
                // anchors on the CUDA cores while the tensor core works (rows of the P^T table in shared memory)
                float acc[64];
                {   // first anchor (nearly every row has one: its maximum is >= 0.5): a product, no zero-fill + FMA
                    const float xv = ak[0] >= 0 ? fabsf(av[0]) : 0.f;
                    const float4 *row = reinterpret_cast<const float4 *>(tab + max(ak[0], 0) * WALK_PT_ROW);
#pragma unroll
                    for (int q = 0; q < 16; q++) {
                        const float4 rr = row[q];
                        acc[4 * q] = xv * rr.x; acc[4 * q + 1] = xv * rr.y; acc[4 * q + 2] = xv * rr.z; acc[4 * q + 3] = xv * rr.w;
                    }
                }
#pragma unroll
                for (int ai = 1; ai < WALK_FAST_ANCHORS; ai++) {
                    if (ak[ai] >= 0) {
                        const float xv = fabsf(av[ai]);
                        const float4 *row = reinterpret_cast<const float4 *>(tab + ak[ai] * WALK_PT_ROW);
#pragma unroll
                        for (int q = 0; q < 16; q++) {
                            const float4 rr = row[q];
                            acc[4 * q] = fmaf(xv, rr.x, acc[4 * q]); acc[4 * q + 1] = fmaf(xv, rr.y, acc[4 * q + 1]);
                            acc[4 * q + 2] = fmaf(xv, rr.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(xv, rr.w, acc[4 * q + 3]);
                        }
                    }
                }
                while (amask) {                  // more than WALK_FAST_ANCHORS entries above the threshold (diffuse vectors): rare
                    const int kk = __ffsll((long long)amask) - 1;
                    amask &= amask - 1;
                    const float xv = fabsf(__ldcg(xrow_f + ((size_t)(kk >> 2) * 128) * 4 + (kk & 3)));
                    const float4 *row = reinterpret_cast<const float4 *>(tab + kk * WALK_PT_ROW);
#pragma unroll
                    for (int q = 0; q < 16; q++) {
                        const float4 rr = row[q];
                        acc[4 * q] = fmaf(xv, rr.x, acc[4 * q]); acc[4 * q + 1] = fmaf(xv, rr.y, acc[4 * q + 1]);
                        acc[4 * q + 2] = fmaf(xv, rr.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(xv, rr.w, acc[4 * q + 3]);
                    }
                }
                wg_wait_all();
                wg_pin(d);
                if (tr) trp[6] = clock64();
                wg_bar();                  // every warp's MMAs are complete: X is dead and D may overwrite it
                wg_store_d(Ds, d, warp_in_wg(), lane);
                wg_bar();                  // (3) every row of D is in the read-back buffer
                {
                    const float4 *drow = reinterpret_cast<const float4 *>(Ds + (size_t)tid * TC_D_ROW);
#pragma unroll
                    for (int q = 0; q < 16; q++) {
                        const float4 dd = drow[q];
                        const int k0 = wg_parent(4 * q), k1 = wg_parent(4 * q + 1), k2 = wg_parent(4 * q + 2), k3 = wg_parent(4 * q + 3);
                        v[k0] *= (dd.x + acc[k0]); v[k1] *= (dd.y + acc[k1]);
                        v[k2] *= (dd.z + acc[k2]); v[k3] *= (dd.w + acc[k3]);
                    }
                }
            }
            // Pinned internal node: only the forced state survives.  Masked after every step of the node and of its side product
            // (slot I + n), not only at its end: renorm_f32 then follows the forced state itself.  Masked at the end only, a
            // forced state far less likely than the node's best one fell below the fp32 range on a node with many children.
            if (a.forced_node >= a.L && a.L + (par >= a.I ? par - a.I : par) == a.forced_node) {
                const int f = __ldg(a.forced + s);
#pragma unroll
                for (int k = 0; k < 64; k++) if (k != f) v[k] = 0.f;
            }
            renorm_f32(v, ex, (flags & STEP_LAST) != 0);
            n_step++;
            if (flags & STEP_LAST) {
                // this tile of the parent: conditionals and exponent, every word tagged with the node's generation bit
                // (consumers in other lanes poll the data itself: no flag, no fence, no barrier); root reduction
                float4 *outp = cond4 + cond_f4(cat, par, tile, 0, tid, w.NI, w.T);
#pragma unroll
                for (int q = 0; q < 16; q++)
                    __stcg(reinterpret_cast<uint4 *>(outp + (size_t)q * 128),
                           make_uint4(__float_as_uint(v[4 * q]) | tagbit, __float_as_uint(v[4 * q + 1]) | tagbit,
                                      __float_as_uint(v[4 * q + 2]) | tagbit, __float_as_uint(v[4 * q + 3]) | tagbit));
                __stcg(a.scal + ((size_t)cat * w.NI + par) * Sp + s, (int)(((uint32_t)ex << 1) | (tagbit >> 31)));
                if (par == a.I - 1) {
                    double rr = 0.0;
#pragma unroll
                    for (int k = 0; k < 64; k++) rr = fma((double)v[k], a.pi[k], rr);
                    a.rootL[(size_t)cat * Sp + s] = rr;
                    a.rootE[(size_t)cat * Sp + s] = ex;
                }
            }
            if (tr) trp[7] = clock64();
            st = nx;
            nx = nx2;
        }
    }
    if (w.trace_cta_times && threadIdx.x == 0) w.trace_cta_times[(size_t)blockIdx.x * 4 + 2] = clock64();
}

}  // namespace hb2

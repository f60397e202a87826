// Microbenchmark: the tensor walk kernel's contraction step on one SM in two wgmma shapes (hb2_kernels_tc.cuh).
//   n64:  X as A, P as B: 2 halves x 3 products x 8 k-steps of m64n64k8 per warpgroup (the kernel before the transpose)
//   n128: P as A, X as B: 3 products x 8 k-steps of m64n128k8 per warpgroup (wg_issue_tf32x3, what the kernel runs)
// Operands are the kernel's own buffers in the canonical no-swizzle K-major layout: a 64 KB Xh|Xl buffer per warpgroup
// and one shared 32 KB Ph|Pl tile.  One CTA on one SM; one or two warpgroups issue a whole step's sequence at once
// (fence .. commit .. wait_group 0), timed with clock64 per warpgroup and sequence.  With "load", two further
// warpgroups stream 16-byte shared-memory loads and stores back to back for as long as the MMAs run: the most
// shared-memory traffic the kernel's split, anchor and read-back phases can put beside the MMAs.
// Numerics: one random non-negative X and P, split hi/lo as the kernel does, contracted in both shapes (the n128
// result read back through the kernel's wg_store_d / wg_parent), compared bitwise and against fp64.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/mb_wgmma tools/microbench_wgmma_shape.cu
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../hyphy_b200/csrc/hb2_kernels_tc.cuh"

using namespace hb2;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

// the m64n64k8 shape with X as the A operand
__device__ __forceinline__ void mma_n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void issue_n64(float (&d)[32], uint32_t xs, uint32_t pb, int m) {
    const uint32_t xh = xs + (uint32_t)m * 1024u, xl = xh + TC_X_BYTES / 2, ph = pb, pl = pb + 16384u;
#pragma unroll
    for (int kk = 0; kk < 8; kk++) mma_n64(d, wg_desc(xl + kk * 4096u, 2048u, 128u), wg_desc(ph + kk * 2048u, 1024u, 128u), kk > 0);
#pragma unroll
    for (int kk = 0; kk < 8; kk++) mma_n64(d, wg_desc(xh + kk * 4096u, 2048u, 128u), wg_desc(pl + kk * 2048u, 1024u, 128u), 1u);
#pragma unroll
    for (int kk = 0; kk < 8; kk++) mma_n64(d, wg_desc(xh + kk * 4096u, 2048u, 128u), wg_desc(ph + kk * 2048u, 1024u, 128u), 1u);
}
__device__ __forceinline__ void pin32(float (&d)[32]) {
#pragma unroll
    for (int i = 0; i < 32; i++) asm volatile("" : "+f"(d[i])::"memory");
}

constexpr int SM_X = 0;                       // 2 x TC_X_BYTES
constexpr int SM_P = 2 * TC_X_BYTES;          // 32 KB Ph|Pl
constexpr int SM_LOAD = SM_P + 32768;         // 2 x 16 KB scratch of the load warpgroups
constexpr int SM_FLAG = SM_LOAD + 32768;
constexpr int SM_BYTES = SM_FLAG + 16;

// X: [2][16][128][4] (Xh, Xl) floats, P: [2][16][64][4] (Ph, Pl); D: [2 warpgroups][128 patterns][64 parents];
// t: [reps][2 warpgroups][2] clock64 stamps; sink: load iterations (keeps the load loop alive)
__global__ void __launch_bounds__(512, 1) shape_kernel(const float *X, const float *P, float *D, long long *t, int *sink,
                                                       int shape, int nwg, int load, int reps) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127, warp = tid >> 5, lane = tid & 31;
    volatile int *flag = reinterpret_cast<volatile int *>(smem + SM_FLAG);
    for (int i = threadIdx.x; i < 2 * 16 * 128 * 4; i += 512) {
        reinterpret_cast<float *>(smem + SM_X)[i] = X[i];
        reinterpret_cast<float *>(smem + SM_X + TC_X_BYTES)[i] = X[i];
    }
    for (int i = threadIdx.x; i < 8192; i += 512) reinterpret_cast<float *>(smem + SM_P)[i] = P[i];
    if (threadIdx.x == 0) *flag = 0;
    fence_proxy_async();
    __syncthreads();
    if (wg < nwg) {
        const uint32_t xs = smem_u32(smem + SM_X + wg * TC_X_BYTES), pb = smem_u32(smem + SM_P);
        float *Ds = reinterpret_cast<float *>(smem + SM_X + wg * TC_X_BYTES);
        if (shape == 128) {
            float d[64];
            for (int r = 0; r < reps; r++) {
                asm volatile("bar.sync 1, %0;" ::"r"(nwg * 128) : "memory");
                const long long t0 = clock64();
                wg_fence();
                wg_issue_tf32x3(d, pb, xs);
                wg_commit();
                wg_wait_all();
                wg_pin(d);
                const long long t1 = clock64();
                if (tid == 0) { t[(r * 2 + wg) * 2] = t0; t[(r * 2 + wg) * 2 + 1] = t1; }
            }
            asm volatile("bar.sync 1, %0;" ::"r"(nwg * 128) : "memory");
            wg_store_d(Ds, d, warp, lane);
            asm volatile("bar.sync 1, %0;" ::"r"(nwg * 128) : "memory");
            for (int x = 0; x < 64; x++) D[((size_t)wg * 128 + tid) * 64 + wg_parent(x)] = Ds[tid * TC_D_ROW + x];
        } else {
            float d0[32], d1[32];
            for (int r = 0; r < reps; r++) {
                asm volatile("bar.sync 1, %0;" ::"r"(nwg * 128) : "memory");
                const long long t0 = clock64();
                wg_fence();
                issue_n64(d0, xs, pb, 0);
                issue_n64(d1, xs, pb, 1);
                wg_commit();
                wg_wait_all();
                pin32(d0);
                pin32(d1);
                const long long t1 = clock64();
                if (tid == 0) { t[(r * 2 + wg) * 2] = t0; t[(r * 2 + wg) * 2 + 1] = t1; }
            }
            // fragment: rows (patterns) 16q + l/4 (+8), columns (parents) 8j + 2(l%4) (+1)
            for (int h = 0; h < 2; h++) {
                const float *d = h ? d1 : d0;
                const int p = 64 * h + 16 * warp + (lane >> 2);
                for (int j = 0; j < 8; j++) {
                    const int c = 8 * j + 2 * (lane & 3);
                    float *o = D + ((size_t)wg * 128 + p) * 64 + c;
                    o[0] = d[4 * j]; o[1] = d[4 * j + 1]; o[8 * 64] = d[4 * j + 2]; o[8 * 64 + 1] = d[4 * j + 3];
                }
            }
        }
        asm volatile("bar.sync 1, %0;" ::"r"(nwg * 128) : "memory");
        if (threadIdx.x == 0) *flag = 1;
    } else if (wg >= 2 && load) {
        uint8_t *buf = smem + SM_LOAD + (wg - 2) * 16384;
        const uint32_t base = smem_u32(buf);
        int n = 0;
        while (!*flag) {
#pragma unroll
            for (int i = 0; i < 8; i++) {
                uint32_t a0, a1, a2, a3;
                const uint32_t src = base + ((i * 128 + tid) & 1023) * 16, dst = base + (((i + 4) * 128 + tid) & 1023) * 16;
                asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a0), "=r"(a1), "=r"(a2), "=r"(a3) : "r"(src) : "memory");
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(dst), "r"(a0 + 1), "r"(a1), "r"(a2), "r"(a3) : "memory");
            }
            n++;
        }
        if (tid == 0) sink[wg - 2] = n;
    }
}

static float tf32_rn_host(float x) {
    uint32_t u;
    memcpy(&u, &x, 4);
    u = (u + 0x1000u) & 0xFFFFE000u;
    float r;
    memcpy(&r, &u, 4);
    return r;
}

struct Stats { double med, p10, p90, mn, mx; };
static Stats stats(std::vector<double> v) {
    std::sort(v.begin(), v.end());
    const size_t n = v.size();
    return {v[n / 2], v[n / 10], v[(9 * n) / 10], v.front(), v.back()};
}

int main(int argc, char **argv) {
    const int reps = argc > 1 ? atoi(argv[1]) : 2000, skip = 20;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    int clk_khz = 0;
    CK(cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0));
    printf("device: %s, %d SMs, max SM clock %.0f MHz\n", prop.name, prop.multiProcessorCount, clk_khz / 1000.0);

    // X: diffuse rows below the anchor threshold (what the tensor core sees); P: row-stochastic
    srand(12345);
    auto u01 = [] { return (rand() + 0.5) / ((double)RAND_MAX + 1.0); };
    std::vector<float> x(128 * 64), p(64 * 64);
    for (auto &e : x) { const double r = u01(); e = (float)(r * r * r * 0.015625); }
    for (int n = 0; n < 64; n++) {
        double s = 0;
        for (int k = 0; k < 64; k++) { p[n * 64 + k] = (float)(u01() * u01()); s += p[n * 64 + k]; }
        for (int k = 0; k < 64; k++) p[n * 64 + k] = (float)(p[n * 64 + k] / s);
    }
    std::vector<float> xb(2 * 8192), pbuf(8192);
    std::vector<float> xh(128 * 64), xl(128 * 64), ph(64 * 64), pl(64 * 64);
    for (int s = 0; s < 128; s++)
        for (int k = 0; k < 64; k++) {
            const float v = x[s * 64 + k], h = tf32_rn_host(v);
            xh[s * 64 + k] = h; xl[s * 64 + k] = v - h;
            xb[(k >> 2) * 512 + s * 4 + (k & 3)] = h;
            xb[8192 + (k >> 2) * 512 + s * 4 + (k & 3)] = v - h;
        }
    for (int n = 0; n < 64; n++)
        for (int k = 0; k < 64; k++) {
            const float v = p[n * 64 + k], h = tf32_rn_host(v);
            ph[n * 64 + k] = h; pl[n * 64 + k] = tf32_rn_host(v - h);
            pbuf[(k >> 2) * 256 + n * 4 + (k & 3)] = h;
            pbuf[4096 + (k >> 2) * 256 + n * 4 + (k & 3)] = tf32_rn_host(v - h);
        }

    float *dX, *dP, *dD;
    long long *dT;
    int *dSink;
    CK(cudaMalloc(&dX, xb.size() * 4));
    CK(cudaMalloc(&dP, pbuf.size() * 4));
    CK(cudaMalloc(&dD, 2 * 128 * 64 * 4));
    CK(cudaMalloc(&dT, (size_t)reps * 4 * 8));
    CK(cudaMalloc(&dSink, 8));
    CK(cudaMemcpy(dX, xb.data(), xb.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dP, pbuf.data(), pbuf.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaFuncSetAttribute(shape_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_BYTES));

    printf("\ncycles per warpgroup and step (3 x 128 x 64 x 64 = 1 572 864 FMA), %d sequences after %d warm-up\n", reps - skip, skip);
    printf("%-6s %-4s %-5s | %8s %8s %8s %8s %8s | %10s | %s\n", "shape", "wgs", "load", "median", "p10", "p90", "min", "max",
           "span med", "FMA/clk/SM");
    double med_wg2[2] = {0, 0};
    std::vector<float> D64(2 * 128 * 64), D128(2 * 128 * 64);
    for (int shape : {64, 128})
        for (int nwg : {1, 2})
            for (int load : {0, 1}) {
                CK(cudaMemset(dT, 0, (size_t)reps * 4 * 8));
                shape_kernel<<<1, 512, SM_BYTES>>>(dX, dP, dD, dT, dSink, shape, nwg, load, reps);
                CK(cudaGetLastError());
                CK(cudaDeviceSynchronize());
                std::vector<long long> t((size_t)reps * 4);
                CK(cudaMemcpy(t.data(), dT, t.size() * 8, cudaMemcpyDeviceToHost));
                std::vector<double> per, span;
                for (int r = skip; r < reps; r++) {
                    long long b = t[r * 4], e = t[r * 4 + 1];
                    per.push_back((double)(t[r * 4 + 1] - t[r * 4]));
                    if (nwg == 2) {
                        per.push_back((double)(t[r * 4 + 3] - t[r * 4 + 2]));
                        b = std::min(b, t[r * 4 + 2]); e = std::max(e, t[r * 4 + 3]);
                    }
                    span.push_back((double)(e - b));
                }
                const Stats s = stats(per), sp = stats(span);
                printf("%-6s %-4d %-5s | %8.0f %8.0f %8.0f %8.0f %8.0f | %10.0f | %.0f\n", shape == 64 ? "n64" : "n128", nwg,
                       load ? "yes" : "no", s.med, s.p10, s.p90, s.mn, s.mx, sp.med, nwg * 1572864.0 / sp.med);
                if (nwg == 2 && load) med_wg2[shape == 128] = sp.med;
                if (nwg == 2 && !load) CK(cudaMemcpy(shape == 64 ? D64.data() : D128.data(), dD, D64.size() * 4, cudaMemcpyDeviceToHost));
            }

    // numerics: both warpgroups contracted the same operands; compare shapes bitwise and against fp64
    int same = 0, wg_same = 0;
    double e64_split = 0, e128_split = 0, e64_exact = 0, e128_exact = 0;
    for (int s = 0; s < 128; s++)
        for (int n = 0; n < 64; n++) {
            double split = 0, exact = 0;
            for (int k = 0; k < 64; k++) {
                split += (double)xl[s * 64 + k] * ph[n * 64 + k] + (double)xh[s * 64 + k] * pl[n * 64 + k] + (double)xh[s * 64 + k] * ph[n * 64 + k];
                exact += (double)x[s * 64 + k] * p[n * 64 + k];
            }
            const float a = D64[s * 64 + n], b = D128[s * 64 + n];
            same += memcmp(&a, &b, 4) == 0;
            wg_same += memcmp(&D128[s * 64 + n], &D128[8192 + s * 64 + n], 4) == 0 && memcmp(&D64[s * 64 + n], &D64[8192 + s * 64 + n], 4) == 0;
            e64_split = std::max(e64_split, std::fabs(a - split) / split);
            e128_split = std::max(e128_split, std::fabs(b - split) / split);
            e64_exact = std::max(e64_exact, std::fabs(a - exact) / exact);
            e128_exact = std::max(e128_exact, std::fabs(b - exact) / exact);
        }
    printf("\nnumerics (128 x 64 outputs): n64 vs n128 bit-identical %d / 8192; both warpgroups identical %d / 8192\n", same, wg_same);
    printf("  max rel. error vs fp64 of the 3 split products: n64 %.3e, n128 %.3e\n", e64_split, e128_split);
    printf("  max rel. error vs fp64 of X * P^T:              n64 %.3e, n128 %.3e\n", e64_exact, e128_exact);
    printf("\ngate (two warpgroups, with load, median step span): n64 %.0f, n128 %.0f cycles -> %s\n", med_wg2[0], med_wg2[1],
           med_wg2[1] < med_wg2[0] ? "n128 faster: PASS" : "n128 not faster: FAIL");
    return 0;
}

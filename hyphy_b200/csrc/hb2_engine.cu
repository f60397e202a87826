// hb2_engine.cu -- C++ host side of libhyphy_b200.so: the C ABI of include/hyphy_b200.h over the CUDA kernels.
//
// Mirrors, for one partition, what the reference does inside _LikelihoodFunction::ComputeBlock
// (likefunc.cpp:10783-11289): keep the per-node caches resident (here: in HBM), take the changed matrices,
// re-exponentiate them, re-prune the dirty part of the tree, reduce at the root, hand back one double.
// No CPU fallback exists on this path: every failure is an error code (fatal for the host).
#include "../../include/hyphy_b200.h"
#include "hb2_kernels_fp64.cuh"
#include "hb2_kernels_tc.cuh"
#include "hb2_kernels_lanes.cuh"

#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <dlfcn.h>
#include <string>
#include <vector>
#include <algorithm>
#include <memory>
#include <mutex>
#include <unordered_map>
#include <type_traits>
#include <utility>

#include <nccl.h>

namespace {

thread_local std::string g_err;

int fail(const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return 1;
}

#define CU(x)                                                                                         \
    do {                                                                                              \
        cudaError_t e_ = (x);                                                                         \
        if (e_ != cudaSuccess) return fail("%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

// The error of a device-side wait that timed out, from the code it left in the partition's error flag (hb2::WaitCode).
int wait_timeout(int code) {
    const char *what = code == hb2::WAIT_TC_STAGING ? "operand staging / tensor pipe"
                       : code == hb2::WAIT_LANE ? "another lane's conditionals"
                       : code == hb2::WAIT_PEER ? "a peer rank's partials"
                       : code == hb2::WAIT_EXPM_POWERS ? "a coefficient matrix of the shared-powers exponential"
                       : "unknown wait";
    return fail("a device-side wait timed out (code %d: %s)", code, what);
}

// ---- Block pool for device and pinned-host memory ----------------------------------------------------------------------
// The site phases of FEL / MEME create and destroy one small likelihood function per site (SURVEY 8f row 3): through the
// patched host that is one hb2_create / hb2_destroy pair each, i.e. ~60 cudaMalloc / cudaMallocHost and as many frees (each
// cudaFree synchronises the device).  Blocks up to 32 MB are rounded up to a power of two and recycled through a
// process-wide free list per device (caps: 1 GB device, 256 MB pinned); larger blocks go straight to the runtime.
// Recycled memory is NOT zero: every buffer whose initial contents matter is cleared explicitly at hb2_create, as it
// always had to be (cudaMalloc gives no such guarantee either).  HB2_POOL=0 switches the pool off.
struct BlockPool {
    struct Info { size_t cls; int dev; bool host; };
    std::mutex mu;
    std::unordered_map<void *, Info> live;
    std::unordered_map<unsigned long long, std::vector<void *>> free_blocks;      // key = (host, device, class)
    size_t pooled_dev = 0, pooled_host = 0;
    static constexpr size_t kMaxClass = (size_t)32 << 20, kDevCap = (size_t)1 << 30, kHostCap = (size_t)256 << 20;
    bool enabled() { static const bool on = !(getenv("HB2_POOL") && getenv("HB2_POOL")[0] == '0'); return on; }
    static size_t size_class(size_t n) { size_t c = 256; while (c < n) c <<= 1; return c; }
    static unsigned long long key(bool host, int dev, size_t cls) { return ((unsigned long long)host << 63) | ((unsigned long long)(dev & 0xff) << 52) | (unsigned long long)cls; }
    cudaError_t alloc(void **p, size_t n, bool host) {
        if (!enabled() || n > kMaxClass) return host ? cudaMallocHost(p, n) : cudaMalloc(p, n);
        int dev = 0;
        cudaGetDevice(&dev);
        const size_t cls = size_class(n);
        {
            std::lock_guard<std::mutex> lk(mu);
            auto it = free_blocks.find(key(host, host ? 0 : dev, cls));
            if (it != free_blocks.end() && !it->second.empty()) {
                *p = it->second.back();
                it->second.pop_back();
                (host ? pooled_host : pooled_dev) -= cls;
                live[*p] = Info{cls, dev, host};
                return cudaSuccess;
            }
        }
        const cudaError_t e = host ? cudaMallocHost(p, cls) : cudaMalloc(p, cls);
        if (e == cudaSuccess) { std::lock_guard<std::mutex> lk(mu); live[*p] = Info{cls, dev, host}; }
        return e;
    }
    cudaError_t release(void *p, bool host) {
        if (!p) return cudaSuccess;
        {
            std::lock_guard<std::mutex> lk(mu);
            auto it = live.find(p);
            if (it != live.end()) {
                const Info in = it->second;
                live.erase(it);
                size_t &pooled = in.host ? pooled_host : pooled_dev;
                if (pooled + in.cls <= (in.host ? kHostCap : kDevCap)) {
                    free_blocks[key(in.host, in.host ? 0 : in.dev, in.cls)].push_back(p);
                    pooled += in.cls;
                    return cudaSuccess;
                }
            }
        }
        return host ? cudaFreeHost(p) : cudaFree(p);
    }
};
BlockPool g_pool;

// Owner of one pool block of n elements of T: device memory, or pinned host memory when Pinned.  Every block of this file
// is held by one, except the peer-exchange buffer, which is exported through CUDA IPC and never pooled.  alloc() and the
// destructor return the block held so far to the pool, which may hand it out again at once: no work queued on any stream
// may still use it by then.
template <typename T, bool Pinned>
class PoolBuffer {
    T *ptr_ = nullptr;
    size_t n_ = 0;
public:
    PoolBuffer() = default;
    PoolBuffer(PoolBuffer &&o) noexcept : ptr_(std::exchange(o.ptr_, nullptr)), n_(std::exchange(o.n_, 0)) {}
    PoolBuffer &operator=(PoolBuffer &&o) noexcept {
        if (this != &o) { g_pool.release(ptr_, Pinned); ptr_ = std::exchange(o.ptr_, nullptr); n_ = std::exchange(o.n_, 0); }
        return *this;
    }
    ~PoolBuffer() { g_pool.release(ptr_, Pinned); }
    // On failure the owner is left empty.
    int alloc(size_t n) {
        g_pool.release(ptr_, Pinned);
        ptr_ = nullptr; n_ = 0;
        void *q = nullptr;
        const cudaError_t e = g_pool.alloc(&q, n * sizeof(T), Pinned);
        if (e != cudaSuccess) return fail("allocating %zu bytes of %s memory failed: %s", n * sizeof(T), Pinned ? "pinned" : "device", cudaGetErrorString(e));
        ptr_ = static_cast<T *>(q); n_ = n;
        return 0;
    }
    // Grows the block to at least n elements; its contents are not kept.  Work queued on `stream` may still use the old
    // block, so the stream is synchronised before it goes back to the pool.
    int reserve(size_t n, cudaStream_t stream) {
        if (n <= n_) return 0;
        CU(cudaStreamSynchronize(stream));
        return alloc(n);
    }
    size_t size() const { return n_; }
    // Clears all n elements on `stream` (device buffers).
    int zero(cudaStream_t stream) {
        CU(cudaMemsetAsync(ptr_, 0, n_ * sizeof(T), stream));
        return 0;
    }
    operator T *() const { return ptr_; }
};
template <typename T> using DeviceBuffer = PoolBuffer<T, false>;
template <typename T> using PinnedBuffer = PoolBuffer<T, true>;

// ---- NCCL through dlopen: single-GPU users never need the library -------------------------------
struct NcclApi {
    void *h = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    bool load() {
        if (h) return true;
        const char *names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char *n : names) {
            h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (h) break;
        }
        if (!h) return false;
        GetUniqueId = (decltype(GetUniqueId))dlsym(h, "ncclGetUniqueId");
        CommInitRank = (decltype(CommInitRank))dlsym(h, "ncclCommInitRank");
        AllReduce = (decltype(AllReduce))dlsym(h, "ncclAllReduce");
        AllGather = (decltype(AllGather))dlsym(h, "ncclAllGather");
        CommDestroy = (decltype(CommDestroy))dlsym(h, "ncclCommDestroy");
        GetErrorString = (decltype(GetErrorString))dlsym(h, "ncclGetErrorString");
        return GetUniqueId && CommInitRank && AllReduce && AllGather && CommDestroy && GetErrorString;
    }
} g_nccl;

int pad_states(int64_t D) {
    if (D <= 4) return 4;
    if (D <= 8) return 8;
    if (D <= 16) return 16;
    if (D <= 24) return 24;
    if (D <= 32) return 32;
    if (D <= 64) return 64;
    return -1;
}

// What a hand-over entry holds: a rate or a transition matrix (the ABI's HB2_MATRIX_* values), or a compiled template's
// formula values.
enum class Kind : signed char { Rate = HB2_MATRIX_RATE, Trans = HB2_MATRIX_TRANS, Compiled = 2 };

// Input of one expm launch: its kind and, for compiled input, the template.
struct Source {
    Kind kind;
    int tmpl = 0;
};

// Matrices handed over since the last flush: entries [0, n) are rows of `row` doubles (D*D matrix entries, or a template's
// formula values), each with its destination slot (-1: retired) and kind.  The pinned rows and slots are uploaded at the
// flush.
struct HandoverQueue {
    int64_t n = 0, cap = 0, row = 0;
    PinnedBuffer<double> h_rows;
    PinnedBuffer<int> h_dst;
    DeviceBuffer<double> d_rows;
    DeviceBuffer<int> d_dst;
    std::vector<Kind> kind;
    int alloc(int64_t cap_, int64_t row_) {
        n = 0; cap = 0; row = row_;
        kind.assign(cap_, Kind::Rate);
        if (h_rows.alloc(cap_ * row_) || h_dst.alloc(cap_) || d_rows.alloc(cap_ * row_) || d_dst.alloc(cap_)) return 1;
        cap = cap_;
        return 0;
    }
};
constexpr int DENSE_QUEUE = -1;               // queue id of the dense queue; a template's compiled queue has the template id

// Where the resident copy of a slot's last matrix is kept (hb2_time_resident replays from it; the classification of the
// shared-powers path compares against it).
enum class Resident : signed char { None, DenseQ, Formula };   // none, dense Q in d_Qres, formula values in a template's d_Vres

// One (class, branch) slot.  A slot handed over again before a flush overwrites its pending entry in place when the new one
// joins the same queue and retires it otherwise (last one wins, like the reference's SetCompExp, calcnode.cpp:714), so one
// expm launch never holds two CTAs with the same destination and the flush order of the queues cannot matter.
struct Slot {
    bool have = false;                        // a matrix was staged or launched (another class group's: handed over)
    Resident res = Resident::None;
    signed char res_tmpl = 0;                 // template whose d_Vres holds the formula values (res == Formula)
    signed char queue = DENSE_QUEUE;          // queue of the pending entry
    int entry = -1;                           // index of the pending entry in that queue, -1 none
};

// Shape of a batch call (batch_shape).
struct BatchShape {
    std::vector<int> row_off;                 // branch b of a set owns component rows row_off[b] .. row_off[b+1]-1
    int64_t R = 0, nF = 0, gk = 0, sets = 0;  // rows per set, formula values per row, groups per set; sets per chunk
    int64_t mat = 4096, vec = 64;             // doubles per P matrix (Dp^2) and per node vector (Dp)
    int64_t ent = 0, in = 0;                  // rows per set through launch_expm (R; 0 for site rates) and input doubles per set
    int64_t side = 0;                         // branches per set with outside scratch (branch rows, leaf support: B; else 0)
    int64_t rows = 0, sup = 0;                // doubles per set of row results (branch rows: R) and of support (leaf support: L*D)
    int64_t joint = 0;                        // internal nodes per set with an argument row and a state (joint ancestors: I)
};

}  // namespace

struct hb2_partition {
    int device = 0, flags = 0;
    cudaStream_t stream = nullptr;
    int64_t S = 0, D = 0, L = 0, I = 0, C = 0, B = 0, nAmb = 0;
    int Dp = 0;
    int64_t Sp = 0;
    std::vector<int64_t> parents;
    std::vector<std::vector<int>> children;   // per internal node, flat ids
    std::vector<int> height;                  // per internal node: 0 = only leaf children
    // device
    DeviceBuffer<int> d_leaf, d_scal, d_rootE, d_child_start, d_child_ids, d_jobs, d_flag;
    DeviceBuffer<double> d_ambig, d_freq, d_cond, d_PT, d_pi, d_rootL, d_weights, d_partial, d_lnL, d_siteL;
    DeviceBuffer<long long> d_siteScale;
    // pinned host staging
    PinnedBuffer<double> h_small;             // pi (Dp) + weights (C) + lnL (1)
    PinnedBuffer<int> h_jobs;
    HandoverQueue dense;                      // dense matrices, one per slot (its d_dst also carries hb2_time_resident's slots)
    std::vector<Slot> slots;                  // [C*B]
    DeviceBuffer<double> d_Qres;              // [C][B][D*D] last rate matrices, resident copy
    // explicit-form mixtures (hb2_set_mixture_matrices): own staging so that nothing is shared with the plain queues
    DeviceBuffer<double> d_mix_scratch, d_mix_Q;   // [cap][Dp*Dp], [cap][D*D] | [cap] weights
    PinnedBuffer<double> h_mix;                    // as d_mix_Q, then 2 cap ints
    DeviceBuffer<int> d_mix_dst;
    // shared-powers expm (64 padded states, hb2_kernels_fp64.cuh "Shared powers"): group = rate class (plain batches) or
    // C + mixture component; per-entry arrays are indexed like the batch
    struct ExBuf {
        int G = 0, stride = 0;                // groups, doubles per cached reference direction
        DeviceBuffer<int> d_int, d_flag;      // d_int: [group cap | ref cap | refs G]
        PinnedBuffer<int> h_int;
        DeviceBuffer<double> d_weight, d_pow, d_refvec;
        DeviceBuffer<hb2::ExpmGroup> d_groups;
        DeviceBuffer<unsigned long long> d_flags;   // generation flags of the coefficient matrices [G][EXPM_POW_TERMS]
        unsigned long long gen = 0;
        std::vector<int> kind;                // host mirror: kind of the reference direction each group holds (0 none)
        int64_t cap = 0;
        // (Re)allocates the buffers for G_ groups and cap_ entries, with no cached direction.
        int alloc(int G_, int64_t cap_, cudaStream_t stream) {
            G = G_; cap = cap_; stride = 4096; gen = 0;
            kind.assign(G, 0);
            return d_int.alloc(2 * cap + G) || h_int.alloc(2 * cap + G) || d_flag.alloc(cap) || d_weight.alloc(cap) ||
                   d_groups.alloc(G) || d_groups.zero(stream) ||
                   d_pow.alloc((size_t)G * hb2::EXPM_POW_TERMS * 4096) || d_flags.alloc((size_t)G * hb2::EXPM_POW_TERMS) ||
                   d_flags.zero(stream) || d_refvec.alloc((size_t)G * stride);
        }
    };
    ExBuf ex;                                 // the partition's own hand-overs
    // Workspace of the batch entry points (hb2_batch_*) for one chunk of `sets` sets: the chunk's P area holds its sets'
    // R rows in [set][row] order; the rows that go through launch_expm are its entries, entry e going to slot e.  The batch
    // calls stage their own root vector, so the staged d_pi stays the evaluations'.
    struct BatchWorkspace {
        ExBuf ex;                             // shared-powers groups of the chunk: [set][groups per set]
        DeviceBuffer<double> PT, V, mixw;     // P area [sets][R][Dp^2], inputs [sets][in] (formula values or rates), weights [sets][rows]
        DeviceBuffer<double> cond, out, pi;   // node vectors [sets][I][Dp], log-likelihoods [sets], root vector [64]
        DeviceBuffer<int> slot, pat, node_ex; // identity slots [entries], patterns [sets], node exponents [sets][I]
        DeviceBuffer<int> row, col;           // first component row of each branch [B+1], caller columns [L][sets]
        PinnedBuffer<int> h_slot, h_pat, h_col;   // staging of slot, pat and col
        // hb2_batch_branch_component_likelihoods and hb2_batch_leaf_support only (sh.side = B; empty for every other call):
        // messages and outside vectors [sets][2][B][64] and their exponents [sets][2][B]; then the row log-likelihoods
        // [sets][R] (branch rows) or the leaf support [sets][L][D] (leaf support)
        DeviceBuffer<double> side, rows, sup;
        DeviceBuffer<int> side_ex;
        // hb2_batch_joint_ancestors only (sh.joint = I; empty for every other call): the argument table [sets][I][64], the
        // node states [sets][I] and the joint log-likelihoods [sets]
        DeviceBuffer<unsigned char> arg;
        DeviceBuffer<long long> states;
        DeviceBuffer<double> jlnl;
        // Sizes the workspace for chunks of `sh`.  A chunk that does not fit re-sizes the whole workspace for this call,
        // after releasing it, so that memory stays at one call's chunk footprint (~8 GB) instead of adding up the largest
        // buffers of different calls' shapes.
        int fit(const BatchShape &sh, int64_t L, int64_t I, cudaStream_t stream) {
            const int64_t sets = sh.sets, nr = sets * sh.R, ne = sets * sh.ent;
            if (sets <= (int64_t)out.size() && ne <= (int64_t)slot.size() && sets * sh.gk <= ex.G && sets * sh.in <= (int64_t)V.size() &&
                nr * sh.mat <= (int64_t)PT.size() && sets * I * sh.vec <= (int64_t)cond.size() && sets * L <= (int64_t)col.size() &&
                sets * sh.side * 128 <= (int64_t)side.size() && sets * sh.rows <= (int64_t)rows.size() &&
                sets * sh.sup <= (int64_t)sup.size() && sets * sh.joint * 64 <= (int64_t)arg.size() &&
                sets * sh.joint <= (int64_t)states.size() && (sh.joint == 0 || sets <= (int64_t)jlnl.size()))
                return 0;
            CU(cudaStreamSynchronize(stream));
            *this = BatchWorkspace();
            if (ex.alloc((int)(sets * sh.gk), ne, stream) || PT.alloc((size_t)nr * sh.mat) || V.alloc((size_t)sets * sh.in) ||
                mixw.alloc(ne) || cond.alloc((size_t)sets * I * sh.vec) || out.alloc(sets) || slot.alloc(ne) || pat.alloc(sets) ||
                node_ex.alloc((size_t)sets * I) || row.alloc(sh.row_off.size()) || col.alloc((size_t)sets * L) || pi.alloc(64) ||
                h_slot.alloc(ne) || h_pat.alloc(sets) || h_col.alloc((size_t)sets * L) ||
                (sh.side && (side.alloc((size_t)sets * sh.side * 128) || side_ex.alloc((size_t)sets * sh.side * 2))) ||
                (sh.rows && rows.alloc((size_t)sets * sh.rows)) || (sh.sup && sup.alloc((size_t)sets * sh.sup)) ||
                (sh.joint && (arg.alloc((size_t)sets * sh.joint * 64) || states.alloc((size_t)sets * sh.joint) || jlnl.alloc(sets)))) {
                *this = BatchWorkspace();     // fits nothing: the next call sizes it again
                return 1;
            }
            for (int64_t e = 0; e < ne; e++) h_slot[e] = (int)e;
            CU(cudaMemcpyAsync(slot, h_slot, (size_t)ne * sizeof(int), cudaMemcpyHostToDevice, stream));
            return 0;
        }
    } batch;
    bool ex_enabled = true;                   // HB2_EXPM_SHARED=0 switches the path off (A/B testing)
    int64_t stage_launches[3] = {0, 0, 0};    // launches per evaluation of the last hb2_time_resident {expm, pruning, root}
    // compiled rate-matrix templates (hb2_set_rate_template*): static scatter map + own queue of per-evaluation formula
    // values.  A tree may carry several models (foreground / background branches, per-branch models of aBSREL): one
    // template each, up to HB2_MAX_TEMPLATES.
    struct Tmpl {
        int64_t nnz = 0, nF = 0;
        bool has_colfreq = false;
        DeviceBuffer<int> d_index, d_formula;
        DeviceBuffer<double> d_colfreq, d_Vres;
        PinnedBuffer<double> h_colfreq;
        HandoverQueue queue;
    };
    std::vector<Tmpl> tmpls;
    // tensor-core path (33..64 states unless HB2_FLAG_FORCE_FP64): fp32 conditionals + split/tiled P operands
    bool use_tc = false;
    DeviceBuffer<float> d_condf, d_PB, d_PTf;
    DeviceBuffer<int> d_err;
    DeviceBuffer<unsigned> d_root_counter;    // ticket counter of the fused root reduction (combine_kernel's last block)
    DeviceBuffer<int> d_forced;               // forced states of the current evaluation (hb2_evaluate_forced)
    PinnedBuffer<int> h_forced;
    int forced_node = -1;
    // persistent walk kernel (one launch per evaluation): plan buffers, generation bits of the tagged hand-over, residency
    int small_ilp = 0, small_resident[2] = {1, 1};   // HB2_SMALL_ILP=1/2 forces one / two patterns per thread (4 states); co-resident CTAs of both
    DeviceBuffer<double> d_cond_side;         // fp64 lanes kernel: side products [C][I][Sp][64] (exponents: second half of d_scal)
    DeviceBuffer<int> d_lane_flags;           // [C][2I][Sp/64] pass id of the last production
    int lane_pass = 0, lanes_resident = 0;    // co-resident CTAs of prune64_lanes_kernel
    int sm_count = 132;
    int walk_max_resident = 0;
    // single-branch shortcut (hb2_branch_cache_*): outside vectors of one branch, all owned classes
    DeviceBuffer<double> d_bc_out; DeviceBuffer<int> d_bc_outE, d_bc_sib; int64_t bc_node = -1;
    int64_t bc_dirty_node = -1;               // first node other than bc_node whose matrix changed since the build
    std::vector<char> plan_jdirty;      // dirty jobs (nodes + side products) of the cached plan
    bool walk_split_nodes = true;       // HB2_WALK_SPLIT_NODES=0: no side products (A/B)
    std::vector<char> plan_dirty;       // cached walk plan (h_walk holds its steps): dirty set, lane count, step count
    int plan_K = 0, plan_steps = 0;
    std::vector<int> walk_gen;          // [C][I] generation bit of each node's resident conditionals (tc walk path)
    bool walk_reset = false;            // a pass was aborted: tags are inconsistent -> wipe and recompute everything
    DeviceBuffer<int> d_walk;
    PinnedBuffer<int> h_walk;
    int walk_lane_cap = 8;              // lanes (CTAs) that share one (class, tile) pair; HB2_WALK_LANES overrides (<= 15)
    bool first_eval_done = false;
    std::vector<char> evaluated_cat;          // [C] whole tree pruned at least once
    int64_t launches = 0;
    ncclComm_t comm = nullptr;
    int n_ranks = 1, rank = 0;
    // class groups (hb2_comm_class_groups): this rank prunes classes [own0, own0 + ownN) only
    int cg_G = 1, cg_g = 0, own0 = 0, ownN = 0, xchg_len = 0;
    DeviceBuffer<double> d_xsend, d_xrecv, d_xfreq, d_xpartial;
    int n_partial_blocks = 0;
    // peer exchange (hb2_kernels_fp64.cuh "Peer exchange"): IPC-mapped buffers of all ranks; falls back to NCCL when the
    // mapping cannot be established (px_ok false)
    bool px_ok = false, px_enabled = true;
    int px_payload = 0;
    unsigned long long px_gen = 0;
    double *px_local = nullptr;               // exported through CUDA IPC: a plain runtime allocation
    std::vector<double *> px_peer;            // host copy of the mapped pointers (entry rank = px_local)
    DeviceBuffer<double *> d_px_peer;
    DeviceBuffer<unsigned> d_px_counter;
    // simulation scratch (hb2_simulate, hb2_batch_site_simulate), grown on demand and used by nothing else: the prefix-sum
    // table, the call's small vectors, and one chunk of leaf / node / class outputs and internal states
    struct SimBuf {
        DeviceBuffer<double> cdf, vec;
        DeviceBuffer<int> ints, cls;
        DeviceBuffer<long long> leaf, node;
        DeviceBuffer<unsigned char> states;
    } sim;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    // side stream of the expm stage: the power tables are built on it while the classification runs on `stream`
    // (launch_expm forks at ev_fork and joins at ev_join)
    cudaStream_t side = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    // recorded after uploads from pinned staging (the queues, ExBuf::h_int, column frequencies, mixtures, the replay's
    // slots): every writer of those buffers waits for it first
    cudaEvent_t ev_staging = nullptr;
    bool staging_busy = false;
};

namespace {

// The pinned staging buffers may still be read by the H2D copies enqueued before the last staged_uploads.
int wait_staging(hb2_partition *p) {
    if (p->staging_busy) {
        CU(cudaEventSynchronize(p->ev_staging));
        p->staging_busy = false;
    }
    return 0;
}

// Called after enqueueing uploads from pinned staging: the next writer waits for them.
int staged_uploads(hb2_partition *p) {
    CU(cudaEventRecord(p->ev_staging, p->stream));
    p->staging_busy = true;
    return 0;
}

HandoverQueue &queue_of(hb2_partition *p, int queue) { return queue == DENSE_QUEUE ? p->dense : p->tmpls[queue].queue; }

// Host half of the shared-powers path for one batch: groups and references of the n entries (h_dst = their slots, < 0
// retired; kind 1 = compiled hand-over, 2 = dense).  A group whose batch holds at least EX_MIN_GROUP live entries gets its
// power table rebuilt from the first of them; smaller groups are compared with the direction the table was last built
// from.  Fills the pinned arrays and enqueues their upload: call BEFORE staged_uploads.
struct SharedPlan {
    bool use = false;
    int kind = 0, n_refs = 0;
    hb2_partition::ExBuf *x = nullptr;
};
constexpr int EX_MIN_GROUP = 24;

int plan_shared(hb2_partition *p, const int *h_dst, int64_t n, int kind, const int *group_override, SharedPlan &sp, int tmpl = 0,
                hb2_partition::ExBuf *bx = nullptr, int min_group = EX_MIN_GROUP) {
    sp = SharedPlan();
    hb2_partition::ExBuf &x = bx ? *bx : p->ex;
    sp.x = &x;
    if (p->Dp != 64 || !p->ex_enabled || !x.d_int || n <= 0 || n > x.cap) return 0;
    if (kind == 1 && !p->tmpls[tmpl].d_Vres) return 0;
    if (wait_staging(p)) return 1;            // an earlier plan's upload may still be reading the pinned arrays
    int *grp = x.h_int, *ref = x.h_int + x.cap, *refs = x.h_int + 2 * x.cap;
    std::vector<int> count(x.G, 0), first(x.G, -1);
    for (int64_t k = 0; k < n; k++) {
        int g = -1;
        if (h_dst[k] >= 0) g = group_override ? group_override[k] : (int)(h_dst[k] / p->B) + tmpl * (int)p->C;   // (template, class)
        if (g >= x.G) g = -1;
        grp[k] = g;
        if (g >= 0) { if (first[g] < 0) first[g] = (int)k; count[g]++; }
    }
    bool any = false;
    int nr = 0;
    for (int g = 0; g < x.G; g++) {
        if (count[g] >= min_group) { refs[nr++] = first[g]; any = true; }
        else { first[g] = -1; if (count[g] > 0 && x.kind[g] == kind) any = true; }
    }
    if (!any) return 0;
    for (int64_t k = 0; k < n; k++) ref[k] = grp[k] >= 0 ? first[grp[k]] : -1;
    // launch_expm rebuilds the power tables beside the classification, and expm_powers_kernel rewrites the cached
    // direction and record of every group it rebuilds, which the classification reads for entries without a reference in
    // the batch: no group may have both in one batch.
    for (int64_t k = 0; k < n; k++)
        if (grp[k] >= 0 && ref[k] < 0 && first[grp[k]] >= 0)
            return fail("plan_shared: entry %lld of group %d has no reference although the group's table is rebuilt", (long long)k, grp[k]);
    for (int r = 0; r < nr; r++) x.kind[grp[refs[r]]] = kind;
    CU(cudaMemcpyAsync(x.d_int, x.h_int, (size_t)(2 * x.cap + x.G) * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    sp.use = true; sp.kind = kind; sp.n_refs = nr;
    return 0;
}

// A template's definition or column frequencies changed.  Its groups' cached power tables were built from matrices the
// template no longer describes, and the classification compares formula values only, so they must not serve another
// entry; the formula values its slots keep for hb2_time_resident no longer assemble to the matrices they hold, so those
// slots cannot be replayed until handed over again.  Stream-ordered after everything flushed so far.
int void_template_cache(hb2_partition *p, int tmpl) {
    for (int c = 0; p->ex.d_groups && c < (int)p->C; c++) {
        const int g = tmpl * (int)p->C + c;
        if (g >= p->ex.G) break;
        CU(cudaMemsetAsync(p->ex.d_groups + g, 0, sizeof(hb2::ExpmGroup), p->stream));
        p->ex.kind[g] = 0;
    }
    for (Slot &s : p->slots) if (s.res == Resident::Formula && s.res_tmpl == tmpl) s.res = Resident::None;
    return 0;
}

constexpr int EXPM64_SMEM = 3 * 64 * hb2::LD64 * sizeof(double);    // expm64_dmma_kernel and expm_powers_kernel

// Launch configuration of expm_poly_kernel: `chunks` clusters of EXPM_POLY_CLUSTER row slices (a non-portable size) that
// share their column sums.
struct PolyLaunch {
    cudaLaunchAttribute attr{};
    cudaLaunchConfig_t cfg{};
    PolyLaunch(unsigned chunks, cudaStream_t stream) {
        attr.id = cudaLaunchAttributeClusterDimension;
        attr.val.clusterDim = {(unsigned)hb2::EXPM_POLY_CLUSTER, 1, 1};
        cfg.gridDim = dim3(hb2::EXPM_POLY_CLUSTER, chunks); cfg.blockDim = dim3(256); cfg.stream = stream;
        cfg.attrs = &attr; cfg.numAttrs = 1;
    }
    PolyLaunch(const PolyLaunch &) = delete;               // cfg points into the object
    PolyLaunch &operator=(const PolyLaunch &) = delete;
};

// Function attributes of the exponential's kernels for padded state count Dp, and the check that one cluster of
// expm_poly_kernel can be resident on the device.
int expm_setup(int Dp, int device) {
    if (Dp == 32) {
        CU(cudaFuncSetAttribute(hb2::expm_small_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hb2::expm_small_smem_bytes(32)));
        CU(cudaFuncSetAttribute(hb2::expm_rates_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hb2::expm_rates_smem_bytes(32)));
    }
    if (Dp != 64) return 0;
    CU(cudaFuncSetAttribute(hb2::expm_powers_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, EXPM64_SMEM));
    CU(cudaFuncSetAttribute(hb2::expm64_dmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, EXPM64_SMEM));
    CU(cudaFuncSetAttribute(hb2::expm64_dmma_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CU(cudaFuncSetAttribute(hb2::expm_poly_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    const PolyLaunch one(1, 0);
    int clusters = 0;
    CU(cudaOccupancyMaxActiveClusters(&clusters, hb2::expm_poly_kernel, &one.cfg));
    if (clusters < 1) return fail("expm_poly_kernel: no cluster of %d CTAs can be resident on device %d", hb2::EXPM_POLY_CLUSTER, device);
    return 0;
}

// Calls f(std::integral_constant<int, DP>{}) for the small-state padded count DP = Dp (4, 8, 16, 24, 32); false otherwise.
template <class F>
bool small_states(int Dp, F &&f) {
    switch (Dp) {
        case 4: f(std::integral_constant<int, 4>{}); return true;
        case 8: f(std::integral_constant<int, 8>{}); return true;
        case 16: f(std::integral_constant<int, 16>{}); return true;
        case 24: f(std::integral_constant<int, 24>{}); return true;
        case 32: f(std::integral_constant<int, 32>{}); return true;
        default: return false;
    }
}

// One CTA per listed matrix of `in` (rows of D*D matrix entries, or of the template's formula values).  The results go to
// the P cache, with the tensor-path operands when use_tc, or, when scratch is given, to scratch alone (mixture components
// and batched site sets).  keep_resident: leave the resident copy of each entry's rate matrix (dense Q, or formula values
// on the shared-powers path), as a flushed hand-over does.  sp: shared-powers plan of the WHOLE batch this run
// [off, off + n) belongs to (in / d_dst already point at the run).
int launch_expm(hb2_partition *p, Source src, const double *in, const int *d_dst, int n, bool keep_resident, const SharedPlan &sp,
                int64_t off = 0, double *scratch = nullptr) {
    if (n <= 0) return 0;
    hb2::ExpmArgs a{};
    a.Q = in; a.dst = d_dst; a.PT = scratch ? scratch : p->d_PT; a.D = (int)p->D;
    a.Qres = keep_resident && src.kind != Kind::Trans ? (double *)p->d_Qres : nullptr;
    a.is_trans = src.kind == Kind::Trans;
    const hb2_partition::Tmpl *t = src.kind == Kind::Compiled ? &p->tmpls[src.tmpl] : nullptr;
    if (t) {
        a.Q = nullptr; a.V = in; a.tmpl_index = t->d_index; a.tmpl_formula = t->d_formula;
        a.tmpl_colfreq = t->has_colfreq ? t->d_colfreq : (double *)nullptr; a.tmpl_nnz = (int)t->nnz; a.nF = (int)t->nF;
    }
    if (p->Dp == 64) {
        hb2::ExpmTcOut tc{nullptr, nullptr};
        if (p->use_tc && !scratch) { tc.PB = p->d_PB; tc.PTf = p->d_PTf; }
        if (sp.use && src.kind != Kind::Trans) {
            hb2_partition::ExBuf &x = *sp.x;
            const int nV = t ? (int)t->nF : (int)(p->D * p->D);
            // references index the whole batch: classification has to see it in one piece (off == 0 for compiled batches
            // and for dense batches that consist of a single run; mixed dense batches fall back below)
            a.group = x.d_int + off; a.flag = x.d_flag + off; a.weight = x.d_weight + off; a.groups = x.d_groups;
            a.pow = x.d_pow;
            a.Qres = nullptr;                    // the classification stage keeps the resident copy
            // the power tables are built on the side stream while the classification runs (plan_shared keeps the two
            // from touching the same group)
            if (sp.n_refs > 0) {
                hb2::ExpmPowersArgs pa{};
                pa.a = a; pa.refs = x.d_int + 2 * x.cap; pa.groups = x.d_groups;
                pa.pow = x.d_pow; pa.refvec = x.d_refvec; pa.refvec_stride = x.stride; pa.nV = nV; pa.kind = sp.kind; pa.Vin = in;
                pa.flags = x.d_flags; pa.gen = ++x.gen; pa.err = p->d_err;
                CU(cudaEventRecord(p->ev_fork, p->stream));
                CU(cudaStreamWaitEvent(p->side, p->ev_fork, 0));
                hb2::expm_powers_kernel<<<dim3(hb2::EXPM_POW_TERMS - 1, (unsigned)sp.n_refs), 256, EXPM64_SMEM, p->side>>>(pa);
                p->launches++;
                CU(cudaEventRecord(p->ev_join, p->side));
            }
            hb2::ExpmClassifyArgs ca{};
            ca.V = in; ca.nV = nV; ca.kind = sp.kind; ca.dst = d_dst; ca.group = x.d_int + off;
            ca.ref = x.d_int + x.cap + off; ca.groups = x.d_groups; ca.refvec = x.d_refvec; ca.refvec_stride = x.stride;
            ca.weight = x.d_weight + off; ca.flag = x.d_flag + off;
            ca.res = !keep_resident ? nullptr : t ? (double *)t->d_Vres : (double *)p->d_Qres;
            if (nV <= 256) hb2::expm_classify_warp_kernel<<<(n + 7) / 8, 256, 0, p->stream>>>(ca, n);
            else hb2::expm_classify_kernel<<<n, 128, 0, p->stream>>>(ca);
            if (sp.n_refs > 0) CU(cudaStreamWaitEvent(p->stream, p->ev_join, 0));
            const PolyLaunch pl((unsigned)((n + hb2::EXPM_POLY_CHUNK - 1) / hb2::EXPM_POLY_CHUNK), p->stream);
            CU(cudaLaunchKernelEx(&pl.cfg, hb2::expm_poly_kernel, a, tc, n));
            p->launches += 2;
        }
        hb2::expm64_dmma_kernel<<<std::min(n, 2 * p->sm_count), 256, EXPM64_SMEM, p->stream>>>(a, tc, n);
    } else if (!small_states(p->Dp, [&](auto dp) {
                   constexpr int DP = decltype(dp)::value;
                   hb2::expm_small_kernel<DP><<<n, 128, hb2::expm_small_smem_bytes(DP), p->stream>>>(a);
               })) {
        return fail("unsupported padded state count %d", p->Dp);
    }
    p->launches++;
    CU(cudaGetLastError());
    return 0;
}

// Uploads a queue and exponentiates its entries, one launch per run of equal kind.  Retired entries (destination -1) are
// skipped by the kernels.  Shared powers apply only when the queue holds no transition matrix.  Each entry leaves its
// slot's resident copy: formula values for a compiled entry on shared powers, none for a transition matrix, dense Q
// otherwise.
int flush_queue(hb2_partition *p, int queue) {
    HandoverQueue &q = queue_of(p, queue);
    const int64_t n = q.n;
    if (n == 0) return 0;
    const int tmpl = std::max(queue, 0);
    CU(cudaMemcpyAsync(q.d_rows, q.h_rows, n * q.row * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    CU(cudaMemcpyAsync(q.d_dst, q.h_dst, n * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    SharedPlan sp;
    const bool any_trans = std::find(q.kind.begin(), q.kind.begin() + n, Kind::Trans) != q.kind.begin() + n;
    if (!any_trans && plan_shared(p, q.h_dst, n, queue == DENSE_QUEUE ? 2 : 1, nullptr, sp, tmpl)) return 1;
    if (staged_uploads(p)) return 1;
    for (int64_t i = 0, j; i < n; i = j) {
        for (j = i + 1; j < n && q.kind[j] == q.kind[i]; j++) {}
        if (launch_expm(p, {q.kind[i], tmpl}, q.d_rows + i * q.row, q.d_dst + i, (int)(j - i), true, sp, i)) return 1;
    }
    for (int64_t k = 0; k < n; k++) {
        if (q.h_dst[k] < 0) continue;
        Slot &s = p->slots[q.h_dst[k]];
        s.entry = -1;
        s.res = q.kind[k] == Kind::Trans ? Resident::None : q.kind[k] == Kind::Compiled && sp.use ? Resident::Formula : Resident::DenseQ;
        s.res_tmpl = (signed char)tmpl;
    }
    q.n = 0;
    return 0;
}

// Flush the compiled queues in ascending template id: one H2D copy and one expm launch sequence each.
int flush_compiled(hb2_partition *p) {
    for (size_t t = 0; t < p->tmpls.size(); t++)
        if (flush_queue(p, (int)t)) return 1;
    return 0;
}

// Flush everything handed over since the last evaluation: the compiled queues, then the dense queue.
int flush_matrices(hb2_partition *p) {
    return flush_compiled(p) || flush_queue(p, DENSE_QUEUE);
}

// Checks a hand-over of n matrices of class `cat` (-1 means 0) as a whole before anything changes: the class, every node
// id and, where the entry point has them, the kind and the matrix pointers.  A refused hand-over changes nothing.  An
// accepted one is noted for the branch cache; `stage` is false for another class group's class, whose slots are marked
// here since nothing is staged for them.
int accept_handover(hb2_partition *p, int64_t &cat, int64_t n, const int64_t *nodeIds, bool &stage, int kind = HB2_MATRIX_RATE,
                    const double *const *M = nullptr) {
    if (cat < 0) cat = 0;
    if (cat >= p->C) return fail("rate class %lld out of range (C=%lld)", (long long)cat, (long long)p->C);
    for (int64_t k = 0; k < n; k++)
        if (nodeIds[k] < 0 || nodeIds[k] >= p->B)
            return fail("node id %lld has no branch (valid 0..%lld)", (long long)nodeIds[k], (long long)p->B - 1);
    if (kind != HB2_MATRIX_RATE && kind != HB2_MATRIX_TRANS) return fail("unknown matrix kind %d", kind);
    for (int64_t k = 0; M && k < n; k++)
        if (!M[k]) return fail("matrix %lld is null", (long long)k);
    // the single-branch cache (if any) only survives changes of ITS branch
    for (int64_t k = 0; k < n && p->bc_node >= 0 && p->bc_dirty_node < 0; k++)
        if (nodeIds[k] != p->bc_node) p->bc_dirty_node = nodeIds[k];
    stage = cat >= p->own0 && cat < p->own0 + p->ownN;
    if (!stage) for (int64_t k = 0; k < n; k++) p->slots[cat * p->B + nodeIds[k]].have = true;
    return 0;
}

// Stages one row for `slot` in a queue (DENSE_QUEUE or a template id).  The slot's pending entry is overwritten when it
// sits in the same queue and retired otherwise.  A full compiled queue flushes the compiled queues; a full dense queue
// flushes everything.
int enqueue(hb2_partition *p, int queue, int64_t slot, const double *row, Kind kind) {
    if (wait_staging(p)) return 1;            // the last flush's H2D copies must have left the pinned buffers
    HandoverQueue &q = queue_of(p, queue);
    Slot &s = p->slots[slot];
    if (s.entry >= 0 && s.queue != queue) {
        queue_of(p, s.queue).h_dst[s.entry] = -1;
        s.entry = -1;
    }
    if (s.entry < 0) {
        if (q.n == q.cap) {
            cudaSetDevice(p->device);
            if ((queue == DENSE_QUEUE ? flush_matrices(p) : flush_compiled(p)) || wait_staging(p)) return 1;
        }
        s.queue = (signed char)queue;
        s.entry = (int)q.n++;
    }
    memcpy(q.h_rows + s.entry * q.row, row, q.row * sizeof(double));
    q.h_dst[s.entry] = (int)slot;
    q.kind[s.entry] = kind;
    s.have = true;
    return 0;
}

// Stages the root vector, zero-padded to Dp (unless null), into d_pi (or dst), and the first nw class weights (when given).
// Every caller synchronises the stream before it returns, so h_small is free again at the next call.
int stage_root(hb2_partition *p, const double *rootFreqs, const double *weights = nullptr, int nw = 0, double *dst = nullptr) {
    double *hs = p->h_small;
    if (rootFreqs) {
        for (int k = 0; k < p->Dp; k++) hs[k] = k < p->D ? rootFreqs[k] : 0.0;
        CU(cudaMemcpyAsync(dst ? dst : (double *)p->d_pi, hs, p->Dp * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    }
    if (weights) {
        for (int c = 0; c < nw; c++) hs[p->Dp + c] = weights[c];
        CU(cudaMemcpyAsync(p->d_weights, hs + p->Dp, nw * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    }
    return 0;
}

// Stages a template's column frequencies through its pinned buffer, so that the caller may reuse colFreq at once.
int stage_colfreq(hb2_partition *p, hb2_partition::Tmpl &t, const double *colFreq) {
    if (wait_staging(p)) return 1;
    memcpy(t.h_colfreq, colFreq, p->D * sizeof(double));
    CU(cudaMemcpyAsync(t.d_colfreq, t.h_colfreq, p->D * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    return staged_uploads(p);
}

// Checks a flat parent list (leaves 0..L-1, then the internal nodes in post-order, the root last with parent -1) and
// fills each internal node's children (flat ids, ascending) and height (0 = only leaf children).
int build_tree(const int64_t *flatParents, int64_t L, int64_t I, std::vector<std::vector<int>> &children, std::vector<int> &height) {
    children.assign(I, {});
    int roots = 0;
    for (int64_t n = 0; n < L + I; n++) {
        const int64_t par = flatParents[n];
        if (par == -1) { roots++; if (n != L + I - 1) return fail("root must be the last node (found -1 parent at %lld)", (long long)n); continue; }
        if (par < 0 || par >= I) return fail("flatParents[%lld]=%lld out of range", (long long)n, (long long)par);
        if (n >= L && par <= n - L) return fail("internal nodes must be in post-order (node %lld has parent %lld)", (long long)n, (long long)par);
        children[par].push_back((int)n);
    }
    if (roots != 1) return fail("tree must have exactly one root");
    height.assign(I, 0);
    for (int64_t i = 0; i < I; i++) {
        if (children[i].empty()) return fail("internal node %lld has no children", (long long)i);
        for (int ch : children[i]) if (ch >= L) height[i] = std::max(height[i], height[ch - L] + 1);
    }
    return 0;
}

// The internal nodes to re-prune when the nodes in `update` changed: the parent of each and all its ancestors.
// update == nullptr or nUpdate < 0 marks every node.  dirty gets one entry per internal node.
int dirty_nodes(const int64_t *flatParents, int64_t L, int64_t I, int64_t nUpdate, const int64_t *update, std::vector<char> &dirty) {
    dirty.assign(I, 0);
    if (update == nullptr || nUpdate < 0) {
        std::fill(dirty.begin(), dirty.end(), 1);
        return 0;
    }
    for (int64_t k = 0; k < nUpdate; k++) {
        const int64_t n = update[k];
        if (n < 0 || n >= L + I) return fail("updateNodes[%lld]=%lld out of range", (long long)k, (long long)n);
        for (int64_t par = flatParents[n]; par >= 0 && !dirty[par]; par = flatParents[L + par]) dirty[par] = 1;
    }
    return 0;
}

hb2::PruneArgs prune_args(hb2_partition *p, int cat0) {
    hb2::PruneArgs a;
    a.PT = p->d_PT; a.cond = p->d_cond; a.scal = p->d_scal; a.leaf = p->d_leaf; a.ambig = p->d_ambig; a.pi = p->d_pi;
    a.rootL = p->d_rootL; a.rootE = p->d_rootE;
    a.tree.child_start = p->d_child_start; a.tree.child_ids = p->d_child_ids;
    a.L = (int)p->L; a.I = (int)p->I; a.B = (int)p->B; a.D = (int)p->D; a.Sp = (int)p->Sp; a.cat0 = cat0;
    a.forced = p->d_forced; a.forced_node = p->forced_node;
    return a;
}

// Pure host code (no CUDA): the walk plan for a dirty set on K lanes.  lane_start[K+1]; steps = 2 ints per step
// (child encoding, job's node slot | flags); jdirty[2I] = jobs of the plan.  Returns the number of steps.  Exposed for
// CPU tests through hb2_plan_walk.
int plan_walk(const std::vector<std::vector<int>> &children, const std::vector<int> &height, int L, int I,
              const std::vector<char> &dirty, int K, bool split_nodes, int *lane_start, int *steps, std::vector<char> &jdirty_out,
              bool canonical_multi = false) {
    // canonical_multi (fp64 lanes kernel): a node with more than two children is neither split nor chained and its children
    // are multiplied in tree order, so its product is associated the same way in every plan; with two children the product
    // is exact-commutative and power-of-two rescalings are exact, hence conditionals do not depend on the plan at all (a
    // partial re-evaluation reproduces the full one bit for bit).
    // Jobs.  Job j < I is node j; job I + n is the SIDE PRODUCT of node n: a node with two or more internal children is
    // split into "contract the child with the deepest subtree" (+ multiply the side product in: no matrix, the cheapest
    // step after a leaf) and a side job that contracts all OTHER children.  Side jobs sit off the root path, so other
    // lanes do them early and the spine of a deep tree carries one contraction per node instead of two (`split`).
    // item list of a job: children to contract (flat ids) and, for a split node, the side job to multiply in.
    const int NJ = 2 * I;
    const bool split_on = split_nodes && K > 1;
    std::vector<std::vector<int>> jch(NJ);       // children (flat ids, leaves and internals) contracted by the job
    std::vector<int> jmul(NJ, -1);               // side job multiplied in by the job (real split nodes only)
    std::vector<char> jdirty(NJ, 0);
    for (int n = 0; n < I; n++) {
        if (!dirty[n]) continue;
        jdirty[n] = 1;
        int heavy = -1, nint = 0;
        for (int ch : children[n]) if (ch >= L) { nint++; if (heavy < 0 || height[ch - L] > height[heavy - L]) heavy = ch; }
        if (split_on && nint >= 2 && !(canonical_multi && children[n].size() > 2)) {
            jch[n].push_back(heavy);
            jmul[n] = I + n;
            jdirty[I + n] = 1;
            for (int ch : children[n]) if (ch != heavy) jch[I + n].push_back(ch);
        } else {
            jch[n] = children[n];
        }
    }
    // Lane assignment = list scheduling of the dirty jobs on K in-order lanes with a rough cost model (cycles per step
    // kind, as HB2_WALK_TRACE reports them): the pass is bound by the busiest lane or by the deepest root path, so the
    // (job, lane) pair that can start first is scheduled next, ties going to the longer remaining path; a job whose
    // contracted internal child was the lane's previous job continues there (register hand-over: the cheapest
    // contraction).  Every lane executes its jobs in the order they were scheduled and a job is scheduled only after
    // the jobs it consumes, so cross-lane waits cannot cycle.
    const double C_LEAF = 1.8e3, C_CHAIN = 4.7e3, C_INT = 7.0e3, C_MUL = 2.5e3, C_NODE = 1.0e3, C_XFER = 1.5e3;
    auto job_of_child = [&](int ch) { return ch - L; };          // internal child (flat id) -> job that produces it
    std::vector<int> lane_of(NJ, -1), lane_last(K, -1), chain_child(NJ, -1), parent_job(NJ, -1);
    std::vector<std::vector<int>> lanes(K);
    int njobs = 0;
    {
        std::vector<double> base(NJ, 0.0), tail(NJ, 0.0), finish(NJ, 0.0), lane_time(K, 0.0);
        std::vector<int> pending(NJ, 0);         // dirty producer jobs not yet scheduled
        std::vector<int> ready;
        for (int j = 0; j < NJ; j++) {
            if (!jdirty[j]) continue;
            njobs++;
            base[j] = C_NODE + (jmul[j] >= 0 ? C_MUL : 0.0);
            for (int ch : jch[j]) {
                base[j] += ch < L ? C_LEAF : C_INT;
                if (ch >= L && dirty[ch - L]) { pending[j]++; parent_job[job_of_child(ch)] = j; }
            }
            if (jmul[j] >= 0) { pending[j]++; parent_job[jmul[j]] = j; }
        }
        // remaining path to the root, parents before children: real nodes by decreasing height, a side job right after
        // its node
        std::vector<int> by_height;
        for (int n = 0; n < I; n++) if (dirty[n]) by_height.push_back(n);
        std::stable_sort(by_height.begin(), by_height.end(), [&](int x, int y) { return height[x] > height[y]; });
        for (int n : by_height) {
            tail[n] = base[n] + (parent_job[n] >= 0 ? tail[parent_job[n]] : 0.0);
            if (jmul[n] >= 0) tail[I + n] = base[I + n] + tail[n];
        }
        for (int j = 0; j < NJ; j++) if (jdirty[j] && pending[j] == 0) ready.push_back(j);
        auto producers = [&](int j, auto &&f) {   // dirty jobs whose output job j consumes
            for (int ch : jch[j]) if (ch >= L && dirty[ch - L]) f(job_of_child(ch));
            if (jmul[j] >= 0) f(jmul[j]);
        };
        for (int done = 0; done < njobs; done++) {
            int best = -1, best_r = 0; double best_start = 0.0;
            for (int j : ready) {
                for (int r = 0; r < K; r++) {
                    double est = lane_time[r];
                    producers(j, [&](int q) { est = std::max(est, finish[q] + (lane_of[q] == r ? 0.0 : C_XFER)); });
                    if (best < 0 || est < best_start || (est == best_start && tail[j] > tail[best])) { best = j; best_r = r; best_start = est; }
                }
            }
            const int j = best, r = best_r;
            double cost = base[j];
            for (int ch : jch[j])
                if (ch >= L && dirty[ch - L] && lane_last[r] == job_of_child(ch) && !(canonical_multi && jch[j].size() > 2)) { chain_child[j] = ch - L; cost -= C_INT - C_CHAIN; break; }
            finish[j] = best_start + cost;
            lane_time[r] = finish[j];
            lane_of[j] = r; lane_last[r] = j;
            lanes[r].push_back(j);
            ready.erase(std::find(ready.begin(), ready.end(), j));
            if (parent_job[j] >= 0 && --pending[parent_job[j]] == 0) ready.push_back(parent_job[j]);
        }
        if (getenv("HB2_DEBUG")) {
            double mx = 0; for (double t : lane_time) mx = std::max(mx, t);
            double deepest = 0; for (int j = 0; j < NJ; j++) if (jdirty[j]) deepest = std::max(deepest, tail[j]);
            fprintf(stderr, "[hb2] walk schedule: %d jobs, modelled makespan %.0f cycles, deepest root path %.0f, lanes (jobs/cycles):", njobs, mx, deepest);
            for (int r = 0; r < K; r++) fprintf(stderr, " %zu/%.0f", lanes[r].size(), lane_time[r]);
            fprintf(stderr, "\n");
        }
    }
    // flatten every lane into steps: chain child first, then leaves, then the other internal children, then the side product
    int ns = 0;
    for (int r = 0; r < K; r++) {
        lane_start[r] = ns;
        for (int j : lanes[r]) {
            const int first = ns;
            auto push = [&](int enc) { steps[2 * ns] = enc; steps[2 * ns + 1] = j; ns++; };
            if (canonical_multi && jch[j].size() > 2) {          // tree order, leaves and internal children interleaved
                for (int ch : jch[j]) push(ch < L ? ch : (ch | ((dirty[ch - L] && lane_of[ch - L] != lane_of[j]) ? hb2::WALK_WAIT : 0)));
            } else {
            if (chain_child[j] >= 0) push((chain_child[j] + L) | hb2::WALK_CHAIN);
            for (int ch : jch[j]) if (ch < L) push(ch);
            for (int ch : jch[j]) {
                if (ch < L || ch - L == chain_child[j]) continue;
                const int ci = ch - L;
                push(ch | ((dirty[ci] && lane_of[ci] != lane_of[j]) ? hb2::WALK_WAIT : 0));
            }
            }
            if (jmul[j] >= 0) push((L + jmul[j]) | hb2::WALK_MUL | (lane_of[jmul[j]] != lane_of[j] ? hb2::WALK_WAIT : 0));
            steps[2 * first + 1] |= hb2::STEP_FIRST;
            steps[2 * (ns - 1) + 1] |= hb2::STEP_LAST;
        }
    }
    lane_start[K] = ns;
    jdirty_out = jdirty;
    return ns;
}

// The walk plan of a dirty set on K lanes, built into h_walk: lane_start[K+1] (16 ints) | steps (int2 each, from int
// offset 16).  The plan depends on the tree, the dirty set and K only, and optimisers re-evaluate the same set again and
// again: when these match the cached plan, h_walk is left as it is.  Returns the step count; *rebuilt tells whether the
// plan was built anew.
int cached_plan(hb2_partition *p, const std::vector<char> &dirty, int K, bool canonical_multi, bool *rebuilt = nullptr) {
    const bool reuse = p->plan_steps > 0 && p->plan_K == K && p->plan_dirty == dirty;
    if (!reuse) {
        p->plan_steps = plan_walk(p->children, p->height, (int)p->L, (int)p->I, dirty, K, p->walk_split_nodes, p->h_walk,
                                  p->h_walk + 16, p->plan_jdirty, canonical_multi);
        p->plan_K = K; p->plan_dirty = dirty;
    }
    if (rebuilt) *rebuilt = !reuse;
    return p->plan_steps;
}

// HB2_WALK_TRACE (bring-up aid): clock stamps of the steps of one CTA (HB2_WALK_TRACE_CTA, 12 per step) and, for the
// tensor walk kernel, 4 stamps of every CTA, written to a text file after the launch.  tools/trace_stats.py and
// tools/trace_stats_lanes.py parse the file.
struct WalkTrace {
    const char *path = getenv("HB2_WALK_TRACE");
    int cta = 0, ns = 0, ctas = 0;
    DeviceBuffer<long long> d;
    size_t n = 0;
    // Stamps of a pass of ns steps; ctas = CTAs that stamp their residence (0: none).  d stays null without a trace.
    int alloc(hb2_partition *p, int ns_, int ctas_) {
        if (!path) return 0;
        if (const char *tc = getenv("HB2_WALK_TRACE_CTA")) cta = atoi(tc);
        ns = ns_; ctas = ctas_;
        n = (size_t)(ns + 1) * 12 + (size_t)ctas * 4;
        return d.alloc(n) || d.zero(p->stream);
    }
    // kernel: header prefix naming the kernel; columns: names of the 12 stamps of a step
    int write(hb2_partition *p, const char *kernel, const char *columns, int K) {
        if (!d) return 0;
        std::vector<long long> ht(n);
        CU(cudaStreamSynchronize(p->stream));
        CU(cudaMemcpy(ht.data(), d, n * sizeof(long long), cudaMemcpyDeviceToHost));
        FILE *f = fopen(path, "w");
        if (!f) return 0;
        const int *lane_start = p->h_walk, r = cta % K;
        fprintf(f, "# %scta %d lane %d steps %d..%d ; columns: %s (cycles rel. to first)\n", kernel, cta, r, lane_start[r],
                lane_start[r + 1], columns);
        const long long t00 = ht[1];
        for (int i = 0; i < lane_start[r + 1] - lane_start[r]; i++) {
            const long long *q = ht.data() + (size_t)i * 12;
            fprintf(f, "%d 0x%x 0x%x", i, (unsigned)(q[0] >> 32), (unsigned)(q[0] & 0xffffffff));
            for (int c = 1; c < 12; c++) fprintf(f, " %lld", q[c] ? q[c] - t00 : -1LL);
            fprintf(f, "\n");
        }
        if (ctas > 0) {   // per-CTA residence: "# C <block> <smid> <cycles> <start ns rel. to the earliest CTA>"
            const long long *ct = ht.data() + (size_t)(ns + 1) * 12;
            long long g0 = ct[3];
            for (int b = 0; b < ctas; b++) g0 = std::min(g0, ct[(size_t)b * 4 + 3]);
            for (int b = 0; b < ctas; b++)
                fprintf(f, "# C %d %lld %lld %lld\n", b, ct[(size_t)b * 4], ct[(size_t)b * 4 + 2] - ct[(size_t)b * 4 + 1], ct[(size_t)b * 4 + 3] - g0);
        }
        fclose(f);
        return 0;
    }
};

// Walk plan for prune64_tc_walk_kernel: K lanes of jobs (nodes and side products, in schedule order), flattened into
// one step per child.  Layout of the int buffer: lane_start[K+1] (16 ints) | steps (int2 each) | generation bits [C][2I]
int run_walk(hb2_partition *p, int cat0, int ncls, const std::vector<char> &dirty) {
    const int I = (int)p->I;
    const int T = (int)(p->Sp / hb2::TC_TILE_P);
    // A CTA runs a unit of two tiles of one class (one per warpgroup) or of one.  Lanes are planned over pairs of tiles.
    int K = std::max(1, std::min(p->walk_lane_cap, p->walk_max_resident / std::max(ncls * ((T + 1) / 2), 1)));
    const int total = (int)std::count(dirty.begin(), dirty.end(), 1);
    if (total == 0) return 0;
    K = std::min(K, total);
    int pairs = T / 2;                           // two-tile units per class; the rest of the tiles are units of one
    if (K == 1) {
        // one lane per unit: split pairs back into single tiles while that leaves no resident CTA without a unit
        const int units = std::min(T, std::max((T + 1) / 2, p->walk_max_resident / std::max(ncls, 1)));
        pairs = T - units;
    }
    const int CT = ncls * (T - pairs);
    const int nslots = (K == 1) ? std::min(CT, p->walk_max_resident) : CT;
    const int ns = cached_plan(p, dirty, K, false);
    // generation bits: every node re-pruned by this pass flips its bit (per class); the kernel tags what it writes with the
    // new bit and awaits cross-lane children on it.  The table travels behind the steps.
    for (int c = cat0; c < cat0 + ncls; c++)
        for (int j = 0; j < 2 * I; j++)
            if (p->plan_jdirty[j]) p->walk_gen[(size_t)c * 2 * I + j] ^= 1;
    const int gen_off = 16 + 2 * ns;
    std::copy(p->walk_gen.begin(), p->walk_gen.end(), p->h_walk + gen_off);
    const int nints = gen_off + (int)p->walk_gen.size();
    CU(cudaMemcpyAsync(p->d_walk, p->h_walk, nints * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    hb2::PruneArgs a = prune_args(p, cat0);
    hb2::WalkArgs w;
    hb2::PruneTcArgs &t = w.a;
    t.PB = p->d_PB; t.PTf = p->d_PTf; t.cond = p->d_condf; t.scal = a.scal; t.leaf = a.leaf; t.ambig = a.ambig; t.pi = a.pi;
    t.rootL = a.rootL; t.rootE = a.rootE; t.tree = a.tree; t.err = p->d_err;
    t.L = a.L; t.I = a.I; t.B = a.B; t.D = a.D; t.Sp = a.Sp; t.cat0 = a.cat0;
    t.forced = a.forced; t.forced_node = a.forced_node;
    w.lane_start = p->d_walk; w.steps = reinterpret_cast<const int2 *>(p->d_walk + 16);
    w.gen = p->d_walk + gen_off; w.NI = 2 * I; w.K = K; w.T = T; w.ncls = ncls; w.nslots = nslots; w.pairs = pairs;
    if (getenv("HB2_DEBUG")) fprintf(stderr, "[hb2] walk: jobs=%d steps=%d K=%d T=%d ncls=%d pairs/class=%d units=%d nslots=%d grid=%d resident=%d\n", total, ns, K, T, ncls, pairs, CT, nslots, nslots * K, p->walk_max_resident);
    { static const float thr = getenv("HB2_ANCHOR_THR") ? (float)atof(getenv("HB2_ANCHOR_THR")) : hb2::TC_ANCHOR_THR; w.anchor_thr = thr; }
    WalkTrace trace;
    if (trace.alloc(p, ns, nslots * K)) return 1;
    w.trace = trace.d; w.trace_cta = trace.cta; w.trace_cta_times = trace.d ? trace.d + (size_t)(ns + 1) * 12 : nullptr;
    hb2::prune64_tc_walk_kernel<<<nslots * K, 256, hb2::WALK_SMEM_BYTES, p->stream>>>(w);
    if (trace.write(p, "", "child_enc parent_flags t_begin bar1 staged/ready tableready|split bar2 bfull mma_done end", K)) return 1;
    p->launches++;
    CU(cudaGetLastError());
    return 0;
}

// The pruning kernels, each of which prunes the dirty nodes of a pass in one launch: the tensor walk (33..64 states), the
// fp64 lanes kernel (33..64 states with HB2_FLAG_FORCE_FP64) and the small-state walks (<= 32 padded states).
enum PruneKernel { TC_WALK, FP64_LANES, SMALL_DMMA, SMALL_WALK_ILP, SMALL_WALK };
// SMALL_WALK_ILP and SMALL_WALK are prune_small_walk_kernel with two and one patterns per thread; they keep their own
// names, which hb2_pruning_kernel reports
const char *const PRUNE_KERNEL_NAME[] = {"prune64_tc_walk_kernel", "prune64_lanes_kernel", "prune_small_dmma_kernel",
                                         "prune_small_walk_ilp_kernel", "prune_small_walk_kernel"};

// The kernel that prunes ncls classes of p.  4 states: one or two patterns per thread -- (passes over the resident
// capacity) x (relative cost of a pass: a two-pattern pass costs about 1.55 one-pattern passes)
PruneKernel pruning_kernel(const hb2_partition *p, int ncls) {
    if (p->use_tc) return TC_WALK;
    if (p->Dp == 64) return FP64_LANES;
    if (p->Dp >= 16) return SMALL_DMMA;
    if (p->Dp != 4 || p->small_ilp == 1) return SMALL_WALK;
    if (p->small_ilp == 2) return SMALL_WALK_ILP;
    const long ct1 = (long)(p->Sp / 128) * ncls, ct2 = (long)((p->Sp + 255) / 256) * ncls;
    return 1.55 * std::ceil((double)ct2 / p->small_resident[1]) < std::ceil((double)ct1 / p->small_resident[0]) ? SMALL_WALK_ILP : SMALL_WALK;
}

// Small state spaces: one launch, every CTA walking the dirty nodes in post-order (internal indices ascending).
int run_small_walk(hb2_partition *p, int cat0, int ncls, const std::vector<char> &dirty, PruneKernel kernel) {
    int n = 0;
    for (int i = 0; i < (int)p->I; i++) if (dirty[i]) p->h_jobs[n++] = i;
    if (n == 0) return 0;
    CU(cudaMemcpyAsync(p->d_jobs, p->h_jobs, n * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    hb2::PruneArgs a = prune_args(p, cat0);
    if (kernel == SMALL_DMMA) {                  // 16 / 24 / 32 padded states: FP64 tensor pipe, 8 patterns per warp
        // every CTA walks the whole tree: the launch is a few long waves.  Shape with the smaller last-wave loss: 8 warps
        // (4 CTAs per SM; 3 at 32 states) or, up to 24 states, 4 warps (9 per SM).
        const double warps = (double)(p->Sp / 8) * ncls;
        const int cap8 = (p->Dp == 32 ? 3 : 4) * 8 * p->sm_count, cap4 = 9 * 4 * p->sm_count;
        auto cost = [&](int cap) { const double wv = warps / cap; return std::ceil(wv - 1e-9) / wv; };      // 1 = no tail loss
        int nw = 8;
        if (p->Dp <= 24 && cost(cap4) < cost(cap8) - 0.05) nw = 4;
        if (const char *ov = getenv("HB2_SMALL_WARPS")) nw = (atoi(ov) == 4 && p->Dp <= 24) ? 4 : 8;
        dim3 g((unsigned)(p->Sp / (8 * nw)), (unsigned)ncls);
        if (nw == 8) {
            switch (p->Dp) {
                case 16: hb2::prune_small_dmma_kernel<16, 8><<<g, 256, 0, p->stream>>>(a, p->d_jobs, n); break;
                case 24: hb2::prune_small_dmma_kernel<24, 8><<<g, 256, 0, p->stream>>>(a, p->d_jobs, n); break;
                case 32: hb2::prune_small_dmma_kernel<32, 8><<<g, 256, 0, p->stream>>>(a, p->d_jobs, n); break;
                default: return fail("unsupported padded state count %d", p->Dp);
            }
        } else {
            if (p->Dp == 16) hb2::prune_small_dmma_kernel<16, 4><<<g, 128, 0, p->stream>>>(a, p->d_jobs, n);
            else hb2::prune_small_dmma_kernel<24, 4><<<g, 128, 0, p->stream>>>(a, p->d_jobs, n);
        }
    } else {                                     // 4 / 8 padded states: PP patterns per thread (two only for 4 states)
        const int PP = kernel == SMALL_WALK_ILP ? 2 : 1;
        dim3 grid((unsigned)((p->Sp + 128 * PP - 1) / (128 * PP)), (unsigned)ncls);
        switch (p->Dp) {
            case 4:
                if (PP == 2) hb2::prune_small_walk_kernel<4, 2><<<grid, 128, 0, p->stream>>>(a, p->d_jobs, n);
                else hb2::prune_small_walk_kernel<4, 1><<<grid, 128, 0, p->stream>>>(a, p->d_jobs, n);
                break;
            case 8: hb2::prune_small_walk_kernel<8, 1><<<grid, 128, 0, p->stream>>>(a, p->d_jobs, n); break;
            default: return fail("unsupported padded state count %d", p->Dp);
        }
    }
    p->launches++;
    CU(cudaGetLastError());
    return 0;
}

// 33..64 states in fp64: one launch, K in-order lanes per (class, 32-pattern tile) (prune64_lanes_kernel).  Same
// planner and plan cache as the tensor walk; the step list travels without a generation table (hand-over by pass id).
int run_fp64_lanes(hb2_partition *p, int cat0, int ncls, const std::vector<char> &dirty) {
    const int I = (int)p->I, L = (int)p->L;
    const int total = (int)std::count(dirty.begin(), dirty.end(), 1);
    if (total == 0) return 0;
    const int T = (int)(p->Sp / hb2::LANES_TILE_P), CT = ncls * T, resident = p->lanes_resident;
    const int K = std::max(1, std::min(std::min(p->walk_lane_cap, total), resident / std::max(CT, 1)));
    const int nslots = (K == 1) ? std::min(CT, resident) : CT;
    int *buf = p->h_walk;
    bool rebuilt = false;
    const int ns = cached_plan(p, dirty, K, true, &rebuilt);
    if (rebuilt) {
        // the kernel's descriptors: (child, job, branch id of the lane's next contraction, -) behind the planner's pairs
        int *d4 = buf + ((16 + 2 * ns + 3) & ~3);
        std::vector<char> awaited(2 * I, 0);                 // jobs some other lane waits for: only those publish a flag
        for (int i = 0; i < ns; i++)
            if (buf[16 + 2 * i] & hb2::WALK_WAIT) awaited[(buf[16 + 2 * i] & hb2::WALK_ID_MASK) - L] = 1;
        for (int r = 0; r < K; r++) {
            int nextb = -1;
            for (int i = buf[r + 1] - 1; i >= buf[r]; i--) {
                const int enc = buf[16 + 2 * i], child = enc & hb2::WALK_ID_MASK;
                const int fl = buf[16 + 2 * i + 1];
                d4[4 * i] = enc; d4[4 * i + 1] = fl; d4[4 * i + 2] = nextb;
                d4[4 * i + 3] = ((fl & hb2::STEP_LAST) && awaited[fl & hb2::WALK_ID_MASK]) ? 1 : 0;
                if (child >= L && !(enc & hb2::WALK_MUL)) nextb = child;
            }
        }
    }
    const int o4 = (16 + 2 * ns + 3) & ~3;
    CU(cudaMemcpyAsync(p->d_walk, p->h_walk, (size_t)(o4 + 4 * ns) * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    hb2::LaneArgs w;
    w.a = prune_args(p, cat0);
    w.cond_side = p->d_cond_side;
    w.scal_side = p->d_scal + (size_t)p->C * I * p->Sp;
    w.lane_start = p->d_walk; w.steps = reinterpret_cast<const int4 *>(p->d_walk + o4);
    w.flags = p->d_lane_flags; w.err = p->d_err;
    w.K = K; w.T = T; w.ncls = ncls; w.nslots = nslots; w.pass = ++p->lane_pass;
    if (getenv("HB2_DEBUG")) fprintf(stderr, "[hb2] fp64 lanes: jobs=%d steps=%d K=%d T=%d ncls=%d nslots=%d grid=%d resident=%d\n", total, ns, K, T, ncls, nslots, nslots * K, resident);
    WalkTrace trace;
    if (trace.alloc(p, ns, 0)) return 1;
    w.trace = trace.d; w.trace_cta = trace.cta;
    hb2::prune64_lanes_kernel<<<nslots * K, hb2::LANES_THREADS, hb2::LANES_SMEM_BYTES, p->stream>>>(w);
    if (trace.write(p, "fp64 lanes kernel, ", "child_enc job_flags begin staged landed barrier product barrier2 body_end stored barrier3 published", K)) return 1;
    p->launches++;
    CU(cudaGetLastError());
    return 0;
}

// One launch per evaluation, of the kernel pruning_kernel chooses.
int run_pruning(hb2_partition *p, int cat0, int ncls, const std::vector<char> &dirty) {
    const PruneKernel kernel = pruning_kernel(p, ncls);
    if (kernel == TC_WALK) return run_walk(p, cat0, ncls, dirty);
    if (kernel == FP64_LANES) return run_fp64_lanes(p, cat0, ncls, dirty);
    return run_small_walk(p, cat0, ncls, dirty, kernel);
}

// (Re)creates the peer-exchange buffers with room for `payload` doubles per rank and maps every other rank's buffer through
// CUDA IPC; the 64-byte handles travel over the partition's NCCL communicator.  Collective: every rank calls it with the
// same payload.  On any failure (IPC not permitted in this container, no peer access) ALL ranks fall back to NCCL.
void peer_teardown(hb2_partition *p) {
    for (size_t r = 0; r < p->px_peer.size(); r++)
        if ((int)r != p->rank && p->px_peer[r]) cudaIpcCloseMemHandle(p->px_peer[r]);
    p->px_peer.clear();
    if (p->px_local) cudaFree(p->px_local);
    p->px_local = nullptr; p->d_px_peer = {}; p->d_px_counter = {}; p->px_ok = false;
}

int peer_setup(hb2_partition *p, int payload) {
    peer_teardown(p);
    { const char *env = getenv("HB2_PEER_XCHG"); p->px_enabled = !(env && env[0] == '0'); }
    if (!p->comm || p->n_ranks < 2 || p->n_ranks > 64) return 0;
    const int R = p->n_ranks;
    const size_t doubles = (size_t)2 * R * payload + (size_t)2 * R;          // data + flags (uint64 = double sized)
    int ok = p->px_enabled ? 1 : 0;
    cudaIpcMemHandle_t mine;
    memset(&mine, 0, sizeof mine);
    if (ok && cudaMalloc(&p->px_local, doubles * sizeof(double)) != cudaSuccess) { cudaGetLastError(); p->px_local = nullptr; ok = 0; }
    if (ok) {
        CU(cudaMemsetAsync(p->px_local, 0, doubles * sizeof(double), p->stream));
        if (cudaIpcGetMemHandle(&mine, p->px_local) != cudaSuccess) { cudaGetLastError(); ok = 0; }
    }
    // exchange {ok, handle} of every rank: one all-gather of 72 bytes per rank
    const size_t rec = 8 + sizeof(cudaIpcMemHandle_t);
    std::vector<unsigned char> sendrec(rec, 0), all(rec * R, 0);
    memcpy(sendrec.data(), &ok, sizeof(int));
    memcpy(sendrec.data() + 8, &mine, sizeof mine);
    DeviceBuffer<unsigned char> d_send, d_all;
    if (d_send.alloc(rec) || d_all.alloc(rec * R)) return 1;
    CU(cudaMemcpyAsync(d_send, sendrec.data(), rec, cudaMemcpyHostToDevice, p->stream));
    ncclResult_t nr = g_nccl.AllGather(d_send, d_all, rec, ncclChar, p->comm, p->stream);
    if (nr != ncclSuccess) return fail("ncclAllGather (IPC handles): %s", g_nccl.GetErrorString(nr));
    CU(cudaMemcpyAsync(all.data(), d_all, rec * R, cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    int all_ok = 1;
    for (int r = 0; r < R; r++) { int o; memcpy(&o, all.data() + rec * r, sizeof(int)); all_ok = all_ok && o; }
    p->px_peer.assign(R, nullptr);
    if (all_ok) {
        for (int r = 0; r < R && all_ok; r++) {
            if (r == p->rank) { p->px_peer[r] = p->px_local; continue; }
            cudaIpcMemHandle_t h;
            memcpy(&h, all.data() + rec * r + 8, sizeof h);
            void *ptr = nullptr;
            if (cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); all_ok = 0; }
            p->px_peer[r] = static_cast<double *>(ptr);
        }
    }
    // the mapping must have worked on EVERY rank: agree with a max-reduce of "failed"
    DeviceBuffer<int> d_flag2;
    if (d_flag2.alloc(1)) return 1;
    int failed = all_ok ? 0 : 1;
    CU(cudaMemcpyAsync(d_flag2, &failed, sizeof(int), cudaMemcpyHostToDevice, p->stream));
    nr = g_nccl.AllReduce(d_flag2, d_flag2, 1, ncclInt32, ncclMax, p->comm, p->stream);
    if (nr != ncclSuccess) return fail("ncclAllReduce (IPC agreement): %s", g_nccl.GetErrorString(nr));
    CU(cudaMemcpyAsync(&failed, d_flag2, sizeof(int), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    if (failed) {
        const bool wanted = p->px_enabled;
        peer_teardown(p);
        if (wanted && getenv("HB2_DEBUG")) fprintf(stderr, "[hb2] rank %d: peer exchange unavailable (CUDA IPC), using NCCL collectives\n", p->rank);
        return 0;
    }
    if (p->d_px_peer.alloc(R)) return 1;
    CU(cudaMemcpyAsync(p->d_px_peer, p->px_peer.data(), R * sizeof(double *), cudaMemcpyHostToDevice, p->stream));
    if (p->d_px_counter.alloc(1) || p->d_px_counter.zero(p->stream)) return 1;
    p->px_payload = payload; p->px_gen = 0; p->px_ok = true;
    return 0;
}

hb2::PeerBuf peer_buf(hb2_partition *p) {
    hb2::PeerBuf b;
    b.peer = p->d_px_peer; b.R = p->n_ranks; b.rank = p->rank; b.payload = p->px_payload; b.gen = ++p->px_gen; b.err = p->d_err;
    return b;
}

int run_root(hb2_partition *p, int c0, int nc, bool use_weights, bool want_sites) {
    if (p->cg_G > 1) CU(cudaMemsetAsync(p->d_flag, 0, sizeof(int), p->stream));
    hb2::CombineArgs c;
    c.counter = nullptr; c.out = nullptr;
    c.rootL = p->d_rootL; c.rootE = p->d_rootE; c.weights = use_weights ? p->d_weights : (double *)nullptr; c.freq = p->d_freq;
    c.partial = p->d_partial; c.flag = p->d_flag; c.siteL = want_sites ? p->d_siteL : (double *)nullptr;
    c.siteScale = want_sites ? p->d_siteScale : (long long *)nullptr;
    c.Sp = (int)p->Sp; c.S = (int)p->S; c.c0 = c0; c.nc = nc;
    if (p->cg_G > 1 && p->px_ok) {
        // class groups over NVLink peer memory: ONE kernel computes this rank's class partials, stores them into every
        // rank's exchange buffer, and (its last block) merges all shards and classes into the complete lnL
        hb2::ClassXchgArgs x;
        x.rootL = p->d_rootL; x.rootE = p->d_rootE; x.weights = p->d_weights; x.Sp = (int)p->Sp; x.S = (int)p->S; x.c0 = p->own0; x.nc = p->ownN;
        x.xs = p->xchg_len; x.pb = peer_buf(p); x.xfreq = p->d_xfreq; x.nShards = p->n_ranks / p->cg_G; x.G = p->cg_G; x.myShard = p->rank / p->cg_G;
        x.lnL = p->d_lnL; x.siteL = c.siteL; x.siteScale = c.siteScale; x.counter = p->d_px_counter;
        const int nblk = std::max(1, std::min(16, (p->xchg_len + 255) / 256));
        hb2::class_exchange_kernel<<<nblk, 256, 0, p->stream>>>(x);
        p->launches++;
        CU(cudaGetLastError());
        return 0;
    }
    if (p->cg_G > 1) {
        // class groups without peer mapping: partial over the owned classes into this rank's slot of a buffer that is zero
        // elsewhere; ONE sum all-reduce then acts as the gather (every rank merges every shard and holds the complete lnL)
        const int xs = p->xchg_len, N = p->n_ranks;
        hb2::class_partial_kernel<<<(xs + 255) / 256, 256, 0, p->stream>>>(p->d_rootL, p->d_rootE, p->d_weights, (int)p->Sp, (int)p->S,
                                                                          p->own0, p->ownN, p->d_xsend + (size_t)p->rank * 2 * xs, xs);
        ncclResult_t r = g_nccl.AllReduce(p->d_xsend, p->d_xrecv, (size_t)2 * xs * N, ncclDouble, ncclSum, p->comm, p->stream);
        if (r != ncclSuccess) return fail("ncclAllReduce (class partials): %s", g_nccl.GetErrorString(r));
        const int nblk = (N / p->cg_G * xs + 255) / 256;
        hb2::class_merge_kernel<<<nblk, 256, 0, p->stream>>>(p->d_xrecv, p->d_xfreq, xs, N / p->cg_G, p->cg_G, p->rank / p->cg_G, p->d_xpartial,
                                                             p->d_flag, c.siteL, c.siteScale, (int)p->S);
        hb2::final_sum_kernel<<<1, 256, 0, p->stream>>>(p->d_xpartial, nblk, p->d_flag, p->d_lnL);
        p->launches += 3;
        CU(cudaGetLastError());
        return 0;
    }
    // single GPU or pattern shards: combine + sum in one kernel (its last block)
    c.counter = p->d_root_counter; c.out = p->d_lnL;
    hb2::combine_kernel<<<p->n_partial_blocks, 256, 0, p->stream>>>(c);
    p->launches += 1;
    CU(cudaGetLastError());
    if (p->comm && p->px_ok) {                // pattern shards: R partial lnL over peer memory, summed in rank order
        hb2::peer_sum_kernel<<<1, 64, 0, p->stream>>>(peer_buf(p), p->d_lnL);
        p->launches++;
        CU(cudaGetLastError());
    } else if (p->comm) {
        ncclResult_t r = g_nccl.AllReduce(p->d_lnL, p->d_lnL, 1, ncclDouble, ncclSum, p->comm, p->stream);
        if (r != ncclSuccess) return fail("ncclAllReduce: %s", g_nccl.GetErrorString(r));
    }
    return 0;
}

int check_ready(hb2_partition *p, int c0, int nc) {
    for (int c = c0; c < c0 + nc; c++)
        for (int64_t b = 0; b < p->B; b++)
            if (!p->slots[c * p->B + b].have)
                return fail("no matrix was ever set for rate class %d, node %lld", c, (long long)b);
    return 0;
}

int evaluate_impl(hb2_partition *p, int c0, int nc, const double *weights, int64_t nUpdate, const int64_t *updateNodes,
                  const double *rootFreqs, double *lnL, double *siteL, int64_t *siteScale, int64_t forcedNode = -1,
                  const int64_t *forcedStates = nullptr) {
    if (!p) return fail("null partition");
    if (!rootFreqs || !lnL) return fail("rootFreqs and lnL must not be null");
    CU(cudaSetDevice(p->device));
    p->forced_node = -1;
    if (forcedNode >= 0) {
        if (forcedNode >= p->L + p->I) return fail("forced node %lld out of range", (long long)forcedNode);
        if (!forcedStates) return fail("forced states are null");
        // keyed on the last of the pair: after a failed allocation the next call allocates both again
        if (!p->h_forced && (p->d_forced.alloc(p->Sp) || p->h_forced.alloc(p->Sp))) return 1;
        CU(cudaStreamSynchronize(p->stream));         // h_forced may still be in flight from the previous forced evaluation
        for (int64_t s = 0; s < p->Sp; s++) {
            const int64_t f = s < p->S ? forcedStates[s] : 0;
            if (f < 0 || f >= p->D) return fail("forced state %lld of pattern %lld out of range", (long long)f, (long long)s);
            p->h_forced[s] = (int)f;
        }
        CU(cudaMemcpyAsync(p->d_forced, p->h_forced, p->Sp * sizeof(int), cudaMemcpyHostToDevice, p->stream));
        p->forced_node = (int)forcedNode;
    }
    if (check_ready(p, c0, nc)) return 1;
    if (p->cg_G > 1) {
        if (!weights || c0 != 0 || nc != (int)p->C) return fail("with class groups only hb2_evaluate_classes is available");
        c0 = p->own0;                          // prune the owned classes; the weights of all C classes are still uploaded
    }
    p->bc_node = -1; p->bc_dirty_node = -1;     // conditionals are about to change: the branch cache is stale
    const int nw = nc;                         // number of class weights the caller passed
    if (p->cg_G > 1) nc = p->ownN;
    if (flush_matrices(p)) return 1;
    if (p->walk_reset) {                      // an earlier pass was aborted half-way: its tags are inconsistent
        if (p->d_condf.zero(p->stream) || p->d_scal.zero(p->stream) || p->d_err.zero(p->stream)) return 1;
        std::fill(p->walk_gen.begin(), p->walk_gen.end(), 0);
        std::fill(p->evaluated_cat.begin(), p->evaluated_cat.end(), 0);
        p->walk_reset = false;
    }
    if (stage_root(p, rootFreqs, weights, nw)) return 1;
    double *hs = p->h_small;
    // classes never pruned before need the whole tree regardless of updateNodes (likefunc.cpp:10965-10967)
    bool all = (updateNodes == nullptr || nUpdate < 0);
    for (int c = c0; c < c0 + nc; c++) if (!p->evaluated_cat[c]) all = true;
    std::vector<char> dirty;
    if (dirty_nodes(p->parents.data(), p->L, p->I, all ? -1 : nUpdate, all ? nullptr : updateNodes, dirty)) return 1;
    // the root must always be recomputed when anything changed; if nothing is dirty (only pi/weights changed)
    // the root tile products are still valid but rootL depends on pi -> recompute the root node
    if (std::count(dirty.begin(), dirty.end(), 1) == 0) dirty[p->I - 1] = 1;
    if (run_pruning(p, c0, nc, dirty)) return 1;
    const bool want_sites = siteL != nullptr || siteScale != nullptr;
    if (run_root(p, c0, nc, weights != nullptr, want_sites)) return 1;
    CU(cudaMemcpyAsync(hs + p->Dp + p->C, p->d_lnL, sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaMemcpyAsync(hs + p->Dp + p->C + 1, p->d_err, sizeof(int), cudaMemcpyDeviceToHost, p->stream));
    if (siteL) CU(cudaMemcpyAsync(siteL, p->d_siteL, p->S * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    if (siteScale) CU(cudaMemcpyAsync(siteScale, p->d_siteScale, p->S * sizeof(long long), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    if (const int code = *reinterpret_cast<int *>(hs + p->Dp + p->C + 1)) {
        p->walk_reset = p->use_tc;          // tags are inconsistent: the next pass starts from scratch
        cudaMemsetAsync(p->d_err, 0, sizeof(int), p->stream);   // on every path, or each later evaluation would fail too
        std::fill(p->evaluated_cat.begin(), p->evaluated_cat.end(), 0);
        return wait_timeout(code);
    }
    *lnL = hs[p->Dp + p->C];
    for (int c = c0; c < c0 + nc; c++) p->evaluated_cat[c] = 1;
    return 0;
}

// CTAs of a lane kernel (the tensor walk or the fp64 lanes kernel) that one SM holds: what the occupancy API reports or,
// where that is more, what the registers and shared memory allow up to `cap` (the API under-reports for the tensor walk
// kernel).  HB2_WALK_CTAS_PER_SM overrides the result.  Correctness does not depend on it: blocks are dispatched in index
// order and a lane only waits for lanes of its own unit -- adjacent block indices -- with time-bounded waits, so fewer
// resident CTAs than planned only make the pass slower.
int lane_ctas_per_sm(const char *name, const void *fn, int threads, int smem, int cap, int device, int &per_sm) {
    CU(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CU(cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, threads, smem));
    cudaFuncAttributes fa;
    CU(cudaFuncGetAttributes(&fa, fn));
    cudaDeviceProp dp;
    CU(cudaGetDeviceProperties(&dp, device));
    const int regs_per_cta = ((fa.numRegs + 7) / 8 * 8) * threads;
    const size_t smem_per_cta = (size_t)smem + fa.sharedSizeBytes + dp.reservedSharedMemPerBlock;
    const int by_res = std::min(dp.regsPerMultiprocessor / std::max(regs_per_cta, 1), (int)(dp.sharedMemPerMultiprocessor / smem_per_cta));
    if (getenv("HB2_DEBUG"))
        fprintf(stderr, "[hb2] %s occupancy: API %d, by resources %d CTAs/SM (regs/thread %d, static smem %zu, dyn smem %d, regs/SM %d, smem/SM %zu, reserved/block %zu)\n",
                name, per_sm, by_res, fa.numRegs, fa.sharedSizeBytes, smem, dp.regsPerMultiprocessor, dp.sharedMemPerMultiprocessor, dp.reservedSharedMemPerBlock);
    per_sm = std::max(per_sm, std::min(by_res, cap));
    if (const char *ov = getenv("HB2_WALK_CTAS_PER_SM")) per_sm = atoi(ov);      // bring-up override
    return 0;
}

// ---- Simulation (hb2_simulate) --------------------------------------------------------------------------------------------
constexpr int64_t SIM_CHUNK = (int64_t)1 << 18;    // sites per simulate_kernel launch
constexpr int SIM_THREADS = 128;
constexpr size_t SIM_SMEM_MAX = 48 << 10;          // internal states of a CTA's sites in shared memory up to this size

// Prefix sums of a weight vector by the draw rule and its last positive index.  False when an entry is negative or NaN or
// the total is not finite and > 0.
bool sim_prefix(const double *v, int64_t m, double *c, int *last) {
    double s = 0.0;
    *last = -1;
    for (int64_t j = 0; j < m; j++) {
        if (!(v[j] >= 0.0)) return false;
        if (v[j] > 0.0) { s += v[j]; *last = (int)j; }
        c[j] = s;
    }
    return s > 0.0 && std::isfinite(s);
}

// Set-up of hb2_simulate and of each chunk of hb2_batch_site_simulate, whose table holds `nblk` blocks (rate classes, or
// sets) of B matrices of a.PT: reserves the scratch for `chunk` columns per launch, uploads the prefix sums `cdf` (class
// weights, if any | root frequencies) and `ints` (active blocks [nblk] | last class | last root state | first bad row),
// fills the fields of `a` both calls share, and builds and checks the table.  A bad row refuses the call before any column
// is drawn, as "<fn>: row r of the transition matrix of <block>", `block` formatting (blk0 + block, branch).
int sim_tables(hb2_partition *p, hb2::SimArgs &a, int64_t nblk, int64_t chunk, uint64_t seed, const std::vector<double> &cdf,
               const std::vector<int> &ints, bool nodes, bool classes, bool mix, const char *fn, const char *block, int64_t blk0) {
    const int64_t B = p->B, D = p->D, L = p->L, I = p->I;
    const bool smem_states = (size_t)I * SIM_THREADS <= SIM_SMEM_MAX;
    hb2_partition::SimBuf &sb = p->sim;
    if (sb.cdf.reserve((size_t)nblk * B * D * p->Dp, p->stream) || sb.vec.reserve(cdf.size(), p->stream) ||
        sb.ints.reserve((size_t)nblk * B * D + ints.size(), p->stream) || sb.leaf.reserve((size_t)L * chunk, p->stream) ||
        (nodes && sb.node.reserve((size_t)I * chunk, p->stream)) || (classes && sb.cls.reserve((size_t)chunk, p->stream)) ||
        (!smem_states && sb.states.reserve((size_t)I * chunk, p->stream)))
        return 1;
    int *d_ints = sb.ints + nblk * B * D;
    CU(cudaMemcpyAsync(sb.vec, cdf.data(), cdf.size() * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    CU(cudaMemcpyAsync(d_ints, ints.data(), ints.size() * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    a.cdf = sb.cdf; a.last = sb.ints; a.class_cdf = sb.vec; a.root_cdf = sb.vec + (cdf.size() - D);
    a.active = d_ints; a.class_last = d_ints + nblk; a.root_last = d_ints + nblk + 1; a.bad = d_ints + nblk + 2;
    a.tree.child_start = p->d_child_start; a.tree.child_ids = p->d_child_ids;
    a.leaf_out = sb.leaf; a.node_out = nodes ? (long long *)sb.node : nullptr; a.class_out = classes ? (int *)sb.cls : nullptr;
    a.states = smem_states ? nullptr : (unsigned char *)sb.states;
    a.L = (int)L; a.I = (int)I; a.B = (int)B; a.D = (int)D; a.Dp = p->Dp; a.chunk = (int)chunk;
    a.key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
    if (mix) hb2::sim_cdf_kernel<true><<<(unsigned)(nblk * B), 64, 0, p->stream>>>(a);
    else hb2::sim_cdf_kernel<false><<<(unsigned)(nblk * B), 64, 0, p->stream>>>(a);
    p->launches++;
    CU(cudaGetLastError());
    int *chk = reinterpret_cast<int *>(p->h_small + p->Dp + p->C + 1);   // first bad row | device-side wait error
    CU(cudaMemcpyAsync(&chk[0], a.bad, sizeof(int), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaMemcpyAsync(&chk[1], p->d_err, sizeof(int), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    if (chk[1]) { cudaMemsetAsync(p->d_err, 0, sizeof(int), p->stream); return wait_timeout(chk[1]); }
    if (chk[0] != INT_MAX) {
        const long long row = chk[0] % D, cb = chk[0] / D;
        const std::string msg = std::string(fn) + ": row %lld of the transition matrix of " + block + " does not have a finite positive total";
        return fail(msg.c_str(), row, (long long)blk0 + cb / B, cb % B);
    }
    return 0;
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

int hb2_abi_version(void) { return HB2_ABI_VERSION; }
const char *hb2_last_error(void) { return g_err.c_str(); }

int hb2_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int hb2_create(hb2_partition **out, int64_t S, int64_t D, int64_t L, int64_t I, int64_t C, const int64_t *flatParents,
               const int64_t *leafState, const double *ambig, int64_t nAmb, const int64_t *patternFreq, int device,
               int flags) {
    if (!out) return fail("out is null");
    *out = nullptr;
    if (S <= 0 || D < 2 || L < 2 || I < 1 || C < 1) return fail("bad sizes S=%lld D=%lld L=%lld I=%lld C=%lld", (long long)S, (long long)D, (long long)L, (long long)I, (long long)C);
    if (!flatParents || !leafState || !patternFreq) return fail("null input array");
    if (nAmb > 0 && !ambig) return fail("nAmb > 0 but ambig is null");
    const int Dp = pad_states(D);
    if (Dp < 0) return fail("state count %lld not supported (max 64)", (long long)D);
    // the kernels sum an ambiguity row's allowed states with the row's weight, which is the reference's only for 0/1 rows
    for (int64_t i = 0; i < nAmb * D; i++)
        if (ambig[i] != 0.0 && ambig[i] != 1.0)
            return fail("ambiguity row %lld, state %lld: weight %g is neither 0 nor 1", (long long)(i / D), (long long)(i % D), ambig[i]);
    int ndev = hb2_device_count();
    if (ndev <= 0) return fail("no CUDA device visible: the engine has no CPU fallback");
    if (device < 0 || device >= ndev) return fail("device %d out of range (%d visible)", device, ndev);
    CU(cudaSetDevice(device));

    std::unique_ptr<hb2_partition, decltype(&hb2_destroy)> p(new hb2_partition(), hb2_destroy);   // destroyed on any early return
    cudaDeviceGetAttribute(&p->sm_count, cudaDevAttrMultiProcessorCount, device);
    p->device = device; p->flags = flags; p->S = S; p->D = D; p->L = L; p->I = I; p->C = C; p->B = L + I - 1; p->nAmb = nAmb;
    p->Dp = Dp;
    p->use_tc = (Dp == 64) && !(flags & HB2_FLAG_FORCE_FP64);
    // pattern padding: fp64 codon partitions to 64 (a multiple of the 32-pattern lanes-kernel tile), all others to 128
    const int64_t tile = (Dp == 64 && !p->use_tc) ? 64 : 128;
    p->Sp = (S + tile - 1) / tile * tile;
    p->parents.assign(flatParents, flatParents + L + I);
    if (build_tree(flatParents, L, I, p->children, p->height)) return 1;
    for (int64_t k = 0; k < L * S; k++) {
        int64_t c = leafState[k];
        if (c >= D || c < -nAmb) return fail("leafState[%lld]=%lld out of range", (long long)k, (long long)c);
    }
    if (const char *ov = getenv("HB2_WALK_LANES")) p->walk_lane_cap = std::max(1, std::min(atoi(ov), 15));
    { const char *ev = getenv("HB2_WALK_SPLIT_NODES"); p->walk_split_nodes = !(ev && ev[0] == '0'); }
    CU(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
    for (auto &e : p->ev) CU(cudaEventCreate(&e));
    CU(cudaEventCreateWithFlags(&p->ev_staging, cudaEventDisableTiming));
    CU(cudaStreamCreateWithFlags(&p->side, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&p->ev_join, cudaEventDisableTiming));
    const size_t Sp = p->Sp, dpdp = (size_t)Dp * Dp, dd = (size_t)D * D;
    cudaStream_t st = p->stream;
    if (p->d_leaf.alloc(L * Sp) || p->d_ambig.alloc(std::max<int64_t>(nAmb, 1) * Dp) || p->d_freq.alloc(Sp)) return 1;
    if (p->use_tc) {
        // 2I node slots per class: I nodes + I side products of the walk kernel
        if (p->d_condf.alloc((size_t)C * 2 * I * Sp * 64) || p->d_PB.alloc((size_t)C * p->B * hb2::TC_PB_FLOATS) ||
            p->d_PTf.alloc((size_t)C * p->B * hb2::TC_PTF_FLOATS) || p->d_condf.zero(st) || p->d_PB.zero(st) || p->d_PTf.zero(st))
            return 1;
        int per_sm = 0;
        if (lane_ctas_per_sm("prune64_tc_walk_kernel", (const void *)hb2::prune64_tc_walk_kernel, 256, hb2::WALK_SMEM_BYTES, 2, device, per_sm)) return 1;
        p->walk_max_resident = std::min(per_sm, 2) * p->sm_count;
        if (p->walk_max_resident < 1)
            return fail("prune64_tc_walk_kernel (%d B of shared memory) cannot be resident on device %d", hb2::WALK_SMEM_BYTES, device);
        p->walk_gen.assign((size_t)C * 2 * I, 0);   // matches the zero-filled conditional and exponent buffers
        const size_t walk_ints = 16 + 2 * (size_t)(L + 2 * I) + (size_t)C * 2 * I;
        if (p->d_walk.alloc(walk_ints) || p->h_walk.alloc(walk_ints)) return 1;
    } else {
        if (p->d_cond.alloc((size_t)C * I * Sp * Dp) || p->d_cond.zero(st)) return 1;
        if (Dp == 64) {
            // lanes kernel: side products, hand-over flags, the step list, and how many CTAs can be co-resident
            const size_t T = Sp / hb2::LANES_TILE_P;
            const size_t walk_ints = 16 + 6 * (size_t)(L + 2 * I) + 4;       // planner's pairs + the kernel's int4 descriptors
            if (p->d_cond_side.alloc((size_t)C * I * Sp * 64) || p->d_cond_side.zero(st) || p->d_lane_flags.alloc((size_t)C * 2 * I * T) ||
                p->d_lane_flags.zero(st) || p->d_walk.alloc(walk_ints) || p->h_walk.alloc(walk_ints))
                return 1;
            int per_sm = 0;
            if (lane_ctas_per_sm("prune64_lanes_kernel", (const void *)hb2::prune64_lanes_kernel, hb2::LANES_THREADS, hb2::LANES_SMEM_BYTES,
                                 hb2::LANES_CTAS_PER_SM, device, per_sm))
                return 1;
            p->lanes_resident = std::max(per_sm, 1) * p->sm_count;
        }
    }
    if (p->d_err.alloc(1) || p->d_err.zero(st)) return 1;
    if (p->d_scal.alloc((size_t)C * 2 * I * Sp) || p->d_PT.alloc((size_t)C * p->B * dpdp) || p->d_Qres.alloc((size_t)C * p->B * dd)) return 1;   // 2I: see d_condf
    if (p->dense.alloc(C * p->B, dd) || p->d_pi.alloc(Dp) || p->d_rootL.alloc((size_t)C * Sp) || p->d_rootE.alloc((size_t)C * Sp) ||
        p->d_weights.alloc(C))
        return 1;
    p->n_partial_blocks = (int)((S + 255) / 256);
    if (p->d_partial.alloc(p->n_partial_blocks) || p->d_lnL.alloc(1) || p->d_flag.alloc(1) || p->d_flag.zero(st) || p->d_root_counter.alloc(1) ||
        p->d_root_counter.zero(st))
        return 1;
    if (p->d_siteL.alloc(Sp) || p->d_siteScale.alloc(Sp) || p->d_jobs.alloc(I) || p->d_child_start.alloc(I + 1) || p->d_child_ids.alloc(L + I)) return 1;
    if (p->h_small.alloc(Dp + C + 8) || p->h_jobs.alloc(I)) return 1;
    if (p->d_scal.zero(st) || p->d_PT.zero(st) || p->d_rootL.zero(st) || p->d_rootE.zero(st)) return 1;
    {   // static uploads (pageable host vectors: released once the copies are enqueued)
        std::vector<int> leaf((size_t)L * Sp, 0);          // padding patterns: state 0 everywhere, frequency 0
        for (int64_t l = 0; l < L; l++)
            for (int64_t s = 0; s < S; s++) leaf[l * Sp + s] = (int)leafState[l * S + s];
        std::vector<double> amb((size_t)std::max<int64_t>(nAmb, 1) * Dp, 0.0);
        for (int64_t a = 0; a < nAmb; a++)
            for (int64_t k = 0; k < D; k++) amb[a * Dp + k] = ambig[a * D + k];
        std::vector<double> fr(Sp, 0.0);
        for (int64_t s = 0; s < S; s++) fr[s] = (double)patternFreq[s];
        std::vector<int> cs(I + 1, 0), ci;
        for (int64_t i = 0; i < I; i++) { cs[i] = (int)ci.size(); for (int ch : p->children[i]) ci.push_back(ch); }
        cs[I] = (int)ci.size();
        CU(cudaMemcpyAsync(p->d_leaf, leaf.data(), leaf.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(p->d_ambig, amb.data(), amb.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(p->d_freq, fr.data(), fr.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(p->d_child_start, cs.data(), cs.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(p->d_child_ids, ci.data(), ci.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    }
    if (expm_setup(Dp, device)) return 1;
    if (Dp == 64) {
        { const char *env = getenv("HB2_EXPM_SHARED"); p->ex_enabled = !(env && env[0] == '0'); }
        if (p->ex.alloc(std::max((int)C + 8, HB2_MAX_TEMPLATES * (int)C), (int64_t)(C + 8) * p->B, st)) return 1;
    }
    if (Dp == 4) {
        if (const char *env = getenv("HB2_SMALL_ILP")) p->small_ilp = atoi(env);
        int b1 = 0, b2 = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b1, hb2::prune_small_walk_kernel<4, 1>, 128, 0);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b2, hb2::prune_small_walk_kernel<4, 2>, 128, 0);
        p->small_resident[0] = std::max(b1, 1) * p->sm_count;
        p->small_resident[1] = std::max(b2, 1) * p->sm_count;
    }
    p->slots.assign(C * p->B, Slot());
    p->evaluated_cat.assign(C, 0);
    p->own0 = 0; p->ownN = (int)C;
    *out = p.release();
    return 0;
}

// Body of both dense entry points: matrix k is at M[k] (pointer array) or at packed + k*D*D.
static int set_dense(hb2_partition *p, int64_t cat, int64_t n, const int64_t *nodeIds, const double *const *M, const double *packed, int kind) {
    if (!p) return fail("null partition");
    if (n < 0 || (n > 0 && (!nodeIds || !(M || packed)))) return fail("bad matrix list");
    bool stage;
    if (accept_handover(p, cat, n, nodeIds, stage, kind, M)) return 1;
    const size_t dd = (size_t)p->D * p->D;
    for (int64_t k = 0; stage && k < n; k++)
        if (enqueue(p, DENSE_QUEUE, cat * p->B + nodeIds[k], M ? M[k] : packed + k * dd, (Kind)kind)) return 1;
    return 0;
}

int hb2_set_matrices(hb2_partition *p, int64_t cat, int64_t n, const int64_t *nodeIds, const double *const *M, int kind) {
    return set_dense(p, cat, n, nodeIds, M, nullptr, kind);
}

int hb2_set_matrices_packed(hb2_partition *p, int64_t cat, int64_t n, const int64_t *nodeIds, const double *M, int kind) {
    return set_dense(p, cat, n, nodeIds, nullptr, M, kind);
}

int hb2_set_mixture_matrices(hb2_partition *p, int64_t cat, int64_t n, const int64_t *nodeIds, int64_t K, const double *M,
                             const double *w) {
    if (!p) return fail("null partition");
    if (n < 0 || K < 1 || (n > 0 && (!nodeIds || !M || !w))) return fail("bad mixture arguments");
    bool stage;
    if (accept_handover(p, cat, n, nodeIds, stage)) return 1;
    if (!stage || n == 0) return 0;
    CU(cudaSetDevice(p->device));
    if (flush_matrices(p)) return 1;         // keep ordering with plain matrices staged earlier (same stream)
    // Two launches, no host synchronisation: all n*K components are exponentiated side by side into a scratch area
    // (one CTA each), then one CTA per node forms sum_k w_k Exp(Q_k) in component order (deterministic) and emits the
    // tensor-path operands.  Own pinned staging: [n*K matrices | n*K weights], then the n destination slots as ints.
    const size_t dd = (size_t)p->D * p->D, dpdp = (size_t)p->Dp * p->Dp;
    const int64_t nk = n * K;
    if (wait_staging(p)) return 1;
    if (p->d_mix_scratch.reserve((size_t)nk * dpdp, p->stream) || p->d_mix_Q.reserve((size_t)nk * (dd + 1), p->stream) ||
        p->d_mix_dst.reserve((size_t)2 * nk, p->stream) ||
        p->h_mix.reserve((size_t)nk * (dd + 2), p->stream))      // 2 nk ints take nk doubles
        return 1;
    memcpy(p->h_mix, M, (size_t)nk * dd * sizeof(double));
    memcpy(p->h_mix + (size_t)nk * dd, w, (size_t)nk * sizeof(double));
    int *h_idx = reinterpret_cast<int *>(p->h_mix + (size_t)nk * (dd + 1));      // [nk] scratch slots 0..nk-1 | [n] P-cache slots
    for (int64_t k = 0; k < nk; k++) h_idx[k] = (int)k;
    for (int64_t i = 0; i < n; i++) h_idx[nk + i] = (int)(cat * p->B + nodeIds[i]);
    CU(cudaMemcpyAsync(p->d_mix_Q, p->h_mix, (size_t)nk * (dd + 1) * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    CU(cudaMemcpyAsync(p->d_mix_dst, h_idx, (size_t)(nk + n) * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    // component k of every node is (in BS-REL / BUSTED models) the same rate matrix up to the branch length: the components
    // form shared-powers groups C + k
    SharedPlan sp;
    if (K <= 8) {
        std::vector<int> grp(nk);
        for (int64_t k = 0; k < nk; k++) grp[k] = (int)(p->C + k % K);
        if (plan_shared(p, h_idx, nk, 2, grp.data(), sp)) return 1;
    }
    if (staged_uploads(p)) return 1;
    if (launch_expm(p, {Kind::Rate}, p->d_mix_Q, p->d_mix_dst, (int)nk, false, sp, 0, p->d_mix_scratch)) return 1;
    hb2::mix_reduce_kernel<<<(unsigned)n, 256, 0, p->stream>>>(p->d_mix_scratch, p->d_mix_Q + (size_t)nk * dd, p->d_mix_dst + nk, (int)K, p->Dp,
                                                              p->d_PT, p->use_tc ? p->d_PB : (float *)nullptr, p->d_PTf);
    p->launches++;
    CU(cudaGetLastError());
    for (int64_t i = 0; i < n; i++) {
        Slot &s = p->slots[cat * p->B + nodeIds[i]];
        s.have = true;
        s.res = Resident::None;
    }
    return 0;
}

int hb2_set_rate_template_id(hb2_partition *p, int64_t templateId, int64_t nnz, const int64_t *entryIndex, const int64_t *entryFormula,
                             int64_t nFormulas, const double *colFreq) {
    if (!p) return fail("null partition");
    if (templateId < 0 || templateId >= HB2_MAX_TEMPLATES) return fail("template id %lld out of range (0..%d)", (long long)templateId, HB2_MAX_TEMPLATES - 1);
    if (nnz < 1 || nFormulas < 1 || !entryIndex || !entryFormula) return fail("bad template arguments");
    CU(cudaSetDevice(p->device));
    if (flush_matrices(p)) return 1;
    CU(cudaStreamSynchronize(p->stream));     // the template's buffers are about to be re-allocated
    std::vector<int> idx(nnz), frm(nnz);
    for (int64_t e = 0; e < nnz; e++) {
        if (entryIndex[e] < 0 || entryIndex[e] >= p->D * p->D) return fail("template entry %lld: index %lld out of range", (long long)e, (long long)entryIndex[e]);
        if (entryFormula[e] < 0 || entryFormula[e] >= nFormulas) return fail("template entry %lld: formula %lld out of range", (long long)e, (long long)entryFormula[e]);
        idx[e] = (int)entryIndex[e]; frm[e] = (int)entryFormula[e];
    }
    if ((int64_t)p->tmpls.size() <= templateId) p->tmpls.resize(templateId + 1);
    hb2_partition::Tmpl &t = p->tmpls[templateId];
    t = hb2_partition::Tmpl();                // undefined until every buffer is in place
    if (t.d_index.alloc(nnz) || t.d_formula.alloc(nnz) || t.d_colfreq.alloc(p->D) || t.h_colfreq.alloc(p->D) ||
        t.queue.alloc(p->C * p->B, nFormulas))
        return 1;
    // resident formula values of every slot (replay, shared-powers classification); cached directions of this template's
    // groups are void now
    if (t.d_Vres.alloc((size_t)p->C * p->B * nFormulas) || void_template_cache(p, (int)templateId)) return 1;
    CU(cudaMemcpyAsync(t.d_index, idx.data(), nnz * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    CU(cudaMemcpyAsync(t.d_formula, frm.data(), nnz * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    t.has_colfreq = colFreq != nullptr;
    if (colFreq && stage_colfreq(p, t, colFreq)) return 1;
    t.nnz = nnz; t.nF = nFormulas;
    return 0;
}

int hb2_set_rate_template(hb2_partition *p, int64_t nnz, const int64_t *entryIndex, const int64_t *entryFormula,
                          int64_t nFormulas, const double *colFreq) {
    return hb2_set_rate_template_id(p, 0, nnz, entryIndex, entryFormula, nFormulas, colFreq);
}

int hb2_set_template_frequencies(hb2_partition *p, int64_t templateId, const double *colFreq) {
    if (!p || !colFreq) return fail("null argument");
    if (templateId < 0 || templateId >= (int64_t)p->tmpls.size() || p->tmpls[templateId].nnz == 0) return fail("template %lld has not been defined", (long long)templateId);
    hb2_partition::Tmpl &t = p->tmpls[templateId];
    if (!t.has_colfreq) return fail("template %lld was defined without column frequencies", (long long)templateId);
    CU(cudaSetDevice(p->device));
    if (flush_matrices(p)) return 1;          // matrices handed over so far were assembled with the old frequencies
    if (stage_colfreq(p, t, colFreq)) return 1;
    return void_template_cache(p, (int)templateId);
}

int hb2_set_matrices_compiled_id(hb2_partition *p, int64_t templateId, int64_t cat, int64_t n, const int64_t *nodeIds, const double *formulaValues) {
    if (!p) return fail("null partition");
    if (templateId < 0 || templateId >= (int64_t)p->tmpls.size() || p->tmpls[templateId].nnz == 0) return fail("hb2_set_rate_template has not been called (template %lld)", (long long)templateId);
    if (n < 0 || (n > 0 && (!nodeIds || !formulaValues))) return fail("bad compiled matrix list");
    bool stage;
    if (accept_handover(p, cat, n, nodeIds, stage)) return 1;
    const int64_t nF = p->tmpls[templateId].nF;
    for (int64_t k = 0; stage && k < n; k++)
        if (enqueue(p, (int)templateId, cat * p->B + nodeIds[k], formulaValues + k * nF, Kind::Compiled)) return 1;
    return 0;
}

int hb2_set_matrices_compiled(hb2_partition *p, int64_t cat, int64_t n, const int64_t *nodeIds, const double *formulaValues) {
    return hb2_set_matrices_compiled_id(p, 0, cat, n, nodeIds, formulaValues);
}

int hb2_evaluate(hb2_partition *p, int64_t cat, int64_t nUpdate, const int64_t *updateNodes, const double *rootFreqs,
                 double *lnL, double *siteL, int64_t *siteScale) {
    if (!p) return fail("null partition");
    if (cat < 0) cat = 0;
    if (cat >= p->C) return fail("rate class %lld out of range", (long long)cat);
    return evaluate_impl(p, (int)cat, 1, nullptr, nUpdate, updateNodes, rootFreqs, lnL, siteL, siteScale);
}

int hb2_evaluate_forced(hb2_partition *p, int64_t cat, int64_t nUpdate, const int64_t *updateNodes, const double *rootFreqs,
                        int64_t forcedNode, const int64_t *forcedStates, double *lnL, double *siteL, int64_t *siteScale) {
    if (!p) return fail("null partition");
    if (cat < 0) cat = 0;
    if (cat >= p->C) return fail("rate class %lld out of range", (long long)cat);
    if (p->cg_G > 1) return fail("forced states are not available with class groups");
    return evaluate_impl(p, (int)cat, 1, nullptr, nUpdate, updateNodes, rootFreqs, lnL, siteL, siteScale, forcedNode, forcedStates);
}

int hb2_evaluate_classes(hb2_partition *p, const double *weights, int64_t nUpdate, const int64_t *updateNodes,
                         const double *rootFreqs, double *lnL, double *siteL, int64_t *siteScale) {
    if (!p) return fail("null partition");
    if (!weights) return fail("weights must not be null");
    return evaluate_impl(p, 0, (int)p->C, weights, nUpdate, updateNodes, rootFreqs, lnL, siteL, siteScale);
}

// A batch call: its entry point, the sets' models, and what it produces -- likelihoods (siteLnL) of partition patterns
// (patternOf) or of caller columns (columns [nSets][L], hb2_create's leaf codes), or nReps simulated columns of every set.
// weights == nullptr: one matrix per branch, row b = branch b (FEL's site model).  Otherwise branch b owns branchK[b]
// (NULL: K) consecutive component rows and its transition matrix is the weighted sum of their exponentials, formed inside
// prune_batch_kernel<true> or sim_cdf_kernel<true> (MEME's site model).
// Rates: set s is pattern patternOf[s] under the resident rate matrices of class `cat`, each multiplied by rates[s]
// (LEISR's site model); its P matrices come from expm_rates_kernel and its likelihood from prune_rates_kernel.
// BranchRows: MixtureSites, and after its pruning every component row of every branch pinned alone (rowLnL [nSets][R],
// branch_rows_kernel; MEME's branch-level empirical Bayes factors).  siteLnL is nullable there.
// LeafSupport: Sites (weights == nullptr) or MixtureSites, and after its pruning every leaf's support [nSets][L][D]
// (leaf_support_kernel; MEME's and PRIME's --impute-states).  siteLnL is nullable there.
// JointAncestors: Sites (weights == nullptr) or MixtureSites, its pruning only when siteLnL is given, then the joint ML
// states of every internal node (nodeStates [nSets][I], jointLnL; joint_ancestors_kernel; ancestral.build at every site
// of FEL, MEME and PRIME).
enum class BatchEntry { Sites, MixtureSites, Columns, Simulate, Rates, BranchRows, LeafSupport, JointAncestors };
struct BatchCall {
    BatchEntry entry;
    int64_t templateId, nSets, K;
    const int64_t *branchK, *branchGroup;
    const double *formulaValues, *weights, *rootFreqs;
    const int64_t *patternOf = nullptr, *columns = nullptr;
    double *siteLnL = nullptr;
    int64_t nReps = 0, firstSet = 0, firstRep = 0;
    uint64_t seed = 0;
    int64_t *leafStates = nullptr, *nodeStates = nullptr;
    int64_t cat = 0;
    const double *rates = nullptr;
    double *rowLnL = nullptr;
    double *support = nullptr;
    double *jointLnL = nullptr;
};

// Sets per chunk of hb2_batch_site_rates, whatever the memory rule allows: at 4 states and 256 taxa a chunk of this many
// sets holds 4.2 GB of P matrices, and its pruning launch fills every SM.
constexpr int64_t RATES_MAX_SETS = 65536;

// Every refusal of the batch entry points, before anything is launched or written.
static int check_batch(const hb2_partition *p, const BatchCall &c) {
    const bool rows = c.entry == BatchEntry::BranchRows, leaves = c.entry == BatchEntry::LeafSupport;
    const bool joint = c.entry == BatchEntry::JointAncestors;
    const bool sites = c.entry == BatchEntry::Sites || c.entry == BatchEntry::MixtureSites || rows || leaves || joint;
    const bool sim = c.entry == BatchEntry::Simulate;
    const char *fn = sim ? "hb2_batch_site_simulate" : "hb2_batch_column_likelihoods";
    if (!p) return fail(c.entry == BatchEntry::Sites ? "null argument" : "null partition");
    if (sites) {
        if (rows && !c.weights)
            return fail("hb2_batch_branch_component_likelihoods: weights must not be null (with one row per branch every row "
                        "would equal siteLnL)");
        if (rows && !c.rowLnL) return fail("hb2_batch_branch_component_likelihoods: rowLnL must not be null");
        if (leaves && !c.support) return fail("hb2_batch_leaf_support: support must not be null");
        if (joint && !c.nodeStates) return fail("hb2_batch_joint_ancestors: nodeStates must not be null");
        if (c.entry == BatchEntry::MixtureSites && !c.weights) return fail("weights must not be null");
        if (c.entry == BatchEntry::MixtureSites && !c.formulaValues) return fail("formulaValues must not be null");
        if (!c.formulaValues || !c.rootFreqs || (!c.siteLnL && !rows && !leaves && !joint) || !c.patternOf) return fail("null argument");
        if (c.nSets < 0) return fail("bad set count");
    } else {
        if (c.nSets < 0) return fail("%s: nSets=%lld is negative", fn, (long long)c.nSets);
        if (sim) {
            if (c.nReps < 0) return fail("%s: nReps=%lld is negative", fn, (long long)c.nReps);
            if (c.firstRep < 0 || c.firstRep > INT64_MAX - c.nReps) return fail("%s: firstRep=%lld out of range", fn, (long long)c.firstRep);
            if (c.firstSet < 0 || c.firstSet > ((int64_t)1 << 32) - c.nSets)
                return fail("%s: firstSet=%lld out of range (firstSet + nSets must not exceed 2^32)", fn, (long long)c.firstSet);
        } else if (!c.columns) {
            return fail("%s: columns must not be null", fn);
        }
        if (!c.formulaValues) return fail("%s: formulaValues must not be null", fn);
        if (!c.rootFreqs) return fail("%s: rootFreqs must not be null", fn);
        if (sim ? !c.leafStates : !c.siteLnL) return fail("%s: %s must not be null", fn, sim ? "leafStates" : "siteLnL");
    }
    // component counts: with weights, K in 1..4 and branchK (nullable) in 1..K; without, one row per branch
    if (!c.weights && (c.K != 1 || c.branchK))
        return fail("K=%lld and branchK need weights: without them every branch has one row (K=1, branchK NULL)", (long long)c.K);
    if (c.weights && (c.K < 1 || c.K > 4)) return fail("K=%lld outside 1..4", (long long)c.K);
    for (int64_t b = 0; c.weights && c.branchK && b < p->B; b++)
        if (c.branchK[b] < 1 || c.branchK[b] > c.K)
            return fail("branchK[%lld]=%lld outside 1..%lld", (long long)b, (long long)c.branchK[b], (long long)c.K);
    if (p->Dp != 64) return fail("hb2_batch_site_likelihoods supports 33..64-state (codon) partitions only");
    if (c.templateId < 0 || c.templateId >= (int64_t)p->tmpls.size() || p->tmpls[c.templateId].nnz == 0)
        return fail("template %lld has not been defined", (long long)c.templateId);
    if (p->cg_G > 1) return fail("hb2_batch_site_likelihoods is not available with class groups (shard the SETS across ranks instead)");
    for (int64_t b = 0; c.branchGroup && b < p->B; b++)
        if (c.branchGroup[b] < 0 || c.branchGroup[b] >= 8) return fail("branchGroup[%lld]=%lld outside 0..7", (long long)b, (long long)c.branchGroup[b]);
    for (int64_t s = 0; c.patternOf && s < c.nSets; s++)
        if (c.patternOf[s] < 0 || c.patternOf[s] >= p->S) return fail("patternOf[%lld]=%lld out of range", (long long)s, (long long)c.patternOf[s]);
    for (int64_t s = 0; c.columns && s < c.nSets; s++)
        for (int64_t l = 0; l < p->L; l++) {
            const int64_t code = c.columns[s * p->L + l];
            if (code >= p->D || code < -p->nAmb)
                return fail("hb2_batch_column_likelihoods: set %lld, leaf %lld: code %lld is neither a state 0..%lld nor an ambiguity row -1..-%lld",
                            (long long)s, (long long)l, (long long)code, (long long)p->D - 1, (long long)p->nAmb);
        }
    double root_cdf[64];
    int root_last;
    if (sim && !sim_prefix(c.rootFreqs, p->D, root_cdf, &root_last))
        return fail("hb2_batch_site_simulate: root frequencies must be >= 0 and not NaN, with a finite positive total");
    return 0;
}

static BatchShape batch_shape(const hb2_partition *p, const BatchCall &c) {
    const int64_t B = p->B, D = p->D;
    BatchShape sh;
    sh.nF = p->tmpls[c.templateId].nF;
    // component k of every tested branch is the same rate matrix up to the branch length, so the shared-powers group of a
    // row is (set, branchGroup[b], k)
    sh.row_off.assign(B + 1, 0);
    for (int64_t b = 0; b < B; b++) sh.row_off[b + 1] = sh.row_off[b] + (int)(c.weights && c.branchK ? c.branchK[b] : c.K);
    sh.R = sh.row_off[B];
    int64_t gps = 1;                            // groups per set and component: branches with the same branchGroup share one
    for (int64_t b = 0; c.branchGroup && b < B; b++) gps = std::max(gps, c.branchGroup[b] + 1);
    sh.gk = gps * c.K;
    // chunk buffers, capped at ~8 GB; a simulation adds the prefix sums and last positive columns of the set's B matrices
    const double sim_bytes = c.entry == BatchEntry::Simulate ? (double)B * D * (64 * 8 + 4) : 0.0;
    double per_set;
    if (!c.weights)                             // P matrices (32 KB per branch)
        per_set = (double)B * (4096 + 1024 + (double)sh.nF) * 8;
    else                                        // a set's R component matrices, formula values and weights,
                                                // the power tables of its groups and its node vectors
        per_set = (double)sh.R * (4096 + (double)sh.nF + 1) * 8 + (double)sh.gk * hb2::EXPM_POW_TERMS * 4096 * 8 + (double)p->I * 64 * 8;
    if (c.entry == BatchEntry::BranchRows) {    // messages and outside vectors with their exponents, and the row results
        sh.side = B;
        per_set += (double)B * 2 * (64 * 8 + 4) + (double)sh.R * 8;
        sh.rows = sh.R;
    }
    if (c.entry == BatchEntry::LeafSupport) {   // messages and outside vectors with their exponents, and the support rows
        sh.side = B;
        sh.sup = p->L * D;
        per_set += (double)B * 2 * (64 * 8 + 4) + (double)sh.sup * 8;
    }
    if (c.entry == BatchEntry::JointAncestors) {    // the argument table and the node states
        sh.joint = p->I;
        per_set += (double)p->I * (64 + 8) + 8;
    }
    sh.sets = std::min<int64_t>({c.nSets, std::max<int64_t>(1, (int64_t)(8.0e9 / (per_set + sim_bytes))), 1024});
    sh.ent = sh.R;
    sh.in = sh.R * sh.nF;
    return sh;
}

// Refusals of hb2_batch_site_rates, before anything is launched or written.  A branch's rate matrix is resident when its
// last hand-over, pending or flushed, was a rate matrix (dense or compiled): that is what d_Qres holds for it.
static int check_rates(const hb2_partition *p, const BatchCall &c) {
    if (!p) return fail("hb2_batch_site_rates: null partition");
    if (!c.patternOf || !c.rates || !c.rootFreqs || !c.siteLnL) return fail("hb2_batch_site_rates: null argument");
    if (c.nSets < 0) return fail("hb2_batch_site_rates: nSets=%lld is negative", (long long)c.nSets);
    if (c.cat < 0 || c.cat >= p->C) return fail("hb2_batch_site_rates: rate class %lld out of range (C=%lld)", (long long)c.cat, (long long)p->C);
    if (p->cg_G > 1) return fail("hb2_batch_site_rates is not available with class groups (shard the SETS across ranks instead)");
    if (p->Dp > 32)
        return fail("hb2_batch_site_rates supports 2..32-state partitions: for 33..64 states use hb2_batch_site_likelihoods with "
                    "formula values multiplied by the rate");
    for (int64_t s = 0; s < c.nSets; s++)
        if (c.patternOf[s] < 0 || c.patternOf[s] >= p->S)
            return fail("hb2_batch_site_rates: set %lld: patternOf=%lld out of range (0..%lld)", (long long)s, (long long)c.patternOf[s], (long long)p->S - 1);
    for (int64_t s = 0; s < c.nSets; s++)
        if (!(c.rates[s] >= 0.0) || std::isinf(c.rates[s]))
            return fail("hb2_batch_site_rates: set %lld: rate %g is not a finite number >= 0", (long long)s, c.rates[s]);
    for (int64_t b = 0; b < p->B; b++) {
        const Slot &s = p->slots[c.cat * p->B + b];
        const HandoverQueue *q = s.entry < 0 ? nullptr : s.queue == DENSE_QUEUE ? &p->dense : &p->tmpls[s.queue].queue;
        if (q ? q->kind[s.entry] == Kind::Trans : s.res != Resident::DenseQ)
            return fail("hb2_batch_site_rates: rate class %lld, branch %lld has no resident rate matrix (its last hand-over was a "
                        "transition matrix or a mixture, or it has none)", (long long)c.cat, (long long)b);
    }
    return 0;
}

// hb2_batch_site_rates: one P matrix per branch and set, read from d_Qres and scaled on the device (no input but the rate),
// and the ~8 GB chunk rule of batch_shape with Dp-sized matrices and node vectors.
static BatchShape rates_shape(const hb2_partition *p, const BatchCall &c) {
    BatchShape sh;
    sh.R = p->B;
    sh.mat = (int64_t)p->Dp * p->Dp;
    sh.vec = p->Dp;
    sh.in = 1;
    // P matrices, node vectors and exponents, rate, pattern and result
    const double per_set = (double)p->B * sh.mat * 8 + (double)p->I * (sh.vec * 8 + 4) + 20;
    sh.sets = std::min<int64_t>({c.nSets, std::max<int64_t>(1, (int64_t)(8.0e9 / per_set)), RATES_MAX_SETS});
    return sh;
}

// The chunk's inside-pass arguments over the batch workspace: set s prunes pattern pat[s] of leaf[L][Sp]; R component rows
// per set (mixtures only).
static hb2::BatchPruneArgs batch_prune_args(const hb2_partition *p, const int *leaf, int Sp, int R) {
    const hb2_partition::BatchWorkspace &ws = p->batch;
    hb2::BatchPruneArgs ba{};
    ba.PT = ws.PT; ba.cond = ws.cond; ba.node_ex = ws.node_ex; ba.pat = ws.pat; ba.leaf = leaf; ba.ambig = p->d_ambig;
    ba.pi = ws.pi; ba.tree.child_start = p->d_child_start; ba.tree.child_ids = p->d_child_ids; ba.out = ws.out;
    ba.L = (int)p->L; ba.I = (int)p->I; ba.B = (int)p->B; ba.D = (int)p->D; ba.Sp = Sp;
    ba.mix_w = ws.mixw; ba.row_off = ws.row; ba.R = R;
    return ba;
}

extern "C++" template <int DP>
void launch_rates(hb2_partition *p, const BatchCall &c, int64_t nb) {
    hb2_partition::BatchWorkspace &ws = p->batch;
    hb2::ExpmRatesArgs ea;
    ea.Q = p->d_Qres + (size_t)c.cat * p->B * p->D * p->D; ea.rate = ws.V; ea.PT = ws.PT;
    ea.D = (int)p->D; ea.B = (int)p->B; ea.n = (long long)nb * p->B;
    constexpr int M = 128 / hb2::expm_rates_team(DP);
    hb2::expm_rates_kernel<DP><<<(unsigned)((ea.n + M - 1) / M), 128, hb2::expm_rates_smem_bytes(DP), p->stream>>>(ea);
    const hb2::BatchPruneArgs ba = batch_prune_args(p, p->d_leaf, (int)p->Sp, 0);
    constexpr int per_block = 128 / (DP <= 16 ? DP : 32);
    hb2::prune_rates_kernel<DP><<<(unsigned)((nb + per_block - 1) / per_block), 128, 0, p->stream>>>(ba, (int)nb);
}

// Sets s0 .. s0+nb-1 of hb2_batch_site_rates: their rates and patterns up, their matrices and likelihoods, the results down.
static int rates_chunk(hb2_partition *p, const BatchCall &c, int64_t s0, int64_t nb) {
    hb2_partition::BatchWorkspace &ws = p->batch;
    for (int64_t s = 0; s < nb; s++) ws.h_pat[s] = (int)c.patternOf[s0 + s];
    CU(cudaMemcpyAsync(ws.pat, ws.h_pat, (size_t)nb * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    CU(cudaMemcpyAsync(ws.V, c.rates + s0, (size_t)nb * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    if (!small_states(p->Dp, [&](auto dp) { launch_rates<decltype(dp)::value>(p, c, nb); }))
        return fail("hb2_batch_site_rates: unsupported padded state count %d", p->Dp);
    p->launches += 2;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(c.siteLnL + s0, ws.out, (size_t)nb * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    return 0;
}

// Uploads the formula values (and weights) of sets s0 .. s0+nb-1, plans their shared-powers groups and exponentiates them
// into the chunk's P area, PT[set][row].
static int exponentiate_chunk(hb2_partition *p, const BatchCall &c, const BatchShape &sh, int64_t s0, int64_t nb) {
    hb2_partition::BatchWorkspace &ws = p->batch;
    const int64_t R = sh.R, ne = nb * R;
    CU(cudaMemcpyAsync(ws.V, c.formulaValues + (size_t)s0 * R * sh.nF, (size_t)ne * sh.nF * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    if (c.weights) CU(cudaMemcpyAsync(ws.mixw, c.weights + (size_t)s0 * R, (size_t)ne * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    std::vector<int> grp(ne);
    for (int64_t s = 0; s < nb; s++)
        for (int64_t b = 0; b < p->B; b++)
            for (int k = 0; k < sh.row_off[b + 1] - sh.row_off[b]; k++)
                grp[s * R + sh.row_off[b] + k] = (int)(s * sh.gk + (c.branchGroup ? c.branchGroup[b] : 0) * c.K + k);
    SharedPlan sp;
    // every chunk rebuilds its tables: a group with fewer than 4 branches must not be compared with a direction cached by
    // an earlier chunk or call, whose table may come from another template or other column frequencies
    std::fill(ws.ex.kind.begin(), ws.ex.kind.end(), 0);
    CU(cudaMemsetAsync(ws.ex.d_groups, 0, (size_t)ws.ex.G * sizeof(hb2::ExpmGroup), p->stream));
    if (plan_shared(p, ws.h_slot, ne, 1, grp.data(), sp, (int)c.templateId, &ws.ex, 4) || staged_uploads(p)) return 1;
    // the chunk's P area is scratch: no resident copy is kept
    return launch_expm(p, {Kind::Compiled, (int)c.templateId}, ws.V, ws.slot, (int)ne, false, sp, 0, ws.PT);
}

// Likelihoods of sets s0 .. s0+nb-1 from the chunk's P area.  Branch rows and leaf support: then branch_rows_kernel or
// leaf_support_kernel on the inside pass's node vectors (so siteLnL stays the likelihood entry point's bit for bit), and the
// chunk's rows or support go down.  Joint ancestors: the inside pass only when siteLnL is given, then
// joint_ancestors_kernel, and the chunk's node states and joint log-likelihoods go down.
static int score_chunk(hb2_partition *p, const BatchCall &c, const BatchShape &sh, int64_t s0, int64_t nb) {
    hb2_partition::BatchWorkspace &ws = p->batch;
    const int64_t L = p->L;
    // set s prunes pattern pat[s] of leaf[L][Sp]: the partition's patterns, or the chunk's columns as leaf[L][nb]
    for (int64_t s = 0; s < nb; s++) ws.h_pat[s] = c.columns ? (int)s : (int)c.patternOf[s0 + s];
    CU(cudaMemcpyAsync(ws.pat, ws.h_pat, (size_t)nb * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    if (c.columns) {
        for (int64_t s = 0; s < nb; s++)
            for (int64_t l = 0; l < L; l++) ws.h_col[l * nb + s] = (int)c.columns[(s0 + s) * L + l];
        CU(cudaMemcpyAsync(ws.col, ws.h_col, (size_t)L * nb * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    }
    const hb2::BatchPruneArgs ba = batch_prune_args(p, c.columns ? (const int *)ws.col : (const int *)p->d_leaf,
                                                    c.columns ? (int)nb : (int)p->Sp, (int)sh.R);
    if (c.entry != BatchEntry::JointAncestors || c.siteLnL) {
        if (c.weights) hb2::prune_batch_kernel<true><<<(unsigned)nb, 64, 0, p->stream>>>(ba);
        else hb2::prune_batch_kernel<false><<<(unsigned)nb, 64, 0, p->stream>>>(ba);
        p->launches++;
        CU(cudaGetLastError());
    }
    if (c.entry == BatchEntry::JointAncestors) {   // after the inside pass, whose cond / node_ex it then reuses
        const hb2::JointArgs g{ba, ws.arg, ws.states, ws.jlnl};
        if (c.weights) hb2::joint_ancestors_kernel<true><<<(unsigned)nb, 64, 0, p->stream>>>(g);
        else hb2::joint_ancestors_kernel<false><<<(unsigned)nb, 64, 0, p->stream>>>(g);
        p->launches++;
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(c.nodeStates + s0 * p->I, ws.states, (size_t)nb * p->I * sizeof(int64_t), cudaMemcpyDeviceToHost, p->stream));
        if (c.jointLnL) CU(cudaMemcpyAsync(c.jointLnL + s0, ws.jlnl, (size_t)nb * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    }
    if (c.rowLnL || c.support) {
        const size_t side = (size_t)nb * p->B;
        hb2::OutsideArgs g{ba, ws.side, ws.side + side * 64, ws.side_ex, ws.side_ex + side, ws.rows, ws.sup};
        if (c.rowLnL) hb2::branch_rows_kernel<<<(unsigned)nb, 64, 0, p->stream>>>(g);
        else if (c.weights) hb2::leaf_support_kernel<true><<<(unsigned)nb, 64, 0, p->stream>>>(g);
        else hb2::leaf_support_kernel<false><<<(unsigned)nb, 64, 0, p->stream>>>(g);
        p->launches++;
        CU(cudaGetLastError());
        if (c.rowLnL)
            CU(cudaMemcpyAsync(c.rowLnL + s0 * sh.R, ws.rows, (size_t)nb * sh.R * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
        else
            CU(cudaMemcpyAsync(c.support + s0 * sh.sup, ws.sup, (size_t)nb * sh.sup * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    }
    if (c.siteLnL) CU(cudaMemcpyAsync(c.siteLnL + s0, ws.out, (size_t)nb * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    return 0;
}

// nReps columns of each of sets s0 .. s0+nb-1 from the chunk's P area: the chunk's table and its check, then launches of
// columns (set-major, a set's replicates consecutive) copied to the caller's [nSets][nReps][L] (and [I]) arrays.
static int simulate_chunk(hb2_partition *p, const BatchCall &c, const BatchShape &sh, int64_t s0, int64_t nb) {
    const int64_t L = p->L, I = p->I;
    const int64_t chunk = c.nReps >= SIM_CHUNK ? SIM_CHUNK : std::min(SIM_CHUNK, sh.sets * c.nReps);   // columns per launch
    std::vector<double> root_cdf(p->D);
    std::vector<int> ints(nb + 3, 1);           // every set of the chunk is active | no class | last root state | first bad row
    sim_prefix(c.rootFreqs, p->D, root_cdf.data(), &ints[nb + 1]);     // checked with the call's arguments
    ints[nb] = 0; ints[nb + 2] = INT_MAX;
    hb2::SimArgs a{};
    a.PT = p->batch.PT; a.mix_w = p->batch.mixw; a.row_off = p->batch.row; a.R = (int)sh.R; a.reps = c.nReps;
    a.g0 = (unsigned long long)c.firstRep; a.t0 = (unsigned)(c.firstSet + s0);
    if (sim_tables(p, a, nb, chunk, c.seed, root_cdf, ints, c.nodeStates, false, c.weights, "hb2_batch_site_simulate",
                   "set %lld, branch %lld", s0))
        return 1;
    const size_t smem = a.states ? 0 : (size_t)I * SIM_THREADS;
    const int64_t ncol = nb * c.nReps;
    for (int64_t c0 = 0; c0 < ncol; c0 += chunk) {
        const int64_t n = std::min(chunk, ncol - c0);
        a.n = (int)n; a.col0 = c0;
        hb2::batch_simulate_kernel<<<(unsigned)((n + SIM_THREADS - 1) / SIM_THREADS), SIM_THREADS, smem, p->stream>>>(a);
        p->launches++;
        CU(cudaGetLastError());
        const size_t col = (size_t)s0 * c.nReps + c0;
        CU(cudaMemcpyAsync(c.leafStates + col * L, a.leaf_out, (size_t)n * L * sizeof(int64_t), cudaMemcpyDeviceToHost, p->stream));
        if (c.nodeStates)
            CU(cudaMemcpyAsync(c.nodeStates + col * I, a.node_out, (size_t)n * I * sizeof(int64_t), cudaMemcpyDeviceToHost, p->stream));
    }
    return 0;
}

// Body of every batch entry point: per chunk of sets, the batched exponential, then the call's consumer.
static int batch_sites(hb2_partition *p, const BatchCall &c) {
    const bool sim = c.entry == BatchEntry::Simulate, rates = c.entry == BatchEntry::Rates;
    if (rates ? check_rates(p, c) : check_batch(p, c)) return 1;
    if (c.nSets == 0 || (sim && c.nReps == 0)) return 0;
    CU(cudaSetDevice(p->device));
    if (rates && flush_matrices(p)) return 1;          // d_Qres holds every matrix handed over so far
    const BatchShape sh = rates ? rates_shape(p, c) : batch_shape(p, c);
    if (p->batch.fit(sh, rates ? 0 : p->L, p->I, p->stream)) return 1;     // site rates score patterns only: no column area
    CU(cudaStreamSynchronize(p->stream));
    if (stage_root(p, c.rootFreqs, nullptr, 0, p->batch.pi)) return 1;
    if (c.weights) CU(cudaMemcpyAsync(p->batch.row, sh.row_off.data(), sh.row_off.size() * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    for (int64_t s0 = 0; s0 < c.nSets; s0 += sh.sets) {
        const int64_t nb = std::min(sh.sets, c.nSets - s0);
        CU(cudaStreamSynchronize(p->stream));          // previous chunk done: buffers and pinned arrays are free again
        if (rates) {
            if (rates_chunk(p, c, s0, nb)) return 1;
        } else if (exponentiate_chunk(p, c, sh, s0, nb) || (sim ? simulate_chunk(p, c, sh, s0, nb) : score_chunk(p, c, sh, s0, nb))) {
            return 1;
        }
    }
    int err = 0;
    CU(cudaMemcpyAsync(&err, p->d_err, sizeof(int), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    if (err) { cudaMemsetAsync(p->d_err, 0, sizeof(int), p->stream); return wait_timeout(err); }
    return 0;
}

int hb2_batch_site_likelihoods(hb2_partition *p, int64_t templateId, int64_t nSets, const int64_t *patternOf,
                               const double *formulaValues, const int64_t *branchGroup, const double *rootFreqs, double *siteLnL) {
    return batch_sites(p, {BatchEntry::Sites, templateId, nSets, 1, nullptr, branchGroup, formulaValues, nullptr, rootFreqs,
                           patternOf, nullptr, siteLnL});
}

int hb2_batch_site_mixture_likelihoods(hb2_partition *p, int64_t templateId, int64_t nSets, const int64_t *patternOf, int64_t K,
                                       const int64_t *branchK, const double *formulaValues, const double *weights,
                                       const int64_t *branchGroup, const double *rootFreqs, double *siteLnL) {
    return batch_sites(p, {BatchEntry::MixtureSites, templateId, nSets, K, branchK, branchGroup, formulaValues, weights, rootFreqs,
                           patternOf, nullptr, siteLnL});
}

int hb2_batch_branch_component_likelihoods(hb2_partition *p, int64_t templateId, int64_t nSets, const int64_t *patternOf,
                                           int64_t K, const int64_t *branchK, const double *formulaValues,
                                           const double *weights, const int64_t *branchGroup, const double *rootFreqs,
                                           double *siteLnL, double *rowLnL) {
    BatchCall c{BatchEntry::BranchRows, templateId, nSets, K, branchK, branchGroup, formulaValues, weights, rootFreqs,
                patternOf, nullptr, siteLnL};
    c.rowLnL = rowLnL;
    return batch_sites(p, c);
}

int hb2_batch_leaf_support(hb2_partition *p, int64_t templateId, int64_t nSets, const int64_t *patternOf, int64_t K,
                           const int64_t *branchK, const double *formulaValues, const double *weights,
                           const int64_t *branchGroup, const double *rootFreqs, double *siteLnL, double *support) {
    BatchCall c{BatchEntry::LeafSupport, templateId, nSets, K, branchK, branchGroup, formulaValues, weights, rootFreqs,
                patternOf, nullptr, siteLnL};
    c.support = support;
    return batch_sites(p, c);
}

int hb2_batch_joint_ancestors(hb2_partition *p, int64_t templateId, int64_t nSets, const int64_t *patternOf, int64_t K,
                              const int64_t *branchK, const double *formulaValues, const double *weights,
                              const int64_t *branchGroup, const double *rootFreqs, double *siteLnL, double *jointLnL,
                              int64_t *nodeStates) {
    BatchCall c{BatchEntry::JointAncestors, templateId, nSets, K, branchK, branchGroup, formulaValues, weights, rootFreqs,
                patternOf, nullptr, siteLnL};
    c.nodeStates = nodeStates;
    c.jointLnL = jointLnL;
    return batch_sites(p, c);
}

int hb2_batch_column_likelihoods(hb2_partition *p, int64_t templateId, int64_t nSets, const int64_t *columns, int64_t K,
                                 const int64_t *branchK, const double *formulaValues, const double *weights,
                                 const int64_t *branchGroup, const double *rootFreqs, double *siteLnL) {
    return batch_sites(p, {BatchEntry::Columns, templateId, nSets, K, branchK, branchGroup, formulaValues, weights, rootFreqs,
                           nullptr, columns, siteLnL});
}

int hb2_batch_site_simulate(hb2_partition *p, int64_t templateId, int64_t nSets, int64_t K, const int64_t *branchK,
                            const double *formulaValues, const double *weights, const int64_t *branchGroup,
                            const double *rootFreqs, int64_t nReps, uint64_t seed, int64_t firstSet, int64_t firstRep,
                            int64_t *leafStates, int64_t *nodeStates) {
    return batch_sites(p, {BatchEntry::Simulate, templateId, nSets, K, branchK, branchGroup, formulaValues, weights, rootFreqs,
                           nullptr, nullptr, nullptr, nReps, firstSet, firstRep, seed, leafStates, nodeStates});
}

int hb2_batch_site_rates(hb2_partition *p, int64_t cat, int64_t nSets, const int64_t *patternOf, const double *rates,
                         const double *rootFreqs, double *siteLnL) {
    BatchCall c{BatchEntry::Rates, 0, nSets, 1, nullptr, nullptr, nullptr, nullptr, rootFreqs, patternOf, nullptr, siteLnL};
    c.cat = cat < 0 ? 0 : cat;
    c.rates = rates;
    return batch_sites(p, c);
}

int hb2_read_conditionals(hb2_partition *p, int64_t cat, int64_t inode, double *cond, int32_t *exp2) {
    if (!p || !cond || !exp2) return fail("null argument");
    if (cat < 0) cat = 0;
    if (cat >= p->C || inode < 0 || inode >= p->I) return fail("index out of range");
    CU(cudaSetDevice(p->device));
    std::vector<double> tmp((size_t)p->Sp * p->Dp);
    std::vector<int> te(p->Sp);
    const int64_t nstride = p->use_tc ? 2 * p->I : p->I;     // node slots per class (tensor walk: + side products)
    CU(cudaStreamSynchronize(p->stream));
    if (p->use_tc) {
        std::vector<float> tf(tmp.size());
        CU(cudaMemcpy(tf.data(), p->d_condf + ((size_t)cat * nstride + inode) * p->Sp * 64, tf.size() * sizeof(float), cudaMemcpyDeviceToHost));
        // device layout per tile of 128 patterns: [16 chunks][128 patterns][4 floats]
        for (int64_t s = 0; s < p->Sp; s++)
            for (int k = 0; k < 64; k++)
                tmp[s * 64 + k] = std::fabs(tf[(((size_t)(s / 128) * 16 + k / 4) * 128 + s % 128) * 4 + k % 4]);   // sign bit = walk tag
    } else
    CU(cudaMemcpy(tmp.data(), p->d_cond + ((size_t)cat * p->I + inode) * p->Sp * p->Dp, tmp.size() * sizeof(double), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(te.data(), p->d_scal + ((size_t)cat * nstride + inode) * p->Sp, te.size() * sizeof(int), cudaMemcpyDeviceToHost));
    for (int64_t s = 0; s < p->S; s++) {
        for (int64_t k = 0; k < p->D; k++) cond[s * p->D + k] = tmp[s * p->Dp + k];
        exp2[s] = p->use_tc ? (te[s] >> 1) : te[s];      // tensor walk: bit 0 is the generation tag
    }
    return 0;
}

int hb2_read_transition(hb2_partition *p, int64_t cat, int64_t node, double *P) {
    if (!p || !P) return fail("null argument");
    if (cat < 0) cat = 0;
    if (cat >= p->C || node < 0 || node >= p->B) return fail("index out of range");
    CU(cudaSetDevice(p->device));
    if (flush_matrices(p)) return 1;
    std::vector<double> tmp((size_t)p->Dp * p->Dp);
    CU(cudaStreamSynchronize(p->stream));
    CU(cudaMemcpy(tmp.data(), p->d_PT + ((size_t)cat * p->B + node) * p->Dp * p->Dp, tmp.size() * sizeof(double), cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < p->D; i++)
        for (int64_t j = 0; j < p->D; j++) P[i * p->D + j] = tmp[j * p->Dp + i];   // stored transposed
    return 0;
}

int hb2_simulate(hb2_partition *p, const double *weights, const double *rootFreqs, int64_t nSites, uint64_t seed, int64_t firstSite,
                 int64_t *leafStates, int64_t *nodeStates, int32_t *siteClass) {
    if (!p) return fail("null partition");
    if (nSites < 0) return fail("hb2_simulate: nSites=%lld is negative", (long long)nSites);
    if (firstSite < 0 || firstSite > INT64_MAX - nSites) return fail("hb2_simulate: firstSite=%lld out of range", (long long)firstSite);
    if (!rootFreqs) return fail("hb2_simulate: rootFreqs must not be null");
    if (nSites > 0 && !leafStates) return fail("hb2_simulate: leafStates must not be null");
    if (p->cg_G > 1) return fail("hb2_simulate is not available with class groups: a rank does not hold the other groups' matrices");
    if (!weights && p->C > 1) return fail("hb2_simulate: weights may be null only with one rate class (C=%lld)", (long long)p->C);
    const int64_t C = p->C, D = p->D, B = p->B, L = p->L, I = p->I;
    std::vector<double> vec(C + D);                 // prefix sums: classes | root states
    std::vector<int> ints(C + 3);                   // active classes [C] | last class | last root state | first bad row
    if (weights) {
        if (!sim_prefix(weights, C, vec.data(), &ints[C]))
            return fail("hb2_simulate: class weights must be >= 0 and not NaN, with a finite positive total");
    } else {
        vec[0] = 1.0; ints[C] = 0;
    }
    if (!sim_prefix(rootFreqs, D, vec.data() + C, &ints[C + 1]))
        return fail("hb2_simulate: root frequencies must be >= 0 and not NaN, with a finite positive total");
    ints[C + 2] = INT_MAX;
    for (int64_t c = 0; c < C; c++) {
        ints[c] = !weights || weights[c] > 0.0;
        for (int64_t b = 0; ints[c] && b < B; b++)
            if (!p->slots[c * B + b].have)
                return fail("hb2_simulate: no matrix was ever set for rate class %lld, node %lld", (long long)c, (long long)b);
    }
    if (nSites == 0) return 0;
    CU(cudaSetDevice(p->device));
    if (flush_matrices(p)) return 1;
    const int64_t chunk = std::min(nSites, SIM_CHUNK);
    hb2::SimArgs a{};
    a.PT = p->d_PT; a.C = (int)C;
    // the table of every drawn class, and its check: a refused call writes nothing
    if (sim_tables(p, a, C, chunk, seed, vec, ints, nodeStates, siteClass, false, "hb2_simulate", "rate class %lld, node %lld", 0))
        return 1;
    const size_t smem = a.states ? 0 : (size_t)I * SIM_THREADS;
    for (int64_t s0 = 0; s0 < nSites; s0 += chunk) {
        const int64_t n = std::min(chunk, nSites - s0);
        a.n = (int)n; a.g0 = (unsigned long long)(firstSite + s0);
        hb2::simulate_kernel<<<(unsigned)((n + SIM_THREADS - 1) / SIM_THREADS), SIM_THREADS, smem, p->stream>>>(a);
        p->launches++;
        CU(cudaGetLastError());
        CU(cudaMemcpy2DAsync(leafStates + s0, nSites * sizeof(int64_t), a.leaf_out, chunk * sizeof(long long), n * sizeof(int64_t), L,
                             cudaMemcpyDeviceToHost, p->stream));
        if (nodeStates)
            CU(cudaMemcpy2DAsync(nodeStates + s0, nSites * sizeof(int64_t), a.node_out, chunk * sizeof(long long), n * sizeof(int64_t), I,
                                 cudaMemcpyDeviceToHost, p->stream));
        if (siteClass) CU(cudaMemcpyAsync(siteClass + s0, a.class_out, n * sizeof(int32_t), cudaMemcpyDeviceToHost, p->stream));
    }
    CU(cudaStreamSynchronize(p->stream));
    return 0;
}

static hb2::BranchCacheArgs bc_args(hb2_partition *p, int c0, int nc) {
    hb2::BranchCacheArgs a{};
    a.cv.c64 = p->use_tc ? nullptr : (double *)p->d_cond;
    a.cv.c32 = p->use_tc ? p->d_condf : (float *)nullptr;
    a.cv.scal = p->d_scal; a.cv.I = (int)(p->use_tc ? 2 * p->I : p->I); a.cv.Sp = (int)p->Sp; a.cv.Dp = p->Dp; a.cv.tagged = p->use_tc ? 1 : 0;
    a.PT = p->d_PT; a.leaf = p->d_leaf; a.ambig = p->d_ambig; a.pi = p->d_pi; a.out = p->d_bc_out; a.outE = p->d_bc_outE;
    a.L = (int)p->L; a.B = (int)p->B; a.D = (int)p->D; a.Dp = p->Dp; a.Sp = (int)p->Sp; a.S = (int)p->S; a.cat0 = c0; a.ncls = nc;
    return a;
}

int hb2_branch_cache_build(hb2_partition *p, int64_t node, const double *rootFreqs) {
    if (!p || !rootFreqs) return fail("null argument");
    if (node < 0 || node >= p->B) return fail("node id %lld has no branch (valid 0..%lld)", (long long)node, (long long)p->B - 1);
    CU(cudaSetDevice(p->device));
    for (int c = p->own0; c < p->own0 + p->ownN; c++)
        if (!p->evaluated_cat[c]) return fail("hb2_branch_cache_build: rate class %d has never been evaluated (no resident conditionals)", c);
    if (flush_matrices(p)) return 1;
    // keyed on the last of the three: after a failed allocation the next build allocates all of them again
    if (!p->d_bc_sib && (p->d_bc_out.alloc((size_t)p->C * p->Sp * p->Dp) || p->d_bc_outE.alloc((size_t)p->C * p->Sp) ||
                         p->d_bc_sib.alloc(3 * (p->L + p->I) + 2)))
        return 1;
    if (stage_root(p, rootFreqs)) return 1;
    // root -> parent(node) path (internal indices) and, per path node, its children that are NOT on the path
    std::vector<int> path;
    for (int64_t u = p->parents[node]; u >= 0; u = p->parents[p->L + u]) path.push_back((int)u);
    std::reverse(path.begin(), path.end());
    std::vector<int> sib, off(path.size() + 1, 0), down(path.size(), -1);
    for (size_t i = 0; i < path.size(); i++) {
        const int on_path = (i + 1 < path.size()) ? (int)p->L + path[i + 1] : (int)node;
        for (int ch : p->children[path[i]]) if (ch != on_path) sib.push_back(ch);
        off[i + 1] = (int)sib.size();
        down[i] = (i + 1 < path.size()) ? on_path : -1;
    }
    // one launch for the whole path: [siblings | sibling offsets (npath+1) | path child below each path node (npath)]
    std::vector<int> pk(sib);
    const int o_off = (int)pk.size();
    pk.insert(pk.end(), off.begin(), off.end());
    const int o_down = (int)pk.size();
    pk.insert(pk.end(), down.begin(), down.end());
    if ((int64_t)pk.size() > 3 * (p->L + p->I) + 2) return fail("branch-cache path does not fit its buffer");
    CU(cudaMemcpyAsync(p->d_bc_sib, pk.data(), pk.size() * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    hb2::BranchCacheArgs a = bc_args(p, p->own0, p->ownN);
    hb2::BranchPathArgs bp;
    bp.sib = p->d_bc_sib; bp.sib_off = p->d_bc_sib + o_off; bp.down = p->d_bc_sib + o_down; bp.npath = (int)path.size();
    dim3 grid((unsigned)p->S, (unsigned)p->ownN);
    if (p->Dp > 32) hb2::bc_path_kernel<64><<<grid, 64, 0, p->stream>>>(a, bp);
    else hb2::bc_path_kernel<32><<<grid, 32, 0, p->stream>>>(a, bp);
    p->launches++;
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(p->stream));
    p->bc_node = node;
    p->bc_dirty_node = -1;
    return 0;
}

int hb2_branch_cache_evaluate(hb2_partition *p, int64_t cat, const double *weights, double *lnL, double *siteL, int64_t *siteScale) {
    if (!p || !lnL) return fail("null argument");
    if (p->bc_node < 0) return fail("hb2_branch_cache_evaluate: no valid branch cache (build it after the last full evaluation)");
    CU(cudaSetDevice(p->device));
    // only the cached branch may have a new matrix (flushed or not, plain, compiled or mixture): anything else needs a
    // regular evaluation
    if (p->bc_dirty_node >= 0)
        return fail("branch cache holds node %lld but a matrix of node %lld changed", (long long)p->bc_node, (long long)p->bc_dirty_node);
    if (flush_matrices(p)) return 1;
    int c0, nc;
    if (weights) { c0 = p->own0; nc = p->ownN; }
    else {
        if (p->cg_G > 1) return fail("with class groups only the all-class form (weights != NULL) is available");
        if (cat < 0) cat = 0;
        if (cat >= p->C) return fail("rate class %lld out of range", (long long)cat);
        c0 = (int)cat; nc = 1;
    }
    if (stage_root(p, nullptr, weights, (int)p->C)) return 1;    // the root vector of the build stays
    double *hs = p->h_small;
    hb2::BranchCacheArgs a = bc_args(p, c0, nc);
    dim3 grid((unsigned)((p->S + 127) / 128), (unsigned)nc);
    hb2::bc_eval_kernel<<<grid, 128, 0, p->stream>>>(a, (int)p->bc_node, p->d_rootL, p->d_rootE);
    p->launches++;
    CU(cudaGetLastError());
    const bool want_sites = siteL != nullptr || siteScale != nullptr;
    if (run_root(p, c0, nc, weights != nullptr, want_sites)) return 1;
    CU(cudaMemcpyAsync(hs + p->Dp + p->C, p->d_lnL, sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    if (siteL) CU(cudaMemcpyAsync(siteL, p->d_siteL, p->S * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    if (siteScale) CU(cudaMemcpyAsync(siteScale, p->d_siteScale, p->S * sizeof(long long), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    *lnL = hs[p->Dp + p->C];
    return 0;
}

int hb2_plan_walk(int64_t L, int64_t I, const int64_t *flatParents, int64_t nUpdate, const int64_t *updateNodes, int lanes,
                  int splitNodes, int32_t *laneStart, int32_t *steps, int64_t stepCapacity, int64_t *nSteps) {
    if (!flatParents || !laneStart || !steps || !nSteps) return fail("null argument");
    if (L < 2 || I < 1 || lanes < 1 || lanes > 15) return fail("bad sizes L=%lld I=%lld lanes=%d", (long long)L, (long long)I, lanes);
    std::vector<std::vector<int>> children;
    std::vector<int> height;
    std::vector<char> dirty;
    if (build_tree(flatParents, L, I, children, height) || dirty_nodes(flatParents, L, I, nUpdate, updateNodes, dirty)) return 1;
    const int total = (int)std::count(dirty.begin(), dirty.end(), 1);
    if (total == 0) { *nSteps = 0; for (int r = 0; r <= lanes; r++) laneStart[r] = 0; return 0; }
    const int K = std::min(lanes, total);
    if (stepCapacity < L + 2 * I) return fail("steps needs room for %lld entries", (long long)(L + 2 * I));
    std::vector<int> ls(K + 1), st(2 * (size_t)(L + 2 * I));
    std::vector<char> jdirty;
    const int ns = plan_walk(children, height, (int)L, (int)I, dirty, K, (splitNodes & 1) != 0, ls.data(), st.data(), jdirty, (splitNodes & 2) != 0);
    for (int r = 0; r <= lanes; r++) laneStart[r] = ls[std::min(r, K)];
    for (int i = 0; i < 2 * ns; i++) steps[i] = st[i];
    *nSteps = ns;
    return 0;
}

int hb2_comm_unique_id(void *uniqueId128) {
    if (!uniqueId128) return fail("null id buffer");
    if (!g_nccl.load()) return fail("cannot load libnccl.so.2: %s", dlerror());
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    ncclResult_t r = g_nccl.GetUniqueId(&id);
    if (r != ncclSuccess) return fail("ncclGetUniqueId: %s", g_nccl.GetErrorString(r));
    memcpy(uniqueId128, &id, 128);
    return 0;
}

int hb2_comm_init(hb2_partition *p, int nRanks, int rank, const void *uniqueId128) {
    if (!p || !uniqueId128) return fail("null argument");
    if (nRanks < 1 || rank < 0 || rank >= nRanks) return fail("bad rank %d of %d", rank, nRanks);
    if (!g_nccl.load()) return fail("cannot load libnccl.so.2: %s", dlerror());
    CU(cudaSetDevice(p->device));
    if (p->comm) { g_nccl.CommDestroy(p->comm); p->comm = nullptr; }      // re-initialisation replaces the communicator
    ncclUniqueId id;
    memcpy(&id, uniqueId128, 128);
    ncclResult_t r = g_nccl.CommInitRank(&p->comm, nRanks, id, rank);
    if (r != ncclSuccess) { p->comm = nullptr; return fail("ncclCommInitRank: %s", g_nccl.GetErrorString(r)); }
    p->n_ranks = nRanks; p->rank = rank;
    return peer_setup(p, 2);
}

int hb2_comm_gather_sites(hb2_partition *p, const double *siteL, const int64_t *siteScale, double *allSiteL, int64_t *allSiteScale,
                          int64_t capacity, int64_t *total) {
    if (!p || !siteL || !siteScale || !allSiteL || !allSiteScale || !total) return fail("null argument");
    if (!p->comm) return fail("hb2_comm_gather_sites needs hb2_comm_init first");
    CU(cudaSetDevice(p->device));
    const int R = p->n_ranks, G = std::max(p->cg_G, 1);
    // 1. every rank's pattern count
    long long mine = (long long)p->S;
    std::vector<long long> cnt(R);
    DeviceBuffer<long long> d_cnt;
    if (d_cnt.alloc(R + 1)) return 1;
    CU(cudaMemcpyAsync(d_cnt + R, &mine, sizeof(long long), cudaMemcpyHostToDevice, p->stream));
    ncclResult_t nr = g_nccl.AllGather(d_cnt + R, d_cnt, sizeof(long long), ncclChar, p->comm, p->stream);
    if (nr != ncclSuccess) return fail("ncclAllGather (pattern counts): %s", g_nccl.GetErrorString(nr));
    CU(cudaMemcpyAsync(cnt.data(), d_cnt, (size_t)R * sizeof(long long), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    long long mx = 0, tot = 0;
    for (int r = 0; r < R; r++) { mx = std::max(mx, cnt[r]); if (r % G == 0) tot += cnt[r]; }    // ranks of one shard hold the same patterns
    *total = (int64_t)tot;
    if (tot > capacity) return fail("hb2_comm_gather_sites: %lld patterns in all shards, room for %lld", tot, (long long)capacity);
    // 2. (likelihood, scaler count) pairs, padded to the largest shard
    const size_t rec = (size_t)mx * 16;
    std::vector<unsigned char> send(rec, 0), all(rec * R);
    for (long long s = 0; s < mine; s++) { memcpy(&send[(size_t)s * 16], siteL + s, 8); memcpy(&send[(size_t)s * 16 + 8], siteScale + s, 8); }
    DeviceBuffer<unsigned char> d_send, d_all;
    if (d_send.alloc(std::max<size_t>(rec, 16)) || d_all.alloc(std::max<size_t>(rec * R, 16))) return 1;
    CU(cudaMemcpyAsync(d_send, send.data(), rec, cudaMemcpyHostToDevice, p->stream));
    nr = g_nccl.AllGather(d_send, d_all, rec, ncclChar, p->comm, p->stream);
    if (nr != ncclSuccess) return fail("ncclAllGather (per-pattern outputs): %s", g_nccl.GetErrorString(nr));
    CU(cudaMemcpyAsync(all.data(), d_all, rec * R, cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    // 3. shard order = rank order of the first rank of every shard
    int64_t at = 0;
    for (int r = 0; r < R; r += G)
        for (long long s = 0; s < cnt[r]; s++, at++) {
            memcpy(allSiteL + at, &all[(size_t)r * rec + (size_t)s * 16], 8);
            memcpy(allSiteScale + at, &all[(size_t)r * rec + (size_t)s * 16 + 8], 8);
        }
    return 0;
}

int hb2_comm_class_groups(hb2_partition *p, int nGroups) {
    if (!p) return fail("null partition");
    if (!p->comm) return fail("hb2_comm_class_groups needs hb2_comm_init first");
    if (nGroups < 1 || p->C % nGroups != 0 || p->n_ranks % nGroups != 0)
        return fail("class groups: %d must divide both the %lld rate classes and the %d ranks", nGroups, (long long)p->C, p->n_ranks);
    for (const Slot &s : p->slots) if (s.have) return fail("hb2_comm_class_groups must be called before matrices are set");
    CU(cudaSetDevice(p->device));
    p->cg_G = nGroups; p->cg_g = p->rank % nGroups;
    p->ownN = (int)(p->C / nGroups); p->own0 = p->cg_g * p->ownN;
    if (nGroups == 1) return 0;
    // exchange length: the longest padded shard among the ranks (shards of the same communicator may differ in size)
    DeviceBuffer<int> d_len;
    if (d_len.alloc(1)) return 1;
    int len = (int)p->Sp;
    CU(cudaMemcpyAsync(d_len, &len, sizeof(int), cudaMemcpyHostToDevice, p->stream));
    ncclResult_t r = g_nccl.AllReduce(d_len, d_len, 1, ncclInt32, ncclMax, p->comm, p->stream);
    if (r != ncclSuccess) return fail("ncclAllReduce(max): %s", g_nccl.GetErrorString(r));
    CU(cudaMemcpyAsync(&len, d_len, sizeof(int), cudaMemcpyDeviceToHost, p->stream));
    CU(cudaStreamSynchronize(p->stream));
    p->xchg_len = len;
    const size_t tot = (size_t)2 * len * p->n_ranks;
    if (p->d_xsend.alloc(tot) || p->d_xrecv.alloc(tot) || p->d_xfreq.alloc((size_t)len * p->n_ranks) ||
        p->d_xpartial.alloc((size_t)len * p->n_ranks / 256 + 2))
        return 1;
    // pattern frequencies of every rank, gathered once with the same zero-elsewhere sum (d_xsend doubles as scratch)
    CU(cudaMemsetAsync(p->d_xsend, 0, tot * sizeof(double), p->stream));
    CU(cudaMemcpyAsync(p->d_xsend + (size_t)p->rank * len, p->d_freq, (size_t)std::min<int64_t>(p->Sp, len) * sizeof(double), cudaMemcpyDeviceToDevice, p->stream));
    r = g_nccl.AllReduce(p->d_xsend, p->d_xfreq, (size_t)len * p->n_ranks, ncclDouble, ncclSum, p->comm, p->stream);
    if (r != ncclSuccess) return fail("ncclAllReduce (frequencies): %s", g_nccl.GetErrorString(r));
    CU(cudaMemsetAsync(p->d_xsend, 0, tot * sizeof(double), p->stream));     // from now on only this rank's slot is written
    CU(cudaStreamSynchronize(p->stream));
    return peer_setup(p, 2 * len);
}

void hb2_destroy(hb2_partition *p) {
    if (!p) return;
    cudaSetDevice(p->device);
    if (p->stream) cudaStreamSynchronize(p->stream);     // first: the pool may hand the released blocks out at once
    if (p->side) cudaStreamSynchronize(p->side);
    peer_teardown(p);
    if (p->comm) g_nccl.CommDestroy(p->comm);
    const cudaStream_t streams[] = {p->stream, p->side};
    const cudaEvent_t events[] = {p->ev[0], p->ev[1], p->ev[2], p->ev[3], p->ev_staging, p->ev_fork, p->ev_join};
    delete p;                                             // releases every buffer
    for (cudaEvent_t e : events) if (e) cudaEventDestroy(e);
    for (cudaStream_t s : streams) if (s) cudaStreamDestroy(s);
}

int64_t hb2_launch_count(const hb2_partition *p) { return p ? p->launches : 0; }
int hb2_precision_mode(const hb2_partition *p) { return (p && p->use_tc) ? 1 : 0; }
int hb2_stage_launches(const hb2_partition *p, int64_t *out3) {
    if (!p || !out3) return fail("null argument");
    for (int k = 0; k < 3; k++) out3[k] = p->stage_launches[k];
    return 0;
}
const char *hb2_pruning_kernel(const hb2_partition *p) { return p ? PRUNE_KERNEL_NAME[pruning_kernel(p, p->ownN)] : ""; }

int hb2_time_resident(hb2_partition *p, const double *weights, const double *rootFreqs, int iters, double *msPerEval,
                      double *stageMs, double *lnL) {
    if (!p || !weights || !rootFreqs || !msPerEval) return fail("null argument");
    if (iters < 1) return fail("iters must be >= 1");
    CU(cudaSetDevice(p->device));
    if (check_ready(p, 0, (int)p->C)) return 1;
    if (flush_matrices(p)) return 1;
    p->bc_node = -1; p->bc_dirty_node = -1;
    // every slot must hold a resident copy of its rate matrix (dense, or the formula values of a compiled hand-over) so
    // that the expm stage can be replayed
    std::vector<int> dst;
    Resident res = Resident::None;
    for (int64_t k = (int64_t)p->own0 * p->B; k < (int64_t)(p->own0 + p->ownN) * p->B; k++) {
        const Slot &s = p->slots[k];
        if (s.res == Resident::None)
            return fail("hb2_time_resident needs a rate matrix (dense or compiled) in every slot, handed over after its template last "
                        "changed: class %lld, branch %lld has none", (long long)(k / p->B), (long long)(k % p->B));
        if (res != Resident::None && res != s.res) return fail("hb2_time_resident: hand all matrices over the same way (dense or compiled) before timing");
        if (s.res == Resident::Formula && s.res_tmpl != 0) return fail("hb2_time_resident replays template 0 only");
        res = s.res;
        dst.push_back((int)k);
    }
    const bool compiled = res == Resident::Formula;
    if (wait_staging(p)) return 1;           // the flush above may still be reading the pinned queues
    HandoverQueue &q = p->dense;             // empty after the flush: its destination slots carry the replay's
    memcpy(q.h_dst, dst.data(), dst.size() * sizeof(int));
    CU(cudaMemcpyAsync(q.d_dst, q.h_dst, dst.size() * sizeof(int), cudaMemcpyHostToDevice, p->stream));
    SharedPlan sp;
    if (plan_shared(p, q.h_dst, (int64_t)dst.size(), compiled ? 1 : 2, nullptr, sp)) return 1;
    if (compiled && !sp.use) return fail("hb2_time_resident: compiled resident copies need the shared-powers path");
    if (staged_uploads(p) || stage_root(p, rootFreqs, weights, (int)p->C)) return 1;
    std::vector<char> dirty;
    if (dirty_nodes(p->parents.data(), p->L, p->I, -1, nullptr, dirty)) return 1;
    const double *in = compiled ? p->tmpls[0].d_Vres + (size_t)p->own0 * p->B * p->tmpls[0].nF : p->d_Qres + (size_t)p->own0 * p->B * p->D * p->D;
    double tot = 0, st[3] = {0, 0, 0};
    for (int it = 0; it < iters; it++) {
        CU(cudaEventRecord(p->ev[0], p->stream));
        const int64_t l0 = p->launches;
        if (launch_expm(p, {compiled ? Kind::Compiled : Kind::Rate}, in, q.d_dst, (int)dst.size(), false, sp)) return 1;
        const int64_t l1 = p->launches;
        CU(cudaEventRecord(p->ev[1], p->stream));
        if (run_pruning(p, p->own0, p->ownN, dirty)) return 1;
        CU(cudaEventRecord(p->ev[2], p->stream));
        const int64_t l2 = p->launches;
        if (run_root(p, p->own0, p->ownN, true, false)) return 1;
        p->stage_launches[0] = l1 - l0; p->stage_launches[1] = l2 - l1; p->stage_launches[2] = p->launches - l2;
        CU(cudaEventRecord(p->ev[3], p->stream));
        CU(cudaEventSynchronize(p->ev[3]));
        float a = 0, b = 0, c = 0;
        CU(cudaEventElapsedTime(&a, p->ev[0], p->ev[1]));
        CU(cudaEventElapsedTime(&b, p->ev[1], p->ev[2]));
        CU(cudaEventElapsedTime(&c, p->ev[2], p->ev[3]));
        st[0] += a; st[1] += b; st[2] += c; tot += a + b + c;
    }
    *msPerEval = tot / iters;
    if (stageMs) for (int k = 0; k < 3; k++) stageMs[k] = st[k] / iters;
    if (lnL) {
        CU(cudaMemcpy(lnL, p->d_lnL, sizeof(double), cudaMemcpyDeviceToHost));
    }
    for (int c = 0; c < p->C; c++) p->evaluated_cat[c] = 1;
    return 0;
}

}  // extern "C"

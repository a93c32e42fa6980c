// c2b_engine.cu -- the sm_90a kernel entry + the C ABI declared in include/c2b200.h.
//
// Build (see __graft_entry__.build):
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -shared -Xcompiler -fPIC \
//        -Iinclude -o crispresso2_b200/libc2b200.so crispresso2_b200/csrc/c2b_engine.cu
// The same file compiles with g++ -DC2B_EMU against tests/emu/warp_emu.h (CPU-only logic tests).
#include <algorithm>
#include <atomic>
#include <mutex>
#ifndef C2B_EMU
#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>
#include <cctype>
#endif
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <memory>
#include <unordered_map>
#include <vector>

#include "c2b_core.cuh"
#include "c2b_split.cuh"
#include "c2b_annotate.cuh"
#include "c2b_vcf.cuh"
#include "c2b_base_edit.cuh"
#include "c2b_amino.cuh"
#include "c2b_fastq_int.h"

using namespace c2b;

// ----------------------------------------------------------------------------------- runtime shim
#ifndef C2B_EMU
#define RT_OK cudaSuccess
typedef cudaStream_t rt_stream;
static const char *rt_errstr(cudaError_t e) { return cudaGetErrorString(e); }
typedef cudaError_t rt_err;
static rt_err rt_malloc(void **p, size_t n) { return cudaMalloc(p, n ? n : 16); }
static rt_err rt_free(void *p) { return cudaFree(p); }
static rt_err rt_h2d(void *d, const void *h, size_t n, rt_stream s) { return n ? cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, s) : cudaSuccess; }
static rt_err rt_d2h(void *h, const void *d, size_t n, rt_stream s) { return n ? cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, s) : cudaSuccess; }
static rt_err rt_zero(void *d, size_t n, rt_stream s) { return cudaMemsetAsync(d, 0, n, s); }
static rt_err rt_d2h_2d(void *h, const void *d, size_t pitch, size_t width, size_t rows, rt_stream s)
{ return (width && rows) ? cudaMemcpy2DAsync(h, pitch, d, pitch, width, rows, cudaMemcpyDeviceToHost, s) : cudaSuccess; }
// A persistent kernel that never finishes (a lost barrier, a spin on a flag nobody sets) would block its host thread for ever and
// nothing can cancel it.  Every blocking wait registers itself; a watchdog thread ends the process with a message when one has lasted
// longer than C2B_WATCHDOG_S seconds (default 1800; 0 = no watchdog) -- a loud failure instead of a silent hang.
static std::atomic<int64_t> g_wait_since[32];
static int64_t wd_now_ms() { return std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
static int64_t wd_limit_ms()
{
    static const int64_t lim = [] { const char *v = getenv("C2B_WATCHDOG_S"); const double s = v ? atof(v) : 1800.0; return (int64_t)(s * 1000.0); }();
    return lim;
}
static void wd_start()
{
    static std::once_flag once;
    std::call_once(once, [] {
        if (wd_limit_ms() <= 0) return;
        std::thread([] {
            const int64_t lim = wd_limit_ms();
            const auto nap = std::chrono::milliseconds(std::max<int64_t>(20, std::min<int64_t>(1000, lim / 4)));
            for (;;) {
                std::this_thread::sleep_for(nap);
                const int64_t now = wd_now_ms();
                for (auto &w : g_wait_since) {
                    const int64_t t = w.load(std::memory_order_relaxed);
                    if (t && now - t > lim) {
                        fprintf(stderr, "c2b200: a wait for the GPU has lasted more than %.3g s (a kernel that does not finish?) -- ending the "
                                        "process; C2B_WATCHDOG_S sets the limit, 0 disables\n", lim / 1000.0);
                        fflush(stderr);
                        _exit(70);
                    }
                }
            }
        }).detach();
    });
}
struct WaitGuard {
    int k = -1;
    WaitGuard()
    {
        wd_start();
        const int64_t now = wd_now_ms();
        for (int i = 0; i < 32; i++) { int64_t z = 0; if (g_wait_since[i].compare_exchange_strong(z, now, std::memory_order_relaxed)) { k = i; break; } }
    }
    ~WaitGuard() { if (k >= 0) g_wait_since[k].store(0, std::memory_order_relaxed); }
};
static rt_err rt_sync(rt_stream s) { WaitGuard g; return cudaStreamSynchronize(s); }
static rt_err cudaMemcpyAsyncOrCopy(void *d, const void *s_, size_t n, rt_stream st) { return cudaMemcpyAsync(d, s_, n, cudaMemcpyDeviceToDevice, st); }
typedef cudaEvent_t rt_event;
static rt_err rt_event_create(rt_event *e) { return cudaEventCreateWithFlags(e, cudaEventDisableTiming); }
static rt_err rt_event_destroy(rt_event e) { return cudaEventDestroy(e); }
static rt_err rt_record(rt_event e, rt_stream s) { return cudaEventRecord(e, s); }
static rt_err rt_wait(rt_stream s, rt_event e) { return cudaStreamWaitEvent(s, e, 0); }
static rt_err rt_event_sync(rt_event e) { WaitGuard g; return cudaEventSynchronize(e); }
static rt_err rt_stream_create(rt_stream *s) { return cudaStreamCreateWithFlags(s, cudaStreamNonBlocking); }
static rt_err rt_stream_destroy(rt_stream s) { return cudaStreamDestroy(s); }
static void *rt_host_alloc(size_t n) { void *p = nullptr; return cudaHostAlloc(&p, n ? n : 16, cudaHostAllocDefault) == cudaSuccess ? p : nullptr; }
static void rt_host_free(void *p) { if (p) cudaFreeHost(p); }
#else
typedef int rt_err;
typedef int rt_stream;
#define RT_OK 0
thread_local emu::Warp *emu::g_warp = nullptr;
static const char *rt_errstr(int) { return "emu"; }
static rt_err rt_malloc(void **p, size_t n) { *p = calloc(1, n ? n : 16); return *p ? 0 : 1; }
static rt_err rt_free(void *p) { free(p); return 0; }
static rt_err rt_h2d(void *d, const void *h, size_t n, rt_stream) { if (n) memcpy(d, h, n); return 0; }
static rt_err rt_d2h(void *h, const void *d, size_t n, rt_stream) { if (n) memcpy(h, d, n); return 0; }
static rt_err rt_zero(void *d, size_t n, rt_stream) { memset(d, 0, n); return 0; }
static rt_err rt_d2h_2d(void *h, const void *d, size_t pitch, size_t width, size_t rows, rt_stream)
{ for (size_t r = 0; r < rows; r++) memcpy((char *)h + r * pitch, (const char *)d + r * pitch, width); return 0; }
static rt_err rt_sync(rt_stream) { return 0; }
static rt_err cudaMemcpyAsyncOrCopy(void *d, const void *s_, size_t n, rt_stream) { memcpy(d, s_, n); return 0; }
typedef int rt_event;
static rt_err rt_event_create(rt_event *e) { *e = 0; return 0; }
static rt_err rt_event_destroy(rt_event) { return 0; }
static rt_err rt_record(rt_event, rt_stream) { return 0; }
static rt_err rt_wait(rt_stream, rt_event) { return 0; }
static rt_err rt_event_sync(rt_event) { return 0; }
static rt_err rt_stream_create(rt_stream *s) { *s = 0; return 0; }
static rt_err rt_stream_destroy(rt_stream) { return 0; }
static void *rt_host_alloc(size_t n) { return malloc(n ? n : 16); }
static void rt_host_free(void *p) { free(p); }
#endif

// ----------------------------------------------------------------------------------------- kernel
constexpr int WARPS_PER_CTA = 8;                                 // general and ALIGN kernels
static_assert(WARPS_PER_CTA % 4 == 0, "the general kernel's phase sets are four warps");
constexpr int MIN_CTAS_PER_SM = 2;                               // general kernel
constexpr int A_MIN_CTAS = 2;                                    // ALIGN kernel
constexpr int B_WARPS_PER_CTA = 4, B_MIN_CTAS = 6;               // CLASSIFY kernel
constexpr int D_WARPS_PER_CTA = 8;                               // diagonal tier

#ifndef C2B_EMU
// TMA-staged reference tile: the packed substitution profile of reference 0, once per CTA (cp.async.bulk + mbarrier);
// every DP step then reads it with two 16-byte LDS.  -> shared-memory address of the tile, or nullptr
__device__ __forceinline__ const uint32_t *stage_profile(const KParams &P, unsigned char *dst)
{
    if (P.stage_bytes <= 0) return nullptr;
    __shared__ __align__(8) unsigned long long mbar;
    const uint32_t mbar_a = (uint32_t)__cvta_generic_to_shared(&mbar), dst_a = (uint32_t)__cvta_generic_to_shared(dst);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbar_a));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar_a), "r"((uint32_t)P.stage_bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(dst_a), "l"(P.stage_src), "r"((uint32_t)P.stage_bytes), "r"(mbar_a) : "memory");
    }
    asm volatile("{\n .reg .pred p;\n C2B_WAIT:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n @p bra C2B_DONE;\n bra C2B_WAIT;\n C2B_DONE:\n}" ::"r"(mbar_a) : "memory");
    return reinterpret_cast<const uint32_t *>(dst);
}

// Each kernel carves up its shared memory, stages the profile tile and runs its loop (c2b_split.cuh, c2b_core.cuh); the
// emulator build runs the same loops as a grid of one warp (run_plan).

// GENERAL kernel: the whole per-read path in one launch (any length within the build limits, any parameters; full-matrix
// DP paths of c2b_core.cuh).  Since r02 it runs after the ALIGN / CLASSIFY pair, over the pairs ALIGN left over (P.n_dev,
// P.pair_order = the left-over list), or alone when the two-kernel form does not apply.
// ONE: every read has one candidate reference (a single amplicon configured, or Pooled ref_id).
// P is a __grid_constant__: the out-of-line device functions take it by reference, and without the qualifier every launch
// copied the struct to each thread's local memory and read its fields back with LDL (slower).
template <bool ONE>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, MIN_CTAS_PER_SM) c2b_align_classify_kernel(const __grid_constant__ KParams P)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    WarpSmem *S = reinterpret_cast<WarpSmem *>(smem_raw) + (threadIdx.x >> 5);
    QuadSmem *Q = reinterpret_cast<QuadSmem *>(smem_raw + (size_t)(blockDim.x >> 5) * sizeof(WarpSmem)) + (threadIdx.x >> 5);
    const int warp_slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const uint32_t *staged_prof = stage_profile(P, smem_raw + (((size_t)(blockDim.x >> 5) * (sizeof(WarpSmem) + sizeof(QuadSmem)) + 127) & ~(size_t)127));
    if (P.n_dev) {
        general_list_loop<ONE>(P, *S, staged_prof, warp_slot);
        return;
    }
    // Phase sets: work groups (8 reads each) are handed out per set of g consecutive warps, one group per warp, one hand-out
    // ahead, so that the loop count -- and with it the number of barriers executed by process_group's phases -- is the same
    // for every warp of the set, and the next group's read bytes are on their way to L2 while this one computes.  This loop
    // needs the warps of a set in step, so it is the one loop the emulator does not share: it runs process_group per group
    // there and checks the barrier count of each (run_plan).  Free-running warps were measured 40-55 % slower on batches whose
    // groups take the ring (DESIGN.md section 3).
    __shared__ unsigned long long next_base[WARPS_PER_CTA];
    const int gs = P.phase_sync, g = gs > 0 ? gs : 1, wib = threadIdx.x >> 5;
    const int set = wib / g, wis = wib % g;
    const int64_t nrd = nreads(P);
    const unsigned long long total = ((unsigned long long)nrd + 7) / 8;
    auto hand_out = [&]() -> unsigned long long {
        if (wis == 0 && (threadIdx.x & 31) == 0) next_base[set] = atomicAdd(P.work_counter, (unsigned long long)g);
        if (g > 1) wp::grp_sync(gs); else __syncwarp();
        const unsigned long long b = next_base[set];
        if (g > 1) wp::grp_sync(gs); else __syncwarp();
        return b;
    };
    unsigned long long base = hand_out();
    while (base < total) {
        const unsigned long long nb = hand_out();
        const unsigned long long wn = nb + wis;
        if (wn < total && !P.pair_order) {
            const int64_t last = (int64_t)(8 * wn + 8) < nrd ? (int64_t)(8 * wn + 8) : nrd;
            const int64_t b0 = P.offsets[8 * wn], b1 = P.offsets[last];
            const int64_t a = b0 + (int64_t)(threadIdx.x & 31) * 128;
            if (a < b1) asm volatile("prefetch.global.L2 [%0];" ::"l"(P.reads + a));
        }
        const unsigned long long w = base + wis;
        if (w < total) process_group<ONE>(P, *S, *Q, staged_prof, (int64_t)w, warp_slot);  // reads 8w .. 8w+7
        else if (P.phase_sync) for (int b = group_phases(P); b > 0; b--) wp::grp_sync(gs);
        __syncwarp();
        base = nb;
    }
}

// ALIGN kernel (c2b_split.cuh: align_loop)
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, A_MIN_CTAS) c2b_align_kernel(const __grid_constant__ KParams P)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    ASmem *S = reinterpret_cast<ASmem *>(smem_raw) + (threadIdx.x >> 5);
    const int nw = blockDim.x >> 5;
    const uint32_t *staged_prof = stage_profile(P, smem_raw + (((size_t)nw * sizeof(ASmem) + 127) & ~(size_t)127));
    align_loop(P, *S, staged_prof, blockIdx.x * nw + (threadIdx.x >> 5));
}

// Diagonal tier (c2b_split.cuh: diag_loop)
__global__ void __launch_bounds__(D_WARPS_PER_CTA * 32) c2b_diag_kernel(const __grid_constant__ KParams P)
{
    __shared__ DSmem smem[D_WARPS_PER_CTA];
    diag_loop(P, smem[threadIdx.x >> 5], (int64_t)blockIdx.x * D_WARPS_PER_CTA + (threadIdx.x >> 5), (int64_t)gridDim.x * D_WARPS_PER_CTA);
}

// CLASSIFY kernel (c2b_split.cuh: classify_loop)
template <bool ONE>
__global__ void __launch_bounds__(B_WARPS_PER_CTA * 32, B_MIN_CTAS) c2b_classify_kernel(const __grid_constant__ KParams P)
{
    __shared__ BSmem smem[B_WARPS_PER_CTA];
    classify_loop<ONE>(P, smem[threadIdx.x >> 5], (int64_t)blockIdx.x * B_WARPS_PER_CTA + (threadIdx.x >> 5), (int64_t)gridDim.x * B_WARPS_PER_CTA);
}
#endif

// ----------------------------------------------------------------------------------------- engine
struct RefHost {
    std::string seq; std::vector<int64_t> gi, inc; double min_aln; std::vector<int64_t> rows;
    std::vector<std::string> fw, rc;
    int64_t sabs = 0, gabs = 0, gsum_abs = 0, gi0_abs = 0;   // largest |score|, largest and summed |gap_incentive|, |gap_incentive[0]|
};

struct DevBuf {
    void *p = nullptr; size_t cap = 0;
};

struct c2b_engine {
    int device = 0;
    rt_stream stream = 0;
    std::string err;
    bool configured = false;
    c2b_params prm;
    int n_refs = 0, max_I = 0, max_nrb = 1, vstride = 0, hstride = 0, hist_zero = 0;
    std::vector<RefHost> refs;
    std::vector<RefDev> refdev;         // host mirror (device pointers inside)
    void *d_tables = nullptr; RefDev *d_refs = nullptr;
    unsigned long long *d_counts = nullptr; size_t counts_n = 0;
    // scratch
    DevBuf tb, tbb, tbq, bnd, ops, rgo, work, lut;
    DevBuf gops, gmeta, left, left2, left0, left1;   // device-pointer API: op streams / meta words / left-over lists of the last launch
    DevBuf pro_tab, pro_in, pro_out, pro_tb, pro_bnd;  // protein alignment (c2b_protein_align): tables, reads, op streams, slabs
    int n_warps = 0, grid = 0, stage_cap = 0;
    int grid_a = 0, grid_b = 0, stage_cap_a = 0;       // ALIGN / CLASSIFY kernels
    int split_ok = 0, split_all = 0;                   // configuration admits the two-kernel form (some / all references)
    int diag_any = 0;                                  // some reference admits the diagonal tier (RefDev::dg_ok)
    int numa_node = -1;                                // NUMA node of the device (-1: unknown / single node)
    int scratch_TS = 0;
    // staging for the host-pointer API: two buffer sets, copy-in / compute / copy-out streams
    struct Stage { DevBuf reads, off, cnt, qw, rid, recs, alns, str, ed, maxlen, ord, gops, gmeta, left, left2, left0, left1; int32_t *h_ord = nullptr; size_t h_ord_cap = 0; int64_t *h_off = nullptr; size_t h_off_cap = 0;
                   // pinned bounce buffers for callers whose arrays are pageable (numpy): copies to / from them run on host
                   // threads while the other set's kernels and DMA are in flight
                   uint8_t *h_in = nullptr, *h_out = nullptr; size_t h_in_cap = 0, h_out_cap = 0;
                   int64_t d_c0 = 0, d_n = 0; size_t d_Wt = 0; bool drain = false;     // chunk waiting in h_out
                   rt_event in_done, k_done, out_done; bool used = false; } stage[2];
    rt_stream s_in = 0, s_out = 0;
    bool pipe_ready = false;
    double last_ms = 0; int64_t launches = 0;
    const uint64_t *forced_ops = nullptr; const int32_t *forced_n = nullptr;
    const int32_t *pair_order = nullptr;
    int64_t band_reruns = 0, ring_pairs = 0, ring_fallbacks = 0;
#ifndef C2B_EMU
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
#endif
};

static std::string g_create_err;

static int fail(c2b_engine *e, int code, const std::string &m) { if (e) e->err = m; else g_create_err = m; return code; }

#define RTCHK(call) do { rt_err _r = (call); if (_r != RT_OK) return fail(e, C2B_E_CUDA, std::string(#call) + ": " + rt_errstr(_r)); } while (0)

static int ensure(c2b_engine *e, DevBuf &b, size_t n)
{
    if (n <= b.cap) return C2B_OK;
    if (b.p) rt_free(b.p);
    b.p = nullptr; b.cap = 0;
    size_t want = n + n / 8 + 256;
    RTCHK(rt_malloc(&b.p, want));
    b.cap = want;
    return C2B_OK;
}

extern "C" {

#ifndef C2B_EMU
// Host side of a rank: run on, and allocate pinned memory from, the NUMA node the GPU hangs off.  On the two-socket
// hosts this engine targets, ranks whose pinned buffers sit on the other socket push every H2D / D2H byte through the
// socket interconnect (r01: e2e efficiency 0.55 at 8 GPUs with un-placed buffers).  Binds the CALLING thread (threads it
// creates later inherit it) unless the process already restricted its CPUs to one node or C2B_NO_NUMA_BIND is set.
static int numa_bind_for_device(int device)
{
    if (getenv("C2B_NO_NUMA_BIND")) return -1;
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) return -1;
    for (char *c = bus; *c; c++) *c = (char)tolower(*c);
    char path[256];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE *f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    if (node < 0) return -1;
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r");
    if (!f) return -1;
    char list[4096] = {0};
    if (!fgets(list, sizeof list, f)) { fclose(f); return -1; }
    fclose(f);
    cpu_set_t want, have;
    CPU_ZERO(&want);
    for (char *tok = strtok(list, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
        int lo = 0, hi = 0;
        if (sscanf(tok, "%d-%d", &lo, &hi) == 2) { for (int c = lo; c <= hi && c < CPU_SETSIZE; c++) CPU_SET(c, &want); }
        else if (sscanf(tok, "%d", &lo) == 1 && lo < CPU_SETSIZE) CPU_SET(lo, &want);
    }
    if (sched_getaffinity(0, sizeof have, &have) != 0) return node;
    cpu_set_t both;
    CPU_AND(&both, &want, &have);
    if (CPU_COUNT(&both) == 0) return node;                 // the caller pinned us elsewhere: leave it
    if (CPU_COUNT(&both) < CPU_COUNT(&have)) sched_setaffinity(0, sizeof both, &both);
    // memory policy of this thread: prefer the device's node (pinned allocations made by this thread follow it)
    unsigned long mask[16] = {0};
    if (node < (int)(sizeof mask * 8)) {
        mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
        syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, sizeof mask * 8);
    }
    return node;
}
#endif

int c2b_create(int device, c2b_engine **out)
{
    if (!out) return C2B_E_ARG;
    c2b_engine *e = new c2b_engine();
    e->device = device;
#ifndef C2B_EMU
    cudaError_t r = cudaSetDevice(device);
    if (r == cudaSuccess) e->numa_node = numa_bind_for_device(device);
    if (r == cudaSuccess) r = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking);
    if (r == cudaSuccess) r = cudaEventCreate(&e->ev0);
    if (r == cudaSuccess) r = cudaEventCreate(&e->ev1);
    int nsm = 0, occ = 0, smem_sm = 0, optin = 0;
    if (r == cudaSuccess) r = cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device);
    if (r == cudaSuccess) r = cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, device);
    if (r == cudaSuccess) r = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    // room for a TMA-staged reference tile next to MIN_CTAS_PER_SM CTAs of per-warp state (1 KB per CTA is reserved by the driver)
    // ... and the kernels' static shared memory (hand-out slots, mbarrier) -- if the sum is a byte too large the
    // occupancy query answers 1 CTA per SM and the persistent grid silently halves
    auto tile_room = [&](size_t per_warp, int ctas) {
        int cap = smem_sm / ctas - 1024 - (int)(per_warp * WARPS_PER_CTA) - 2048;
        const int fixed = (int)(per_warp * WARPS_PER_CTA) + 128;
        if (cap > optin - fixed) cap = optin - fixed;
        if (cap < 0) cap = 0;
        return cap & ~127;
    };
    e->stage_cap = tile_room(sizeof(WarpSmem) + sizeof(QuadSmem), MIN_CTAS_PER_SM);
    const int dyn_smem = (int)((sizeof(WarpSmem) + sizeof(QuadSmem)) * WARPS_PER_CTA) + 128 + e->stage_cap;
    {
        const void *kernels[2] = {(const void *)c2b_align_classify_kernel<true>, (const void *)c2b_align_classify_kernel<false>};
        occ = 1 << 20;
        for (const void *k : kernels) {                    // both instantiations must fit the same persistent grid
            int o = 0;
            if (r == cudaSuccess) r = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_smem);
            if (r == cudaSuccess) r = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k, WARPS_PER_CTA * 32, dyn_smem);
            occ = std::min(occ, o);
        }
    }
    // ALIGN kernel: its own (smaller) per-warp state; CTAs per SM from the occupancy query
    int occ_a = 0, occ_b = 0;
    e->stage_cap_a = tile_room(sizeof(ASmem), A_MIN_CTAS);
    const int dyn_a = (int)(sizeof(ASmem) * WARPS_PER_CTA) + 128 + e->stage_cap_a;
    if (r == cudaSuccess) r = cudaFuncSetAttribute((const void *)c2b_align_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_a);
    if (r == cudaSuccess) r = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_a, (const void *)c2b_align_kernel, WARPS_PER_CTA * 32, dyn_a);
    if (r == cudaSuccess) r = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_b, (const void *)c2b_classify_kernel<true>, B_WARPS_PER_CTA * 32, 0);
    {
        int o = 0;
        if (r == cudaSuccess) r = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, (const void *)c2b_classify_kernel<false>, B_WARPS_PER_CTA * 32, 0);
        occ_b = std::min(occ_b, o);
    }
    if (r != cudaSuccess) { g_create_err = std::string("c2b_create: ") + cudaGetErrorString(r); delete e; return C2B_E_CUDA; }
    if (occ < 1) occ = 1;
    if (occ_a < 1) occ_a = 1;
    if (occ_b < 1) occ_b = 1;
    if (occ < MIN_CTAS_PER_SM)
        fprintf(stderr, "[c2b] warning: only %d CTA(s) of the general kernel fit an SM (built for %d)\n", occ, MIN_CTAS_PER_SM);
    if (occ_a > A_MIN_CTAS) occ_a = A_MIN_CTAS;
    e->grid = nsm * occ;                 // persistent: one wave of CTAs, warps pull work items from a counter
    e->grid_a = nsm * occ_a;
    e->grid_b = nsm * std::min(occ_b, 8);
    e->n_warps = std::max(e->grid, e->grid_a) * WARPS_PER_CTA;  // scratch slabs are per resident warp of whichever kernel is larger
    if (getenv("C2B_VERBOSE"))
        fprintf(stderr, "[c2b] device %d (NUMA node %d): general kernel %d CTAs/SM, ALIGN %d CTAs/SM (tile room %d B), CLASSIFY %d CTAs/SM x %d warps\n",
                device, e->numa_node, occ, occ_a, e->stage_cap_a, std::min(occ_b, 8), B_WARPS_PER_CTA);
#else
    e->grid = 1; e->n_warps = 1;
#endif
    *out = e;
    return C2B_OK;
}

void c2b_destroy(c2b_engine *e)
{
    if (!e) return;
    DevBuf *bufs[] = {&e->tb, &e->tbb, &e->tbq, &e->bnd, &e->ops, &e->rgo, &e->work, &e->lut, &e->gops, &e->gmeta, &e->left, &e->left2, &e->left0, &e->left1,
                      &e->pro_tab, &e->pro_in, &e->pro_out, &e->pro_tb, &e->pro_bnd};
    for (DevBuf *b : bufs) if (b->p) rt_free(b->p);
    for (auto &st : e->stage) {
        DevBuf *sb[] = {&st.reads, &st.off, &st.cnt, &st.qw, &st.rid, &st.recs, &st.alns, &st.str, &st.ed, &st.maxlen, &st.ord, &st.gops, &st.gmeta, &st.left, &st.left2, &st.left0, &st.left1};
        if (st.h_ord) rt_host_free(st.h_ord);
        for (DevBuf *b : sb) if (b->p) rt_free(b->p);
        if (st.h_off) rt_host_free(st.h_off);
        if (st.h_in) rt_host_free(st.h_in);
        if (st.h_out) rt_host_free(st.h_out);
        if (e->pipe_ready) { rt_event_destroy(st.in_done); rt_event_destroy(st.k_done); rt_event_destroy(st.out_done); }
    }
    if (e->pipe_ready) { rt_stream_destroy(e->s_in); rt_stream_destroy(e->s_out); }
    if (e->d_tables) rt_free(e->d_tables);
    if (e->d_counts) rt_free(e->d_counts);
#ifndef C2B_EMU
    if (e->ev0) cudaEventDestroy(e->ev0);
    if (e->ev1) cudaEventDestroy(e->ev1);
    if (e->stream) cudaStreamDestroy(e->stream);
#endif
    delete e;
}

const char *c2b_last_error(const c2b_engine *e) { return e ? e->err.c_str() : g_create_err.c_str(); }

static uint64_t pack_seed(const c2b_params &p, const std::string &s)
{
    uint64_t v = 0;
    for (size_t c = 0; c < s.size(); c++) {
        int code = -1;
        for (int q = 0; q < p.nq; q++) if (s[c] == p.alphabet[q]) code = q;
        if (code < 0) return ~0ull;                     // can never equal a read k-mer
        v |= (uint64_t)code << (3 * c);
    }
    return v;
}

int c2b_configure(c2b_engine *e, const c2b_params *p, int32_t n_refs, const c2b_ref *refs)
{
    if (!e || !p || !refs || n_refs < 1) return fail(e, C2B_E_ARG, "c2b_configure: bad argument");
    if (n_refs > C2B_MAX_POOLED_REFS) return fail(e, C2B_E_LIMIT, "c2b_configure: more than C2B_MAX_POOLED_REFS references");
    if (p->nq < 1 || p->nq > C2B_MAX_Q) return fail(e, C2B_E_ARG, "c2b_configure: alphabet size out of range");
    if (p->seed_count < 0 || p->edit_cap < 0) return fail(e, C2B_E_ARG, "c2b_configure: negative seed_count/edit_cap");
    e->configured = false;
    e->prm = *p;
    e->n_refs = n_refs;
    e->refs.assign(n_refs, RefHost());
    e->refdev.assign(n_refs, RefDev());
    int maxI = 0, max_nrb = 1;
    size_t bytes = 0;
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    std::vector<size_t> base(n_refs);
    for (int r = 0; r < n_refs; r++) {
        const c2b_ref &rf = refs[r];
        if (!rf.seq || rf.len < 1 || !rf.gap_incentive || !rf.score_rows) return fail(e, C2B_E_ARG, "c2b_configure: incomplete reference");
        if (rf.len > C2B_MAX_REF_LEN) return fail(e, C2B_E_LIMIT, "c2b_configure: reference longer than C2B_MAX_REF_LEN");
        if (rf.n_seeds > 0 && (!rf.fw_seeds || !rf.rc_seeds)) return fail(e, C2B_E_ARG, "c2b_configure: seeds missing");
        maxI = std::max(maxI, rf.len);
        const int nrb = (rf.len + 255) / 256, Ipad = nrb * 256;
        max_nrb = std::max(max_nrb, nrb);
        base[r] = bytes;
        bytes += al((size_t)p->nq * Ipad * 4) + 2 * al((size_t)Ipad * 4) + 2 * al(Ipad) + al(Ipad + 1) + 3 * al((size_t)(Ipad + 2) * 2);
        bytes += al((size_t)p->nq * p->nq * Ipad * 4) + 2 * al((size_t)Ipad * 4);      // packed-path tables
        bytes += al((size_t)(Ipad / 32 + 2) * 16);                                      // routing test's bit planes
    }
    const size_t refs_off = bytes;
    bytes += al(sizeof(RefDev) * n_refs);
    std::vector<unsigned char> blob(bytes, 0);
    if (e->d_tables) { rt_free(e->d_tables); e->d_tables = nullptr; }
    RTCHK(rt_malloc(&e->d_tables, bytes));
    e->vstride = (maxI + 31) & ~31;
    {   // histogram buckets: sizes 0..I, effective lengths 0..I+J, frame keys -I+tem..J+tem around hist_zero
        int max_tem = 0;
        for (int r = 0; r < n_refs; r++) max_tem = std::max(max_tem, std::abs((int)refs[r].tot_exon_len_mod));
        if (max_tem > 4 * C2B_MAX_REF_LEN) return fail(e, C2B_E_LIMIT, "c2b_configure: tot_exon_len_mod out of range");
        e->hist_zero = maxI + max_tem;
        const int need = std::max(e->hist_zero + C2B_MAX_READ_LEN + max_tem, std::min(maxI + C2B_MAX_READ_LEN, C2B_MAX_ALN_LEN)) + 1;
        e->hstride = (need + 31) & ~31;
    }
    const size_t per_ref = C2B_NVEC * (size_t)e->vstride + C2B_NHIST * (size_t)e->hstride + C2B_NSCAL;
    e->counts_n = (size_t)n_refs * per_ref;
    if (e->d_counts) { rt_free(e->d_counts); e->d_counts = nullptr; }
    RTCHK(rt_malloc((void **)&e->d_counts, e->counts_n * 8));
    RTCHK(rt_zero(e->d_counts, e->counts_n * 8, e->stream));

    for (int r = 0; r < n_refs; r++) {
        const c2b_ref &rf = refs[r];
        const int I = rf.len, nrb = (I + 255) / 256, Ipad = nrb * 256;
        RefDev &d = e->refdev[r];
        e->refs[r].seq.assign(rf.seq, (size_t)rf.len);
        d.I = I; d.nrb = nrb; d.Ipad = Ipad; d.kstar = (I - 1) & 7; d.lstar = ((I - 1) >> 3) & 31;
        d.min_aln = rf.min_aln_score;
        unsigned char *hb = blob.data() + base[r];
        unsigned char *db = (unsigned char *)e->d_tables + base[r];
        size_t o = 0;
        int32_t *prof = (int32_t *)(hb + o); d.prof = (const int32_t *)(db + o); o += al((size_t)p->nq * Ipad * 4);
        int32_t *cIe = (int32_t *)(hb + o); d.cIe = (const int32_t *)(db + o); o += al((size_t)Ipad * 4);
        int32_t *g4 = (int32_t *)(hb + o); d.g4 = (const int32_t *)(db + o); o += al((size_t)Ipad * 4);
        uint8_t *asc = hb + o; d.asc = db + o; o += al(Ipad);
        uint8_t *rcode = hb + o; d.rcode = db + o; o += al(Ipad);
        uint8_t *incl = hb + o; d.incl = db + o; o += al(Ipad + 1);
        uint16_t *cum = (uint16_t *)(hb + o); d.cum = (const uint16_t *)(db + o); o += al((size_t)(Ipad + 2) * 2);
        uint16_t *cumx = (uint16_t *)(hb + o); d.cumx = (const uint16_t *)(db + o); o += al((size_t)(Ipad + 2) * 2);
        uint16_t *cums = (uint16_t *)(hb + o); d.cums = (const uint16_t *)(db + o); o += al((size_t)(Ipad + 2) * 2);
        uint32_t *prof2 = (uint32_t *)(hb + o); d.prof2 = (const uint32_t *)(db + o); o += al((size_t)p->nq * p->nq * Ipad * 4);
        uint32_t *cIe2 = (uint32_t *)(hb + o); d.cIe2 = (const uint32_t *)(db + o); o += al((size_t)Ipad * 4);
        uint32_t *g42 = (uint32_t *)(hb + o); d.g42 = (const uint32_t *)(db + o); o += al((size_t)Ipad * 4);
        uint4 *rt_pl = (uint4 *)(hb + o); d.rt_pl = (const uint4 *)(db + o); o += al((size_t)(Ipad / 32 + 2) * 16);
        const int64_t lim = (1ll << 27);
        for (int q = 0; q < p->nq; q++)
            for (int i = 0; i < I; i++) {
                const int64_t v = rf.score_rows[(size_t)q * I + i];
                if (v > lim || v < -lim) return fail(e, C2B_E_LIMIT, "c2b_configure: substitution score out of range");
                prof[(size_t)q * Ipad + i] = (int32_t)(4 * v);
            }
        for (int i = 0; i <= I; i++) if (rf.gap_incentive[i] > lim || rf.gap_incentive[i] < -lim) return fail(e, C2B_E_LIMIT, "c2b_configure: gap incentive out of range");
        {   // extrema for the per-batch score range check (score_range_ok)
            RefHost &h = e->refs[r];
            h.sabs = h.gabs = h.gsum_abs = 0; h.gi0_abs = std::abs(rf.gap_incentive[0]);
            for (size_t k = 0; k < (size_t)p->nq * I; k++) h.sabs = std::max<int64_t>(h.sabs, std::abs(rf.score_rows[k]));
            for (int i = 0; i <= I; i++) { h.gabs = std::max<int64_t>(h.gabs, std::abs(rf.gap_incentive[i])); h.gsum_abs += std::abs(rf.gap_incentive[i]); }
        }
        for (int row = 0; row < I; row++) {
            cIe[row] = (int32_t)(4 * (p->gap_extend + rf.gap_incentive[row + 1]));
            g4[row] = (int32_t)(4 * rf.gap_incentive[row]);
            asc[row] = (uint8_t)rf.seq[row];
            int code = 255;
            for (int q = 0; q < p->nq; q++) if (rf.seq[row] == p->alphabet[q]) code = q;
            rcode[row] = (uint8_t)code;
        }
        d.gi0_4 = (int32_t)(4 * rf.gap_incentive[0]);
        {   // packed 16-bit path: biased scores (beta = -gap_extend per unit of i+j) + offset; see DESIGN.md section 6
            const int64_t go = p->gap_open, ge = p->gap_extend, beta = -ge, OFFu = 512;
            int64_t gmin = rf.gap_incentive[0], gmax = rf.gap_incentive[0], smin = rf.score_rows[0], smax = rf.score_rows[0];
            for (int i = 0; i <= I; i++) { gmin = std::min(gmin, rf.gap_incentive[i]); gmax = std::max(gmax, rf.gap_incentive[i]); }
            for (size_t k = 0; k < (size_t)p->nq * I; k++) { smin = std::min(smin, rf.score_rows[k]); smax = std::max(smax, rf.score_rows[k]); }
            bool ok = go <= ge && ge <= 0 && gmin >= 0 && gmax <= 64 && smin + 2 * beta >= 0 && smax + 2 * beta <= 1000 &&
                      (go - ge) > -1900 && 4 * (OFFu + (go - ge)) > 256 + 4 * gmax + 3 + 64 && !(p->flags & C2B_F_NO_PAIRING);
            d.pk_maxJ = 0;
            if (ok) {
                for (int J = 1; J <= C2B_MAX_READ_LEN && I + J <= PK_MAX_ALN2; J++) {      // device paths that hold 512 columns add I + J <= PK_MAX_ALN
                    const int64_t bound = 4 * ((smax + 2 * beta) * std::min(I, J) + gmax * (I + J + 2) + OFFu) + 3;
                    if (bound > 32000) break;
                    d.pk_maxJ = J;
                }
            }
            const uint32_t rep = 0x00010001u;
            d.pk_XB = (uint32_t)((4 * (rf.gap_incentive[0] + OFFu)) | 2) * rep;
            d.pk_YB = (uint32_t)((4 * (rf.gap_incentive[0] + OFFu)) | 1) * rep;
            d.pk_M00 = (uint32_t)(4 * OFFu) * rep;
            {   // ring-banded path: the out-of-band score bound (ring_bound) must be decreasing in the number of gap columns
                int64_t gsum = 0;
                for (int i = 0; i <= I; i++) gsum += rf.gap_incentive[i];
                d.rg_smax = (int32_t)smax; d.rg_gmax = (int32_t)gmax; d.rg_gsum = (int32_t)std::min<int64_t>(gsum, 1 << 24);
                d.rg_ok = d.pk_maxJ > 0 && nrb == 1 && smax >= 0 && 2 * ge + gmax <= smax && gsum < (1 << 24) && !(p->flags & C2B_F_NO_RING);
            }
            if (d.pk_maxJ > 0) {
                for (int qa = 0; qa < p->nq; qa++)
                    for (int qb = 0; qb < p->nq; qb++)
                        for (int i = 0; i < I; i++) {
                            const uint32_t a = (uint32_t)(4 * (rf.score_rows[(size_t)qa * I + i] + 2 * beta));
                            const uint32_t b = (uint32_t)(4 * (rf.score_rows[(size_t)qb * I + i] + 2 * beta));
                            const int rbk = i >> 8, ln = (i >> 3) & 31, hf = (i >> 2) & 1, wd = i & 3;
                            prof2[((size_t)qa * p->nq + qb) * Ipad + rbk * 256 + hf * 128 + ln * 4 + wd] = a | (b << 16);
                        }
                for (int row = 0; row < I; row++) {
                    cIe2[row] = (uint32_t)(4 * rf.gap_incentive[row + 1]) * rep;
                    g42[row] = (uint32_t)(4 * rf.gap_incentive[row]) * rep;
                }
            }
        }
        for (int k = 0; k < rf.n_include; k++) {
            const int64_t v = rf.include_idx[k];
            if (v >= 0 && v < I) incl[v] = 1;
        }
        cum[0] = 0;
        for (int q = 0; q <= Ipad; q++) cum[q + 1] = (uint16_t)(cum[q] + (q < I && incl[q] ? 1 : 0));
        d.coding = rf.coding_mask != nullptr; d.tem = rf.tot_exon_len_mod; d.hist_zero = e->hist_zero;
        {   // diagonal tier (c2b_diag_kernel): score bounds of every path other than the main diagonal, DESIGN.md section 3
            const int64_t go = p->gap_open, ge = p->gap_extend, gi0 = rf.gap_incentive[0], gI = rf.gap_incentive[I];
            int64_t gmin = gi0, gp = 0, smax = rf.score_rows[0];
            for (int i = 0; i <= I; i++) { gmin = std::min(gmin, rf.gap_incentive[i]); gp = std::max(gp, rf.gap_incentive[i]); }
            for (size_t k = 0; k < (size_t)p->nq * I; k++) smax = std::max(smax, rf.score_rows[k]);
            // (b) an interior gap run (one gap_open): smax (I - g) + 2 g (ge + gp) + go - ge, largest at g = 1 when 2 (ge + gp) <= smax
            int64_t thr = smax * (I - 1) + go + ge + 2 * gp;
            // (c) a path through a border cell that holds the reference's min_score = gap_open * I * J
            thr = std::max(thr, go * I * I + std::max<int64_t>(smax, 0) * I + 2 * (int64_t)I * gp);
            // (a) offset diagonal t = |s| with its two edge runs: at most smax (I - t) + t (2 ge + gp) + gp, decreasing in t;
            // offsets up to dg_S are scored exactly, the bound covers the rest
            auto edge_bound = [&](int64_t t) { return smax * (I - t) + t * (2 * ge + gp) + gp; };
            int S = 0;
            while (S < 4 && S + 1 < I && edge_bound(S + 1) > thr) S++;
            if (S + 1 < I) thr = std::max(thr, edge_bound(S + 1));
            thr = std::max<int64_t>(thr, -(1ll << 28));
            d.dg_ok = d.rg_ok && !d.coding && go <= ge && ge <= 0 && gmin >= 0 && 2 * (ge + gp) <= smax && I >= 2 && thr < (1ll << 28) &&
                      !(p->flags & C2B_F_NO_RING);
            d.dg_S = S; d.dg_thr4 = (int32_t)(4 * thr);
            for (int s = -4; s <= 4; s++) {
                const int64_t t = s < 0 ? -s : s;
                d.dg_c4[s + 4] = (int32_t)(4 * (s == 0 ? 0 : 2 * ge * t + gi0 + (s > 0 ? rf.gap_incentive[I - std::min<int64_t>(t, I)] : t * gI)));
            }
            if (!d.dg_ok) { d.dg_S = 0; d.dg_thr4 = 0; }
            // two-valued scores over codes 0..3 (EDNAFULL over ACGT: 5 / -4): the tier's sums become match counts
            const int nq4 = std::min(p->nq, 4);
            int64_t a = 0, b = 0;
            bool two = d.dg_ok && I <= 256, have_b = false;
            for (int i = 0; i < I && two; i++) {
                if (rcode[i] >= nq4) { two = false; break; }
                for (int q = 0; q < nq4; q++) {
                    const int64_t v = rf.score_rows[(size_t)q * I + i];
                    if (q == rcode[i]) { if (i == 0) a = v; else if (v != a) two = false; }
                    else if (!have_b) { b = v; have_b = true; }
                    else if (v != b) two = false;
                }
            }
            two = two && 4 * (std::abs(a) + std::abs(b)) * I < (1ll << 30);      // the grouped sums stay inside int32
            d.dg_two = two; d.dg_a4 = two ? (int32_t)(4 * a) : 0; d.dg_b4 = two ? (int32_t)(4 * b) : 0;
        }
        {   // routing of the diagonal tier's unproved reads (route_read, DESIGN.md section 3)
            const int nq4 = std::min(p->nq, 4);
            for (int i = 0; i < I; i++) {                    // bit planes: codes 0..3 match when equal, every other code never
                const int q = rcode[i];
                if (q >= nq4) continue;
                uint4 &w = rt_pl[i >> 5];
                const uint32_t bit = 1u << (i & 31);
                if (q & 1) w.x |= bit;
                if (q & 2) w.y |= bit;
                w.z |= bit;
            }
            // least score of a matched column (reference code < 4, read base equal) and of any other column
            int64_t m = INT64_MAX, x = INT64_MAX;
            for (int q = 0; q < p->nq; q++)
                for (int i = 0; i < I; i++) {
                    const int64_t v = rf.score_rows[(size_t)q * I + i];
                    if (q == rcode[i] && q < nq4) m = std::min(m, v); else x = std::min(x, v);
                }
            // the narrow tier's bound, ring_bound(P, R, I, RN_DLO, RN_DHI) at J == I
            const int64_t ge = p->gap_extend, go = p->gap_open, smax = d.rg_smax, gmax = d.rg_gmax, gsum = d.rg_gsum;
            int64_t thr = -(1 << 28);
            if (RN_DHI + 1 <= I) thr = std::max(thr, smax * (I - RN_DHI - 1) + (RN_DHI + 1) * (ge + gmax) + (RN_DHI + 1) * ge + gsum);
            if (RN_DLO + 1 <= I) thr = std::max(thr, smax * (I - RN_DLO - 1) + (RN_DLO + 1) * (ge + gmax) + (RN_DLO + 1) * ge + gsum);
            const int64_t gI = rf.gap_incentive[I];
            // every estimate must stay far inside int32: |score| x columns, gap costs, incentives
            const int64_t big = std::max<int64_t>({std::abs(m == INT64_MAX ? 0 : m), std::abs(x == INT64_MAX ? 0 : x), std::abs(go), std::abs(ge), e->refs[r].gabs});
            d.rt_ok = d.dg_ok && I <= 256 && m != INT64_MAX && x != INT64_MAX && m > x && big * (4 * I + 64) < (1ll << 28);
            d.rt_thr = d.rt_ok ? (int32_t)thr : 0;
            d.rt_mx = d.rt_ok ? (int32_t)(m - x) : 0;
            for (int k = 0; k < 32; k++) {
                // offset s = k - 16, t = |s| gap columns; only offsets whose one-gap paths lie inside the narrow band
                const int s = k - 16, t = s < 0 ? -s : s;
                const bool on = d.rt_ok && s != 0 && t < I && (s < 0 ? t <= RN_DLO : t <= RN_DHI);
                // interior gap run (gap_open, then gap_extend) + edge run (s < 0: insertion in row I, gap_extend and
                // gap_incentive[I] per column; s > 0: deletion in column J, gap_extend per column, gap_incentive[I - t] once)
                d.rt_c[k] = RT_OFF;
                if (on) d.rt_c[k] = (int32_t)(go + (t - 1) * ge + (s < 0 ? t * (ge + gI) : t * ge + rf.gap_incentive[I - t]) + x * (I - t));
            }
        }
        if (rf.coding_mask)
            for (int q = 0; q < I; q++) incl[q] |= (uint8_t)((rf.coding_mask[q] & 3) << 1);   // after cum[]: bit 0 stays the window
        cumx[0] = cums[0] = 0;
        for (int q = 0; q <= Ipad; q++) {
            cumx[q + 1] = (uint16_t)(cumx[q] + (q < I && (incl[q] & 2) ? 1 : 0));
            cums[q + 1] = (uint16_t)(cums[q] + (q < I && (incl[q] & 4) ? 1 : 0));
        }
        const int ns = std::min({(int)rf.n_seeds, (int)p->seed_count, (int)C2B_MAX_SEEDS});
        if (rf.n_seeds > 0 && std::min((int)rf.n_seeds, (int)p->seed_count) > C2B_MAX_SEEDS)
            return fail(e, C2B_E_LIMIT, "c2b_configure: more seeds than C2B_MAX_SEEDS");
        d.nseeds = ns; d.seed_len = 0;
        for (int s = 0; s < C2B_MAX_SEEDS; s++) { d.fw_seed[s] = ~0ull; d.rc_seed[s] = ~0ull; }
        for (int s = 0; s < ns; s++) {
            const std::string f = rf.fw_seeds[s], c = rf.rc_seeds[s];
            if (f.size() != c.size() || f.empty() || f.size() > C2B_MAX_SEED_LEN) return fail(e, C2B_E_LIMIT, "c2b_configure: seed length unsupported");
            if (s && (int)f.size() != d.seed_len) return fail(e, C2B_E_LIMIT, "c2b_configure: seeds of unequal length");
            d.seed_len = (int)f.size();
            d.fw_seed[s] = pack_seed(*p, f); d.rc_seed[s] = pack_seed(*p, c);
        }
        d.vec = e->d_counts + (size_t)r * per_ref;
        d.hist = d.vec + C2B_NVEC * (size_t)e->vstride;
        d.scal = d.hist + C2B_NHIST * (size_t)e->hstride;
    }
    memcpy(blob.data() + refs_off, e->refdev.data(), sizeof(RefDev) * n_refs);
    e->d_refs = (RefDev *)((unsigned char *)e->d_tables + refs_off);
    RTCHK(rt_h2d(e->d_tables, blob.data(), bytes, e->stream));
    RTCHK(rt_sync(e->stream));
    {
        unsigned char lut[256];
        memset(lut, 255, sizeof lut);
        for (int q = 0; q < p->nq; q++) lut[(unsigned char)p->alphabet[q]] = (unsigned char)q;
        int rc2;
        if ((rc2 = ensure(e, e->lut, 256))) return rc2;
        RTCHK(rt_h2d(e->lut.p, lut, 256, e->stream));
        RTCHK(rt_sync(e->stream));
    }
    e->max_I = maxI; e->max_nrb = max_nrb;
    {   // two-kernel form (c2b_split.cuh): the ring-banded DP must be admissible -- for one reference at least when every
        // read has one candidate, for all of them when every read is tried against every reference
        int n_ok = 0;
        for (int r = 0; r < n_refs; r++) n_ok += (e->refdev[r].pk_maxJ > 0 && !e->refdev[r].coding) ? 1 : 0;     // the packed DP is admissible
        e->split_ok = !(p->flags & (C2B_F_NO_PAIRING | C2B_F_NO_RING)) && n_ok > 0;
        e->split_all = n_ok == n_refs;
        e->diag_any = 0;
        for (int r = 0; r < n_refs; r++) e->diag_any |= e->refdev[r].dg_ok ? 1 : 0;
    }
    e->scratch_TS = 0;
    e->configured = true;
    return C2B_OK;
}

int c2b_set_edit_cap(c2b_engine *e, int32_t edit_cap)
{
    if (!e || !e->configured || edit_cap < 0) return fail(e, C2B_E_ARG, "c2b_set_edit_cap: bad argument");
    e->prm.edit_cap = edit_cap;
    return C2B_OK;
}

int c2b_string_width(const c2b_engine *e, int32_t max_read_len)
{
    if (!e || !e->configured) return C2B_E_STATE;
    return (e->max_I + max_read_len + 31) & ~31;
}

static int ensure_scratch(c2b_engine *e, int maxJ)
{
    const int TS = ((maxJ + 32 + 31) & ~31);
    if (TS <= e->scratch_TS) return C2B_OK;
    int rc;
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    if ((rc = ensure(e, e->tb, al((size_t)e->n_warps * e->max_nrb * TS * 64 * 4)))) return rc;      // 64: a pair stores two words per lane
    if ((rc = ensure(e, e->tbb, al((size_t)e->n_warps * PK_BAND_SLOTS * 64 * 4)))) return rc;        // banded slabs (packed path)
    if ((rc = ensure(e, e->tbq, al((size_t)e->n_warps * TS * 64 * 4 + 64)))) return rc;              // ring-banded path: (step, lane) entries
    if ((rc = ensure(e, e->bnd, al((size_t)e->n_warps * 2 * 3 * TS * 4)))) return rc;
    if ((rc = ensure(e, e->ops, al((size_t)e->n_warps * std::min(e->n_refs, (int)C2B_MAX_REFS) * 32 * 8)))) return rc;
    if ((rc = ensure(e, e->rgo, al((size_t)e->n_warps * RG_MAX_REFS * 4 * RG_OPS_STRIDE * 8)))) return rc;
    const bool fresh_work = !e->work.p;
    if ((rc = ensure(e, e->work, WORK_BYTES))) return rc;
    if (fresh_work) RTCHK(rt_zero(e->work.p, WORK_BYTES, e->stream));
    e->scratch_TS = TS;
    return C2B_OK;
}

// Every DP value is stored as 4 * score + tag in int32, where the reference keeps the raw score in a C int: refuse a batch whose
// scores could wrap here while the reference still computes them exactly.  A cell of reference r's matrix for reads up to maxJ
// holds a path score from the origin or from a min_score border (gap_open * I * J).  On the way there are at most min(I, J)
// substitutions and I + J gap columns, each with one gap_open or gap_extend term; an inserted read base adds its row's
// incentive (at most J of them), an opened deletion that of the row it leaves (distinct rows), a border cell gap_incentive[0].
static bool score_fits(int64_t gap_open, int64_t gap_extend, int64_t I, int64_t maxJ, const RefHost &h)
{
    const int64_t go = std::abs(gap_open), gap = std::max(go, std::abs(gap_extend)), J = std::max<int64_t>(maxJ, 1);
    const int64_t bound = go * I * J + std::min(I, J) * h.sabs + (I + J) * gap + J * h.gabs + h.gsum_abs + h.gi0_abs;
    return 4 * bound + 3 <= (int64_t)INT32_MAX;
}
static int score_range_ok(c2b_engine *e, int64_t maxJ, const char *who)
{
    for (int r = 0; r < e->n_refs; r++)
        if (!score_fits(e->prm.gap_open, e->prm.gap_extend, (int64_t)e->refs[r].seq.size(), maxJ, e->refs[r]))
            return fail(e, C2B_E_LIMIT, std::string(who) + ": scores, gap penalties and incentives can exceed the int32 range of the DP");
    return C2B_OK;
}

// One batch's device arrays.  gops / gmeta / left: op streams [n_reads * R * W/32] u64, meta words [n_reads * R], left-over
// list [n_reads + 8] i32; left2 / left0 / left1: the tier-2 list, the diagonal tier's list and the narrow tier's list after
// routing, each [n_reads + 16] i32 (nullptr: that tier / routing is off).
struct Batch {
    const uint8_t *reads; const int64_t *offsets; int64_t n_reads; int32_t max_read_len;
    const int32_t *count, *qweight, *ref_id;
    c2b_read_rec *recs; c2b_aln_rec *alns; uint8_t *strings; c2b_edit *edits;
    uint64_t *gops; uint32_t *gmeta; int32_t *left, *left2, *left0, *left1;
};

// Launch switches, read once per batch (tests toggle them between batches on one engine): the launch sequence without the
// diagonal tier, without its routing, with every unproved read routed, without the narrow first tier, the general kernel alone.
struct Switches { bool no_diag, no_route, route_all, no_narrow, no_split; };
static Switches read_switches()
{
    return {getenv("C2B_NO_DIAG") != nullptr, getenv("C2B_NO_ROUTE") != nullptr, getenv("C2B_ROUTE_ALL") != nullptr,
            getenv("C2B_NO_NARROW") != nullptr, getenv("C2B_NO_SPLIT") != nullptr};
}

// A batch's launch sequence: the kernels in order, each with its parameters and launch geometry.
enum StepKind { STEP_DIAG, STEP_ALIGN, STEP_CLASSIFY, STEP_GENERAL };
struct Step { StepKind kind; KParams P; int grid, block; size_t smem; };
struct Plan { Step step[5]; int n = 0; bool one = false; };      // one: CLASSIFY / GENERAL in their one-candidate form

// The only place that decides a batch's launch sequence: the two-kernel form (ALIGN -> CLASSIFY, then the general kernel over
// what ALIGN left over) or the general kernel alone; in the two-kernel form the narrow first tier with its second-tier launch,
// the diagonal tier ahead of it and the diagonal tier's routing.
static Plan plan_batch(const c2b_engine *e, const Batch &b, const Switches &sw)
{
    Plan plan;
    WorkBlock *wb = (WorkBlock *)e->work.p;
    KParams P;
    memset(&P, 0, sizeof P);
    P.reads = b.reads; P.offsets = b.offsets; P.n_reads = b.n_reads; P.count = b.count; P.qweight = b.qweight; P.ref_id = b.ref_id;
    P.recs = b.recs; P.alns = b.alns; P.strings = b.strings; P.edits = b.edits;
    P.W = (e->max_I + b.max_read_len + 31) & ~31; P.edit_cap = b.edits ? e->prm.edit_cap : 0;
    if (P.edit_cap == 0) P.edits = nullptr;
    P.refs = e->d_refs; P.n_refs = e->n_refs;
    P.out_refs = b.ref_id ? 1 : e->n_refs; P.ops_refs = std::min(e->n_refs, (int)C2B_MAX_REFS);
    P.go = e->prm.gap_open; P.ge = e->prm.gap_extend; P.seed_count = e->prm.seed_count; P.seed_min = e->prm.seed_min;
    P.flags = e->prm.flags; P.nq = e->prm.nq;
    memcpy(P.alpha, e->prm.alphabet, C2B_MAX_Q); memcpy(P.comp, e->prm.complement, C2B_MAX_Q);
    P.TS = e->scratch_TS;
    P.tb = (uint32_t *)e->tb.p; P.tb_words_per_warp = (int64_t)e->max_nrb * P.TS * 64;
    P.tbb = (uint32_t *)e->tbb.p; P.tbb_words_per_warp = (int64_t)PK_BAND_SLOTS * 64;
    P.tbq = (uint32_t *)e->tbq.p;
    P.bnd = (int32_t *)e->bnd.p; P.bnd_words_per_warp = 2 * 3 * (int64_t)P.TS;
    P.opsbuf = (uint64_t *)e->ops.p;
    P.rgops = (uint64_t *)e->rgo.p;
    P.wb = wb; P.work_counter = &wb->launch.align_next;
    P.vstride = e->vstride; P.hstride = e->hstride;
    P.forced_ops = e->forced_ops; P.forced_n = e->forced_n;
    P.gops = b.gops; P.gmeta = b.gmeta; P.NW = P.W / 32;
    P.pair_order = e->pair_order;
    P.lut = (const uint8_t *)e->lut.p;
    plan.one = e->n_refs == 1 || b.ref_id != nullptr;       // one candidate reference per read
    // two-kernel form: the configuration admits the ring-banded DP, op-stream buffers were supplied, nothing forces the
    // general kernel (caller-supplied op streams, C2B_NO_SPLIT)
    const bool split = e->split_ok && b.gops && b.gmeta && b.left && !e->forced_ops && !sw.no_split &&
                       (plan.one || (e->n_refs <= RG_MAX_REFS && e->split_all));
    P.phase_sync = split ? 0 : 4;                         // one-kernel form: the warps of a phase set move in step
    // reference 0's packed profile, staged into shared memory where it fits next to the kernel's per-warp state
    const RefDev &r0 = e->refdev[0];
    const size_t tile = (size_t)e->prm.nq * e->prm.nq * r0.Ipad * 4;
    const bool can_stage = r0.pk_maxJ > 0 && !e->forced_ops;
    auto add = [&](StepKind kind, const KParams &K, int grid, int block, size_t smem) { plan.step[plan.n++] = Step{kind, K, grid, block, smem}; };
    if (split) {
        KParams A = P;
        A.left = b.left;
        if (can_stage && tile <= (size_t)e->stage_cap_a) { A.stage_bytes = (int32_t)tile; A.stage_src = r0.prof2; }
        const size_t smem_a = sizeof(ASmem) * WARPS_PER_CTA + 128 + (size_t)A.stage_bytes;
        // narrow first tier (align_narrow16): reads in their given order (no pairing order = the caller's reads are of one
        // length, or unsorted -- then hardly any unit of sixteen qualifies), one candidate reference per read
        const bool narrow = b.left2 && !P.pair_order && plan.one && !sw.no_narrow;
        if (narrow) A.left2 = b.left2;
        // diagonal tier ahead of the narrow one: reads it proves are done, the narrow tier works through the rest.
        // A batch smaller than one narrow unit (16 reads) goes through the groups of eight anyway and keeps them whole.
        const bool diag = narrow && b.left0 && e->diag_any && b.n_reads >= 16 && !sw.no_diag;
        // routing: the diagonal tier puts the reads the narrow band cannot prove straight on the tier-2 list and the rest on
        // the narrow tier's list; CLASSIFY still takes all its unproved reads
        const bool route = diag && b.left1 && !sw.no_route;
        if (diag) {
            KParams D = P;
            D.left0 = b.left0;
            if (route) { D.left1 = b.left1; D.left2 = b.left2; D.route = sw.route_all ? 2 : 1; }
            const int64_t units = (b.n_reads + 31) / 32;
            add(STEP_DIAG, D, (int)std::min<int64_t>((units + D_WARPS_PER_CTA - 1) / D_WARPS_PER_CTA, (int64_t)e->grid_a * 16), D_WARPS_PER_CTA * 32, 0);
            A.pair_order = route ? b.left1 : b.left0; A.n_dev = route ? &wb->launch.narrow_n : &wb->launch.diag_n;
        }
        add(STEP_ALIGN, A, e->grid_a, WARPS_PER_CTA * 32, smem_a);
        if (narrow) {                                         // second tier: what the narrow band did not settle, eight reads per group
            KParams A2 = A;
            A2.left2 = nullptr;
            A2.pair_order = b.left2; A2.n_dev = &wb->launch.tier2_n; A2.work_counter = &wb->launch.tier2_next;
            add(STEP_ALIGN, A2, e->grid_a, WARPS_PER_CTA * 32, smem_a);
        }
        KParams B = P;                                        // CLASSIFY: every read in batch order, or the diagonal tier's list
        B.pair_order = diag ? b.left0 : nullptr; B.n_dev = diag ? &wb->launch.diag_n : nullptr;
        add(STEP_CLASSIFY, B, e->grid_b, B_WARPS_PER_CTA * 32, 0);
        // the general kernel over ALIGN's left-over pairs (free-running warps, no ring-banded attempt); these pairs left the
        // ring band: the banded slab would only cost a second DP
        P.pair_order = b.left; P.n_dev = &wb->launch.left_n; P.work_counter = &wb->launch.general_next;
        P.tbq = nullptr; P.rgops = nullptr; P.tbb = nullptr;
    }
    if (can_stage && tile <= (size_t)e->stage_cap) { P.stage_bytes = (int32_t)tile; P.stage_src = r0.prof2; }
    add(STEP_GENERAL, P, e->grid, WARPS_PER_CTA * 32, (sizeof(WarpSmem) + sizeof(QuadSmem)) * WARPS_PER_CTA + 128 + (size_t)P.stage_bytes);
    return plan;
}

#ifndef C2B_EMU
static int run_plan(c2b_engine *e, const Plan &plan, rt_stream cs)
{
    cudaEventRecord(e->ev0, cs);
    for (int k = 0; k < plan.n; k++) {
        const Step &s = plan.step[k];
        switch (s.kind) {
        case STEP_DIAG: c2b_diag_kernel<<<s.grid, s.block, s.smem, cs>>>(s.P); break;
        case STEP_ALIGN: c2b_align_kernel<<<s.grid, s.block, s.smem, cs>>>(s.P); break;
        case STEP_CLASSIFY:
            if (plan.one) c2b_classify_kernel<true><<<s.grid, s.block, s.smem, cs>>>(s.P);
            else c2b_classify_kernel<false><<<s.grid, s.block, s.smem, cs>>>(s.P);
            break;
        case STEP_GENERAL:
            if (plan.one) c2b_align_classify_kernel<true><<<s.grid, s.block, s.smem, cs>>>(s.P);
            else c2b_align_classify_kernel<false><<<s.grid, s.block, s.smem, cs>>>(s.P);
            break;
        }
    }
    cudaEventRecord(e->ev1, cs);
    RTCHK(cudaGetLastError());
    return C2B_OK;
}
#else
// The kernels' loops, each as a grid of one warp: the launch sequence's counters start at zero, so the warp's hand-outs walk
// every item in order.
static void run_phase_sets(const KParams &P, bool one, WarpSmem &S, QuadSmem &Q)
{
    // the general kernel's phase-set loop needs the warps of a set in step: here each group runs alone, and every path through
    // a work group must execute the same number of phase barriers (a mismatch deadlocks the GPU)
    for (int64_t w = 0; 8 * w < P.n_reads; w++) {
        wp::g_grp_syncs = 0;
        if (one) emu::run_warp([&]() { process_group<true>(P, S, Q, nullptr, w, 0); });
        else emu::run_warp([&]() { process_group<false>(P, S, Q, nullptr, w, 0); });
        if (P.phase_sync && wp::g_grp_syncs != group_phases(P)) {
            fprintf(stderr, "warp_emu: work group %lld executed %ld phase barriers, expected %d\n", (long long)w, wp::g_grp_syncs, group_phases(P));
            abort();
        }
    }
}

static int run_plan(c2b_engine *, const Plan &plan, rt_stream)
{
    static WarpSmem S; static QuadSmem Q; static ASmem AS; static BSmem BS; static DSmem DS;
    for (int k = 0; k < plan.n; k++) {
        const KParams &P = plan.step[k].P;
        switch (plan.step[k].kind) {
        case STEP_DIAG: emu::run_warp([&]() { diag_loop(P, DS, 0, 1); }); break;
        case STEP_ALIGN: emu::run_warp([&]() { align_loop(P, AS, nullptr, 0); }); break;
        case STEP_CLASSIFY:
            if (plan.one) emu::run_warp([&]() { classify_loop<true>(P, BS, 0, 1); });
            else emu::run_warp([&]() { classify_loop<false>(P, BS, 0, 1); });
            break;
        case STEP_GENERAL:
            if (P.n_dev && plan.one) emu::run_warp([&]() { general_list_loop<true>(P, S, nullptr, 0); });
            else if (P.n_dev) emu::run_warp([&]() { general_list_loop<false>(P, S, nullptr, 0); });
            else run_phase_sets(P, plan.one, S, Q);
            break;
        }
    }
    return C2B_OK;
}
#endif

// One batch on compute stream `cs`: the launch sequence of plan_batch.
static int launch_on(c2b_engine *e, rt_stream cs, Batch b)
{
    if (!e || !e->configured) return fail(e, C2B_E_STATE, "c2b_align_batch: engine not configured");
    if (b.n_reads < 0 || !b.recs || !b.alns || (b.n_reads && (!b.reads || !b.offsets))) return fail(e, C2B_E_ARG, "c2b_align_batch: bad argument");
    if (b.n_reads >= (1ll << 31)) return fail(e, C2B_E_LIMIT, "c2b_align_batch: more than 2^31 reads in one batch");
    if (b.max_read_len < 1) b.max_read_len = 1;
    if (b.max_read_len > C2B_MAX_READ_LEN) return fail(e, C2B_E_LIMIT, "c2b_align_batch: read longer than C2B_MAX_READ_LEN");
    if ((int64_t)std::abs((long long)e->prm.gap_open) * b.max_read_len * e->max_I >= (1ll << 28))
        return fail(e, C2B_E_LIMIT, "c2b_align_batch: gap_open * lengths exceeds the int32 score range");
    if (int rc0 = score_range_ok(e, b.max_read_len, "c2b_align_batch")) return rc0;
    if (!b.ref_id && e->n_refs > C2B_MAX_REFS)
        return fail(e, C2B_E_LIMIT, "c2b_align_batch: more than C2B_MAX_REFS references need a per-read ref_id");
    int rc = ensure_scratch(e, b.max_read_len);
    if (rc) return rc;
    if (b.n_reads == 0) return C2B_OK;
    const Plan plan = plan_batch(e, b, read_switches());
    RTCHK(rt_zero(&((WorkBlock *)e->work.p)->launch, sizeof(WorkBlock::Launch), cs));
    if (b.gmeta) RTCHK(rt_zero(b.gmeta, (size_t)b.n_reads * (b.ref_id ? 1 : e->n_refs) * 4, cs));
    if ((rc = run_plan(e, plan, cs))) return rc;
    e->launches += plan.n;
    return C2B_OK;
}

// op-stream buffers of the device-pointer API (engine-owned, sized for the batch)
static int ensure_ops(c2b_engine *e, DevBuf &gops, DevBuf &gmeta, DevBuf &left, DevBuf &left2, DevBuf &left0, DevBuf &left1, int64_t n_reads,
                      int nr, int W)
{
    int rc;
    if ((rc = ensure(e, gops, (size_t)n_reads * nr * (W / 32) * 8))) return rc;
    if ((rc = ensure(e, gmeta, (size_t)n_reads * nr * 4))) return rc;
    if ((rc = ensure(e, left, (size_t)(n_reads + 8) * 4))) return rc;
    if ((rc = ensure(e, left2, (size_t)(n_reads + 16) * 4))) return rc;
    if ((rc = ensure(e, left0, (size_t)(n_reads + 16) * 4))) return rc;
    if ((rc = ensure(e, left1, (size_t)(n_reads + 16) * 4))) return rc;
    return C2B_OK;
}

int c2b_align_batch_device(c2b_engine *e, const uint8_t *d_reads, const int64_t *d_offsets, int64_t n_reads,
                           int32_t max_read_len, const int32_t *d_count, const int32_t *d_qweight,
                           const int32_t *d_ref_id, c2b_read_rec *d_recs, c2b_aln_rec *d_alns,
                           uint8_t *d_strings, c2b_edit *d_edits)
{
    if (!e || !e->configured) return fail(e, C2B_E_STATE, "c2b_align_batch_device: engine not configured");
#ifndef C2B_EMU
    cudaSetDevice(e->device);
#endif
    if (max_read_len < 1) max_read_len = 1;
    const int W = (e->max_I + max_read_len + 31) & ~31, nr = d_ref_id ? 1 : e->n_refs;
    int rc = ensure_ops(e, e->gops, e->gmeta, e->left, e->left2, e->left0, e->left1, n_reads, nr, W);
    if (rc) return rc;
    return launch_on(e, e->stream, Batch{d_reads, d_offsets, n_reads, max_read_len, d_count, d_qweight, d_ref_id, d_recs,
                     d_alns, d_strings, d_edits, (uint64_t *)e->gops.p, (uint32_t *)e->gmeta.p, (int32_t *)e->left.p, (int32_t *)e->left2.p,
                     (int32_t *)e->left0.p, (int32_t *)e->left1.p});
}

int c2b_ops_device(c2b_engine *e, void **d_ops, void **d_meta)
{
    if (!e) return C2B_E_ARG;
    if (d_ops) *d_ops = e->gops.p;
    if (d_meta) *d_meta = e->gmeta.p;
    return C2B_OK;
}

int64_t c2b_band_reruns(c2b_engine *e) { return e ? e->band_reruns : 0; }

int c2b_set_pair_order(c2b_engine *e, const int32_t *d_order)
{
    if (!e) return C2B_E_ARG;
    e->pair_order = d_order;
    return C2B_OK;
}

int c2b_sync(c2b_engine *e)
{
    if (!e) return C2B_E_ARG;
    RTCHK(rt_sync(e->stream));
    return C2B_OK;
}

void *c2b_stream(c2b_engine *e) { return e ? (void *)(uintptr_t)e->stream : nullptr; }

double c2b_last_kernel_ms(c2b_engine *e)
{
#ifndef C2B_EMU
    if (!e || !e->launches) return 0.0;
    float ms = 0.f;
    if (cudaEventSynchronize(e->ev1) != cudaSuccess) return 0.0;
    if (cudaEventElapsedTime(&ms, e->ev0, e->ev1) != cudaSuccess) return 0.0;
    return (double)ms;
#else
    (void)e; return 0.0;
#endif
}

int64_t c2b_launch_count(const c2b_engine *e) { return e ? e->launches : 0; }

int c2b_path_counts(c2b_engine *e, int64_t *pair_items, int64_t *single_items)
{
    if (!e || !e->work.p) return fail(e, C2B_E_STATE, "c2b_path_counts: nothing launched yet");
    WorkBlock v;
    RTCHK(rt_d2h(&v, e->work.p, sizeof v, e->stream));
    RTCHK(rt_sync(e->stream));
    // the ALIGN kernel counts reads (kept by the ring, sent on, fully aligned); reported in pairs
    e->band_reruns = (int64_t)v.band_reruns; e->ring_pairs = (int64_t)(v.ring_kept + 1) / 2; e->ring_fallbacks = (int64_t)(v.ring_sent + 1) / 2;
    if (getenv("C2B_VERBOSE"))
        fprintf(stderr, "[c2b] counters: general kernel %lld pair items + %lld single items; ALIGN: %lld read x reference combinations kept "
                        "by the ring, %lld sent to the full matrix, %lld reads settled\n", (long long)v.pair_items, (long long)v.single_items,
                (long long)v.ring_kept, (long long)v.ring_sent, (long long)v.align_settled);
    if (pair_items) *pair_items = (int64_t)(v.pair_items + (v.align_settled + 1) / 2);
    if (single_items) *single_items = (int64_t)v.single_items;
    return C2B_OK;
}

int c2b_diag_counts(c2b_engine *e, int64_t *proved, int64_t *tier1, int64_t *tier2)
{
    if (!e || !e->work.p) return fail(e, C2B_E_STATE, "c2b_diag_counts: nothing launched yet");
    WorkBlock v;
    RTCHK(rt_d2h(&v, e->work.p, sizeof v, e->stream));
    RTCHK(rt_sync(e->stream));
    if (proved) *proved = (int64_t)v.diag_proved;
    if (tier1) *tier1 = (int64_t)v.diag_listed;
    if (tier2) *tier2 = (int64_t)v.tier2;
    return C2B_OK;
}

int c2b_diag_popcount_reads(c2b_engine *e, int64_t *reads)
{
    if (!e || !e->work.p) return fail(e, C2B_E_STATE, "c2b_diag_popcount_reads: nothing launched yet");
    WorkBlock v;
    RTCHK(rt_d2h(&v, e->work.p, sizeof v, e->stream));
    RTCHK(rt_sync(e->stream));
    if (reads) *reads = (int64_t)v.diag_popc;
    return C2B_OK;
}

int c2b_route_counts(c2b_engine *e, int64_t *routed, int64_t *kept)
{
    if (!e || !e->work.p) return fail(e, C2B_E_STATE, "c2b_route_counts: nothing launched yet");
    WorkBlock v;
    RTCHK(rt_d2h(&v, e->work.p, sizeof v, e->stream));
    RTCHK(rt_sync(e->stream));
    if (routed) *routed = (int64_t)v.routed;
    if (kept) *kept = (int64_t)v.kept;
    return C2B_OK;
}

int c2b_ring_counts(c2b_engine *e, int64_t *ring_pairs, int64_t *ring_fallbacks)
{
    if (!e) return C2B_E_ARG;
    if (ring_pairs) *ring_pairs = e->ring_pairs;
    if (ring_fallbacks) *ring_fallbacks = e->ring_fallbacks;
    return C2B_OK;
}

// true when `p` is ordinary pageable host memory (cudaMemcpyAsync on it is staged by the driver and blocks the host thread)
static bool is_pageable(const void *p)
{
#ifndef C2B_EMU
    if (!p) return false;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
#else
    (void)p; return false;
#endif
}

// rows x width bytes between buffers of different pitch, split over a few host threads
static void par_copy2d(void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t rows)
{
    if (!rows || !width) return;
    const size_t bytes = width * rows;
    int T = bytes > (8u << 20) ? 4 : bytes > (1u << 20) ? 2 : 1;
    auto work = [&](int t) {
        const size_t lo = rows * t / T, hi = rows * (t + 1) / T;
        if (dpitch == width && spitch == width) memcpy((char *)dst + lo * width, (const char *)src + lo * width, (hi - lo) * width);
        else for (size_t r = lo; r < hi; r++) memcpy((char *)dst + r * dpitch, (const char *)src + r * spitch, width);
    };
    std::vector<std::thread> th;
    for (int t = 1; t < T; t++) th.emplace_back(work, t);
    work(0);
    for (auto &x : th) x.join();
}
static void par_copy(void *dst, const void *src, size_t bytes) { par_copy2d(dst, bytes, src, bytes, bytes, 1 == 1 ? (bytes ? 1 : 0) : 0); }

static int ensure_pinned(c2b_engine *e, uint8_t *&p, size_t &cap, size_t n)
{
    if (n <= cap) return C2B_OK;
    if (p) rt_host_free(p);
    const size_t want = n + n / 8 + 4096;
    p = (uint8_t *)rt_host_alloc(want); cap = p ? want : 0;
    return p ? C2B_OK : fail(e, C2B_E_CUDA, "c2b_align_batch: pinned allocation failed");
}

// Host buffers in, host buffers out: chunks pipeline through two staging sets and three streams -- H2D of chunk c+1 and
// D2H of chunk c-1 overlap the kernels of chunk c.  strings (two W-byte slots per (read, reference)) and / or the compact
// form (ops: W/32 words of 32 two-bit ops per slot, meta: one word per slot) are produced as requested; of either only the
// part the chunk's widest alignment needs crosses PCIe.
static int align_batch_host(c2b_engine *e, const uint8_t *reads, const int64_t *offsets, int64_t n_reads,
                            const int32_t *count, const int32_t *qweight, const int32_t *ref_id,
                            c2b_read_rec *recs, c2b_aln_rec *alns, uint8_t *strings, uint64_t *ops, uint32_t *meta, c2b_edit *edits)
{
    if (!e || !e->configured) return fail(e, C2B_E_STATE, "c2b_align_batch: engine not configured");
    if (n_reads < 0 || !recs || !alns || (n_reads && (!reads || !offsets))) return fail(e, C2B_E_ARG, "c2b_align_batch: bad argument");
    if ((ops == nullptr) != (meta == nullptr)) return fail(e, C2B_E_ARG, "c2b_align_batch: ops and meta go together");
#ifndef C2B_EMU
    cudaSetDevice(e->device);                              // the current device is per host thread: callers may use a worker thread
#endif
    if (n_reads == 0) return C2B_OK;
    int64_t maxJ = 1, minJ = 0;                            // branch-free reductions (vectorised): this scan runs before anything is queued
    for (int64_t r = 0; r < n_reads; r++) {
        const int64_t L = offsets[r + 1] - offsets[r];
        maxJ = L > maxJ ? L : maxJ;
        minJ = L < minJ ? L : minJ;
    }
    if (minJ < 0) return fail(e, C2B_E_ARG, "c2b_align_batch: offsets not monotone");
    if (maxJ > C2B_MAX_READ_LEN) return fail(e, C2B_E_LIMIT, "c2b_align_batch: read longer than C2B_MAX_READ_LEN");
    if (int rc0 = score_range_ok(e, maxJ, "c2b_align_batch")) return rc0;     // before anything is queued
    if (!e->pipe_ready) {
        RTCHK(rt_stream_create(&e->s_in));
        RTCHK(rt_stream_create(&e->s_out));
        for (auto &st : e->stage) { RTCHK(rt_event_create(&st.in_done)); RTCHK(rt_event_create(&st.k_done)); RTCHK(rt_event_create(&st.out_done)); }
        e->pipe_ready = true;
    }
    const int W = (e->max_I + (int)maxJ + 31) & ~31, NW = W / 32;
    const int cap = edits ? e->prm.edit_cap : 0;
    const int nr = ref_id ? 1 : e->n_refs;                 // output slots per read (compact when ref_id is given)
    const int64_t per_read = (int64_t)nr * (2 * (int64_t)W * (strings ? 1 : 0) + NW * 8 + (int64_t)cap * 8 + 36) + 16 + maxJ + 28;
    // 256 Ki reads per chunk: every chunk's launches end in a tail of partly idle SMs (persistent kernels, a second-tier launch of
    // one or two waves), so fewer, larger chunks win until the exposed first copy-in / last copy-out take over (256 Ki
    // measured fastest end to end of 128 / 256 / 512 Ki)
    int64_t chunk = std::max<int64_t>(4096, std::min<int64_t>((int64_t)(1536ll << 20) / per_read, 1 << 18));
    if (n_reads < 4 * chunk) chunk = std::max<int64_t>(4096, (n_reads + 3) / 4);
    if (const char *v = getenv("C2B_CHUNK")) chunk = std::max<int64_t>(2, atoll(v));     // test hook: force many small chunks
    for (auto &st : e->stage) st.used = false;
    int rc = C2B_OK;
    // D2H of a chunk is queued one iteration late: by then its kernels have finished and the widest alignment of the
    // chunk is known, so only the right-hand `Wt` bytes of every W-byte string slot (the first Wt/32 op words) cross PCIe.
    // Pageable caller arrays (numpy): cudaMemcpyAsync on them is staged by the driver and blocks this thread -- more than
    // twenty times the cost of the same copies from pinned arrays.  Then every
    // chunk goes through the set's pinned bounce buffers; the copies between them and the caller's arrays run on host threads
    // while the other set's kernels and DMA are in flight.
    const bool bounce = getenv("C2B_FORCE_BOUNCE") ? atoi(getenv("C2B_FORCE_BOUNCE")) != 0 : (is_pageable(reads) || is_pageable(recs));
    auto al256 = [](size_t x) { return (x + 255) & ~(size_t)255; };
    struct OutLay { size_t recs, alns, ed, meta, str, ops, total; };
    auto out_layout = [&](int64_t n) {
        OutLay L; size_t o = 0;
        L.recs = o; o = al256(o + (size_t)n * sizeof(c2b_read_rec));
        L.alns = o; o = al256(o + (size_t)n * nr * sizeof(c2b_aln_rec));
        L.ed = o; o = al256(o + (size_t)n * nr * cap * sizeof(c2b_edit));
        L.meta = o; o = al256(o + (meta ? (size_t)n * nr * 4 : 0));
        L.str = o; o = al256(o + (strings ? (size_t)n * nr * 2 * W : 0));
        L.ops = o; o = al256(o + (ops ? (size_t)n * nr * NW * 8 : 0));
        L.total = o;
        return L;
    };
    struct Pending { bool any = false; int64_t c0 = 0, n = 0; int set = 0; } pend;
    auto flush = [&](const Pending &q) -> int {
        c2b_engine::Stage &st = e->stage[q.set];
        const OutLay L = out_layout(q.n);
        int rc2;
        if (bounce && (rc2 = ensure_pinned(e, st.h_out, st.h_out_cap, L.total))) return rc2;
        uint8_t *ho = st.h_out;
        RTCHK(rt_wait(e->s_out, st.k_done));
        RTCHK(rt_d2h(bounce ? (void *)(ho + L.recs) : (void *)(recs + q.c0), st.recs.p, (size_t)q.n * sizeof(c2b_read_rec), e->s_out));
        RTCHK(rt_d2h(bounce ? (void *)(ho + L.alns) : (void *)(alns + q.c0 * nr), st.alns.p, (size_t)q.n * nr * sizeof(c2b_aln_rec), e->s_out));
        if (cap) RTCHK(rt_d2h(bounce ? (void *)(ho + L.ed) : (void *)(edits + q.c0 * nr * cap), st.ed.p, (size_t)q.n * nr * cap * sizeof(c2b_edit), e->s_out));
        if (meta) RTCHK(rt_d2h(bounce ? (void *)(ho + L.meta) : (void *)(meta + q.c0 * nr), st.gmeta.p, (size_t)q.n * nr * 4, e->s_out));
        size_t Wt = 0;
        if (strings || ops) {
            RTCHK(rt_event_sync(st.k_done));
            long long wmax = 0;
            RTCHK(rt_d2h(&wmax, (const char *)st.maxlen.p, 8, e->s_out));
            RTCHK(rt_sync(e->s_out));
            Wt = ((size_t)wmax + 31) & ~(size_t)31;
            if (Wt > (size_t)W) Wt = W;
            if (strings) RTCHK(rt_d2h_2d((bounce ? ho + L.str : strings + q.c0 * nr * 2 * W) + (W - Wt), (const uint8_t *)st.str.p + (W - Wt), W, Wt, (size_t)q.n * nr * 2, e->s_out));
            if (ops) RTCHK(rt_d2h_2d(bounce ? (void *)(ho + L.ops) : (void *)(ops + q.c0 * nr * NW), st.gops.p, (size_t)NW * 8, Wt / 32 * 8, (size_t)q.n * nr, e->s_out));
        }
        RTCHK(rt_record(st.out_done, e->s_out));
        st.drain = bounce; st.d_c0 = q.c0; st.d_n = q.n; st.d_Wt = Wt;
        return C2B_OK;
    };
    // bounce buffers -> the caller's arrays, once the set's D2H is done
    auto drain = [&](c2b_engine::Stage &st) -> int {
        if (!st.drain) return C2B_OK;
        RTCHK(rt_event_sync(st.out_done));
        const int64_t c0 = st.d_c0, n = st.d_n;
        const OutLay L = out_layout(n);
        const uint8_t *ho = st.h_out;
        par_copy(recs + c0, ho + L.recs, (size_t)n * sizeof(c2b_read_rec));
        par_copy(alns + c0 * nr, ho + L.alns, (size_t)n * nr * sizeof(c2b_aln_rec));
        if (cap) par_copy(edits + c0 * nr * cap, ho + L.ed, (size_t)n * nr * cap * sizeof(c2b_edit));
        if (meta) par_copy(meta + c0 * nr, ho + L.meta, (size_t)n * nr * 4);
        if (strings) par_copy2d(strings + c0 * nr * 2 * W + (W - st.d_Wt), W, ho + L.str + (W - st.d_Wt), W, st.d_Wt, (size_t)n * nr * 2);
        if (ops) par_copy2d(ops + c0 * nr * NW, (size_t)NW * 8, ho + L.ops, (size_t)NW * 8, st.d_Wt / 32 * 8, (size_t)n * nr);
        st.drain = false;
        return C2B_OK;
    };
    // chunk boundaries: a small first chunk (its H2D is exposed) and a small last chunk (its D2H is exposed)
    std::vector<int64_t> cuts;
    {
        const int64_t edge = getenv("C2B_CHUNK") ? std::max<int64_t>(2, chunk / 2) : std::max<int64_t>(4096, chunk / 8);
        int64_t pos = 0;
        cuts.push_back(0);
        if (n_reads > 4 * edge) { pos = edge; cuts.push_back(pos); }
        const int64_t tail = (n_reads - pos > 2 * edge) ? edge : 0;
        while (n_reads - tail - pos > 0) { pos += std::min(chunk, n_reads - tail - pos); cuts.push_back(pos); }
        if (tail) cuts.push_back(n_reads);
    }
    if ((rc = ensure_scratch(e, (int)maxJ))) return rc;
    for (int ci = 0; ci + 1 < (int)cuts.size(); ci++) {
        c2b_engine::Stage &st = e->stage[ci & 1];
        const int64_t c0 = cuts[ci], n = cuts[ci + 1] - cuts[ci];
        const int64_t b0 = offsets[c0], b1 = offsets[c0 + n];
        if (st.used) RTCHK(rt_event_sync(st.out_done));        // set is being reused: the D2H of chunk ci-2 must be done
        if ((rc = drain(st))) return rc;
        if ((rc = ensure(e, st.reads, (size_t)(b1 - b0) + 16))) return rc;
        if ((rc = ensure(e, st.off, (size_t)(n + 1) * 8))) return rc;
        if ((rc = ensure(e, st.recs, (size_t)n * sizeof(c2b_read_rec)))) return rc;
        if ((rc = ensure(e, st.alns, (size_t)n * nr * sizeof(c2b_aln_rec)))) return rc;
        if ((rc = ensure(e, st.maxlen, 8))) return rc;
        if (strings && (rc = ensure(e, st.str, (size_t)n * nr * 2 * W))) return rc;
        if (cap && (rc = ensure(e, st.ed, (size_t)n * nr * cap * sizeof(c2b_edit)))) return rc;
        if (count && (rc = ensure(e, st.cnt, (size_t)n * 4))) return rc;
        if (qweight && (rc = ensure(e, st.qw, (size_t)n * 4))) return rc;
        if (ref_id && (rc = ensure(e, st.rid, (size_t)n * 4))) return rc;
        if ((rc = ensure_ops(e, st.gops, st.gmeta, st.left, st.left2, st.left0, st.left1, n, nr, W))) return rc;
        if (st.h_off_cap < (size_t)(n + 1)) {
            if (st.h_off) rt_host_free(st.h_off);
            st.h_off = (int64_t *)rt_host_alloc((size_t)(n + 1) * 8); st.h_off_cap = st.h_off ? (size_t)(n + 1) : 0;
            if (!st.h_off) return fail(e, C2B_E_CUDA, "c2b_align_batch: pinned allocation failed");
        }
        for (int64_t k = 0; k <= n; k++) st.h_off[k] = offsets[c0 + k] - b0;      // chunk-relative offsets
        const uint8_t *src_reads = reads + b0;
        const int32_t *src_cnt = count ? count + c0 : nullptr, *src_qw = qweight ? qweight + c0 : nullptr, *src_rid = ref_id ? ref_id + c0 : nullptr;
        if (bounce) {
            const size_t rb = al256((size_t)(b1 - b0)), ib = al256((size_t)n * 4);
            if ((rc = ensure_pinned(e, st.h_in, st.h_in_cap, rb + 3 * ib))) return rc;
            par_copy(st.h_in, src_reads, (size_t)(b1 - b0)); src_reads = st.h_in;
            if (count) { memcpy(st.h_in + rb, src_cnt, (size_t)n * 4); src_cnt = (const int32_t *)(st.h_in + rb); }
            if (qweight) { memcpy(st.h_in + rb + ib, src_qw, (size_t)n * 4); src_qw = (const int32_t *)(st.h_in + rb + ib); }
            if (ref_id) { memcpy(st.h_in + rb + 2 * ib, src_rid, (size_t)n * 4); src_rid = (const int32_t *)(st.h_in + rb + 2 * ib); }
        }
        RTCHK(rt_h2d(st.reads.p, src_reads, (size_t)(b1 - b0), e->s_in));
        RTCHK(rt_h2d(st.off.p, st.h_off, (size_t)(n + 1) * 8, e->s_in));
        if (count) RTCHK(rt_h2d(st.cnt.p, src_cnt, (size_t)n * 4, e->s_in));
        if (qweight) RTCHK(rt_h2d(st.qw.p, src_qw, (size_t)n * 4, e->s_in));
        if (ref_id) RTCHK(rt_h2d(st.rid.p, src_rid, (size_t)n * 4, e->s_in));
        // pairing order: counting sort of the chunk by (reference id, length) when reads differ, so equal ones are adjacent
        bool need_order = false;
        for (int64_t k = 1; k < n && !need_order; k++)
            need_order = (st.h_off[k + 1] - st.h_off[k] != st.h_off[1] - st.h_off[0]) || (ref_id && ref_id[c0 + k] != ref_id[c0]);
        e->pair_order = nullptr;
        if (need_order) {
            if ((rc = ensure(e, st.ord, (size_t)n * 4))) return rc;
            if (st.h_ord_cap < (size_t)n) {
                if (st.h_ord) rt_host_free(st.h_ord);
                st.h_ord = (int32_t *)rt_host_alloc((size_t)n * 4); st.h_ord_cap = st.h_ord ? (size_t)n : 0;
                if (!st.h_ord) return fail(e, C2B_E_CUDA, "c2b_align_batch: pinned allocation failed");
            }
            const int64_t nb = (int64_t)(C2B_MAX_READ_LEN + 1) * (ref_id ? e->n_refs : 1);
            std::vector<int64_t> start((size_t)nb + 1, 0);
            auto key = [&](int64_t k) -> int64_t {
                const int64_t L = st.h_off[k + 1] - st.h_off[k];
                const int64_t r = ref_id ? std::min<int64_t>(std::max<int32_t>(ref_id[c0 + k], 0), e->n_refs - 1) : 0;
                return r * (C2B_MAX_READ_LEN + 1) + L;
            };
            for (int64_t k = 0; k < n; k++) start[(size_t)key(k) + 1]++;
            for (int64_t b = 0; b < nb; b++) start[(size_t)b + 1] += start[(size_t)b];
            for (int64_t k = 0; k < n; k++) st.h_ord[start[(size_t)key(k)]++] = (int32_t)k;
            RTCHK(rt_h2d(st.ord.p, st.h_ord, (size_t)n * 4, e->s_in));
            e->pair_order = (const int32_t *)st.ord.p;
        }
        RTCHK(rt_record(st.in_done, e->s_in));
        RTCHK(rt_wait(e->stream, st.in_done));
        rc = launch_on(e, e->stream, Batch{(const uint8_t *)st.reads.p, (const int64_t *)st.off.p, n, (int32_t)maxJ,
                       count ? (const int32_t *)st.cnt.p : nullptr, qweight ? (const int32_t *)st.qw.p : nullptr,
                       ref_id ? (const int32_t *)st.rid.p : nullptr, (c2b_read_rec *)st.recs.p,
                       (c2b_aln_rec *)st.alns.p, strings ? (uint8_t *)st.str.p : nullptr,
                       cap ? (c2b_edit *)st.ed.p : nullptr, (uint64_t *)st.gops.p, (uint32_t *)st.gmeta.p, (int32_t *)st.left.p, (int32_t *)st.left2.p, (int32_t *)st.left0.p,
                       (int32_t *)st.left1.p});
        e->pair_order = nullptr;
        if (rc) return rc;
        // keep this batch's "widest alignment" before the next launch sequence resets it
        RTCHK(cudaMemcpyAsyncOrCopy(st.maxlen.p, &((WorkBlock *)e->work.p)->launch.widest, 8, e->stream));
        RTCHK(rt_record(st.k_done, e->stream));
        st.used = true;
        if (pend.any && (rc = flush(pend))) return rc;           // chunk ci-1: overlaps this chunk's kernels
        pend.any = true; pend.c0 = c0; pend.n = n; pend.set = ci & 1;
    }
    if (pend.any && (rc = flush(pend))) return rc;
    RTCHK(rt_sync(e->s_out));
    RTCHK(rt_sync(e->stream));
    for (auto &st : e->stage) if ((rc = drain(st))) return rc;
    return C2B_OK;
}

int c2b_align_batch(c2b_engine *e, const uint8_t *reads, const int64_t *offsets, int64_t n_reads,
                    const int32_t *count, const int32_t *qweight, const int32_t *ref_id,
                    c2b_read_rec *recs, c2b_aln_rec *alns, uint8_t *strings, c2b_edit *edits)
{
    return align_batch_host(e, reads, offsets, n_reads, count, qweight, ref_id, recs, alns, strings, nullptr, nullptr, edits);
}

int c2b_align_batch_compact(c2b_engine *e, const uint8_t *reads, const int64_t *offsets, int64_t n_reads,
                            const int32_t *count, const int32_t *qweight, const int32_t *ref_id,
                            c2b_read_rec *recs, c2b_aln_rec *alns, uint64_t *ops, uint32_t *meta, c2b_edit *edits)
{
    if (!ops || !meta) return fail(e, C2B_E_ARG, "c2b_align_batch_compact: ops / meta missing");
    return align_batch_host(e, reads, offsets, n_reads, count, qweight, ref_id, recs, alns, nullptr, ops, meta, edits);
}

int c2b_ops_words(const c2b_engine *e, int32_t max_read_len)
{
    if (!e || !e->configured) return C2B_E_STATE;
    return ((e->max_I + max_read_len + 31) & ~31) / 32;
}

// Aligned strings of one (read, reference) slot from its op stream: host code, no device work.  Column q from the RIGHT
// end of the alignment is op (ops[q >> 5] >> 2 (q & 31)) & 3: 0 = both consume, 1 = gap in the read, 2 = gap in the
// reference.  strand 1: the read was aligned as its reverse complement (comp256: the complement of every byte).
static int expand_slot(const uint8_t *comp256, const uint64_t *ops, uint32_t meta, const char *read, int32_t read_len,
                       const char *ref, int32_t ref_len, char *out_read, char *out_ref)
{
    const int n = (int)(meta & 0xffffu), strand = (int)((meta >> 16) & 1u);
    int i = ref_len, j = read_len;
    for (int q = 0; q < n; q++) {
        const int op = (int)((ops[q >> 5] >> (2 * (q & 31))) & 3ull);
        char rd = '-', rf = '-';
        if (op != OP_J) { if (j < 1) return C2B_E_ARG; j--; rd = strand ? (char)comp256[(unsigned char)read[read_len - 1 - j]] : read[j]; }
        if (op != OP_I) { if (i < 1) return C2B_E_ARG; i--; rf = ref[i]; }
        if (op == OP_NONE) return C2B_E_ARG;
        out_read[n - 1 - q] = rd; out_ref[n - 1 - q] = rf;
    }
    return (i == 0 && j == 0) ? C2B_OK : C2B_E_ARG;
}

// the engine's complement table (c2b_params.complement) over all bytes, identity outside the alphabet
static void engine_comp256(const c2b_engine *e, uint8_t *comp)
{
    for (int c = 0; c < 256; c++) comp[c] = (uint8_t)c;
    for (int q = 0; q < e->prm.nq; q++) comp[(unsigned char)e->prm.alphabet[q]] = (uint8_t)e->prm.alphabet[e->prm.complement[q]];
}

int c2b_expand_alignment(const c2b_engine *e, const uint64_t *ops, uint32_t meta, const char *read, int32_t read_len,
                         const char *ref, int32_t ref_len, char *out_read, char *out_ref)
{
    if (!e || !ops || !read || !ref || !out_read || !out_ref) return C2B_E_ARG;
    uint8_t comp[256];
    engine_comp256(e, comp);
    return expand_slot(comp, ops, meta, read, read_len, ref, ref_len, out_read, out_ref);
}

// Batch form over explicit tables: strings[n_reads][R][2][W], right-aligned like c2b_align_batch's; host threads.  Nothing is
// read from an engine, so a batch's results spell the same strings whatever their engine was configured with since.
int c2b_expand_batch_tables(const uint8_t *reads, const int64_t *offsets, int64_t n_reads, const int32_t *ref_id,
                            const uint64_t *ops, const uint32_t *meta, int32_t R, int32_t W, int32_t n_refs,
                            const char *const *ref_seqs, const int32_t *ref_lens, const uint8_t *comp256,
                            uint8_t *strings, int32_t n_threads)
{
    if (n_reads < 0 || (n_reads && (!reads || !offsets || !ops || !meta || !strings)) || !ref_seqs || !ref_lens || !comp256)
        return C2B_E_ARG;
    if (W < 32 || (W & 31) || n_refs < 1 || R < 1 || (ref_id ? R != 1 : R > n_refs)) return C2B_E_ARG;
    for (int r = 0; r < n_refs; r++) if (!ref_seqs[r] || ref_lens[r] < 1) return C2B_E_ARG;
    const int NW = W / 32;
    if (n_threads <= 0) n_threads = (int)std::max(1u, std::thread::hardware_concurrency());
    n_threads = (int)std::min<int64_t>(n_threads, std::max<int64_t>(1, n_reads / 1024));
    std::vector<int> bad((size_t)n_threads, 0);
    auto work = [&](int t) {
        const int64_t lo = n_reads * t / n_threads, hi = n_reads * (t + 1) / n_threads;
        for (int64_t rd = lo; rd < hi; rd++)
            for (int k = 0; k < R; k++) {
                const int r = ref_id ? ref_id[rd] : k;
                const int64_t slot = rd * R + k;
                const uint32_t m = meta[slot];
                const int n = (int)(m & 0xffffu);
                if ((m >> 24) == 0 || n == 0 || n > W) continue;      // no alignment in this slot
                if (r < 0 || r >= n_refs) { bad[(size_t)t]++; continue; }
                uint8_t *o = strings + slot * 2 * (int64_t)W;
                if (expand_slot(comp256, ops + slot * NW, m, (const char *)reads + offsets[rd], (int32_t)(offsets[rd + 1] - offsets[rd]),
                                ref_seqs[r], ref_lens[r], (char *)o + W - n, (char *)o + 2 * W - n)) bad[(size_t)t]++;
            }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < n_threads; t++) th.emplace_back(work, t);
    work(0);
    for (auto &x : th) x.join();
    for (int b : bad) if (b) return C2B_E_ARG;
    return C2B_OK;
}

// Batch form over the engine's current configuration (the batch must have run under it)
int c2b_expand_batch(const c2b_engine *e, const uint8_t *reads, const int64_t *offsets, int64_t n_reads, const int32_t *ref_id,
                     const uint64_t *ops, const uint32_t *meta, int32_t max_read_len, uint8_t *strings, int32_t n_threads)
{
    if (!e || !e->configured || !reads || !offsets || !ops || !meta || !strings) return C2B_E_ARG;
    const int W = (e->max_I + max_read_len + 31) & ~31, nr = ref_id ? 1 : e->n_refs;
    std::vector<const char *> seqs((size_t)e->n_refs);
    std::vector<int32_t> lens((size_t)e->n_refs);
    for (int r = 0; r < e->n_refs; r++) { seqs[(size_t)r] = e->refs[(size_t)r].seq.data(); lens[(size_t)r] = (int32_t)e->refs[(size_t)r].seq.size(); }
    uint8_t comp[256];
    engine_comp256(e, comp);
    return c2b_expand_batch_tables(reads, offsets, n_reads, ref_id, ops, meta, nr, W, e->n_refs, seqs.data(), lens.data(), comp,
                                   strings, n_threads);
}

int c2b_counts_layout(const c2b_engine *e, int32_t *n_refs, int32_t *n_vec, int32_t *stride, int32_t *n_scal)
{
    if (!e || !e->configured) return C2B_E_STATE;
    if (n_refs) *n_refs = e->n_refs;
    if (n_vec) *n_vec = C2B_NVEC;
    if (stride) *stride = e->vstride;
    if (n_scal) *n_scal = C2B_NSCAL;
    return C2B_OK;
}

int c2b_counts_hist_layout(const c2b_engine *e, int32_t *n_hist, int32_t *hstride, int32_t *hist_zero)
{
    if (!e || !e->configured) return C2B_E_STATE;
    if (n_hist) *n_hist = C2B_NHIST;
    if (hstride) *hstride = e->hstride;
    if (hist_zero) *hist_zero = e->hist_zero;
    return C2B_OK;
}

int c2b_counts_reset(c2b_engine *e)
{
    if (!e || !e->configured) return fail(e, C2B_E_STATE, "c2b_counts_reset: engine not configured");
    RTCHK(rt_zero(e->d_counts, e->counts_n * 8, e->stream));
    if (e->work.p) RTCHK(rt_zero(e->work.p, WORK_BYTES, e->stream));
    RTCHK(rt_sync(e->stream));
    return C2B_OK;
}

int c2b_counts_read(c2b_engine *e, int64_t *out, size_t n_int64)
{
    if (!e || !e->configured || !out) return fail(e, C2B_E_STATE, "c2b_counts_read: engine not configured");
    if (n_int64 < e->counts_n) return fail(e, C2B_E_ARG, "c2b_counts_read: buffer too small");
    RTCHK(rt_d2h(out, e->d_counts, e->counts_n * 8, e->stream));
    RTCHK(rt_sync(e->stream));
    return C2B_OK;
}

int c2b_counts_device(c2b_engine *e, void **d_ptr, size_t *n_int64)
{
    if (!e || !e->configured) return C2B_E_STATE;
    if (d_ptr) *d_ptr = e->d_counts;
    if (n_int64) *n_int64 = e->counts_n;
    return C2B_OK;
}

int c2b_global_align(c2b_engine *e, const char *read, int32_t read_len, const char *ref, int32_t ref_len,
                     const char *alphabet, int32_t nq, const int64_t *score_rows, const int64_t *gap_incentive,
                     int32_t gap_open, int32_t gap_extend,
                     char *out_read, char *out_ref, int32_t *aln_len, int32_t *n_match)
{
    if (!e || !read || !ref || !alphabet || !score_rows || !gap_incentive || !out_read || !out_ref || !aln_len || !n_match)
        return fail(e, C2B_E_ARG, "c2b_global_align: bad argument");
    c2b_params p; memset(&p, 0, sizeof p);
    p.gap_open = gap_open; p.gap_extend = gap_extend; p.flags = C2B_F_NO_STRAND_SEARCH; p.nq = nq;
    if (nq < 1 || nq > C2B_MAX_Q) return fail(e, C2B_E_LIMIT, "c2b_global_align: alphabet larger than C2B_MAX_Q");
    memcpy(p.alphabet, alphabet, nq);
    for (int q = 0; q < nq; q++) p.complement[q] = (uint8_t)q;
    c2b_ref r; memset(&r, 0, sizeof r);
    r.seq = ref; r.len = ref_len; r.gap_incentive = gap_incentive; r.score_rows = score_rows; r.min_aln_score = -1.0;
    int rc = c2b_configure(e, &p, 1, &r);
    if (rc) return rc;
    const int W = c2b_string_width(e, read_len);
    std::vector<uint8_t> str((size_t)2 * W);
    int64_t off[2] = {0, read_len};
    c2b_read_rec rec; c2b_aln_rec a;
    rc = c2b_align_batch(e, (const uint8_t *)read, off, 1, nullptr, nullptr, nullptr, &rec, &a, str.data(), nullptr);
    if (rc) return rc;
    if (a.status) { e->err = "c2b_global_align: alignment status " + std::to_string(a.status); return 100 + a.status; }
    memcpy(out_read, str.data() + W - a.aln_len, a.aln_len);
    memcpy(out_ref, str.data() + 2 * W - a.aln_len, a.aln_len);
    *aln_len = a.aln_len; *n_match = a.n_match;
    return C2B_OK;
}

int c2b_classify_aligned(c2b_engine *e, const char *read_al, const char *ref_al, int32_t n_cols,
                         const char *alphabet, int32_t nq, const int64_t *include_idx, int32_t n_include,
                         c2b_aln_rec *out, c2b_edit *edits)
{
    return c2b_classify_aligned_flags(e, read_al, ref_al, n_cols, alphabet, nq, include_idx, n_include, 0u, out, edits);
}

int c2b_classify_aligned_flags(c2b_engine *e, const char *read_al, const char *ref_al, int32_t n_cols,
                               const char *alphabet, int32_t nq, const int64_t *include_idx, int32_t n_include,
                               uint32_t flags, c2b_aln_rec *out, c2b_edit *edits)
{
    if (!e || !read_al || !ref_al || !alphabet || !out || !edits || n_cols < 1) return fail(e, C2B_E_ARG, "c2b_classify_aligned: bad argument");
    if (n_cols > C2B_MAX_ALN_LEN) return fail(e, C2B_E_LIMIT, "c2b_classify_aligned: alignment longer than C2B_MAX_ALN_LEN");
    if (nq < 1 || nq > C2B_MAX_Q) return fail(e, C2B_E_LIMIT, "c2b_classify_aligned: alphabet larger than C2B_MAX_Q");
    std::string read, ref;
    std::vector<uint64_t> ops(32, ~0ull);
    int prev = -1;
    for (int c = n_cols - 1, n = 0; c >= 0; c--, n++) {           // op n = n-th column from the right
        const bool gq = read_al[c] == '-', gr = ref_al[c] == '-';
        if (gq && gr) return fail(e, C2B_E_ARG, "c2b_classify_aligned: column with two gaps");
        const int op = gq ? OP_J : gr ? OP_I : OP_M;
        if ((op == OP_I && prev == OP_J) || (op == OP_J && prev == OP_I))
            return fail(e, C2B_E_ARG, "c2b_classify_aligned: insertion column adjacent to a deletion column");
        prev = op;
        ops[n >> 5] &= ~(3ull << (2 * (n & 31)));
        ops[n >> 5] |= (uint64_t)op << (2 * (n & 31));
    }
    for (int c = 0; c < n_cols; c++) { if (read_al[c] != '-') read.push_back(read_al[c]); if (ref_al[c] != '-') ref.push_back(ref_al[c]); }
    if (read.empty() || ref.empty()) return fail(e, C2B_E_ARG, "c2b_classify_aligned: empty sequence");
    if ((int)read.size() > C2B_MAX_READ_LEN || (int)ref.size() > C2B_MAX_REF_LEN) return fail(e, C2B_E_LIMIT, "c2b_classify_aligned: sequence too long");
    c2b_params p; memset(&p, 0, sizeof p);
    p.gap_open = -1; p.gap_extend = -1; p.flags = C2B_F_NO_STRAND_SEARCH | (flags & C2B_F_LEGACY_INS); p.nq = nq; p.edit_cap = n_cols + 1;
    memcpy(p.alphabet, alphabet, nq);
    for (int q = 0; q < nq; q++) p.complement[q] = (uint8_t)q;
    std::vector<int64_t> gi(ref.size() + 1, 0), rows((size_t)nq * ref.size(), 0);
    c2b_ref r; memset(&r, 0, sizeof r);
    r.seq = ref.c_str(); r.len = (int32_t)ref.size(); r.gap_incentive = gi.data(); r.score_rows = rows.data();
    r.include_idx = include_idx; r.n_include = n_include; r.min_aln_score = -1.0;
    int rc = c2b_configure(e, &p, 1, &r);
    if (rc) return rc;
    DevBuf d_ops, d_n;
    if ((rc = ensure(e, d_ops, 32 * 8)) || (rc = ensure(e, d_n, 4))) return rc;
    const int32_t n32 = n_cols;
    RTCHK(rt_h2d(d_ops.p, ops.data(), 32 * 8, e->stream));
    RTCHK(rt_h2d(d_n.p, &n32, 4, e->stream));
    e->forced_ops = (const uint64_t *)d_ops.p; e->forced_n = (const int32_t *)d_n.p;
    int64_t off[2] = {0, (int64_t)read.size()};
    c2b_read_rec rec;
    rc = c2b_align_batch(e, (const uint8_t *)read.data(), off, 1, nullptr, nullptr, nullptr, &rec, out, nullptr, edits);
    e->forced_ops = nullptr; e->forced_n = nullptr;
    rt_free(d_ops.p); rt_free(d_n.p);
    return rc;
}

// Read annotations (c2b_annotate.cuh) for unique reads in chunks: the chunk's inputs go up through one pinned buffer, a size
// pass, a scan and a write pass run on the engine's stream, the texts come back through a second pinned buffer.  Device memory
// is bounded by the chunk, whatever the number of reads.
int c2b_annotate_build(c2b_engine *e, const uint8_t *reads, const int64_t *offsets, int64_t n_unique, const int32_t *bidx,
                       int32_t R, int32_t NW, int32_t edit_cap, const c2b_read_rec *recs, const c2b_aln_rec *alns,
                       const uint64_t *ops, const uint32_t *meta, const c2b_edit *edits,
                       const uint32_t *amask, const int16_t *aname, const int32_t *label,
                       int32_t n_names, const char *const *names, const uint8_t *name_rev,
                       int32_t n_labels, const char *const *labels,
                       const char *const *ref_seqs, const int32_t *ref_lens, const uint8_t *comp256, uint32_t flags,
                       int64_t chunk, c2b_annotation **out)
{
    if (!e || !out || n_unique < 0 || (n_unique && (!offsets || !bidx)) || R < 1 || R > C2B_MAX_REFS || NW < 1 || edit_cap < 0 ||
        n_names < R || !names || !name_rev || n_labels < 0 || (n_labels && !labels) || !ref_seqs || !ref_lens || !comp256)
        return fail(e, C2B_E_ARG, "c2b_annotate_build: bad argument");
    *out = nullptr;
    int64_t nb = 0;                                               // batch reads referenced
    for (int64_t u = 0; u < n_unique; u++) if (bidx[u] >= 0) nb = std::max<int64_t>(nb, (int64_t)bidx[u] + 1);
    if (nb && (!recs || !alns || !ops || !meta || !amask || !aname || !label || (edit_cap && !edits)))
        return fail(e, C2B_E_ARG, "c2b_annotate_build: batch arrays missing");
    for (int64_t k = 0; k < nb; k++) {
        if (label[k] < -1 || label[k] >= n_labels || aname[k] >= n_names) return fail(e, C2B_E_ARG, "c2b_annotate_build: label / name id out of range");
        if (amask[k] && label[k] < 0) return fail(e, C2B_E_ARG, "c2b_annotate_build: aligned read without a class label");
        // widened before the shift: a 32-bit shift by R = C2B_MAX_REFS = 32 is undefined (x86 shifts by 0 and refused every read)
        if ((uint64_t)amask[k] >> R) return fail(e, C2B_E_ARG, "c2b_annotate_build: listed slot out of range");
        for (int r = 0; r < R; r++) {
            const uint32_t m = meta[k * R + r];
            if ((m >> 24) && ((int)(m & 0xffffu) > std::min(32 * NW, (int)C2B_MAX_ALN_LEN) || alns[k * R + r].n_edits > edit_cap))
                return fail(e, C2B_E_ARG, "c2b_annotate_build: alignment wider than the op words, or an incomplete edit list");
        }
    }
    if (chunk <= 0) chunk = 1 << 16;
    // constant tables: names, labels, reference sequences, complement table
    std::string tab;
    std::vector<int32_t> name_off(1, 0), label_off(1, 0), ref_off(1, 0);
    std::string nm, lb, rs;
    for (int i = 0; i < n_names; i++) { nm += names[i]; name_off.push_back((int32_t)nm.size()); }
    for (int i = 0; i < n_labels; i++) { lb += labels[i]; label_off.push_back((int32_t)lb.size()); }
    for (int r = 0; r < R; r++) { rs.append(ref_seqs[r], (size_t)ref_lens[r]); ref_off.push_back((int32_t)rs.size()); }
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    size_t t_names = 0, t_noff = al(nm.size()), t_rev = t_noff + al(name_off.size() * 4), t_lab = t_rev + al((size_t)n_names),
           t_loff = t_lab + al(lb.size()), t_ref = t_loff + al(label_off.size() * 4), t_roff = t_ref + al(rs.size()),
           t_comp = t_roff + al(ref_off.size() * 4), t_end = t_comp + 256;
    tab.assign(t_end, '\0');
    memcpy(&tab[t_names], nm.data(), nm.size()); memcpy(&tab[t_noff], name_off.data(), name_off.size() * 4);
    memcpy(&tab[t_rev], name_rev, (size_t)n_names); memcpy(&tab[t_lab], lb.data(), lb.size());
    memcpy(&tab[t_loff], label_off.data(), label_off.size() * 4); memcpy(&tab[t_ref], rs.data(), rs.size());
    memcpy(&tab[t_roff], ref_off.data(), ref_off.size() * 4); memcpy(&tab[t_comp], comp256, 256);
    DevBuf d_tab, d_in, d_len, d_out;
    uint8_t *h_in = nullptr, *h_out = nullptr; size_t h_in_cap = 0, h_out_cap = 0;
    auto cleanup = [&]() { rt_free(d_tab.p); rt_free(d_in.p); rt_free(d_len.p); rt_free(d_out.p); rt_host_free(h_in); rt_host_free(h_out); };
    auto grow_host = [](uint8_t *&p, size_t &cap, size_t n) {
        if (n <= cap) return true;
        rt_host_free(p); cap = n + n / 4 + 4096; p = (uint8_t *)rt_host_alloc(cap);
        return p != nullptr;
    };
    std::unique_ptr<c2b_annotation> A(new c2b_annotation());
    A->n = n_unique;
    A->ann_off.assign(1, 0); A->cig_off.assign(1, 0);
    A->flag.resize((size_t)n_unique); A->mapq.resize((size_t)n_unique); A->first.resize((size_t)n_unique);
    int rc = ensure(e, d_tab, t_end);
    if (!rc) { rt_err r = rt_h2d(d_tab.p, tab.data(), t_end, e->stream); if (r != RT_OK) rc = fail(e, C2B_E_CUDA, "c2b_annotate_build: copy of the tables"); }
    const size_t ER = (size_t)R, OW = (size_t)R * NW * 8, EW = (size_t)R * edit_cap * sizeof(c2b_edit);
    auto one_chunk = [&](int64_t u0) -> int {
        const int64_t u1 = std::min(n_unique, u0 + chunk), m = u1 - u0;
        int64_t k0 = -1, k1 = 0;
        for (int64_t u = u0; u < u1; u++) if (bidx[u] >= 0) { if (k0 < 0) k0 = bidx[u]; k1 = (int64_t)bidx[u] + 1; }
        if (k0 < 0) k0 = k1 = 0;
        const int64_t mk = k1 - k0;
        const size_t rb = (size_t)(offsets[u1] - offsets[u0]);
        // chunk input layout (device): reads | roff | bidx | recs | alns | ops | meta | edits | amask | aname | label
        size_t o_reads = 0, o_roff = al(rb), o_bidx = o_roff + al((size_t)(m + 1) * 8), o_recs = o_bidx + al((size_t)m * 4),
               o_alns = o_recs + al((size_t)mk * sizeof(c2b_read_rec)), o_ops = o_alns + al((size_t)mk * ER * sizeof(c2b_aln_rec)),
               o_meta = o_ops + al((size_t)mk * OW), o_ed = o_meta + al((size_t)mk * ER * 4), o_am = o_ed + al((size_t)mk * EW),
               o_an = o_am + al((size_t)mk * 4), o_lb = o_an + al((size_t)mk * 2), o_end = o_lb + al((size_t)mk * 4);
        if (!grow_host(h_in, h_in_cap, o_end)) return fail(e, C2B_E_CUDA, "c2b_annotate_build: pinned allocation");
        if (rb) memcpy(h_in + o_reads, reads + offsets[u0], rb);
        int64_t *hro = (int64_t *)(h_in + o_roff);
        for (int64_t u = 0; u <= m; u++) hro[u] = offsets[u0 + u] - offsets[u0];
        int32_t *hb = (int32_t *)(h_in + o_bidx);
        for (int64_t u = 0; u < m; u++) hb[u] = bidx[u0 + u] >= 0 ? (int32_t)(bidx[u0 + u] - k0) : -1;
        if (mk) {
            memcpy(h_in + o_recs, recs + k0, (size_t)mk * sizeof(c2b_read_rec));
            memcpy(h_in + o_alns, alns + k0 * R, (size_t)mk * ER * sizeof(c2b_aln_rec));
            memcpy(h_in + o_ops, ops + k0 * R * NW, (size_t)mk * OW);
            memcpy(h_in + o_meta, meta + k0 * R, (size_t)mk * ER * 4);
            if (EW) memcpy(h_in + o_ed, edits + k0 * R * edit_cap, (size_t)mk * EW);
            memcpy(h_in + o_am, amask + k0, (size_t)mk * 4);
            memcpy(h_in + o_an, aname + k0, (size_t)mk * 2);
            memcpy(h_in + o_lb, label + k0, (size_t)mk * 4);
        }
        // lengths (2m) + offsets (2(m+1)) + flag / mapq / first
        const size_t l_len = 0, l_aoff = al((size_t)2 * m * 8), l_coff = l_aoff + al((size_t)(m + 1) * 8),
                     l_flag = l_coff + al((size_t)(m + 1) * 8), l_mapq = l_flag + al((size_t)m), l_first = l_mapq + al((size_t)m * 4),
                     l_end = l_first + al((size_t)m * 2);
        int rc2;
        if ((rc2 = ensure(e, d_in, o_end)) || (rc2 = ensure(e, d_len, l_end))) return rc2;
        RTCHK(rt_h2d(d_in.p, h_in, o_end, e->stream));
        char *di = (char *)d_in.p, *dl = (char *)d_len.p, *dt = (char *)d_tab.p;
        c2b::ann::AParams P;
        memset(&P, 0, sizeof P);
        P.reads = (const uint8_t *)(di + o_reads); P.roff = (const int64_t *)(di + o_roff); P.n = m;
        P.bidx = (const int32_t *)(di + o_bidx); P.R = R; P.NW = NW; P.cap = edit_cap; P.flags = flags;
        P.recs = (const c2b_read_rec *)(di + o_recs); P.alns = (const c2b_aln_rec *)(di + o_alns); P.ops = (const uint64_t *)(di + o_ops);
        P.meta = (const uint32_t *)(di + o_meta); P.edits = (const c2b_edit *)(di + o_ed);
        P.amask = (const uint32_t *)(di + o_am); P.aname = (const int16_t *)(di + o_an); P.label = (const int32_t *)(di + o_lb);
        P.names = dt + t_names; P.name_off = (const int32_t *)(dt + t_noff); P.name_rev = (const uint8_t *)(dt + t_rev);
        P.labels = dt + t_lab; P.label_off = (const int32_t *)(dt + t_loff);
        P.refseq = dt + t_ref; P.ref_off = (const int32_t *)(dt + t_roff); P.comp = (const uint8_t *)(dt + t_comp);
        P.ann_len = (int64_t *)(dl + l_len); P.cig_len = P.ann_len + m;
        P.ann_off = (const int64_t *)(dl + l_aoff); P.cig_off = (const int64_t *)(dl + l_coff);
        P.flag = (uint8_t *)(dl + l_flag); P.mapq = (int32_t *)(dl + l_mapq); P.first = (int16_t *)(dl + l_first);
        int64_t tot[2] = {0, 0};
#ifndef C2B_EMU
        const int grid = (int)std::min<int64_t>((m + 7) / 8, 8192);
        c2b_annotate_size_kernel<<<grid, 256, 0, e->stream>>>(P);
        c2b_annotate_scan_kernel<<<1, 32, 0, e->stream>>>(P.ann_len, (int64_t *)P.ann_off, P.cig_len, (int64_t *)P.cig_off, m);
        RTCHK(cudaGetLastError());
        RTCHK(rt_d2h(&tot[0], P.ann_off + m, 8, e->stream));
        RTCHK(rt_d2h(&tot[1], P.cig_off + m, 8, e->stream));
        RTCHK(rt_sync(e->stream));
#else
        for (int64_t u = 0; u < m; u++) emu::run_warp([&]() { c2b::ann::annotate_one<false>(P, u); });
        emu::run_warp([&]() { c2b::ann::scan_sizes(P.ann_len, (int64_t *)P.ann_off, m); c2b::ann::scan_sizes(P.cig_len, (int64_t *)P.cig_off, m); });
        tot[0] = P.ann_off[m]; tot[1] = P.cig_off[m];
#endif
        if ((rc2 = ensure(e, d_out, (size_t)(tot[0] + tot[1]) + 16))) return rc2;
        P.ann = (char *)d_out.p; P.cig = (char *)d_out.p + tot[0];
#ifndef C2B_EMU
        c2b_annotate_write_kernel<<<grid, 256, 0, e->stream>>>(P);
        RTCHK(cudaGetLastError());
#else
        for (int64_t u = 0; u < m; u++) emu::run_warp([&]() { c2b::ann::annotate_one<true>(P, u); });
#endif
        const size_t l_tail = l_end - l_aoff, bytes = (size_t)(tot[0] + tot[1]);
        if (!grow_host(h_out, h_out_cap, l_tail + bytes)) return fail(e, C2B_E_CUDA, "c2b_annotate_build: pinned allocation");
        RTCHK(rt_d2h(h_out, dl + l_aoff, l_tail, e->stream));
        RTCHK(rt_d2h(h_out + l_tail, d_out.p, bytes, e->stream));
        RTCHK(rt_sync(e->stream));
        const int64_t *ao = (const int64_t *)(h_out + 0), *co = (const int64_t *)(h_out + (l_coff - l_aoff));
        const int64_t abase = A->ann_off.back(), cbase = A->cig_off.back();
        for (int64_t u = 1; u <= m; u++) { A->ann_off.push_back(abase + ao[u]); A->cig_off.push_back(cbase + co[u]); }
        A->ann.resize((size_t)(abase + tot[0])); A->cig.resize((size_t)(cbase + tot[1]));
        if (tot[0]) memcpy(A->ann.data() + abase, h_out + l_tail, (size_t)tot[0]);
        if (tot[1]) memcpy(A->cig.data() + cbase, h_out + l_tail + tot[0], (size_t)tot[1]);
        memcpy(A->flag.data() + u0, h_out + (l_flag - l_aoff), (size_t)m);
        memcpy(A->mapq.data() + u0, h_out + (l_mapq - l_aoff), (size_t)m * 4);
        memcpy(A->first.data() + u0, h_out + (l_first - l_aoff), (size_t)m * 2);
        return C2B_OK;
    };
    for (int64_t u0 = 0; !rc && u0 < n_unique; u0 += chunk) rc = one_chunk(u0);
    cleanup();
    if (rc) return rc;
    *out = A.release();
    return C2B_OK;
}

void c2b_annotate_free(c2b_annotation *a) { delete a; }
int64_t c2b_annotate_n(const c2b_annotation *a) { return a ? a->n : 0; }
const uint8_t *c2b_annotate_arena(const c2b_annotation *a) { return a ? a->ann.data() : nullptr; }
const int64_t *c2b_annotate_offsets(const c2b_annotation *a) { return a ? a->ann_off.data() : nullptr; }
const uint8_t *c2b_annotate_cigar_arena(const c2b_annotation *a) { return a ? a->cig.data() : nullptr; }
const int64_t *c2b_annotate_cigar_offsets(const c2b_annotation *a) { return a ? a->cig_off.data() : nullptr; }
const uint8_t *c2b_annotate_flags(const c2b_annotation *a) { return a ? a->flag.data() : nullptr; }
const int32_t *c2b_annotate_mapq(const c2b_annotation *a) { return a ? a->mapq.data() : nullptr; }
const int16_t *c2b_annotate_first(const c2b_annotation *a) { return a ? a->first.data() : nullptr; }
const int64_t *c2b_annotate_last_record(const c2b_annotation *a) { return a && !a->last_rec.empty() ? a->last_rec.data() : nullptr; }
const uint8_t *c2b_annotate_record_arena(const c2b_annotation *a) { return a ? (const uint8_t *)a->rec.data() : nullptr; }
const int64_t *c2b_annotate_record_offsets(const c2b_annotation *a) { return a && !a->rec_off.empty() ? a->rec_off.data() : nullptr; }

}  // extern "C"

// ----------------------------------------------------------------------------------------- packed allele rows in chunks
// --vcf_output and --base_editor_output pass allele rows to the device as packed columns, a chunk of rows at a time: the
// chunk's columns go up through one pinned buffer, per-row sizes and scans live in a second device buffer, results come back
// through a second pinned buffer.

// one packed column: `width` bytes per row (off == nullptr), or per row the items [off[r], off[r+1]) of `width` bytes each
struct RowCol { const void *val; const int64_t *off; size_t width; };

struct ChunkPipe {
    c2b_engine *e;
    DevBuf d_in, d_len, d_out, d_fixed;
    uint8_t *h_in = nullptr, *h_out = nullptr; size_t h_in_cap = 0, h_out_cap = 0;
    explicit ChunkPipe(c2b_engine *e_) : e(e_) {}
    ~ChunkPipe() { rt_free(d_in.p); rt_free(d_len.p); rt_free(d_out.p); rt_free(d_fixed.p); rt_host_free(h_in); rt_host_free(h_out); }
    static size_t al(size_t x) { return (x + 255) & ~(size_t)255; }
    static bool grow(uint8_t *&p, size_t &cap, size_t n)
    {
        if (n <= cap) return true;
        rt_host_free(p); cap = n + n / 4 + 4096; p = (uint8_t *)rt_host_alloc(cap);
        return p != nullptr;
    }
    // rows [r0, r1) of the columns to the device: dev[c] their values, doff[c] their offsets rebased to the chunk (ragged columns)
    int upload(const RowCol *cols, int nc, int64_t r0, int64_t r1, const char **dev, const int64_t **doff)
    {
        const int64_t m = r1 - r0;
        std::vector<size_t> o_val((size_t)nc), o_off((size_t)nc);
        size_t o = 0;
        for (int c = 0; c < nc; c++) {
            o_val[(size_t)c] = o;
            o += al(cols[c].off ? (size_t)(cols[c].off[r1] - cols[c].off[r0]) * cols[c].width : (size_t)m * cols[c].width);
            o_off[(size_t)c] = o;
            if (cols[c].off) o += al((size_t)(m + 1) * 8);
        }
        if (!grow(h_in, h_in_cap, o)) return fail(e, C2B_E_CUDA, "packed rows: pinned allocation");
        for (int c = 0; c < nc; c++) {
            const RowCol &k = cols[c];
            const int64_t b = k.off ? k.off[r0] : r0;
            const size_t nb = (size_t)((k.off ? k.off[r1] : r1) - b) * k.width;
            if (nb) memcpy(h_in + o_val[(size_t)c], (const uint8_t *)k.val + (size_t)b * k.width, nb);
            if (k.off) {
                int64_t *ho = (int64_t *)(h_in + o_off[(size_t)c]);
                for (int64_t r = 0; r <= m; r++) ho[r] = k.off[r0 + r] - b;
            }
        }
        int rc;
        if ((rc = ensure(e, d_in, o))) return rc;
        RTCHK(rt_h2d(d_in.p, h_in, o, e->stream));
        for (int c = 0; c < nc; c++) {
            dev[c] = (const char *)d_in.p + o_val[(size_t)c];
            if (doff) doff[c] = cols[c].off ? (const int64_t *)((const char *)d_in.p + o_off[(size_t)c]) : nullptr;
        }
        return C2B_OK;
    }
    // data every chunk reads, to the device once
    int fixed(const void *src, size_t n, const char **dev)
    {
        int rc;
        if ((rc = ensure(e, d_fixed, n))) return rc;
        RTCHK(rt_h2d(d_fixed.p, src, n, e->stream));
        *dev = (const char *)d_fixed.p;
        return C2B_OK;
    }
    // d_out[0 .. n) to pinned host memory once the stream's work is done
    int download(size_t n, const uint8_t **h)
    {
        if (!grow(h_out, h_out_cap, n)) return fail(e, C2B_E_CUDA, "packed rows: pinned allocation");
        RTCHK(rt_d2h(h_out, d_out.p, n, e->stream));
        RTCHK(rt_sync(e->stream));
        *h = h_out;
        return C2B_OK;
    }
};

// the records of all chunks of a record pass, in row order
struct RecordSink { std::vector<uint8_t> keys; std::vector<int64_t> rec_pos, rec_w; };

// One chunk of m rows through a record pass (c2b_vcf.cuh, c2b_base_edit.cuh), P's inputs set: the size pass notes every row's
// records, bytes and exception, a one-warp scan places them and finds the first exception, the write pass builds the records in
// d_out and, after them, `extra` bytes of per-row output (*extra_out: their pinned host copy, at the P.* pointer that `write`
// sets from its second argument).  -> C2B_OK; 1 with first[0..2] = chunk row, kind, value of the chunk's first exception; or an
// error code.
template <class PT, class Size, class Write>
static int record_chunk(c2b_engine *e, ChunkPipe &cp, PT &P, int64_t m, size_t extra, Size size_pass, Write write_pass,
                        RecordSink &S, int64_t *first, const uint8_t **extra_out)
{
    auto al = ChunkPipe::al;
    // per row: nrec | nbytes | err (2) | rec_base (m + 1) | key_off (m + 1) | first (3)
    const size_t l_nrec = 0, l_nbytes = al((size_t)m * 8), l_err = l_nbytes + al((size_t)m * 8), l_rb = l_err + al((size_t)m * 16),
                 l_ko = l_rb + al((size_t)(m + 1) * 8), l_first = l_ko + al((size_t)(m + 1) * 8), l_end = l_first + 3 * 8;
    int rc;
    if ((rc = ensure(e, cp.d_len, l_end))) return rc;
    char *dl = (char *)cp.d_len.p;
    P.nrec = (int64_t *)(dl + l_nrec); P.nbytes = (int64_t *)(dl + l_nbytes); P.err = (int64_t *)(dl + l_err);
    P.rec_base = (const int64_t *)(dl + l_rb); P.key_off = (const int64_t *)(dl + l_ko);
    int64_t tot[2] = {0, 0};
    first[0] = -1; first[1] = 0; first[2] = 0;
    size_pass(P);
#ifndef C2B_EMU
    c2b_vcf_scan_kernel<<<1, 32, 0, e->stream>>>(P.nrec, (int64_t *)P.rec_base, P.nbytes, (int64_t *)P.key_off, P.err,
                                                 (int64_t *)(dl + l_first), m);
    RTCHK(cudaGetLastError());
    RTCHK(rt_d2h(first, dl + l_first, 24, e->stream));
    RTCHK(rt_d2h(&tot[0], P.rec_base + m, 8, e->stream));
    RTCHK(rt_d2h(&tot[1], P.key_off + m, 8, e->stream));
    RTCHK(rt_sync(e->stream));
#else
    emu::run_warp([&]() {
        c2b::ann::scan_sizes(P.nrec, (int64_t *)P.rec_base, m);
        c2b::ann::scan_sizes(P.nbytes, (int64_t *)P.key_off, m);
        c2b::vcf::first_error(P.err, m, (int64_t *)(dl + l_first));
    });
    memcpy(first, dl + l_first, 24);
    tot[0] = P.rec_base[m]; tot[1] = P.key_off[m];
#endif
    if (first[0] >= 0) return 1;
    const size_t o_keys = 0, o_rpos = al((size_t)tot[1]), o_rw = o_rpos + al((size_t)tot[0] * 8), o_x = o_rw + al((size_t)tot[0] * 8),
                 out_end = o_x + extra;
    if ((rc = ensure(e, cp.d_out, out_end + 16))) return rc;
    char *dout = (char *)cp.d_out.p;
    P.keys = (uint8_t *)(dout + o_keys); P.rec_pos = (int64_t *)(dout + o_rpos); P.rec_w = (int64_t *)(dout + o_rw);
    write_pass(P, dout + o_x);
#ifndef C2B_EMU
    RTCHK(cudaGetLastError());
#endif
    const uint8_t *h;
    if ((rc = cp.download(out_end, &h))) return rc;
    const int64_t kb = (int64_t)S.keys.size();
    S.keys.insert(S.keys.end(), h + o_keys, h + o_keys + tot[1]);
    const int64_t *hp = (const int64_t *)(h + o_rpos), *hw = (const int64_t *)(h + o_rw);
    for (int64_t i = 0; i < tot[0]; i++) S.rec_pos.push_back(kb + hp[i]);
    S.rec_w.insert(S.rec_w.end(), hw, hw + tot[0]);
    if (extra_out) *extra_out = h + o_x;
    return C2B_OK;
}

// every offset array starts at 0 and does not decrease
static bool offsets_ok(const int64_t *const *offs, int n_offs, int64_t n_rows)
{
    for (int c = 0; c < n_offs; c++) {
        if (offs[c][0] != 0) return false;
        for (int64_t r = 0; r < n_rows; r++) if (offs[c][r + 1] < offs[c][r]) return false;
    }
    return true;
}

#ifndef C2B_EMU
static int row_grid(int64_t m) { return (int)std::min<int64_t>((m + 7) / 8, 8192); }
#endif

extern "C" {

// --vcf_output edit counts (c2b_vcf.cuh) for packed allele rows in chunks (ChunkPipe, record_chunk).  The records of all chunks
// are then summed on the host (c2b_vcf_sum_records).
int c2b_vcf_edit_counts(c2b_engine *e, int64_t n_rows, const int32_t *chrom, const int64_t *pos, const int64_t *reads,
                        const uint8_t *ref, const int64_t *ref_off, const uint8_t *aln, const int64_t *aln_off,
                        const int64_t *rp, const int64_t *rp_off, const int64_t *del, const int64_t *del_off,
                        const int64_t *ins, const int64_t *ins_off, const int64_t *isz, const int64_t *isz_off,
                        const int64_t *sub, const int64_t *sub_off, int64_t chunk, int64_t *err, c2b_vcf_counts **out)
{
    if (!e || !out || !err || n_rows < 0 || !ref_off || !aln_off || !rp_off || !del_off || !ins_off || !isz_off || !sub_off)
        return fail(e, C2B_E_ARG, "c2b_vcf_edit_counts: bad argument");
    *out = nullptr;
    err[0] = -1; err[1] = 0; err[2] = 0;
    const int64_t *offs[7] = {ref_off, aln_off, rp_off, del_off, ins_off, isz_off, sub_off};
    if (!offsets_ok(offs, 7, n_rows)) return fail(e, C2B_E_ARG, "c2b_vcf_edit_counts: offsets must start at 0 and not decrease");
    if (n_rows && (!chrom || !pos || !reads || (ref_off[n_rows] && !ref) || (aln_off[n_rows] && !aln) || (rp_off[n_rows] && !rp) ||
                   (del_off[n_rows] && !del) || (ins_off[n_rows] && !ins) || (isz_off[n_rows] && !isz) || (sub_off[n_rows] && !sub)))
        return fail(e, C2B_E_ARG, "c2b_vcf_edit_counts: row arrays missing");
    if (chunk <= 0) chunk = 1 << 14;
    const auto t0 = std::chrono::steady_clock::now();
    const RowCol cols[10] = {{chrom, nullptr, 4}, {pos, nullptr, 8}, {reads, nullptr, 8}, {ref, ref_off, 1}, {aln, aln_off, 1},
                             {rp, rp_off, 8}, {del, del_off, 16}, {ins, ins_off, 16}, {isz, isz_off, 8}, {sub, sub_off, 8}};
    RecordSink S;
    int rc = C2B_OK;
    {
        ChunkPipe cp(e);
        for (int64_t r0 = 0; !rc && r0 < n_rows; r0 += chunk) {
            const int64_t r1 = std::min(n_rows, r0 + chunk), m = r1 - r0;
            const char *d[10]; const int64_t *o[10];
            if ((rc = cp.upload(cols, 10, r0, r1, d, o))) break;
            c2b::vcf::VParams P;
            memset(&P, 0, sizeof P);
            P.n = m;
            P.chrom = (const int32_t *)d[0]; P.pos = (const int64_t *)d[1]; P.reads = (const int64_t *)d[2];
            P.ref = (const uint8_t *)d[3]; P.ref_off = o[3]; P.aln = (const uint8_t *)d[4]; P.aln_off = o[4];
            P.rp = (const int64_t *)d[5]; P.rp_off = o[5]; P.del = (const int64_t *)d[6]; P.del_off = o[6];
            P.ins = (const int64_t *)d[7]; P.ins_off = o[7]; P.isz = (const int64_t *)d[8]; P.isz_off = o[8];
            P.sub = (const int64_t *)d[9]; P.sub_off = o[9];
            auto size_pass = [&](const c2b::vcf::VParams &Q) {
#ifndef C2B_EMU
                c2b_vcf_size_kernel<<<row_grid(m), 256, 0, e->stream>>>(Q);
#else
                for (int64_t r = 0; r < m; r++) emu::run_warp([&]() { c2b::vcf::edits_one<false>(Q, r); });
#endif
            };
            auto write_pass = [&](const c2b::vcf::VParams &Q, char *) {
#ifndef C2B_EMU
                c2b_vcf_write_kernel<<<row_grid(m), 256, 0, e->stream>>>(Q);
#else
                for (int64_t r = 0; r < m; r++) emu::run_warp([&]() { c2b::vcf::edits_one<true>(Q, r); });
#endif
            };
            int64_t first[3];
            rc = record_chunk(e, cp, P, m, 0, size_pass, write_pass, S, first, nullptr);
            if (rc == 1) {
                static const char *what[5] = {"", "KeyError", "ValueError: value is not in list", "IndexError: string index out of range",
                                              "ValueError: max() iterable argument is empty"};
                err[0] = r0 + first[0]; err[1] = first[1]; err[2] = first[2];
                char msg[160];
                snprintf(msg, sizeof msg, "c2b_vcf_edit_counts: row %lld raises %s (value %lld)", (long long)err[0],
                         what[first[1] >= 1 && first[1] <= 4 ? first[1] : 0], (long long)err[2]);
                rc = fail(e, C2B_E_ARG, msg);
            }
        }
    }
    if (rc) return rc;
    const auto t1 = std::chrono::steady_clock::now();
    S.rec_pos.push_back((int64_t)S.keys.size());
    std::unique_ptr<c2b_vcf_counts> V(new c2b_vcf_counts());
    if (!c2b_vcf_sum_records(S.keys.data(), S.rec_pos.data(), S.rec_w.data(), (int64_t)S.rec_w.size(), V.get()))
        return fail(e, C2B_E_LIMIT, "c2b_vcf_edit_counts: a summed #Reads leaves int64");
    const auto t2 = std::chrono::steady_clock::now();
    V->device_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    V->sum_ms = std::chrono::duration<double, std::milli>(t2 - t1).count();
    *out = V.release();
    return C2B_OK;
}

void c2b_vcf_free(c2b_vcf_counts *v) { delete v; }
int64_t c2b_vcf_n(const c2b_vcf_counts *v) { return v ? (int64_t)v->reads.size() : 0; }
const uint8_t *c2b_vcf_keys(const c2b_vcf_counts *v) { return v ? v->keys.get() : nullptr; }
const int64_t *c2b_vcf_key_offsets(const c2b_vcf_counts *v) { return v ? v->key_off.data() : nullptr; }
const int64_t *c2b_vcf_reads(const c2b_vcf_counts *v) { return v ? v->reads.data() : nullptr; }
int64_t c2b_vcf_n_records(const c2b_vcf_counts *v) { return v ? v->n_records : 0; }
int c2b_vcf_timings(const c2b_vcf_counts *v, double *device_ms, double *sum_ms)
{
    if (!v || !device_ms || !sum_ms) return C2B_E_ARG;
    *device_ms = v->device_ms; *sum_ms = v->sum_ms;
    return C2B_OK;
}

}  // extern "C"

// --base_editor_output upset counts: the summed keys (tag byte | key text, c2b_base_edit.cuh) and the totals of
// c2b_be_upset_totals
struct c2b_be_upset {
    c2b_vcf_counts keys;
    std::vector<int64_t> totals;
};

// --base_editor_output quilt table: the projections of all rows (arena), Reference_Sequence projections (nuc repeated) and the
// sorted groups, whose strings point into them
struct c2b_be_quilt {
    std::vector<uint8_t> arena, nucs;
    std::vector<c2b_cut_group> groups;
    double device_ms = 0, group_ms = 0;
};

extern "C" {

// get_upset_plot_counts (c2b_base_edit.cuh) for packed allele rows in chunks (ChunkPipe, record_chunk); the records are summed on
// the host (c2b_vcf_sum_records), the category codes give the per-position counts and the totals.
int c2b_be_upset_counts(c2b_engine *e, int64_t n_rows, const uint8_t *flags, const int64_t *reads, const uint8_t *ref,
                        const int64_t *ref_off, const uint8_t *aln, const int64_t *aln_off, int32_t n_targets, const int64_t *tpos,
                        const uint8_t *tstr, const int64_t *toff, int64_t chunk, int64_t *err, c2b_be_upset **out)
{
    if (!e || !out || !err || n_rows < 0 || !ref_off || !aln_off || n_targets < 0 || (n_targets && (!tpos || !toff)))
        return fail(e, C2B_E_ARG, "c2b_be_upset_counts: bad argument");
    *out = nullptr;
    err[0] = -1; err[1] = 0;
    const int64_t *offs[2] = {ref_off, aln_off};
    if (!offsets_ok(offs, 2, n_rows)) return fail(e, C2B_E_ARG, "c2b_be_upset_counts: offsets must start at 0 and not decrease");
    if (n_rows && (!flags || !reads || (ref_off[n_rows] && !ref) || (aln_off[n_rows] && !aln)))
        return fail(e, C2B_E_ARG, "c2b_be_upset_counts: row arrays missing");
    const int nt = n_targets;
    const int64_t ts = nt ? toff[2 * nt] : 0;
    if (nt && (toff[0] != 0 || (ts && !tstr))) return fail(e, C2B_E_ARG, "c2b_be_upset_counts: target strings missing");
    for (int k = 0; k < 2 * nt; k++) if (toff[k + 1] < toff[k]) return fail(e, C2B_E_ARG, "c2b_be_upset_counts: target offsets decrease");
    if (chunk <= 0) chunk = 1 << 14;
    const auto t0 = std::chrono::steady_clock::now();
    const RowCol cols[4] = {{flags, nullptr, 1}, {reads, nullptr, 8}, {ref, ref_off, 1}, {aln, aln_off, 1}};
    // targets: positions (nt) | offsets (2 nt + 1) | strings
    std::vector<uint8_t> fixed((size_t)(8 * nt + 8 * (2 * nt + 1) + ts));
    if (nt) {
        memcpy(fixed.data(), tpos, (size_t)nt * 8);
        memcpy(fixed.data() + 8 * nt, toff, (size_t)(2 * nt + 1) * 8);
        if (ts) memcpy(fixed.data() + 8 * nt + 8 * (2 * nt + 1), tstr, (size_t)ts);
    }
    RecordSink S;
    std::vector<uint8_t> codes((size_t)n_rows * nt);
    int rc = C2B_OK;
    {
        ChunkPipe cp(e);
        const char *df = nullptr;
        rc = cp.fixed(fixed.data(), fixed.size(), &df);
        for (int64_t r0 = 0; !rc && r0 < n_rows; r0 += chunk) {
            const int64_t r1 = std::min(n_rows, r0 + chunk), m = r1 - r0;
            const char *d[4]; const int64_t *o[4];
            if ((rc = cp.upload(cols, 4, r0, r1, d, o))) break;
            c2b::be::UParams P;
            memset(&P, 0, sizeof P);
            P.n = m; P.flags = (const uint8_t *)d[0]; P.reads = (const int64_t *)d[1];
            P.ref = (const uint8_t *)d[2]; P.ref_off = o[2]; P.aln = (const uint8_t *)d[3]; P.aln_off = o[3];
            P.nt = nt; P.tpos = (const int64_t *)df; P.toff = (const int64_t *)(df + 8 * nt);
            P.tstr = (const uint8_t *)(df + 8 * nt + 8 * (2 * nt + 1));
            auto size_pass = [&](const c2b::be::UParams &Q) {
#ifndef C2B_EMU
                c2b_be_upset_size_kernel<<<row_grid(m), 256, 0, e->stream>>>(Q);
#else
                for (int64_t r = 0; r < m; r++) emu::run_warp([&]() { c2b::be::upset_one<false>(Q, r); });
#endif
            };
            auto write_pass = [&](c2b::be::UParams &Q, char *x) {
                Q.codes = (uint8_t *)x;
#ifndef C2B_EMU
                c2b_be_upset_write_kernel<<<row_grid(m), 256, 0, e->stream>>>(Q);
#else
                for (int64_t r = 0; r < m; r++) emu::run_warp([&]() { c2b::be::upset_one<true>(Q, r); });
#endif
            };
            int64_t first[3];
            const uint8_t *hc = nullptr;
            rc = record_chunk(e, cp, P, m, (size_t)m * nt, size_pass, write_pass, S, first, &hc);
            if (rc == 1) {
                err[0] = r0 + first[0]; err[1] = first[1];
                char msg[160];
                snprintf(msg, sizeof msg, "c2b_be_upset_counts: row %lld raises IndexError: string index out of range", (long long)err[0]);
                rc = fail(e, C2B_E_ARG, msg);
            } else if (!rc && m * nt) {
                memcpy(codes.data() + (size_t)r0 * nt, hc, (size_t)(m * nt));
            }
        }
    }
    if (rc) return rc;
    const auto t1 = std::chrono::steady_clock::now();
    std::unique_ptr<c2b_be_upset> U(new c2b_be_upset());
    S.rec_pos.push_back((int64_t)S.keys.size());
    bool ok = c2b_vcf_sum_records(S.keys.data(), S.rec_pos.data(), S.rec_w.data(), (int64_t)S.rec_w.size(), &U->keys);
    // totals (C2B_BE_T_*), then per category (C2B_BE_CAT_*) the #Reads of every target position
    std::vector<int64_t> &T = U->totals;
    T.assign((size_t)(10 + 5 * nt), 0);
    int64_t *pc = T.data() + 10;
    auto add = [&](int64_t &a, int64_t b) { if (__builtin_add_overflow(a, b, &a)) ok = false; };
    T[0] = n_rows;
    for (int64_t r = 0; r < n_rows; r++) {
        const int64_t w = reads[r];
        add(T[1], w);
        if (!(flags[r] & 1)) continue;
        T[2]++;
        add(T[3], w);
        const uint8_t *c = codes.data() + (size_t)r * nt;
        bool all_r = true, all_t = true;
        for (int t = 0; t < nt; t++) {
            add(pc[(size_t)c[t] * nt + t], w);
            all_r = all_r && c[t] == c2b::be::CAT_R;
            all_t = all_t && c[t] == c2b::be::CAT_T;
        }
        add(T[4 + 2 * (all_r ? 0 : all_t ? 1 : 2) + ((flags[r] & 2) ? 1 : 0)], w);
    }
    if (!ok) return fail(e, C2B_E_LIMIT, "c2b_be_upset_counts: a summed #Reads leaves int64");
    const auto t2 = std::chrono::steady_clock::now();
    U->keys.device_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    U->keys.sum_ms = std::chrono::duration<double, std::milli>(t2 - t1).count();
    *out = U.release();
    return C2B_OK;
}

void c2b_be_upset_free(c2b_be_upset *u) { delete u; }
int64_t c2b_be_upset_n(const c2b_be_upset *u) { return u ? (int64_t)u->keys.reads.size() : 0; }
const uint8_t *c2b_be_upset_keys(const c2b_be_upset *u) { return u ? u->keys.keys.get() : nullptr; }
const int64_t *c2b_be_upset_key_offsets(const c2b_be_upset *u) { return u ? u->keys.key_off.data() : nullptr; }
const int64_t *c2b_be_upset_reads(const c2b_be_upset *u) { return u ? u->keys.reads.data() : nullptr; }
const int64_t *c2b_be_upset_totals(const c2b_be_upset *u) { return u ? u->totals.data() : nullptr; }
int c2b_be_upset_timings(const c2b_be_upset *u, double *device_ms, double *sum_ms)
{
    if (!u || !device_ms || !sum_ms) return C2B_E_ARG;
    *device_ms = u->keys.device_ms; *sum_ms = u->keys.sum_ms;
    return C2B_OK;
}

// get_base_edit_dataframe_around_cut (c2b_base_edit.cuh) for packed allele rows in chunks (ChunkPipe): one pass writes each
// row's projection at its Reference_Sequence offset, its length and its error; the projections are then grouped and sorted on
// the host (c2b_group_around_cut).
int c2b_be_quilt_table(c2b_engine *e, int64_t n_rows, int32_t nuc, const uint8_t *ref, const int64_t *ref_off, const uint8_t *aln,
                 const int64_t *aln_off, const uint8_t *unedited, const int64_t *n_deleted, const int64_t *n_inserted,
                 const int64_t *n_mutated, const int64_t *reads, const double *pct, int64_t chunk, int64_t *err, c2b_be_quilt **out)
{
    if (!e || !out || !err || n_rows < 0 || !ref_off || !aln_off || nuc > 255) return fail(e, C2B_E_ARG, "c2b_be_quilt_table: bad argument");
    *out = nullptr;
    err[0] = -1;
    const int64_t *offs[2] = {ref_off, aln_off};
    if (!offsets_ok(offs, 2, n_rows)) return fail(e, C2B_E_ARG, "c2b_be_quilt_table: offsets must start at 0 and not decrease");
    if (n_rows && (!unedited || !n_deleted || !n_inserted || !n_mutated || !reads || !pct || (ref_off[n_rows] && !ref) ||
                   (aln_off[n_rows] && !aln)))
        return fail(e, C2B_E_ARG, "c2b_be_quilt_table: row arrays missing");
    if (chunk <= 0) chunk = 1 << 14;
    const auto t0 = std::chrono::steady_clock::now();
    const RowCol cols[2] = {{ref, ref_off, 1}, {aln, aln_off, 1}};
    std::unique_ptr<c2b_be_quilt> Q(new c2b_be_quilt());
    std::vector<int64_t> plen((size_t)n_rows), pstart((size_t)n_rows);
    int rc = C2B_OK;
    {
        ChunkPipe cp(e);
        auto al = ChunkPipe::al;
        for (int64_t r0 = 0; !rc && r0 < n_rows; r0 += chunk) {
            const int64_t r1 = std::min(n_rows, r0 + chunk), m = r1 - r0, rb = ref_off[r1] - ref_off[r0];
            const char *d[2]; const int64_t *o[2];
            if ((rc = cp.upload(cols, 2, r0, r1, d, o))) break;
            // out: projections (at the chunk's Reference_Sequence offsets) | len (m) | err (m)
            const size_t o_len = al((size_t)rb), o_err = o_len + al((size_t)m * 8), o_end = o_err + (size_t)m * 8;
            if ((rc = ensure(e, cp.d_out, o_end + 16))) break;
            char *dout = (char *)cp.d_out.p;
            c2b::be::QParams P;
            memset(&P, 0, sizeof P);
            P.n = m; P.nuc = nuc; P.ref = (const uint8_t *)d[0]; P.ref_off = o[0]; P.aln = (const uint8_t *)d[1]; P.aln_off = o[1];
            P.out = (uint8_t *)dout; P.len = (int64_t *)(dout + o_len); P.err = (int64_t *)(dout + o_err);
#ifndef C2B_EMU
            c2b_be_quilt_kernel<<<row_grid(m), 256, 0, e->stream>>>(P);
            if (cudaGetLastError() != cudaSuccess) { rc = fail(e, C2B_E_CUDA, "c2b_be_quilt_table: launch failed"); break; }
#else
            for (int64_t r = 0; r < m; r++) emu::run_warp([&]() { c2b::be::quilt_one(P, r); });
#endif
            const uint8_t *h;
            if ((rc = cp.download(o_end, &h))) break;
            const int64_t *hl = (const int64_t *)(h + o_len), *he = (const int64_t *)(h + o_err);
            for (int64_t r = 0; r < m; r++)
                if (he[r]) {
                    err[0] = r0 + r;
                    char msg[160];
                    snprintf(msg, sizeof msg, "c2b_be_quilt_table: row %lld raises IndexError: string index out of range", (long long)err[0]);
                    rc = fail(e, C2B_E_ARG, msg);
                    break;
                }
            if (rc) break;
            for (int64_t r = 0; r < m; r++) {
                const int64_t s = ref_off[r0 + r] - ref_off[r0];
                pstart[(size_t)(r0 + r)] = (int64_t)Q->arena.size();
                plen[(size_t)(r0 + r)] = hl[r];
                Q->arena.insert(Q->arena.end(), h + s, h + s + hl[r]);
            }
        }
    }
    if (rc) return rc;
    const auto t1 = std::chrono::steady_clock::now();
    int64_t longest = 0;
    for (int64_t r = 0; r < n_rows; r++) longest = std::max(longest, plen[(size_t)r]);
    Q->nucs.assign((size_t)longest + 1, (uint8_t)(nuc < 0 ? 0 : nuc));
    std::vector<c2b_cut_group> rows((size_t)n_rows);
    for (int64_t r = 0; r < n_rows; r++) {
        c2b_cut_group &G = rows[(size_t)r];
        G.seq = Q->arena.data() + pstart[(size_t)r]; G.ref = Q->nucs.data(); G.len = plen[(size_t)r];
        G.unedited = unedited[r] ? 1 : 0; G.ndel = n_deleted[r]; G.nins = n_inserted[r]; G.nmut = n_mutated[r];
        G.reads = reads[r]; G.pct = pct[r];
    }
    Q->groups = c2b_group_around_cut(rows);
    const auto t2 = std::chrono::steady_clock::now();
    Q->device_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    Q->group_ms = std::chrono::duration<double, std::milli>(t2 - t1).count();
    *out = Q.release();
    return C2B_OK;
}

void c2b_be_quilt_free(c2b_be_quilt *q) { delete q; }
int64_t c2b_be_quilt_n(const c2b_be_quilt *q) { return q ? (int64_t)q->groups.size() : 0; }
int64_t c2b_be_quilt_bytes(const c2b_be_quilt *q)
{
    int64_t n = 0;
    if (q) for (const c2b_cut_group &G : q->groups) n += G.len;
    return n;
}
int c2b_be_quilt_fetch(const c2b_be_quilt *q, uint8_t *seq, int64_t *seq_off, uint8_t *unedited, int64_t *n_deleted, int64_t *n_inserted,
                       int64_t *n_mutated, int64_t *reads, double *pct)
{
    if (!q || !seq_off || !unedited || !n_deleted || !n_inserted || !n_mutated || !reads || !pct) return C2B_E_ARG;
    int64_t o = 0;
    seq_off[0] = 0;
    for (size_t g = 0; g < q->groups.size(); g++) {
        const c2b_cut_group &G = q->groups[g];
        if (G.len) { if (!seq) return C2B_E_ARG; memcpy(seq + o, G.seq, (size_t)G.len); }
        o += G.len; seq_off[g + 1] = o;
        unedited[g] = G.unedited; n_deleted[g] = G.ndel; n_inserted[g] = G.nins; n_mutated[g] = G.nmut; reads[g] = G.reads; pct[g] = G.pct;
    }
    return C2B_OK;
}
int c2b_be_quilt_timings(const c2b_be_quilt *q, double *device_ms, double *group_ms)
{
    if (!q || !device_ms || !group_ms) return C2B_E_ARG;
    *device_ms = q->device_ms; *group_ms = q->group_ms;
    return C2B_OK;
}

}  // extern "C"

// ----------------------------------------------------------------------------------------- protein alignment
// The reference protein's tables in the layout of c2b_configure (RefDev: prof [nq][Ipad] = 4 * score, cIe, g4), uploaded to
// e->pro_tab.  `rows` is [nq][I] = matrix[ord(ref[i])][ord(alphabet[q])].
static int protein_ref(c2b_engine *e, const char *who, int I, int nq, const int64_t *rows, const int64_t *gi, int gap_extend, RefDev &d,
                       RefHost &h)
{
    const int nrb = (I + 255) / 256, Ipad = nrb * 256;
    memset(&d, 0, sizeof d);
    d.I = I; d.nrb = nrb; d.Ipad = Ipad; d.kstar = (I - 1) & 7; d.lstar = ((I - 1) >> 3) & 31;
    d.gi0_4 = (int32_t)(4 * gi[0]);
    const int64_t lim = (1ll << 27);
    h.sabs = h.gabs = h.gsum_abs = 0; h.gi0_abs = std::abs(gi[0]);
    for (size_t k = 0; k < (size_t)nq * I; k++) {
        if (rows[k] > lim || rows[k] < -lim) return fail(e, C2B_E_LIMIT, std::string(who) + ": substitution score out of range");
        h.sabs = std::max<int64_t>(h.sabs, std::abs(rows[k]));
    }
    for (int i = 0; i <= I; i++) {
        if (gi[i] > lim || gi[i] < -lim) return fail(e, C2B_E_LIMIT, std::string(who) + ": gap incentive out of range");
        h.gabs = std::max<int64_t>(h.gabs, std::abs(gi[i])); h.gsum_abs += std::abs(gi[i]);
    }
    std::vector<int32_t> blob((size_t)(nq + 2) * Ipad, 0);
    int32_t *prof = blob.data(), *cIe = prof + (size_t)nq * Ipad, *g4 = cIe + Ipad;
    for (int q = 0; q < nq; q++)
        for (int i = 0; i < I; i++) prof[(size_t)q * Ipad + i] = (int32_t)(4 * rows[(size_t)q * I + i]);
    for (int i = 0; i < I; i++) { cIe[i] = (int32_t)(4 * (gap_extend + gi[i + 1])); g4[i] = (int32_t)(4 * gi[i]); }
    int rc;
    if ((rc = ensure(e, e->pro_tab, blob.size() * 4))) return rc;
    RTCHK(rt_h2d(e->pro_tab.p, blob.data(), blob.size() * 4, e->stream));
    const int32_t *dp = (const int32_t *)e->pro_tab.p;
    d.prof = dp; d.cIe = dp + (size_t)nq * Ipad; d.g4 = d.cIe + Ipad;
    return C2B_OK;
}

// global_align of n reads (alphabet codes codes[off[r] .. off[r+1])) against one reference protein: ops [n][32] (column k from
// the right: bits 2 (k & 31) of word k >> 5), nops[n] = alignment columns.  Limits first, nothing launched past one.
static int protein_batch(c2b_engine *e, const char *who, int I, int nq, const int64_t *rows, const int64_t *gi, int go, int ge,
                         const uint8_t *codes, const int64_t *off, int64_t n, uint64_t *ops, int32_t *nops, int64_t *bad = nullptr)
{
    if (I < 1 || I > C2B_MAX_REF_LEN) return fail(e, C2B_E_LIMIT, std::string(who) + ": reference empty or longer than C2B_MAX_REF_LEN");
    if (nq < 1 || nq > C2B_AA_MAX_Q) return fail(e, C2B_E_LIMIT, std::string(who) + ": alphabet larger than C2B_AA_MAX_Q");
    int64_t maxJ = 0;
    for (int64_t r = 0; r < n; r++) {
        const int64_t J = off[r + 1] - off[r];
        if (J < 1 || J > C2B_MAX_READ_LEN || I + J > C2B_MAX_ALN_LEN)
            return fail(e, C2B_E_LIMIT, std::string(who) + ": read " + std::to_string(r) + " empty or beyond C2B_MAX_READ_LEN / C2B_MAX_ALN_LEN");
        maxJ = std::max(maxJ, J);
    }
    for (int64_t k = 0; k < off[n]; k++)
        if (codes[k] >= nq) return fail(e, C2B_E_ARG, std::string(who) + ": read symbol outside the alphabet");
    RefDev d; RefHost h;
    int rc;
    if ((rc = protein_ref(e, who, I, nq, rows, gi, ge, d, h))) return rc;
    if (!score_fits(go, ge, I, maxJ, h))
        return fail(e, C2B_E_LIMIT, std::string(who) + ": scores, gap penalties and incentives can exceed the int32 range of the DP");
    if (n == 0) return C2B_OK;
    const int TS = (int)((maxJ + 32 + 31) & ~31);
    const int64_t nw = std::min<int64_t>(n, std::max(e->n_warps, 1));
    aa::PParams P;
    memset(&P, 0, sizeof P);
    P.K.go = go; P.K.ge = ge; P.K.TS = TS;
    P.K.tb_words_per_warp = (int64_t)d.nrb * TS * 32; P.K.bnd_words_per_warp = 2 * 3 * (int64_t)TS;
    if ((rc = ensure(e, e->pro_tb, (size_t)(nw * P.K.tb_words_per_warp * 4)))) return rc;
    if ((rc = ensure(e, e->pro_bnd, (size_t)(nw * P.K.bnd_words_per_warp * 4)))) return rc;
    const size_t o_off = ChunkPipe::al((size_t)off[n]), in_end = o_off + (size_t)(n + 1) * 8;
    const size_t o_n = (size_t)n * 32 * 8, out_end = o_n + (size_t)n * 4;
    if ((rc = ensure(e, e->pro_in, in_end))) return rc;
    if ((rc = ensure(e, e->pro_out, out_end))) return rc;
    RTCHK(rt_h2d(e->pro_in.p, codes, (size_t)off[n], e->stream));
    RTCHK(rt_h2d((char *)e->pro_in.p + o_off, off, (size_t)(n + 1) * 8, e->stream));
    P.K.tb = (uint32_t *)e->pro_tb.p; P.K.bnd = (int32_t *)e->pro_bnd.p;
    P.R = d;
    P.codes = (const uint8_t *)e->pro_in.p; P.off = (const int64_t *)((const char *)e->pro_in.p + o_off); P.n = n;
    P.ops = (uint64_t *)e->pro_out.p; P.nops = (int32_t *)((char *)e->pro_out.p + o_n);
#ifndef C2B_EMU
    c2b_protein_kernel<<<(int)((nw + 7) / 8), 256, 0, e->stream>>>(P);
    RTCHK(cudaGetLastError());
#else
    for (int64_t r = 0; r < n; r++) emu::run_warp([&]() { aa::protein_one(P, r, 0); });
#endif
    RTCHK(rt_d2h(ops, P.ops, o_n, e->stream));
    RTCHK(rt_d2h(nops, P.nops, (size_t)n * 4, e->stream));
    RTCHK(rt_sync(e->stream));
    for (int64_t r = 0; r < n; r++)
        if (nops[r] < 0) {
            if (bad) *bad = r;
            return fail(e, C2B_E_STATE, std::string(who) + ": the traceback of read " + std::to_string(r) +
                                            " leaves the zone where global_align is defined (SURVEY 3.2)");
        }
    return C2B_OK;
}

// the aligned strings of one op stream (right to left), written left-justified to out_read / out_ref -> matched columns
static int32_t spell_ops(const uint64_t *ops, int32_t n, const uint8_t *read, int64_t J, const uint8_t *ref, int64_t I, uint8_t *out_read,
                         uint8_t *out_ref)
{
    int64_t j = J, i = I;
    int32_t m = 0;
    for (int32_t k = 0, c = n - 1; k < n; k++, c--) {
        const int op = (int)((ops[k >> 5] >> (2 * (k & 31))) & 3u);
        const uint8_t a = op == OP_J ? '-' : read[--j], b = op == OP_I ? '-' : ref[--i];
        out_read[c] = a; out_ref[c] = b;
        m += op == OP_M && a == b;
    }
    return m;
}

// --coding_seq amino-acid table: every row's aligned strings (arena) and the sorted groups, whose strings point into it
struct c2b_amino {
    std::vector<uint8_t> arena;
    std::vector<c2b_cut_group> groups;
    std::vector<int64_t> ref_len;                              // per row: residues of the reference protein
    int64_t n_pairs = 0;
    double row_ms = 0, align_ms = 0, group_ms = 0;
};

// the standard genetic code, codon index 16 a + 4 b + c over A C G T (CRISPRessoShared.CODON_TO_AMINO_ACID_SINGLE_CHAR)
static const char AA_TABLE[65] = "KNKNTTTTRSRSIIMIQHQHPPPPRRRRLLLLEDEDAAAAGGGGVVVV*Y*YSSSS*CWCLFLF";

extern "C" {

int c2b_protein_align(c2b_engine *e, const char *ref, int32_t ref_len, const char *reads, const int64_t *offsets, int64_t n,
                      const char *alphabet, int32_t nq, const int64_t *score_rows, const int64_t *gap_incentive, int32_t gap_open,
                      int32_t gap_extend, uint64_t *ops, int32_t *aln_len, int32_t *n_match)
{
    if (!e || !ref || !offsets || n < 0 || !alphabet || !score_rows || !gap_incentive || (n && (!ops || !aln_len || !n_match)) ||
        (n && offsets[n] && !reads))
        return fail(e, C2B_E_ARG, "c2b_protein_align: bad argument");
    const int64_t *offs[1] = {offsets};
    if (!offsets_ok(offs, 1, n)) return fail(e, C2B_E_ARG, "c2b_protein_align: offsets must start at 0 and not decrease");
    if (nq < 1 || nq > C2B_AA_MAX_Q) return fail(e, C2B_E_LIMIT, "c2b_protein_align: alphabet larger than C2B_AA_MAX_Q");
    uint8_t lut[256];
    memset(lut, 255, sizeof lut);
    for (int q = 0; q < nq; q++) lut[(uint8_t)alphabet[q]] = (uint8_t)q;
    std::vector<uint8_t> codes((size_t)offsets[n]);
    for (int64_t k = 0; k < offsets[n]; k++) codes[(size_t)k] = lut[(uint8_t)reads[k]];
    int rc = protein_batch(e, "c2b_protein_align", ref_len, nq, score_rows, gap_incentive, gap_open, gap_extend, codes.data(), offsets, n,
                           ops, aln_len);
    if (rc) return rc;
    std::vector<uint8_t> a((size_t)C2B_MAX_ALN_LEN), b((size_t)C2B_MAX_ALN_LEN);
    for (int64_t r = 0; r < n; r++)
        n_match[r] = spell_ops(ops + r * 32, aln_len[r], (const uint8_t *)reads + offsets[r], offsets[r + 1] - offsets[r],
                               (const uint8_t *)ref, ref_len, a.data(), b.data());
    return C2B_OK;
}

// get_amino_acid_dataframe over packed allele rows: the row pass in chunks (ChunkPipe, c2b_amino.cuh), one global_align per
// distinct (read protein, reference protein) pair (c2b_vcf_sum_records' exact hash; one protein_batch per reference protein),
// silent edits and truncation per row on host threads, then c2b_group_around_cut.
int c2b_amino_table(c2b_engine *e, int64_t n_rows, int64_t plot_left_idx, const uint8_t *ref, const int64_t *ref_off, const uint8_t *aln,
                    const int64_t *aln_off, const int64_t *rp, const int64_t *rp_off, const int64_t *matrix, int32_t msize,
                    int64_t cut_point, int64_t seq_len, const uint8_t *unedited, const int64_t *n_deleted, const int64_t *n_inserted,
                    const int64_t *n_mutated, const int64_t *reads, const double *pct, int64_t chunk, int64_t *err, c2b_amino **out)
{
    if (!e || !out || !err || n_rows < 0 || !ref_off || !aln_off || !rp_off || !matrix || msize < 1)
        return fail(e, C2B_E_ARG, "c2b_amino_table: bad argument");
    *out = nullptr;
    err[0] = -1; err[1] = 0;
    const int64_t *offs[3] = {ref_off, aln_off, rp_off};
    if (!offsets_ok(offs, 3, n_rows)) return fail(e, C2B_E_ARG, "c2b_amino_table: offsets must start at 0 and not decrease");
    if (n_rows && (!unedited || !n_deleted || !n_inserted || !n_mutated || !reads || !pct || (ref_off[n_rows] && !ref) ||
                   (aln_off[n_rows] && !aln) || (rp_off[n_rows] && !rp)))
        return fail(e, C2B_E_ARG, "c2b_amino_table: row arrays missing");
    if (chunk <= 0) chunk = 1 << 14;
    const auto t0 = std::chrono::steady_clock::now();
    std::unique_ptr<c2b_amino> A(new c2b_amino());
    A->ref_len.assign((size_t)n_rows, 0);
    // per row: key = read protein | 0 | reference protein, and at the same offsets the codon indices
    std::vector<uint8_t> key, cod;
    std::vector<int64_t> koff(1, 0), na((size_t)n_rows);
    const RowCol cols[3] = {{ref, ref_off, 1}, {aln, aln_off, 1}, {rp, rp_off, 8}};
    int rc = C2B_OK;
    {
        ChunkPipe cp(e);
        auto al = ChunkPipe::al;
        const char *dt = nullptr;
        rc = cp.fixed(AA_TABLE, 64, &dt);
        for (int64_t r0 = 0; !rc && r0 < n_rows; r0 += chunk) {
            const int64_t r1 = std::min(n_rows, r0 + chunk), m = r1 - r0;
            const int64_t ab = aln_off[r1] - aln_off[r0], fb = ref_off[r1] - ref_off[r0];
            const char *d[3]; const int64_t *o[3];
            if ((rc = cp.upload(cols, 3, r0, r1, d, o))) break;
            // out: read protein | read codons (at aln offsets) | reference protein | reference codons (at ref offsets) | len | err
            const size_t o_rc = al((size_t)ab), o_fa = o_rc + al((size_t)ab), o_fc = o_fa + al((size_t)fb), o_len = o_fc + al((size_t)fb),
                         o_err = o_len + al((size_t)m * 16), o_end = o_err + (size_t)m * 8;
            if ((rc = ensure(e, cp.d_out, o_end + 16))) break;
            char *dout = (char *)cp.d_out.p;
            aa::RParams P;
            memset(&P, 0, sizeof P);
            P.n = m; P.left = plot_left_idx; P.table = (const uint8_t *)dt;
            P.ref = (const uint8_t *)d[0]; P.ref_off = o[0]; P.aln = (const uint8_t *)d[1]; P.aln_off = o[1];
            P.rp = (const int64_t *)d[2]; P.rp_off = o[2];
            P.raa = (uint8_t *)dout; P.rcod = (uint8_t *)dout + o_rc; P.faa = (uint8_t *)dout + o_fa; P.fcod = (uint8_t *)dout + o_fc;
            P.len = (int64_t *)(dout + o_len); P.err = (int64_t *)(dout + o_err);
#ifndef C2B_EMU
            c2b_amino_codons_kernel<<<row_grid(m), 256, 0, e->stream>>>(P);
            if (cudaGetLastError() != cudaSuccess) { rc = fail(e, C2B_E_CUDA, "c2b_amino_table: launch failed"); break; }
#else
            for (int64_t r = 0; r < m; r++) emu::run_warp([&]() { aa::codons_one(P, r); });
#endif
            const uint8_t *h;
            if ((rc = cp.download(o_end, &h))) break;
            const int64_t *hl = (const int64_t *)(h + o_len), *he = (const int64_t *)(h + o_err);
            for (int64_t r = 0; r < m && err[0] < 0; r++)
                if (he[r]) { err[0] = r0 + r; err[1] = he[r]; }
            if (err[0] >= 0) break;
            for (int64_t r = 0; r < m; r++) {
                const int64_t a0 = aln_off[r0 + r] - aln_off[r0], f0 = ref_off[r0 + r] - ref_off[r0], a = hl[2 * r], f = hl[2 * r + 1];
                na[(size_t)(r0 + r)] = a;
                A->ref_len[(size_t)(r0 + r)] = f;
                key.insert(key.end(), h + a0, h + a0 + a); key.push_back(0); key.insert(key.end(), h + o_fa + f0, h + o_fa + f0 + f);
                cod.insert(cod.end(), h + o_rc + a0, h + o_rc + a0 + a); cod.push_back(0);
                cod.insert(cod.end(), h + o_fc + f0, h + o_fc + f0 + f);
                koff.push_back((int64_t)key.size());
            }
        }
    }
    if (rc) return rc;
    if (err[0] >= 0) {
        static const char *what[4] = {"", "ValueError: plot_left_idx is not in ref_positions", "KeyError: a codon outside the table",
                                      "a translation shorter than one codon (global_align is undefined on an empty sequence)"};
        char msg[200];
        snprintf(msg, sizeof msg, "c2b_amino_table: row %lld raises %s", (long long)err[0], what[err[1] >= 1 && err[1] <= 3 ? err[1] : 0]);
        return fail(e, C2B_E_ARG, msg);
    }
    const auto t1 = std::chrono::steady_clock::now();
    // distinct pairs, first-seen order; one batch per distinct reference protein
    c2b_vcf_counts U;
    std::vector<int64_t> uix((size_t)n_rows);
    c2b_vcf_sum_records(key.data(), koff.data(), nullptr, n_rows, &U, uix.data());
    const int64_t nu = (int64_t)U.key_off.size() - 1;
    A->n_pairs = nu;
    const uint8_t *uk = U.keys.get();
    std::vector<int64_t> ualn_off((size_t)nu + 1, 0), ucols((size_t)nu);
    std::vector<uint8_t> ualn;                               // per pair: aligned read | aligned reference
    {
        std::vector<std::pair<std::string, std::vector<int64_t>>> by_ref;
        std::unordered_map<std::string, size_t> ref_at;
        std::vector<int64_t> sep((size_t)nu);
        for (int64_t u = 0; u < nu; u++) {
            const uint8_t *p = uk + U.key_off[(size_t)u];
            const int64_t len = U.key_off[(size_t)u + 1] - U.key_off[(size_t)u];
            sep[(size_t)u] = (int64_t)((const uint8_t *)memchr(p, 0, (size_t)len) - p);
            std::string f((const char *)p + sep[(size_t)u] + 1, (size_t)(len - sep[(size_t)u] - 1));
            auto it = ref_at.find(f);
            if (it == ref_at.end()) { it = ref_at.emplace(f, by_ref.size()).first; by_ref.push_back({f, {}}); }
            by_ref[it->second].second.push_back(u);
        }
        std::vector<std::vector<uint64_t>> uops((size_t)nu);
        std::vector<int32_t> un((size_t)nu);
        for (auto &br : by_ref) {
            const std::string &f = br.first;
            const std::vector<int64_t> &us = br.second;
            const int I = (int)std::min<size_t>(f.size(), (size_t)C2B_MAX_REF_LEN + 1);
            bool seen[256] = {false};
            for (int64_t u : us) for (int64_t x = 0; x < sep[(size_t)u]; x++) seen[uk[U.key_off[(size_t)u] + x]] = true;
            std::string alpha;
            for (int c = 0; c < 256; c++) if (seen[c]) alpha.push_back((char)c);
            const int nq = (int)alpha.size();
            if (nq > C2B_AA_MAX_Q) return fail(e, C2B_E_LIMIT, "c2b_amino_table: read alphabet larger than C2B_AA_MAX_Q");
            for (char c : alpha + f)
                if ((uint8_t)c >= (uint32_t)msize) return fail(e, C2B_E_ARG, "c2b_amino_table: amino acid outside the substitution matrix");
            std::vector<int64_t> rows((size_t)nq * I), gi((size_t)I + 1, 0);
            for (int q = 0; q < nq; q++)
                for (int i = 0; i < I; i++) rows[(size_t)q * I + i] = matrix[(size_t)(uint8_t)f[(size_t)i] * msize + (uint8_t)alpha[(size_t)q]];
            if (cut_point >= 0 && cut_point <= I) gi[(size_t)cut_point] = 1;
            uint8_t lut[256];
            for (int q = 0; q < nq; q++) lut[(uint8_t)alpha[(size_t)q]] = (uint8_t)q;
            std::vector<uint8_t> codes;
            std::vector<int64_t> off(1, 0);
            for (int64_t u : us) {
                for (int64_t x = 0; x < sep[(size_t)u]; x++) codes.push_back(lut[uk[U.key_off[(size_t)u] + x]]);
                off.push_back((int64_t)codes.size());
            }
            const int64_t nb = (int64_t)us.size();
            std::vector<uint64_t> ops((size_t)nb * 32);
            std::vector<int32_t> nops((size_t)nb);
            int64_t bad = -1;
            if ((rc = protein_batch(e, "c2b_amino_table", I, nq, rows.data(), gi.data(), -1, -1, codes.data(), off.data(), nb, ops.data(),
                                    nops.data(), &bad))) {
                if (bad < 0) return rc;
                for (int64_t r = 0; r < n_rows && err[0] < 0; r++) if (uix[(size_t)r] == us[(size_t)bad]) err[0] = r;
                err[1] = aa::E_UNDEFINED;
                return fail(e, C2B_E_ARG, "c2b_amino_table: row " + std::to_string(err[0]) +
                                              ": global_align's traceback leaves the zone where it is defined (SURVEY 3.2)");
            }
            for (int64_t k = 0; k < nb; k++) {
                uops[(size_t)us[(size_t)k]].assign(ops.begin() + k * 32, ops.begin() + k * 32 + 32);
                un[(size_t)us[(size_t)k]] = nops[(size_t)k];
            }
        }
        for (int64_t u = 0; u < nu; u++) { ucols[(size_t)u] = un[(size_t)u]; ualn_off[(size_t)u + 1] = ualn_off[(size_t)u] + 2 * un[(size_t)u]; }
        ualn.resize((size_t)ualn_off[(size_t)nu]);
        for (int64_t u = 0; u < nu; u++) {
            const uint8_t *p = uk + U.key_off[(size_t)u];
            const int64_t s = sep[(size_t)u], len = U.key_off[(size_t)u + 1] - U.key_off[(size_t)u];
            uint8_t *o = ualn.data() + ualn_off[(size_t)u];
            spell_ops(uops[(size_t)u].data(), un[(size_t)u], p, s, p + s + 1, len - s - 1, o, o + un[(size_t)u]);
        }
    }
    const auto t2 = std::chrono::steady_clock::now();
    // per row: get_silent_edits (a read residue equal to the reference's but from another codon is lower-cased), then
    // [:sequence_length] with Python's slice bounds
    std::vector<int64_t> roff((size_t)n_rows + 1, 0);
    auto cut_len = [&](int64_t n) { int64_t k = seq_len < 0 ? std::max<int64_t>(0, n + seq_len) : seq_len; return std::min(k, n); };
    for (int64_t r = 0; r < n_rows; r++) roff[(size_t)r + 1] = roff[(size_t)r] + 2 * cut_len(ucols[(size_t)uix[(size_t)r]]);
    A->arena.resize((size_t)roff[(size_t)n_rows] + 1);
    std::vector<c2b_cut_group> rows((size_t)n_rows);
    {
        const int T = (int)std::max<int64_t>(1, std::min<int64_t>({(int64_t)std::thread::hardware_concurrency(), 32, n_rows / 4096 + 1}));
        auto work = [&](int t) {
            for (int64_t r = n_rows * t / T; r < n_rows * (t + 1) / T; r++) {
                const int64_t u = uix[(size_t)r], n = ucols[(size_t)u], L = cut_len(n);
                const uint8_t *sa = ualn.data() + ualn_off[(size_t)u], *sb = sa + n;
                const uint8_t *rc_ = cod.data() + koff[(size_t)r], *fc = rc_ + na[(size_t)r] + 1;
                uint8_t *o = A->arena.data() + roff[(size_t)r];
                int64_t x = 0, y = 0;
                for (int64_t c = 0; c < n; c++) {
                    const bool ga = sa[c] == '-', gb = sb[c] == '-';
                    if (c < L) { o[c] = (!ga && !gb && sa[c] == sb[c] && rc_[x] != fc[y]) ? (uint8_t)tolower(sa[c]) : sa[c]; o[L + c] = sb[c]; }
                    x += !ga; y += !gb;
                }
                c2b_cut_group &G = rows[(size_t)r];
                G.seq = o; G.ref = o + L; G.len = L;
                G.unedited = unedited[r] ? 1 : 0; G.ndel = n_deleted[r]; G.nins = n_inserted[r]; G.nmut = n_mutated[r];
                G.reads = reads[r]; G.pct = pct[r];
            }
        };
        std::vector<std::thread> th;
        for (int t = 1; t < T; t++) th.emplace_back(work, t);
        work(0);
        for (auto &x : th) x.join();
    }
    A->groups = c2b_group_around_cut(rows);
    const auto t3 = std::chrono::steady_clock::now();
    A->row_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    A->align_ms = std::chrono::duration<double, std::milli>(t2 - t1).count();
    A->group_ms = std::chrono::duration<double, std::milli>(t3 - t2).count();
    *out = A.release();
    return C2B_OK;
}

void c2b_amino_free(c2b_amino *a) { delete a; }
int64_t c2b_amino_n(const c2b_amino *a) { return a ? (int64_t)a->groups.size() : 0; }
int64_t c2b_amino_bytes(const c2b_amino *a)
{
    int64_t n = 0;
    if (a) for (const c2b_cut_group &G : a->groups) n += G.len;
    return n;
}
const int64_t *c2b_amino_ref_lens(const c2b_amino *a) { return a && !a->ref_len.empty() ? a->ref_len.data() : nullptr; }
int c2b_amino_fetch(const c2b_amino *a, uint8_t *seq, uint8_t *ref, int64_t *seq_off, uint8_t *unedited, int64_t *n_deleted,
                    int64_t *n_inserted, int64_t *n_mutated, int64_t *reads, double *pct)
{
    if (!a || !seq_off || !unedited || !n_deleted || !n_inserted || !n_mutated || !reads || !pct) return C2B_E_ARG;
    int64_t o = 0;
    seq_off[0] = 0;
    for (size_t g = 0; g < a->groups.size(); g++) {
        const c2b_cut_group &G = a->groups[g];
        if (G.len) {
            if (!seq || !ref) return C2B_E_ARG;
            memcpy(seq + o, G.seq, (size_t)G.len); memcpy(ref + o, G.ref, (size_t)G.len);
        }
        o += G.len; seq_off[g + 1] = o;
        unedited[g] = G.unedited; n_deleted[g] = G.ndel; n_inserted[g] = G.nins; n_mutated[g] = G.nmut; reads[g] = G.reads; pct[g] = G.pct;
    }
    return C2B_OK;
}
int c2b_amino_timings(const c2b_amino *a, double *row_ms, double *align_ms, double *group_ms, int64_t *n_pairs)
{
    if (!a || !row_ms || !align_ms || !group_ms || !n_pairs) return C2B_E_ARG;
    *row_ms = a->row_ms; *align_ms = a->align_ms; *group_ms = a->group_ms; *n_pairs = a->n_pairs;
    return C2B_OK;
}

// pinned host memory for callers that want full-speed copies (bench.py, the Python wrapper)
void *c2b_host_alloc(size_t n)
{
#ifndef C2B_EMU
    void *p = nullptr;
    if (cudaHostAlloc(&p, n ? n : 16, cudaHostAllocDefault) != cudaSuccess) return nullptr;
    return p;
#else
    return malloc(n ? n : 16);
#endif
}
void c2b_host_free(void *p)
{
#ifndef C2B_EMU
    if (p) cudaFreeHost(p);
#else
    free(p);
#endif
}

}  // extern "C"

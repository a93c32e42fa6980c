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
#include <vector>

#include "c2b_core.cuh"
#include "c2b_split.cuh"
#include "c2b_annotate.cuh"
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
#ifndef C2B_EMU
#ifndef C2B_WARPS_PER_CTA
#define C2B_WARPS_PER_CTA 8
#endif
#ifndef C2B_MIN_CTAS_PER_SM
#define C2B_MIN_CTAS_PER_SM 2
#endif
constexpr int WARPS_PER_CTA = C2B_WARPS_PER_CTA;      // launch-bounds maximum; the launch may use fewer (env C2B_WARPS_PER_CTA)
#ifndef C2B_B_WARPS
#define C2B_B_WARPS 4
#endif
constexpr int B_WARPS_PER_CTA = C2B_B_WARPS;                    // CLASSIFY kernel
#ifndef C2B_B_MIN_CTAS
#define C2B_B_MIN_CTAS 6
#endif

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

// GENERAL kernel: the whole per-read path in one launch (any length within the build limits, any parameters; full-matrix
// DP paths of c2b_core.cuh).  Since r02 it runs after the ALIGN / CLASSIFY pair, over the pairs ALIGN left over (P.n_dev,
// P.pair_order = the left-over list), or alone when the two-kernel form does not apply.
// ONE: every read has one candidate reference (a single amplicon configured, or Pooled ref_id).
// P is a __grid_constant__: the out-of-line device functions take it by reference, and without the qualifier every launch
// copied the struct to each thread's local memory and read its fields back with LDL (slower).
template <bool ONE>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, C2B_MIN_CTAS_PER_SM) c2b_align_classify_kernel(const __grid_constant__ KParams P)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    WarpSmem *S = reinterpret_cast<WarpSmem *>(smem_raw) + (threadIdx.x >> 5);
    QuadSmem *Q = reinterpret_cast<QuadSmem *>(smem_raw + (size_t)(blockDim.x >> 5) * sizeof(WarpSmem)) + (threadIdx.x >> 5);
    const int warp_slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const uint32_t *staged_prof = stage_profile(P, smem_raw + (((size_t)(blockDim.x >> 5) * (sizeof(WarpSmem) + sizeof(QuadSmem)) + 127) & ~(size_t)127));
    // Work groups (8 reads each) are handed out per phase set (g consecutive warps, one group per warp), one hand-out
    // ahead, so that the loop count -- and with it the number of barriers executed by process_group's phases -- is the
    // same for every warp of the set, and the next group's read bytes are on their way to L2 while this one computes.
    __shared__ unsigned long long next_base[WARPS_PER_CTA];
    const int gs = P.phase_sync, g = gs > 0 ? gs : gs < 0 ? -gs : 1, wib = threadIdx.x >> 5, nsets = (int)(blockDim.x >> 5) / g;
    const int set = gs < 0 ? wib % nsets : wib / g, wis = gs < 0 ? wib / nsets : wib % g;
    const int64_t nrd = nreads(P);
    if (P.n_dev) {
        // over the ALIGN kernel's left-over list: one pair per hand-out (a warp that drew four hard pairs in a row was the
        // critical path of the whole launch)
        const unsigned total = (unsigned)((nrd + 1) / 2);
        for (;;) {
            unsigned w = 0;
            if ((threadIdx.x & 31) == 0) w = (unsigned)atomicAdd(P.work_counter, 1ull);
            w = __shfl_sync(0xffffffffu, w, 0);
            if (w >= total) break;
            process_item<ONE>(P, *S, staged_prof, (int64_t)w, warp_slot);
            __syncwarp();
        }
        return;
    }
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

// ALIGN kernel (c2b_split.cuh: align_group): persistent, free-running warps pull work groups of 8 reads from a counter.
#ifndef C2B_A_MIN_CTAS
#define C2B_A_MIN_CTAS 2
#endif
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, C2B_A_MIN_CTAS) c2b_align_kernel(const __grid_constant__ KParams P)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    ASmem *S = reinterpret_cast<ASmem *>(smem_raw) + (threadIdx.x >> 5);
    const int nw = blockDim.x >> 5;
    const int warp_slot = blockIdx.x * nw + (threadIdx.x >> 5);
    const uint32_t *staged_prof = stage_profile(P, smem_raw + (((size_t)nw * sizeof(ASmem) + 127) & ~(size_t)127));
    asmem_init(P, *S);
    const int64_t nrd = nreads(P);
    const unsigned ahead = gridDim.x * nw;
    if (P.left2) {
        // narrow first tier: work in units of sixteen reads; units it does not take run as two ordinary groups of eight
        const unsigned total = (unsigned)((nrd + 15) / 16);
        for (;;) {
            unsigned w = 0;
            if ((threadIdx.x & 31) == 0) w = (unsigned)atomicAdd(P.work_counter, 1ull);
            w = __shfl_sync(0xffffffffu, w, 0);
            if (w >= total) break;
            if (w + ahead < total) {                            // the unit this warp is likely to get next: bytes towards L2
                const int64_t g = (int64_t)w + ahead;
                const int64_t last = 16 * g + 16 < nrd ? 16 * g + 16 : nrd;
                const int64_t a = P.offsets[16 * g] + (int64_t)(threadIdx.x & 31) * 128;
                if (a < P.offsets[last]) asm volatile("prefetch.global.L2 [%0];" ::"l"(P.reads + a));
            }
            if (!align_narrow16(P, *S, staged_prof, (int64_t)w, warp_slot)) {
                align_group(P, *S, staged_prof, 2 * (int64_t)w, warp_slot);
                __syncwarp();
                if (8 * (2 * (int64_t)w + 1) < nrd) align_group(P, *S, staged_prof, 2 * (int64_t)w + 1, warp_slot);
            }
            __syncwarp();
        }
        return;
    }
    const unsigned total = (unsigned)((nrd + 7) / 8);
    for (;;) {
        unsigned w = 0;
        if ((threadIdx.x & 31) == 0) w = (unsigned)atomicAdd(P.work_counter, 1ull);
        w = __shfl_sync(0xffffffffu, w, 0);
        if (w >= total) break;
        if (w + ahead < total && !P.pair_order) {           // the group this warp is likely to get next: bytes towards L2
            const int64_t g = (int64_t)w + ahead;
            const int64_t last = 8 * g + 8 < nrd ? 8 * g + 8 : nrd;
            const int64_t a = P.offsets[8 * g] + (int64_t)(threadIdx.x & 31) * 128;
            if (a < P.offsets[last]) asm volatile("prefetch.global.L2 [%0];" ::"l"(P.reads + a));
        }
        align_group(P, *S, staged_prof, (int64_t)w, warp_slot);
        __syncwarp();
    }
}

// CLASSIFY kernel (c2b_split.cuh: classify_read): one aligned read per warp, reads strided over the grid.
template <bool ONE>
__global__ void __launch_bounds__(B_WARPS_PER_CTA * 32, C2B_B_MIN_CTAS) c2b_classify_kernel(const __grid_constant__ KParams P)
{
    __shared__ BSmem smem[B_WARPS_PER_CTA];
    BSmem &S = smem[threadIdx.x >> 5];
    const int64_t nw = (int64_t)gridDim.x * B_WARPS_PER_CTA;
    const int64_t total_bytes = P.offsets[P.n_reads];
    int64_t rd = (int64_t)blockIdx.x * B_WARPS_PER_CTA + (threadIdx.x >> 5);
    if (rd >= P.n_reads) return;
    ScAcc<ONE ? 1 : RG_MAX_REFS> acc;
    sc_init(acc);
    // two-deep input pipeline: stage A of read rd + 2 nw and stage B of read rd + nw are in flight while read rd is classified
    BPreA a1 = classify_pre_a(P, rd);
    BPre pre = classify_pre_b<ONE>(P, rd, a1, total_bytes);
    if (rd + nw < P.n_reads) a1 = classify_pre_a(P, rd + nw);
    while (rd < P.n_reads) {
        const BPre cur = pre;
        if (cur.go) classify_stage<ONE>(cur, S);
        __syncwarp();
        const int64_t nxt = rd + nw;
        if (nxt < P.n_reads) {
            pre = classify_pre_b<ONE>(P, nxt, a1, total_bytes);
            if (nxt + nw < P.n_reads) a1 = classify_pre_a(P, nxt + nw);
        }
        if (cur.go) classify_read<ONE>(P, rd, cur, S, acc);
        __syncwarp();
        rd = nxt;
    }
    sc_flush(acc, P);
}
#endif

// ----------------------------------------------------------------------------------------- engine
struct RefHost {
    std::string seq; std::vector<int64_t> gi, inc; double min_aln; std::vector<int64_t> rows;
    std::vector<std::string> fw, rc;
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
    DevBuf gops, gmeta, left, left2;   // device-pointer API: op streams / meta words / left-over list of the last launch
    int n_warps = 0, grid = 0, wpc = 8, stage_cap = 0;
    int grid_a = 0, grid_b = 0, stage_cap_a = 0;       // ALIGN / CLASSIFY kernels
    int split_ok = 0, split_all = 0;                   // configuration admits the two-kernel form (some / all references)
    int numa_node = -1;                                // NUMA node of the device (-1: unknown / single node)
    int scratch_TS = 0;
    // staging for the host-pointer API: two buffer sets, copy-in / compute / copy-out streams
    struct Stage { DevBuf reads, off, cnt, qw, rid, recs, alns, str, ed, maxlen, ord, gops, gmeta, left, left2; int32_t *h_ord = nullptr; size_t h_ord_cap = 0; int64_t *h_off = nullptr; size_t h_off_cap = 0;
                   // pinned bounce buffers for callers whose arrays are pageable (numpy): copies to / from them run on host
                   // threads while the other set's kernels and DMA are in flight
                   uint8_t *h_in = nullptr, *h_out = nullptr; size_t h_in_cap = 0, h_out_cap = 0;
                   int64_t d_c0 = 0, d_n = 0; size_t d_Wt = 0; bool drain = false;     // chunk waiting in h_out
                   rt_event in_done, k_done, out_done; bool used = false; } stage[2];
    rt_stream s_in = 0, s_out = 0, stream2 = 0;     // stream2: second compute stream, kernels of odd chunks
    rt_event fork_ev = 0;                           // orders stream2 after what is already queued on `stream`
    size_t set_tb = 0, set_tbb = 0, set_tbq = 0, set_bnd = 0, set_ops = 0, set_rgo = 0;   // bytes per scratch set (two sets: kernels of
                                                    // consecutive chunks overlap their tail / head on the two streams)
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
    if (r == cudaSuccess) r = cudaStreamCreateWithFlags(&e->stream2, cudaStreamNonBlocking);
    if (r == cudaSuccess) r = cudaEventCreateWithFlags(&e->fork_ev, cudaEventDisableTiming);
    if (r == cudaSuccess) r = cudaEventCreate(&e->ev0);
    if (r == cudaSuccess) r = cudaEventCreate(&e->ev1);
    int nsm = 0, occ = 0, smem_sm = 0, optin = 0;
    if (r == cudaSuccess) r = cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device);
    if (r == cudaSuccess) r = cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, device);
    if (r == cudaSuccess) r = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    // room for a TMA-staged reference tile next to C2B_MIN_CTAS_PER_SM CTAs of per-warp state (1 KB per CTA is reserved by the driver)
    // ... and the kernels' static shared memory (hand-out slots, mbarrier) -- if the sum is a byte too large the
    // occupancy query answers 1 CTA per SM and the persistent grid silently halves
    auto tile_room = [&](size_t per_warp, int ctas) {
        int cap = smem_sm / ctas - 1024 - (int)(per_warp * WARPS_PER_CTA) - 2048;
        const int fixed = (int)(per_warp * WARPS_PER_CTA) + 128;
        if (cap > optin - fixed) cap = optin - fixed;
        if (cap < 0) cap = 0;
        return cap & ~127;
    };
    e->stage_cap = tile_room(sizeof(WarpSmem) + sizeof(QuadSmem), C2B_MIN_CTAS_PER_SM);
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
    // ALIGN kernel: its own (smaller) per-warp state; CTAs per SM from the occupancy query, optionally capped (C2B_A_CTAS_PER_SM)
    int occ_a = 0, occ_b = 0;
    e->stage_cap_a = tile_room(sizeof(ASmem), C2B_A_MIN_CTAS);
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
    if (occ < C2B_MIN_CTAS_PER_SM && !getenv("C2B_CTAS_PER_SM"))
        fprintf(stderr, "[c2b] warning: only %d CTA(s) of the general kernel fit an SM (built for %d)\n", occ, C2B_MIN_CTAS_PER_SM);
    e->wpc = WARPS_PER_CTA;
    if (const char *v = getenv("C2B_WARPS_PER_CTA")) { int k = atoi(v); if (k >= 1 && k <= WARPS_PER_CTA) e->wpc = k; }
    if (const char *v = getenv("C2B_CTAS_PER_SM")) { int k = atoi(v); if (k >= 1 && k <= occ) occ = k; }
    if (const char *v = getenv("C2B_A_CTAS_PER_SM")) { int k = atoi(v); if (k >= 1 && k <= occ_a) occ_a = k; }
    if (occ_a > C2B_A_MIN_CTAS) occ_a = C2B_A_MIN_CTAS;
    e->grid = nsm * occ;                 // persistent: one wave of CTAs, warps pull work items from a counter
    e->grid_a = nsm * occ_a;
    e->grid_b = nsm * std::min(occ_b, 8);
    e->n_warps = std::max(e->grid, e->grid_a) * e->wpc;  // scratch slabs are per resident warp of whichever kernel is larger
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
    DevBuf *bufs[] = {&e->tb, &e->tbb, &e->tbq, &e->bnd, &e->ops, &e->rgo, &e->work, &e->lut, &e->gops, &e->gmeta, &e->left, &e->left2};
    for (DevBuf *b : bufs) if (b->p) rt_free(b->p);
    for (auto &st : e->stage) {
        DevBuf *sb[] = {&st.reads, &st.off, &st.cnt, &st.qw, &st.rid, &st.recs, &st.alns, &st.str, &st.ed, &st.maxlen, &st.ord, &st.gops, &st.gmeta, &st.left, &st.left2};
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
    if (e->stream2) cudaStreamDestroy(e->stream2);
    if (e->fork_ev) cudaEventDestroy(e->fork_ev);
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
        const int64_t lim = (1ll << 27);
        for (int q = 0; q < p->nq; q++)
            for (int i = 0; i < I; i++) {
                const int64_t v = rf.score_rows[(size_t)q * I + i];
                if (v > lim || v < -lim) return fail(e, C2B_E_LIMIT, "c2b_configure: substitution score out of range");
                prof[(size_t)q * Ipad + i] = (int32_t)(4 * v);
            }
        for (int i = 0; i <= I; i++) if (rf.gap_incentive[i] > lim || rf.gap_incentive[i] < -lim) return fail(e, C2B_E_LIMIT, "c2b_configure: gap incentive out of range");
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

// work block (u64): [2..6] cumulative path statistics; set s: [8 + 8 s] work hand-out counter, [9 + 8 s] widest alignment
constexpr size_t WORK_BYTES = 24 * 8;

static int ensure_scratch(c2b_engine *e, int maxJ)
{
    const int TS = ((maxJ + 32 + 31) & ~31);
    if (TS <= e->scratch_TS) return C2B_OK;
    int rc;
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    e->set_tb = al((size_t)e->n_warps * e->max_nrb * TS * 64 * 4);      // 64: a pair stores two words per lane
    e->set_tbb = al((size_t)e->n_warps * PK_BAND_SLOTS * 64 * 4);        // banded slabs (packed path)
    e->set_tbq = al((size_t)e->n_warps * TS * 64 * 4 + 64);              // ring-banded path: (step, lane) entries
    e->set_bnd = al((size_t)e->n_warps * 2 * 3 * TS * 4);
    e->set_ops = al((size_t)e->n_warps * std::min(e->n_refs, (int)C2B_MAX_REFS) * 32 * 8);
    if ((rc = ensure(e, e->tb, 2 * e->set_tb))) return rc;
    if ((rc = ensure(e, e->tbb, 2 * e->set_tbb))) return rc;
    if ((rc = ensure(e, e->tbq, 2 * e->set_tbq))) return rc;
    if ((rc = ensure(e, e->bnd, 2 * e->set_bnd))) return rc;
    if ((rc = ensure(e, e->ops, 2 * e->set_ops))) return rc;
    e->set_rgo = al((size_t)e->n_warps * RG_MAX_REFS * 4 * RG_OPS_STRIDE * 8);
    if ((rc = ensure(e, e->rgo, 2 * e->set_rgo))) return rc;
    const bool fresh_work = !e->work.p;
    if ((rc = ensure(e, e->work, WORK_BYTES))) return rc;
    if (fresh_work) RTCHK(rt_zero(e->work.p, WORK_BYTES, e->stream));
    e->scratch_TS = TS;
#ifndef C2B_EMU
    {   // L2 policy for the traceback slabs (written once, read back by the same warp microseconds later).  C2B_L2_PERSIST:
        //   unset / "none": no set-aside -- the whole L2 serves every access (r02 default: the ALIGN kernel's ring slabs are
        //                   the hot set now, and a set-aside sized for the general kernel's banded slabs took 60 % of L2 away);
        //   "ring"        : persisting window over the ring slabs (hit ratio = set-aside / slab bytes);
        //   "band"        : the r01 setting, persisting window over the general kernel's banded slabs.
        cudaDeviceProp prop;
        const char *mode = getenv("C2B_L2_PERSIST");
        if (cudaGetDeviceProperties(&prop, e->device) == cudaSuccess && prop.persistingL2CacheMaxSize > 0) {
            cudaStreamAttrValue av; memset(&av, 0, sizeof av);
            size_t carve = 0;
            if (mode && (!strcmp(mode, "ring") || !strcmp(mode, "band"))) {
                const bool ring = !strcmp(mode, "ring");
                const size_t slab = ring ? e->set_tbq : 2 * e->set_tbb;
                carve = std::min((size_t)prop.persistingL2CacheMaxSize, slab);
                av.accessPolicyWindow.base_ptr = ring ? e->tbq.p : e->tbb.p;
                av.accessPolicyWindow.num_bytes = std::min(slab, (size_t)prop.accessPolicyMaxWindowSize);
                av.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)carve / (double)std::max<size_t>(1, av.accessPolicyWindow.num_bytes));
                av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
                av.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
            }
            cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, carve);
            cudaStreamSetAttribute(e->stream, cudaStreamAttributeAccessPolicyWindow, &av);
            cudaGetLastError();
            if (getenv("C2B_VERBOSE"))
                fprintf(stderr, "[c2b] scratch for %d warps: ring slabs %.1f MB, L2 %.1f MB, persisting set-aside %.1f MB (%s)\n",
                        e->n_warps, e->set_tbq / 1e6, prop.l2CacheSize / 1e6, carve / 1e6, mode ? mode : "none");
        }
    }
#endif
    return C2B_OK;
}

// One batch on compute stream `cs` using scratch set `set` (0 or 1): the ALIGN / CLASSIFY pair followed by the general
// kernel over what ALIGN left over -- or the general kernel alone where the two-kernel form does not apply.  Launches that
// may overlap in time must use different sets; launches on the same stream are ordered.
// d_gops / d_gmeta / d_left: op streams [n_reads * R * W/32] u64, meta words [n_reads * R], left-over list [n_reads + 8] i32.
static int launch_on(c2b_engine *e, rt_stream cs, int set, const uint8_t *d_reads, const int64_t *d_offsets, int64_t n_reads,
                     int32_t max_read_len, const int32_t *d_count, const int32_t *d_qweight,
                     const int32_t *d_ref_id, c2b_read_rec *d_recs, c2b_aln_rec *d_alns,
                     uint8_t *d_strings, c2b_edit *d_edits, uint64_t *d_gops, uint32_t *d_gmeta, int32_t *d_left, int32_t *d_left2 = nullptr)
{
    if (!e || !e->configured) return fail(e, C2B_E_STATE, "c2b_align_batch: engine not configured");
    if (n_reads < 0 || !d_recs || !d_alns || (n_reads && (!d_reads || !d_offsets))) return fail(e, C2B_E_ARG, "c2b_align_batch: bad argument");
    if (n_reads >= (1ll << 31)) return fail(e, C2B_E_LIMIT, "c2b_align_batch: more than 2^31 reads in one batch");
    if (max_read_len < 1) max_read_len = 1;
    if (max_read_len > C2B_MAX_READ_LEN) return fail(e, C2B_E_LIMIT, "c2b_align_batch: read longer than C2B_MAX_READ_LEN");
    if ((int64_t)std::abs((long long)e->prm.gap_open) * max_read_len * e->max_I >= (1ll << 28))
        return fail(e, C2B_E_LIMIT, "c2b_align_batch: gap_open * lengths exceeds the int32 score range");
    if (!d_ref_id && e->n_refs > C2B_MAX_REFS)
        return fail(e, C2B_E_LIMIT, "c2b_align_batch: more than C2B_MAX_REFS references need a per-read ref_id");
    int rc = ensure_scratch(e, max_read_len);
    if (rc) return rc;
    if (n_reads == 0) return C2B_OK;
    KParams P;
    memset(&P, 0, sizeof P);
    P.reads = d_reads; P.offsets = d_offsets; P.n_reads = n_reads; P.count = d_count; P.qweight = d_qweight; P.ref_id = d_ref_id;
    P.recs = d_recs; P.alns = d_alns; P.strings = d_strings; P.edits = d_edits;
    P.W = (e->max_I + max_read_len + 31) & ~31; P.edit_cap = d_edits ? e->prm.edit_cap : 0;
    if (P.edit_cap == 0) P.edits = nullptr;
    P.refs = e->d_refs; P.n_refs = e->n_refs;
    P.out_refs = d_ref_id ? 1 : e->n_refs; P.ops_refs = std::min(e->n_refs, (int)C2B_MAX_REFS);
    P.go = e->prm.gap_open; P.ge = e->prm.gap_extend; P.seed_count = e->prm.seed_count; P.seed_min = e->prm.seed_min;
    P.flags = e->prm.flags; P.nq = e->prm.nq;
    memcpy(P.alpha, e->prm.alphabet, C2B_MAX_Q); memcpy(P.comp, e->prm.complement, C2B_MAX_Q);
    P.TS = e->scratch_TS;
    auto at = [&](const DevBuf &b, size_t per_set) { return (char *)b.p + (size_t)set * per_set; };
    P.tb = (uint32_t *)at(e->tb, e->set_tb); P.tb_words_per_warp = (int64_t)e->max_nrb * P.TS * 64;
    P.tbb = getenv("C2B_NO_BAND") ? nullptr : (uint32_t *)at(e->tbb, e->set_tbb); P.tbb_words_per_warp = (int64_t)PK_BAND_SLOTS * 64;
    P.tbq = getenv("C2B_NO_RING") ? nullptr : (uint32_t *)at(e->tbq, e->set_tbq);
    P.bnd = (int32_t *)at(e->bnd, e->set_bnd); P.bnd_words_per_warp = 2 * 3 * (int64_t)P.TS;
    P.opsbuf = (uint64_t *)at(e->ops, e->set_ops);
    P.rgops = getenv("C2B_NO_MULTI_RING") ? nullptr : (uint64_t *)at(e->rgo, e->set_rgo);
    P.stats = (unsigned long long *)e->work.p;
    unsigned long long *wk = P.stats + 8 + 8 * set;       // [0] ALIGN / general hand-out counter, [1] widest alignment, [2] general kernel's counter after ALIGN, [3] left-over count
    P.work_counter = wk; P.widest = wk + 1;
    P.vstride = e->vstride; P.hstride = e->hstride;
    P.forced_ops = e->forced_ops; P.forced_n = e->forced_n;
    P.gops = d_gops; P.gmeta = d_gmeta; P.NW = P.W / 32;
    P.pair_order = e->pair_order;
    P.lut = (const uint8_t *)e->lut.p;
    P.stage_bytes = 0; P.stage_src = nullptr;
    // two-kernel form: the configuration admits the ring-banded DP, op-stream buffers were supplied, nothing forces the
    // general kernel (caller-supplied op streams, the A/B switches)
    const bool split = e->split_ok && d_gops && d_gmeta && d_left && P.tbq && !e->forced_ops && !getenv("C2B_NO_SPLIT") &&
                       (e->n_refs == 1 || d_ref_id != nullptr || (e->n_refs <= RG_MAX_REFS && e->split_all));
    P.phase_sync = 0;
    if (!split) {                                         // one-kernel form: warps of a phase set move in step (C2B_PHASE_WARPS: 0/1 = free-running, 2, 4, 8)
        P.phase_sync = 4;
        if (const char *v = getenv("C2B_PHASE_WARPS")) { const int k = atoi(v), a = k < 0 ? -k : k; P.phase_sync = (a == 2 || a == 4 || a == 8 || a == 16) ? k : 0; }
        const int a = P.phase_sync < 0 ? -P.phase_sync : P.phase_sync;
        const int nsets = a ? e->wpc / a : 0;
        if (a > e->wpc || (a && e->wpc % a) || (P.phase_sync < 0 && (nsets & (nsets - 1)))) P.phase_sync = 0;
        if (e->n_refs > 1 && !d_ref_id && getenv("C2B_NO_MULTI_PHASE")) P.phase_sync = 0;
    }
    const bool one = (e->n_refs == 1 || d_ref_id != nullptr) && !getenv("C2B_GENERIC_KERNEL");      // one candidate reference per read
    RTCHK(rt_zero(wk, 64, cs));                           // this set's counters and widest alignment ([4], [5]: second-tier ALIGN launch)
    if (d_gmeta) RTCHK(rt_zero(d_gmeta, (size_t)n_reads * P.out_refs * 4, cs));
#ifndef C2B_EMU
    const RefDev &r0 = e->refdev[0];
    const size_t tile = (size_t)e->prm.nq * e->prm.nq * r0.Ipad * 4;        // reference 0's packed profile
    const bool can_stage = r0.pk_maxJ > 0 && !e->forced_ops && !getenv("C2B_NO_TMA_STAGE");
    cudaEventRecord(e->ev0, cs);
    if (split) {
        KParams A = P;
        A.left = d_left; A.left_n = wk + 3;
        A.discard_slab = getenv("C2B_NO_DISCARD") ? 0 : 1;
        if (can_stage && tile <= (size_t)e->stage_cap_a) { A.stage_bytes = (int32_t)tile; A.stage_src = r0.prof2; }
        const size_t smem_a = sizeof(ASmem) * e->wpc + 128 + (size_t)A.stage_bytes;
        // narrow first tier (align_narrow16): reads in their given order (no pairing order = the caller's reads are of one
        // length, or unsorted -- then hardly any unit of sixteen qualifies), one candidate reference per read
        const bool narrow = d_left2 && !P.pair_order && (e->n_refs == 1 || d_ref_id != nullptr) && !getenv("C2B_NO_NARROW");
        if (narrow) { A.left2 = d_left2; A.left2_n = wk + 5; }
        c2b_align_kernel<<<e->grid_a, e->wpc * 32, smem_a, cs>>>(A);
        if (narrow) {                                         // second tier: what the narrow band did not settle, eight reads per group
            KParams A2 = A;
            A2.left2 = nullptr; A2.left2_n = nullptr;
            A2.pair_order = d_left2; A2.n_dev = wk + 5; A2.work_counter = wk + 4;
            c2b_align_kernel<<<e->grid_a, e->wpc * 32, smem_a, cs>>>(A2);
            e->launches++;
        }
        if (one) c2b_classify_kernel<true><<<e->grid_b, B_WARPS_PER_CTA * 32, 0, cs>>>(P);
        else c2b_classify_kernel<false><<<e->grid_b, B_WARPS_PER_CTA * 32, 0, cs>>>(P);
        // the general kernel over ALIGN's left-over pairs (free-running warps, no ring-banded attempt)
        P.pair_order = d_left; P.n_dev = wk + 3; P.work_counter = wk + 2; P.tbq = nullptr; P.rgops = nullptr;
        P.tbb = nullptr;                                      // these pairs left the ring band: the banded slab would only cost a second DP
        e->launches += 2;
    }
    {
        if (can_stage && tile <= (size_t)e->stage_cap) { P.stage_bytes = (int32_t)tile; P.stage_src = r0.prof2; }
        const size_t smem = (sizeof(WarpSmem) + sizeof(QuadSmem)) * e->wpc + 128 + (size_t)P.stage_bytes;
        if (one) c2b_align_classify_kernel<true><<<e->grid, e->wpc * 32, smem, cs>>>(P);
        else c2b_align_classify_kernel<false><<<e->grid, e->wpc * 32, smem, cs>>>(P);
    }
    cudaEventRecord(e->ev1, cs);
    RTCHK(cudaGetLastError());
#else
    {
        static WarpSmem S; static QuadSmem Q; static ASmem AS;
        if (split) {
            KParams A = P;
            A.left = d_left; A.left_n = wk + 3;
            emu::run_warp([&]() { asmem_init(A, AS); });
            const bool narrow = d_left2 && !P.pair_order && (e->n_refs == 1 || d_ref_id != nullptr) && !getenv("C2B_NO_NARROW");
            if (narrow) {
                A.left2 = d_left2; A.left2_n = wk + 5;
                for (int64_t w = 0; 16 * w < n_reads; w++)
                    emu::run_warp([&]() {
                        if (!align_narrow16(A, AS, nullptr, w, 0)) {
                            align_group(A, AS, nullptr, 2 * w, 0);
                            wp::sync();
                            if (8 * (2 * w + 1) < n_reads) align_group(A, AS, nullptr, 2 * w + 1, 0);
                        }
                    });
                KParams A2 = A;
                A2.left2 = nullptr; A2.left2_n = nullptr; A2.pair_order = d_left2; A2.n_dev = wk + 5; A2.work_counter = wk + 4;
                const int64_t n2 = (int64_t)*A2.n_dev;
                for (int64_t w = 0; 8 * w < n2; w++) emu::run_warp([&]() { align_group(A2, AS, nullptr, w, 0); });
            } else
            for (int64_t w = 0; 8 * w < n_reads; w++) emu::run_warp([&]() { align_group(A, AS, nullptr, w, 0); });
            static BSmem BS;
            const int64_t total_bytes = d_offsets[n_reads];
            for (int64_t rd = 0; rd < n_reads; rd++) {
                if (one) emu::run_warp([&]() { ScAcc<1> acc; sc_init(acc); const BPreA a = classify_pre_a(P, rd); const BPre b = classify_pre_b<true>(P, rd, a, total_bytes);
                                               if (b.go) { classify_stage<true>(b, BS); wp::sync(); classify_read<true>(P, rd, b, BS, acc); } sc_flush(acc, P); });
                else emu::run_warp([&]() { ScAcc<RG_MAX_REFS> acc; sc_init(acc); const BPreA a = classify_pre_a(P, rd); const BPre b = classify_pre_b<false>(P, rd, a, total_bytes);
                                            if (b.go) { classify_stage<false>(b, BS); wp::sync(); classify_read<false>(P, rd, b, BS, acc); } sc_flush(acc, P); });
            }
            P.pair_order = d_left; P.n_dev = wk + 3; P.work_counter = wk + 2; P.tbq = nullptr; P.rgops = nullptr; P.tbb = nullptr;
        }
        const int64_t nrd = P.n_dev ? (int64_t)*P.n_dev : n_reads;
        if (P.n_dev) {                                      // left-over list: one pair per hand-out, like the kernel
            for (int64_t w = 0; 2 * w < nrd; w++) {
                if (one) emu::run_warp([&]() { process_item<true>(P, S, nullptr, w, 0); });
                else emu::run_warp([&]() { process_item<false>(P, S, nullptr, w, 0); });
            }
        } else
        for (int64_t w = 0; 8 * w < nrd; w++) {
            wp::g_grp_syncs = 0;
            if (one) emu::run_warp([&]() { process_group<true>(P, S, Q, nullptr, w, 0); });
            else emu::run_warp([&]() { process_group<false>(P, S, Q, nullptr, w, 0); });
            // every path through a work group must execute the same number of phase barriers (a mismatch deadlocks the GPU)
            if (P.phase_sync && wp::g_grp_syncs != group_phases(P)) {
                fprintf(stderr, "warp_emu: work group %lld executed %ld phase barriers, expected %d\n", (long long)w, wp::g_grp_syncs, group_phases(P));
                abort();
            }
        }
    }
#endif
    e->launches++;
    return C2B_OK;
}

// op-stream buffers of the device-pointer API (engine-owned, sized for the batch)
static int ensure_ops(c2b_engine *e, DevBuf &gops, DevBuf &gmeta, DevBuf &left, DevBuf &left2, int64_t n_reads, int nr, int W)
{
    int rc;
    if ((rc = ensure(e, gops, (size_t)n_reads * nr * (W / 32) * 8))) return rc;
    if ((rc = ensure(e, gmeta, (size_t)n_reads * nr * 4))) return rc;
    if ((rc = ensure(e, left, (size_t)(n_reads + 8) * 4))) return rc;
    if ((rc = ensure(e, left2, (size_t)(n_reads + 16) * 4))) return rc;
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
    int rc = ensure_ops(e, e->gops, e->gmeta, e->left, e->left2, n_reads, nr, W);
    if (rc) return rc;
    return launch_on(e, e->stream, 0, d_reads, d_offsets, n_reads, max_read_len, d_count, d_qweight, d_ref_id, d_recs,
                     d_alns, d_strings, d_edits, (uint64_t *)e->gops.p, (uint32_t *)e->gmeta.p, (int32_t *)e->left.p, (int32_t *)e->left2.p);
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
    int64_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    RTCHK(rt_d2h(v, e->work.p, 64, e->stream));
    RTCHK(rt_sync(e->stream));
    // the ALIGN kernel counts reads ([5] kept by the ring, [6] sent on, [7] fully aligned); reported in pairs
    e->band_reruns = v[4]; e->ring_pairs = (v[5] + 1) / 2; e->ring_fallbacks = (v[6] + 1) / 2;
    if (getenv("C2B_VERBOSE"))
        fprintf(stderr, "[c2b] counters: general kernel %lld pair items + %lld single items; ALIGN: %lld read x reference combinations kept "
                        "by the ring, %lld sent to the full matrix, %lld reads settled\n", (long long)v[2], (long long)v[3], (long long)v[5],
                (long long)v[6], (long long)v[7]);
    if (pair_items) *pair_items = v[2] + (v[7] + 1) / 2;
    if (single_items) *single_items = v[3];
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
        if ((rc = ensure_ops(e, st.gops, st.gmeta, st.left, st.left2, n, nr, W))) return rc;
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
        // C2B_TWO_STREAMS=1: consecutive chunks alternate between two compute streams (and the two scratch sets) so that the
        // head of chunk c+1's ALIGN launch could fill the SMs the tails of chunk c's launches leave idle.  Measured slower
        // end to end than one stream (two sets of ring slabs in flight, far more than the L2 holds) -- off.
        const int set = (e->stream2 && getenv("C2B_TWO_STREAMS")) ? (ci & 1) : 0;
        rt_stream cs = set ? e->stream2 : e->stream;
        RTCHK(rt_wait(cs, st.in_done));
        rc = launch_on(e, cs, set, (const uint8_t *)st.reads.p, (const int64_t *)st.off.p, n, (int32_t)maxJ,
                       count ? (const int32_t *)st.cnt.p : nullptr, qweight ? (const int32_t *)st.qw.p : nullptr,
                       ref_id ? (const int32_t *)st.rid.p : nullptr, (c2b_read_rec *)st.recs.p,
                       (c2b_aln_rec *)st.alns.p, strings ? (uint8_t *)st.str.p : nullptr,
                       cap ? (c2b_edit *)st.ed.p : nullptr, (uint64_t *)st.gops.p, (uint32_t *)st.gmeta.p, (int32_t *)st.left.p, (int32_t *)st.left2.p);
        e->pair_order = nullptr;
        if (rc) return rc;
        // keep this batch's "widest alignment" before the next launch sequence resets it
        RTCHK(cudaMemcpyAsyncOrCopy(st.maxlen.p, (const char *)e->work.p + (9 + 8 * set) * 8, 8, cs));
        RTCHK(rt_record(st.k_done, cs));
        st.used = true;
        if (pend.any && (rc = flush(pend))) return rc;           // chunk ci-1: overlaps this chunk's kernels
        pend.any = true; pend.c0 = c0; pend.n = n; pend.set = ci & 1;
    }
    if (pend.any && (rc = flush(pend))) return rc;
    RTCHK(rt_sync(e->s_out));
    RTCHK(rt_sync(e->stream));
    if (e->stream2) RTCHK(rt_sync(e->stream2));
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
// reference.  strand 1: the read was aligned as its reverse complement (engine's complement table).
int c2b_expand_alignment(const c2b_engine *e, const uint64_t *ops, uint32_t meta, const char *read, int32_t read_len,
                         const char *ref, int32_t ref_len, char *out_read, char *out_ref)
{
    if (!e || !ops || !read || !ref || !out_read || !out_ref) return C2B_E_ARG;
    const int n = (int)(meta & 0xffffu), strand = (int)((meta >> 16) & 1u);
    unsigned char comp[256];
    if (strand) {
        for (int c = 0; c < 256; c++) comp[c] = (unsigned char)c;
        for (int q = 0; q < e->prm.nq; q++) comp[(unsigned char)e->prm.alphabet[q]] = (unsigned char)e->prm.alphabet[e->prm.complement[q]];
    }
    int i = ref_len, j = read_len;
    for (int q = 0; q < n; q++) {
        const int op = (int)((ops[q >> 5] >> (2 * (q & 31))) & 3ull);
        char rd = '-', rf = '-';
        if (op != OP_J) { if (j < 1) return C2B_E_ARG; j--; rd = strand ? (char)comp[(unsigned char)read[read_len - 1 - j]] : read[j]; }
        if (op != OP_I) { if (i < 1) return C2B_E_ARG; i--; rf = ref[i]; }
        if (op == OP_NONE) return C2B_E_ARG;
        out_read[n - 1 - q] = rd; out_ref[n - 1 - q] = rf;
    }
    return (i == 0 && j == 0) ? C2B_OK : C2B_E_ARG;
}

// Batch form: strings[n_reads][R][2][W], right-aligned like c2b_align_batch's, from the compact outputs; host threads.
int c2b_expand_batch(const c2b_engine *e, const uint8_t *reads, const int64_t *offsets, int64_t n_reads, const int32_t *ref_id,
                     const uint64_t *ops, const uint32_t *meta, int32_t max_read_len, uint8_t *strings, int32_t n_threads)
{
    if (!e || !e->configured || !reads || !offsets || !ops || !meta || !strings) return C2B_E_ARG;
    const int W = (e->max_I + max_read_len + 31) & ~31, NW = W / 32, nr = ref_id ? 1 : e->n_refs;
    if (n_threads <= 0) n_threads = (int)std::max(1u, std::thread::hardware_concurrency());
    n_threads = (int)std::min<int64_t>(n_threads, std::max<int64_t>(1, n_reads / 1024));
    std::vector<int> bad((size_t)n_threads, 0);
    auto work = [&](int t) {
        const int64_t lo = n_reads * t / n_threads, hi = n_reads * (t + 1) / n_threads;
        for (int64_t rd = lo; rd < hi; rd++)
            for (int k = 0; k < nr; k++) {
                const int r = ref_id ? ref_id[rd] : k;
                const int64_t slot = rd * nr + k;
                const uint32_t m = meta[slot];
                const int n = (int)(m & 0xffffu);
                if ((m >> 24) == 0 || n == 0 || n > W) continue;      // no alignment in this slot
                uint8_t *o = strings + slot * 2 * (int64_t)W;
                const RefHost &R = e->refs[(size_t)r];
                if (c2b_expand_alignment(e, ops + slot * NW, m, (const char *)reads + offsets[rd], (int32_t)(offsets[rd + 1] - offsets[rd]),
                                         R.seq.data(), (int32_t)R.seq.size(), (char *)o + W - n, (char *)o + 2 * W - n)) bad[(size_t)t]++;
            }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < n_threads; t++) th.emplace_back(work, t);
    work(0);
    for (auto &x : th) x.join();
    for (int b : bad) if (b) return C2B_E_ARG;
    return C2B_OK;
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
        if (amask[k] >> R) return fail(e, C2B_E_ARG, "c2b_annotate_build: listed slot out of range");
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

// sage_b200.cu — host runtime and C ABI (include/sage_b200.h) of the H100-native search-and-score library.
//
// Host side of the boundary, written in C++ because the reference (Rust) toolchain is absent in this image; it
// mirrors the reference's call structure: IndexedDatabase (database.rs:384-395) -> sage_b200_db, Scorer
// (scoring.rs:210-232) -> sage_b200_scorer, `par_iter().flat_map(|s| scorer.score(s))` (runner.rs:311-325) ->
// sage_b200_score_batch. No CPU fallback exists: every entry point fails loudly when CUDA is unavailable.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_merge_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_segmented_sort.cuh>
#include <cuda_runtime.h>
#include <thrust/iterator/counting_iterator.h>

#include <pthread.h>
#include <sched.h>

#include <algorithm>
#include <atomic>
#include <cctype>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <chrono>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <thread>
#include <string>
#include <vector>

#include "../../include/sage_b200.h"
#include "kernels.cuh"
#include "lfq.cuh"
#include "fdr.cuh"
#include "rt.cuh"
#include "picked.cuh"
#include "protein_groups.cuh"
#include "digest.cuh"
#include "prefilter.cuh"
#include "spectra.cuh"
#include "write.cuh"
#include "mgf.cuh"

using namespace sb;

// ------------------------------------------------------------------------------------------------ errors
static thread_local std::string g_last_error;
static int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}
#define CUDA_TRY(expr)                                                                                         \
    do {                                                                                                       \
        cudaError_t _e = (expr);                                                                               \
        if (_e != cudaSuccess) return fail(SAGE_B200_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

// mass.rs:64-76
static const float kResidueMass[26] = {71.03711f, 0.0f,      103.00919f, 115.02694f, 129.04259f, 147.0684f, 57.02146f,  137.05891f, 113.08406f,
                                       0.0f,      128.09496f, 113.08406f, 131.0405f,  114.04293f, 237.14774f, 97.05276f, 128.05858f, 156.1011f,
                                       87.03203f, 101.04768f, 150.95363f, 99.06841f,  186.07932f, 0.0f,       163.06332f, 0.0f};

// Every entry point that takes a device: one must exist (there is no CPU fallback) and the index must name one; then it is selected.
static int select_device(int device) {
    int ndev = 0;
    const cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(SAGE_B200_ECUDA, "no CUDA device available (%s): sage_b200 has no CPU fallback", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    }
    if (device < 0 || device >= ndev) return fail(SAGE_B200_EINVAL, "device %d out of range (0..%d)", device, ndev - 1);
    CUDA_TRY(cudaSetDevice(device));
    return 0;
}

// ------------------------------------------------------------------------------------------- device buffers
// A growable buffer (25 % + 256 B of headroom) that lives as long as its owner.
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
    int reserve(size_t bytes) {
        if (bytes <= cap) return 0;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) return fail(SAGE_B200_ECUDA, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
        cap = want;
        return 0;
    }
    // cub's two-phase call f(tmp, bytes) with this buffer as its temporary storage: f(nullptr, bytes) sizes it, then f runs.
    template <class F>
    cudaError_t two_phase(F f) {
        size_t b = 0;
        if (cudaError_t e = f(nullptr, b)) return e;
        if (reserve(b)) return cudaErrorMemoryAllocation;
        return f(p, b);
    }
    template <class T>
    T* as() const { return reinterpret_cast<T*>(p); }
};
struct PinBuf {
    void* p = nullptr;
    size_t cap = 0;
    PinBuf() = default;
    PinBuf(const PinBuf&) = delete;
    PinBuf& operator=(const PinBuf&) = delete;
    ~PinBuf() { if (p) cudaFreeHost(p); }
    int reserve(size_t bytes) {
        if (bytes <= cap) return 0;
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaHostAlloc(&p, want, cudaHostAllocPortable);
        if (e != cudaSuccess) return fail(SAGE_B200_ECUDA, "cudaHostAlloc(%zu) failed: %s", want, cudaGetErrorString(e));
        cap = want;
        return 0;
    }
};

// Exact-size device allocations freed together when the arena goes (the temporaries of one call, or arrays that live as long as their
// owner), and one growable buffer for the temporary storage of cub's two-phase calls.
struct DevArena {
    std::vector<void*> ps;
    uint64_t bytes = 0;
    void* tmp = nullptr;
    size_t tmp_bytes = 0;
    DevArena() = default;
    DevArena(const DevArena&) = delete;
    DevArena& operator=(const DevArena&) = delete;
    ~DevArena() { for (void* p : ps) cudaFree(p); }
    template <class T>
    cudaError_t alloc(T** out, size_t count) {
        const size_t b = count ? count * sizeof(T) : 16;
        void* p = nullptr;
        cudaError_t e = cudaMalloc(&p, b);
        if (e == cudaSuccess) { ps.push_back(p); bytes += b; *out = (T*)p; }
        return e;
    }
    // alloc(out, count + pad), then the copy of `count` items from `host` queued on st.
    template <class T>
    cudaError_t upload(T** out, const T* host, size_t count, cudaStream_t st, size_t pad = 0) {
        cudaError_t e = alloc(out, count + pad);
        if (e == cudaSuccess && count) e = cudaMemcpyAsync(*out, host, count * sizeof(T), cudaMemcpyHostToDevice, st);
        return e;
    }
    // alloc(out, count), then zeroed on st.
    template <class T>
    cudaError_t zeros(T** out, size_t count, cudaStream_t st) {
        cudaError_t e = alloc(out, count);
        if (e == cudaSuccess && count) e = cudaMemsetAsync(*out, 0, count * sizeof(T), st);
        return e;
    }
    // A larger request allocates a new buffer; the old one stays until the arena goes (work queued on a stream may still use it).
    cudaError_t reserve_tmp(size_t b) {
        if (tmp && b <= tmp_bytes) return cudaSuccess;
        cudaError_t e = alloc((char**)&tmp, b);
        if (e == cudaSuccess) tmp_bytes = b;
        return e;
    }
    // cub's two-phase call f(tmp, bytes) on the growable buffer: f(nullptr, bytes) sizes it (plus `pad` bytes reserved), then f runs.
    template <class F>
    cudaError_t two_phase(F f, size_t pad = 0) {
        size_t b = 0;
        if (cudaError_t e = f(nullptr, b)) return e;
        if (cudaError_t e = reserve_tmp(b + pad)) return e;
        return f(tmp, b);
    }
};

// A non-blocking stream and an event, each destroyed with its owner (with the owner's device current) and created by create(). The stream
// waits for its queued work before it goes: declared after the DevArena and host buffers that work uses, it keeps them alive until it ends.
struct Stream {
    cudaStream_t s = nullptr;
    Stream() = default;
    Stream(const Stream&) = delete;
    Stream& operator=(const Stream&) = delete;
    ~Stream() {
        if (!s) return;
        cudaStreamSynchronize(s);
        cudaStreamDestroy(s);
    }
    cudaError_t create() { return cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking); }
    operator cudaStream_t() const { return s; }
};
struct Event {
    cudaEvent_t e = nullptr;
    Event() = default;
    Event(const Event&) = delete;
    Event& operator=(const Event&) = delete;
    ~Event() { if (e) cudaEventDestroy(e); }
    cudaError_t create() { return cudaEventCreate(&e); }
    operator cudaEvent_t() const { return e; }
};

// Blocks of 256 threads that cover n items.
static unsigned grid256(uint64_t n) { return (unsigned)((n + 255) / 256); }

// A kernel launch and its check: LAUNCH(k<<<grid, block, smem, st>>>(args)).
#define LAUNCH(...)                         \
    do {                                    \
        __VA_ARGS__;                        \
        CUDA_TRY(cudaGetLastError());       \
    } while (0)
// `kernel` over n items in blocks of 256 on stream st, checked; n == 0 launches nothing.
#define LAUNCH_N(kernel, n, st, ...)                                                  \
    do {                                                                              \
        if ((n) > 0) LAUNCH(kernel<<<grid256(n), 256, 0, st>>>(__VA_ARGS__));         \
    } while (0)

// Copies `bytes` from the device to the host on st and waits for the stream.
static int read_back(cudaStream_t st, void* host, const void* dev, size_t bytes) {
    CUDA_TRY(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

// Host -> device copy of a PAGEABLE array (a Rust Vec<f32>, a numpy array) through a pinned staging buffer: a few pool threads copy 2 MB pieces
// into the staging buffer while the calling thread submits each piece's DMA as soon as it is staged, so the memcpy (one core copies
// slower than the PCIe link) overlaps the transfer instead of preceding it. The pool threads are persistent (one pool per pipeline lane, started by
// the first pageable chunk): creating the threads per array was a visible share of the call. 6 threads x 2 MB pieces chosen by A/B on cfg2
// against 3..24 threads and 512 KB..2 MB pieces (more copy threads only fight the DMA reads for the memory controllers).
struct StagePool {
    std::vector<std::thread> th;
    std::mutex mu;
    std::condition_variable cv;
    uint64_t gen = 0;
    bool quit = false;
    const char* src = nullptr;
    char* dst = nullptr;
    size_t bytes = 0, piece = 0, np = 0, done_cap = 0;
    std::atomic<size_t> next{0};
    std::atomic<int> busy{0};
    std::unique_ptr<std::atomic<unsigned char>[]> done;

    void worker() {
        uint64_t seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return quit || gen != seen; });
                if (quit) return;
                seen = gen;
            }
            for (;;) {
                const size_t i = next.fetch_add(1, std::memory_order_relaxed);
                if (i >= np) break;
                const size_t off = i * piece, len = std::min(piece, bytes - off);
                memcpy(dst + off, src + off, len);
                done[i].store(1, std::memory_order_release);
            }
            busy.fetch_sub(1, std::memory_order_release);
        }
    }
    // Copies src -> stage in pieces with the pool and submits piece i's DMA (stage -> device) as soon as pieces 0..i are staged.
    cudaError_t run(void* dev, const void* s, size_t n, void* stage, size_t piece_bytes, size_t nthreads, cudaStream_t st) {
        if (th.size() < nthreads) {
            const size_t have = th.size();
            for (size_t t = have; t < nthreads; t++) th.emplace_back([this] { worker(); });
        }
        const size_t pieces = (n + piece_bytes - 1) / piece_bytes;
        if (pieces > done_cap) { done.reset(new std::atomic<unsigned char>[pieces]); done_cap = pieces; }
        for (size_t i = 0; i < pieces; i++) done[i].store(0, std::memory_order_relaxed);
        {
            std::lock_guard<std::mutex> lk(mu);
            src = (const char*)s; dst = (char*)stage; bytes = n; piece = piece_bytes; np = pieces;
            next.store(0, std::memory_order_relaxed);
            busy.store((int)th.size(), std::memory_order_relaxed);
            gen++;
        }
        cv.notify_all();
        cudaError_t e = cudaSuccess;
        for (size_t i = 0; i < pieces; i++) {
            while (!done[i].load(std::memory_order_acquire)) std::this_thread::yield();
            const size_t off = i * piece_bytes, len = std::min(piece_bytes, n - off);
            if (e == cudaSuccess) e = cudaMemcpyAsync((char*)dev + off, (char*)stage + off, len, cudaMemcpyHostToDevice, st);
        }
        while (busy.load(std::memory_order_acquire) != 0) std::this_thread::yield();   // every worker has left the job: its fields may change
        return e;
    }
    ~StagePool() {
        {
            std::lock_guard<std::mutex> lk(mu);
            quit = true;
        }
        cv.notify_all();
        for (auto& t : th) t.join();
    }
};

static int staged_h2d(void* dst, const void* src, size_t bytes, PinBuf& stage, StagePool& pool, cudaStream_t st) {
    if (bytes == 0) return 0;
    int rc = stage.reserve(bytes);
    if (rc) return rc;
    static const size_t piece = []() { const char* e = getenv("SAGE_B200_STAGE_PIECE_KB"); return (size_t)std::max(64, e ? atoi(e) : 2048) << 10; }();
    static const size_t max_threads = []() { const char* e = getenv("SAGE_B200_STAGE_THREADS"); return (size_t)std::max(1, e ? atoi(e) : 6); }();
    const size_t np = (bytes + piece - 1) / piece;
    if (np <= 2) {   // small: a plain copy is cheaper than waking threads
        memcpy(stage.p, src, bytes);
        CUDA_TRY(cudaMemcpyAsync(dst, stage.p, bytes, cudaMemcpyHostToDevice, st));
        return 0;
    }
    const unsigned hw = std::max(2u, std::thread::hardware_concurrency());
    const size_t nthreads = std::min<size_t>(max_threads, (size_t)hw - 1);
    const cudaError_t e = pool.run(dst, src, bytes, stage.p, piece, nthreads, st);
    if (e != cudaSuccess) return fail(SAGE_B200_ECUDA, "staged host-to-device copy failed: %s", cudaGetErrorString(e));
    return 0;
}

static bool is_pinned(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeHost;
}

// ------------------------------------------------------------------------------------------------ db
// Runs f() (0 or an error code) for work whose failure only turns an optimisation off: the error is cleared and the thread's last error
// message is kept, since the calling entry point still succeeds.
template <class F>
static bool optional_work(F f) {
    const std::string msg = g_last_error;
    if (f() == 0) return true;
    cudaGetLastError();
    g_last_error = msg;
    return false;
}

// One lazily built block-major copy of the fragments: its view and the device arrays behind it.
template <class View>
struct BlockIndexSlot {
    View v{};
    std::unique_ptr<DevArena> mem;   // the arrays of the current build
    int failed = 0;
    uint64_t bytes = 0;
    std::vector<std::unique_ptr<DevArena>> retired;   // arrays of earlier builds: another scorer of the same db may still hold a view of them (freed with the db)
    uint64_t retired_bytes = 0;
    // A rebuild with another block size keeps the old arrays alive: a chunk of another scorer, queued with the old view, may still run.
    void retire() {
        if (mem) retired.push_back(std::move(mem));
        retired_bytes += bytes;
        v = View{};
        bytes = 0;
    }
    // build(arena, view, bytes) makes the copy's arrays in a fresh arena and returns 0 once they are finished on the device; only then is
    // the view published. A failed build frees its arrays and leaves an empty view for good (the kernels then read the page index).
    template <class F>
    View rebuild(F build) {
        retire();
        std::unique_ptr<DevArena> fresh(new DevArena);
        View nv{};
        uint64_t nbytes = 0;
        if (!optional_work([&] { return build(*fresh, nv, nbytes); })) {
            failed = 1;
            return View{};
        }
        mem = std::move(fresh);
        v = nv;
        bytes = nbytes;
        return v;
    }
};

struct sage_b200_db {
    int device = 0;
    DbView v{};
    DevArena mem;   // the arrays the view points at, exact-size
    uint64_t total_residues = 0;
    int sm_count = 132;   // H100 SXM; replaced by the device's multiProcessorCount in db_new
    // secondary copies of the fragments in peptide-block-major order, built lazily and guarded by wmu: `wide` (WideIndexView: blocks = the
    // open-search count tile, built by the first scorer that meets a wide window) and `narrow` (NarrowIndexView: small blocks, built by the
    // first narrow chunk)
    mutable std::mutex wmu;
    mutable BlockIndexSlot<WideIndexView> wide;
    mutable BlockIndexSlot<NarrowIndexView> narrow;
};

static uint32_t ceil_log2_u64(uint64_t n) {
    uint32_t l = 0;
    while ((1ull << l) < n) l++;
    return l;
}

// The ion kinds of an index, validated.
static int db_set_kinds(sage_b200_db* db, const uint8_t* kinds, uint64_t n_kinds) {
    if (n_kinds == 0 || n_kinds > MAX_KINDS) return fail(SAGE_B200_EINVAL, "ion_kinds: need 1..%d kinds", MAX_KINDS);
    db->v.n_kinds = (uint32_t)n_kinds;
    for (uint64_t k = 0; k < n_kinds; k++) {
        if (kinds[k] > 5) return fail(SAGE_B200_EINVAL, "ion kind %u out of range", kinds[k]);
        db->v.kinds[k] = kinds[k];
        if (kinds[k] <= 2) db->v.nterm_mask |= 1u << k;
    }
    return 0;
}

// The per-peptide arrays of an index, writable (the view holds them read-only).
struct PeptideArrays {
    float* mono = nullptr;
    uint8_t *len = nullptr, *flags = nullptr, *missed = nullptr;
    uint32_t* ion_off = nullptr;
};

// The per-peptide arrays of an n-peptide index (mono, length, flags, missed cleavages, ion offsets), allocated and placed in the view.
static int db_alloc_peptides(sage_b200_db* db, uint64_t n, PeptideArrays& p) {
    CUDA_TRY(db->mem.alloc(&p.mono, n));
    CUDA_TRY(db->mem.alloc(&p.len, n));
    CUDA_TRY(db->mem.alloc(&p.flags, n));
    CUDA_TRY(db->mem.alloc(&p.missed, n));
    CUDA_TRY(db->mem.alloc(&p.ion_off, n + 1));
    db->v.n_pep = (uint32_t)n;
    db->v.pep_mono = p.mono;
    db->v.pep_len = p.len;
    db->v.pep_flags = p.flags;
    db->v.pep_missed = p.missed;
    db->v.ion_off = p.ion_off;
    return 0;
}

// The per-peptide ion tables (n_ions entries at the ion offsets already on the device) from the table's device arrays, finished on st.
static int db_build_ions(sage_b200_db* db, uint64_t n, uint64_t n_ions, const uint32_t* off, const uint8_t* seq, const float* mods, const float* nterm,
                         cudaStream_t st) {
    float* ions = nullptr;
    CUDA_TRY(db->mem.alloc(&ions, n_ions));
    db->v.ions = ions;
    DevArena A;
    float* t_res = nullptr;
    CUDA_TRY(A.upload(&t_res, kResidueMass, sizeof kResidueMass / sizeof(float), st));
    if (n) LAUNCH(k_build_ions<<<(unsigned)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, off, seq, mods, nterm, db->v.pep_mono, db->v.ion_off, db->v.n_kinds, db->v, ions, t_res));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

// Uploads the peptide table and builds the per-peptide ion tables on st.
static int db_upload_peptides(sage_b200_db* db, const sage_b200_peptides* P, const uint8_t* kinds, uint64_t n_kinds, cudaStream_t st) {
    if (!P || (P->n_peptides && (!P->residue_offsets || !P->sequence || !P->modifications || !P->nterm || !P->monoisotopic || !P->decoy || !P->missed_cleavages)))
        return fail(SAGE_B200_EINVAL, "peptides: null array");
    if (int rc = db_set_kinds(db, kinds, n_kinds)) return rc;
    if (P->n_peptides >= 0xFFFFFFFEull) return fail(SAGE_B200_ELIMIT, "too many peptides for u32 PeptideIx");
    const uint64_t n = P->n_peptides;
    const uint64_t nres = n ? P->residue_offsets[n] : 0;
    db->total_residues = nres;
    std::vector<uint8_t> len(n), flags(n);
    std::vector<uint32_t> ion_off(n + 1);
    uint64_t acc = 0;
    for (uint64_t i = 0; i < n; i++) {
        const uint64_t L = P->residue_offsets[i + 1] - P->residue_offsets[i];
        if (L == 0 || L > 255) return fail(SAGE_B200_ELIMIT, "peptide %llu has length %llu (supported 1..255)", (unsigned long long)i, (unsigned long long)L);
        len[i] = (uint8_t)L;
        flags[i] = P->decoy[i] ? 1 : 0;
        ion_off[i] = (uint32_t)acc;
        acc += n_kinds * (L - 1);
        if (acc > 0xFFFFFFFFull) return fail(SAGE_B200_ELIMIT, "ion table exceeds 2^32 entries");
    }
    ion_off[n] = (uint32_t)acc;
    PeptideArrays p;
    if (int rc = db_alloc_peptides(db, n, p)) return rc;
    if (n) {
        CUDA_TRY(cudaMemcpyAsync(p.mono, P->monoisotopic, 4 * n, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(p.len, len.data(), n, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(p.flags, flags.data(), n, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(p.missed, P->missed_cleavages, n, cudaMemcpyHostToDevice, st));
    }
    CUDA_TRY(cudaMemcpyAsync(p.ion_off, ion_off.data(), 4 * (n + 1), cudaMemcpyHostToDevice, st));
    // device copies of the arrays ion generation reads
    DevArena A;
    uint32_t* t_off = nullptr;
    uint8_t* t_seq = nullptr;
    float *t_mods = nullptr, *t_nterm = nullptr;
    CUDA_TRY(A.alloc(&t_off, n + 5));
    CUDA_TRY(A.alloc(&t_seq, nres + 16));
    CUDA_TRY(A.alloc(&t_mods, nres + 4));
    CUDA_TRY(A.alloc(&t_nterm, n + 4));
    if (n) {
        CUDA_TRY(cudaMemcpyAsync(t_off, P->residue_offsets, 4 * (n + 1), cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(t_seq, P->sequence, nres, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(t_mods, P->modifications, 4 * nres, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(t_nterm, P->nterm, 4 * n, cudaMemcpyHostToDevice, st));
    }
    return db_build_ions(db, n, acc, t_off, t_seq, t_mods, t_nterm, st);   // it waits for st: the host and device arrays above outlive the copies
}

// A handle under construction: destroyed (by its C destroy function) unless released to the caller.
template <class T>
using Guard = std::unique_ptr<T, void (*)(T*)>;

static int db_new(int device, Guard<sage_b200_db>& out) {
    if (int rc = select_device(device)) return rc;
    out.reset(new sage_b200_db());
    out->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) out->sm_count = prop.multiProcessorCount;
    return 0;
}

extern "C" int sage_b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

extern "C" void sage_b200_db_destroy(sage_b200_db* db) {
    if (!db) return;
    cudaSetDevice(db->device);
    delete db;
}

// Search directories over the finished index (see DbView), built on st. Skipped (plain binary searches are used) when the shapes do not fit.
static int db_build_directories(sage_b200_db* db, cudaStream_t st) {
    DbView& v = db->v;
    v.page_grid = nullptr; v.bucket_lut = nullptr; v.pep_lut = nullptr;
    if (v.n_frag == 0 || v.n_bucket == 0 || v.n_pep == 0 || (getenv("SAGE_B200_NO_DIRECTORIES") && getenv("SAGE_B200_NO_DIRECTORIES")[0] == '1')) return 0;
    int rc;
    uint16_t* page_grid = nullptr;
    uint32_t *bucket_lut = nullptr, *pep_lut = nullptr;
    if (v.bucket_size <= 65535u) {
        // cells per page ~ bucket_size / entries-per-cell: the in-cell search that follows a grid lookup is a chain of dependent loads
        uint32_t epc = 2;   // chosen by A/B on cfg2 against 4..32 entries per cell (+6 % index memory)
        if (const char* e = getenv("SAGE_B200_GRID_ENTRIES")) epc = (uint32_t)std::min(1024, std::max(1, atoi(e)));
        uint32_t cells = 64;
        while (cells < 16384 && (uint64_t)cells * epc < v.bucket_size) cells <<= 1;
        uint32_t shift = 0;
        while (((uint64_t)v.n_pep >> shift) >= cells) shift++;
        const uint32_t gn = (uint32_t)(((uint64_t)v.n_pep - 1) >> shift) + 1;   // cells 0..gn-1 cover every PeptideIx
        const uint64_t total = (uint64_t)v.n_bucket * (gn + 1);
        CUDA_TRY(db->mem.alloc(&page_grid, total));
        LAUNCH(k_build_page_grid<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(v, shift, gn, page_grid));
        v.grid_shift = shift; v.grid_n = gn;
    }
    float ends[2] = {0.f, 0.f};
    if ((rc = read_back(st, &ends[0], v.bucket_min, 4))) return rc;
    if ((rc = read_back(st, &ends[1], v.bucket_min + (v.n_bucket - 1), 4))) return rc;
    bool lut_ok = ends[0] > 0.0f && std::isfinite(ends[0]) && std::isfinite(ends[1]);   // positive finite m/z: float order == total_cmp order
    if (lut_ok) {
        const float w = (ends[1] - ends[0]) / (float)BUCKET_LUT_CELLS;
        const float inv_w = (w > 0.0f && w < 3.0e38f) ? 1.0f / w : 0.0f;
        CUDA_TRY(db->mem.alloc(&bucket_lut, BUCKET_LUT_CELLS));
        LAUNCH(k_build_bucket_lut<<<BUCKET_LUT_CELLS / 256, 256, 0, st>>>(v, ends[0], inv_w, bucket_lut));
        v.blut_base = ends[0]; v.blut_inv_w = inv_w;
    }
    // precursor-mass LUT over peptides[].monoisotopic (sorted ascending; needs positive finite ends like the bucket LUT)
    float pe[2] = {0.f, 0.f};
    if ((rc = read_back(st, &pe[0], v.pep_mono, 4))) return rc;
    if ((rc = read_back(st, &pe[1], v.pep_mono + (v.n_pep - 1), 4))) return rc;
    const float pw = (pe[1] - pe[0]) / (float)PEP_LUT_CELLS;
    bool plut_ok = pe[0] > 0.0f && std::isfinite(pe[1]) && pw > 0.0f && pw < 3.0e38f;
    if (plut_ok) {   // only for a table the reference's binary search is well defined on: ascending, positive, finite
        DevArena A;
        uint32_t* d_bad = nullptr;
        uint32_t h_bad = 1;
        CUDA_TRY(A.zeros(&d_bad, 1, st));
        LAUNCH_N(k_check_ascending, v.n_pep, st, v.n_pep, v.pep_mono, d_bad);
        if ((rc = read_back(st, &h_bad, d_bad, 4))) return rc;
        plut_ok = h_bad == 0;
    }
    if (plut_ok) {
        CUDA_TRY(db->mem.alloc(&pep_lut, PEP_LUT_CELLS + 1));
        LAUNCH(k_build_pep_lut<<<(PEP_LUT_CELLS + 256) / 256, 256, 0, st>>>(v, pe[0], 1.0f / pw, pep_lut));
        v.plut_base = pe[0]; v.plut_inv_w = 1.0f / pw;
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    if (plut_ok) v.pep_lut = pep_lut;
    if (page_grid) v.page_grid = page_grid;
    if (lut_ok) v.bucket_lut = bucket_lut;
    return 0;
}

extern "C" int sage_b200_db_create(const sage_b200_peptides* peptides, const sage_b200_index* index, int device, sage_b200_db** out) {
    if (!out || !index) return fail(SAGE_B200_EINVAL, "db_create: null argument");
    if (index->bucket_size == 0 || index->bucket_size > 0x7FFFFFFFull) return fail(SAGE_B200_EINVAL, "bucket_size out of range");
    if (index->n_fragments && (!index->fragment_peptide || !index->fragment_mz || !index->bucket_min)) return fail(SAGE_B200_EINVAL, "index: null array");
    const uint64_t nb_expect = (index->n_fragments + index->bucket_size - 1) / index->bucket_size;
    if (index->n_buckets != nb_expect) return fail(SAGE_B200_EINVAL, "n_buckets %llu != ceil(n_fragments/bucket_size) %llu", (unsigned long long)index->n_buckets, (unsigned long long)nb_expect);
    Guard<sage_b200_db> guard(nullptr, sage_b200_db_destroy);
    if (int rc = db_new(device, guard)) return rc;
    sage_b200_db* db = guard.get();
    Stream st;
    CUDA_TRY(st.create());
    if (int rc = db_upload_peptides(db, peptides, index->ion_kinds, index->n_ion_kinds, st)) return rc;
    const uint64_t nf = index->n_fragments;
    db->v.n_frag = nf;
    db->v.n_bucket = (uint32_t)index->n_buckets;
    db->v.bucket_size = (uint32_t)index->bucket_size;
    uint2* frag = nullptr;
    float* bucket_min = nullptr;
    CUDA_TRY(db->mem.alloc(&frag, nf + 8));
    CUDA_TRY(db->mem.alloc(&bucket_min, index->n_buckets));
    if (nf) {
        DevArena A;
        uint32_t* t_pep = nullptr;
        float* t_mz = nullptr;
        // these errors are not sticky: a later synchronize would not report them and the index would be garbage
        CUDA_TRY(A.upload(&t_pep, index->fragment_peptide, nf, st));
        CUDA_TRY(A.upload(&t_mz, index->fragment_mz, nf, st));
        CUDA_TRY(cudaMemcpyAsync(bucket_min, index->bucket_min, 4 * index->n_buckets, cudaMemcpyHostToDevice, st));
        LAUNCH_N(k_pack_fragments_soa, nf, st, nf, t_pep, t_mz, frag);
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    db->v.frag = frag;
    db->v.bucket_min = bucket_min;
    // IndexedDatabase does not carry min_ion_index (it lives in Parameters, database.rs:128): infer it from the fragment count and
    // verify the index content against the ion table; only then may narrow windows be counted peptide-centrically.
    db->v.pep_centric_ok = 0;
    db->v.min_ion_index = 0;
    if (peptides->n_peptides && nf) {
        const uint64_t n = peptides->n_peptides;
        int found = -1;
        for (uint32_t m = 0; m <= 64 && found < 0; m++) {
            uint64_t tot = 0;
            for (uint64_t i = 0; i < n; i++) {
                const uint64_t L = peptides->residue_offsets[i + 1] - peptides->residue_offsets[i];
                tot += index->n_ion_kinds * ((L - 1) > m ? (L - 1) - m : 0);
            }
            if (tot == nf) found = (int)m;
            if (tot < nf) break;
        }
        uint32_t mismatch = 1;
        if (found >= 0 && optional_work([&] {   // any failure here only leaves the peptide-centric path off
                DevArena A;
                uint32_t *acc = nullptr, *mis = nullptr;
                CUDA_TRY(A.zeros(&acc, 2 * n, st));
                CUDA_TRY(A.zeros(&mis, 1, st));
                LAUNCH_N(k_index_signature, nf, st, nf, db->v.frag, (uint32_t)n, acc);
                LAUNCH(k_index_verify<<<(unsigned)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, db->v.pep_len, db->v.ion_off, db->v.ions, db->v.n_kinds, db->v,
                                                                                  (uint32_t)found, acc, mis));
                return read_back(st, &mismatch, mis, 4);
            }) && mismatch == 0) {
            db->v.min_ion_index = (uint32_t)found;
            db->v.pep_centric_ok = 1;
        }
    }
    if (int rc = db_build_directories(db, st)) return rc;
    *out = guard.release();
    return 0;
}

// The fragment index of a db whose ion tables are built: fragments kept per peptide at d_off (u64, n + 1; nf in all), the global sort by
// fragment m/z, bucketing, the per-bucket sort by PeptideIx and the search directories (database.rs:281-365), all on st.
static int db_build_fragments(sage_b200_db* db, const uint64_t* d_off, uint64_t nf, uint64_t bucket_size, uint64_t min_ion_index, cudaStream_t st) {
    const uint64_t n = db->v.n_pep;
    const uint32_t shift = ceil_log2_u64(bucket_size);
    const uint64_t nb = (nf + bucket_size - 1) / bucket_size;
    if (nb > 0xFFFFFFFFull) return fail(SAGE_B200_ELIMIT, "too many buckets");
    db->v.n_frag = nf;
    db->v.n_bucket = (uint32_t)nb;
    db->v.bucket_size = (uint32_t)bucket_size;
    db->v.min_ion_index = (uint32_t)std::min<uint64_t>(min_ion_index, 0xFFFFFFFFull);
    db->v.pep_centric_ok = 1;  // the index is generated from the ion table with this filter by construction
    uint2* frag = nullptr;
    float* bucket_min = nullptr;
    CUDA_TRY(db->mem.alloc(&frag, nf + 8));
    CUDA_TRY(db->mem.alloc(&bucket_min, nb));
    db->v.frag = frag;
    db->v.bucket_min = bucket_min;
    if (nf == 0) return 0;
    if (nf > 0x7FFFFFFFull) return fail(SAGE_B200_ELIMIT, "more than 2^31 fragments: sort in slabs not implemented");

    {
        DevArena A;   // freed before the directories are built
        uint32_t *k32b = nullptr, *pb = nullptr;
        CUDA_TRY(A.alloc(&k32b, nf)); CUDA_TRY(A.alloc(&pb, nf));
        {   // (1) stable LSD radix sort by fragment m/z (par_sort_unstable_by fragment_mz, database.rs:301; ties keep PeptideIx order); its
            // inputs are freed before step (2) allocates
            DevArena S;
            uint32_t *k32a = nullptr, *pa = nullptr;
            CUDA_TRY(S.alloc(&k32a, nf)); CUDA_TRY(S.alloc(&pa, nf));
            LAUNCH(k_gen_fragments<<<(unsigned)((n + 127) / 128), 128, 0, st>>>((uint32_t)n, db->v.pep_len, db->v.ion_off, db->v.ions, db->v.n_kinds, db->v,
                                                                               (uint32_t)std::min<uint64_t>(min_ion_index, 0xFFFFFFFFull), nullptr, d_off, k32a, pa));
            CUDA_TRY(S.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, (const uint32_t*)k32a, k32b, (const uint32_t*)pa, pb, (int)nf, 0, 32, st); },
                                 16));
            CUDA_TRY(cudaStreamSynchronize(st));
        }
        // (2) bucket minima + (bucket, PeptideIx) keys, then a stable sort inside buckets (database.rs:337-346)
        uint64_t *k64a = nullptr, *k64b = nullptr;
        uint32_t *mza = nullptr, *mzb = nullptr;
        CUDA_TRY(A.alloc(&k64a, nf)); CUDA_TRY(A.alloc(&k64b, nf));
        CUDA_TRY(A.alloc(&mza, nf)); CUDA_TRY(A.alloc(&mzb, nf));
        LAUNCH_N(k_bucket_keys, nf, st, nf, shift, k32b, pb, k64a, mza, bucket_min);
        const int end_bit = std::min<int>(64, 32 + (int)ceil_log2_u64(nb + 1) + 1);
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, (const uint64_t*)k64a, k64b, (const uint32_t*)mza, mzb, (int)nf, 0, end_bit, st); },
                             16));
        LAUNCH_N(k_pack_fragments, nf, st, nf, k64b, mzb, frag);
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    return db_build_directories(db, st);
}

static int db_check_bucket_size(uint64_t bucket_size) {
    if (bucket_size == 0 || (bucket_size & (bucket_size - 1)) || bucket_size > (1ull << 30))
        return fail(SAGE_B200_EINVAL, "bucket_size must be a power of two (Builder::make_parameters rounds up, database.rs:97)");
    return 0;
}

extern "C" int sage_b200_db_build(const sage_b200_peptides* peptides, uint64_t bucket_size, const uint8_t* ion_kinds, uint64_t n_ion_kinds,
                                  uint64_t min_ion_index, int device, sage_b200_db** out) {
    if (!out || !peptides || !ion_kinds) return fail(SAGE_B200_EINVAL, "db_build: null argument");
    if (int rc = db_check_bucket_size(bucket_size)) return rc;
    Guard<sage_b200_db> guard(nullptr, sage_b200_db_destroy);
    if (int rc = db_new(device, guard)) return rc;
    sage_b200_db* db = guard.get();
    std::vector<uint64_t> frag_off;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    if (int rc = db_upload_peptides(db, peptides, ion_kinds, n_ion_kinds, st)) return rc;
    const uint64_t n = peptides->n_peptides;
    // fragments kept per peptide: n_kinds * max(0, L-1-min_ion_index)   (database.rs:281-291)
    frag_off.resize(n + 1);
    uint64_t nf = 0;
    for (uint64_t i = 0; i < n; i++) {
        frag_off[i] = nf;
        const uint64_t L = peptides->residue_offsets[i + 1] - peptides->residue_offsets[i];
        const uint64_t keep = (L - 1) > min_ion_index ? (L - 1) - min_ion_index : 0;
        nf += n_ion_kinds * keep;
    }
    frag_off[n] = nf;
    uint64_t* d_off = nullptr;
    CUDA_TRY(A.upload(&d_off, frag_off.data(), n + 1, st));
    if (int rc = db_build_fragments(db, d_off, nf, bucket_size, min_ion_index, st)) return rc;
    *out = guard.release();
    return 0;
}

// A peptide table held on the device in the digest's export layout (the prefilter's chunk tables and its merged table).
struct DevTable {
    uint64_t n = 0, n_res = 0, n_ref = 0;
    const uint32_t *res_off = nullptr, *ref_off = nullptr, *ids = nullptr;
    const uint8_t *seq = nullptr, *decoy = nullptr, *missed = nullptr, *semi = nullptr;
    const float *mods = nullptr, *nterm = nullptr, *cterm = nullptr, *mono = nullptr;
    PfRows rows() const { return PfRows{res_off, ref_off, seq, mods, nterm, cterm, mono, decoy, missed, semi, ids}; }
};

// Parameters::build_from_peptides (database.rs:265-365) from a table already on the device: lengths, flags, ion and fragment offsets come
// from kernels and scans, the limits are read back once, and nothing crosses PCIe. The table's work must be finished before the call.
static int db_build_device(const DevTable& T, uint64_t bucket_size, const uint8_t* kinds, uint64_t n_kinds, uint64_t min_ion_index, int device,
                           sage_b200_db** out) {
    if (int rc = db_check_bucket_size(bucket_size)) return rc;
    Guard<sage_b200_db> guard(nullptr, sage_b200_db_destroy);
    if (int rc = db_new(device, guard)) return rc;
    sage_b200_db* db = guard.get();
    if (int rc = db_set_kinds(db, kinds, n_kinds)) return rc;
    if (T.n >= 0xFFFFFFFEull) return fail(SAGE_B200_ELIMIT, "too many peptides for u32 PeptideIx");
    const uint64_t n = T.n;
    db->total_residues = T.n_res;
    PeptideArrays p;
    if (int rc = db_alloc_peptides(db, n, p)) return rc;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    uint64_t *d_nion = nullptr, *d_ion_off = nullptr, *d_nfrag = nullptr, *d_frag_off = nullptr;
    uint32_t* d_bad = nullptr;
    CUDA_TRY(A.zeros(&d_nion, n + 1, st));
    CUDA_TRY(A.zeros(&d_nfrag, n + 1, st));
    CUDA_TRY(A.alloc(&d_ion_off, n + 1));
    CUDA_TRY(A.alloc(&d_frag_off, n + 1));
    CUDA_TRY(A.zeros(&d_bad, 1, st));
    LAUNCH_N(k_pf_pep_meta, n, st, T.res_off, T.decoy, (uint32_t)n, (uint32_t)n_kinds, min_ion_index, p.len, p.flags, d_nion, d_nfrag, d_bad);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_nion, d_ion_off, (int)(n + 1), st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_nfrag, d_frag_off, (int)(n + 1), st); }));
    uint64_t tail[2] = {0, 0};
    uint32_t bad = 0;
    CUDA_TRY(cudaMemcpyAsync(&tail[0], d_ion_off + n, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&tail[1], d_frag_off + n, 8, cudaMemcpyDeviceToHost, st));
    if (int rc = read_back(st, &bad, d_bad, 4)) return rc;
    if (bad) return fail(SAGE_B200_ELIMIT, "a peptide has length 0 or over 255 (supported 1..255)");
    if (tail[0] > 0xFFFFFFFFull) return fail(SAGE_B200_ELIMIT, "ion table exceeds 2^32 entries");
    LAUNCH_N(k_dg_u64_to_u32, n + 1, st, d_ion_off, n + 1, p.ion_off);
    if (n) {
        CUDA_TRY(cudaMemcpyAsync(p.mono, T.mono, 4 * n, cudaMemcpyDeviceToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(p.missed, T.missed, n, cudaMemcpyDeviceToDevice, st));
    }
    if (int rc = db_build_ions(db, n, tail[0], T.res_off, T.seq, T.mods, T.nterm, st)) return rc;
    if (int rc = db_build_fragments(db, d_frag_off, tail[1], bucket_size, min_ion_index, st)) return rc;
    *out = guard.release();
    return 0;
}

extern "C" int sage_b200_db_get_info(const sage_b200_db* db, sage_b200_db_info* info) {
    if (!db || !info) return fail(SAGE_B200_EINVAL, "db_info: null argument");
    info->n_peptides = db->v.n_pep; info->n_fragments = db->v.n_frag; info->n_buckets = db->v.n_bucket; info->bucket_size = db->v.bucket_size;
    info->n_ion_kinds = db->v.n_kinds; info->total_residues = db->total_residues; info->device = db->device;
    {   // + the lazily built block-major copies (open search / narrow search), as far as they exist now
        std::lock_guard<std::mutex> lock(db->wmu);
        info->device_bytes = db->mem.bytes + db->wide.bytes + db->narrow.bytes + db->wide.retired_bytes + db->narrow.retired_bytes;
    }
    return 0;
}

extern "C" int sage_b200_db_export_index(const sage_b200_db* db, uint32_t* fragment_peptide, float* fragment_mz, float* bucket_min) {
    if (!db) return fail(SAGE_B200_EINVAL, "db_export_index: null db");
    CUDA_TRY(cudaSetDevice(db->device));
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    const uint64_t nf = db->v.n_frag;
    if (nf && (fragment_peptide || fragment_mz)) {
        uint32_t* t_pep = nullptr;
        float* t_mz = nullptr;
        CUDA_TRY(A.alloc(&t_pep, nf));
        CUDA_TRY(A.alloc(&t_mz, nf));
        LAUNCH_N(k_unpack_fragments, nf, st, nf, db->v.frag, t_pep, t_mz);
        if (fragment_peptide) CUDA_TRY(cudaMemcpyAsync(fragment_peptide, t_pep, 4 * nf, cudaMemcpyDeviceToHost, st));
        if (fragment_mz) CUDA_TRY(cudaMemcpyAsync(fragment_mz, t_mz, 4 * nf, cudaMemcpyDeviceToHost, st));
    }
    if (bucket_min && db->v.n_bucket) CUDA_TRY(cudaMemcpyAsync(bucket_min, db->v.bucket_min, 4ull * db->v.n_bucket, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

// Both block-major copies of the fragments start alike: fragments keyed by (PeptideIx / block, m/z), one LSD radix sort, block offsets, and
// the m/z range of the index, on st. On success *keys / *peps hold the sorted keys and PeptideIx; every temporary is in A.
static int sort_block_major(const sage_b200_db* db, DevArena& A, cudaStream_t st, uint32_t block, uint32_t n_block, uint64_t* blk_off, uint64_t** keys,
                            uint32_t** peps, float& lo, float& hi) {
    const uint64_t nf = db->v.n_frag;
    if (nf > 0x7FFFFFFFull) return fail(SAGE_B200_ELIMIT, "more than 2^31 fragments");
    uint64_t* k_a = nullptr;
    uint32_t *p_a = nullptr, *d_rng = nullptr;
    CUDA_TRY(A.alloc(&k_a, nf));
    CUDA_TRY(A.alloc(keys, nf));
    CUDA_TRY(A.alloc(&p_a, nf));
    CUDA_TRY(A.alloc(peps, nf));
    LAUNCH_N(k_wide_keys, nf, st, nf, db->v.frag, block, k_a, p_a);
    int nb_bits = 1;
    while (nb_bits < 32 && (n_block >> nb_bits)) nb_bits++;
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, (const uint64_t*)k_a, *keys, (const uint32_t*)p_a, *peps, (int)nf, 0, 32 + nb_bits, st); },
                         16));
    LAUNCH_N(k_wide_block_offsets, (uint64_t)n_block + 1, st, nf, *keys, n_block, blk_off);
    // m/z range of the index (positive floats order like their bit patterns)
    const uint32_t rng0[2] = {0xFFFFFFFFu, 0u};
    CUDA_TRY(A.upload(&d_rng, rng0, 2, st));
    LAUNCH(k_frag_mz_range<<<(unsigned)std::min<uint64_t>((nf + 255) / 256, 4096), 256, 0, st>>>(nf, db->v.frag, d_rng));
    uint32_t rng[2];
    if (int rc = read_back(st, rng, d_rng, 8)) return rc;
    memcpy(&lo, &rng[0], 4); memcpy(&hi, &rng[1], 4);
    return 0;
}

// Directory cells of `cells` equal m/z steps over [lo, hi] (the same for every block): base and inverse width, or inv_w = 0 (every walk
// starts at the block start) when the range is degenerate.
template <class View>
static void set_mz_cells(View& v, float lo, float hi, uint32_t cells) {
    v.cells = cells;
    const float width = (hi - lo) / (float)cells;
    v.base = (std::isfinite(lo) && lo > 0.0f) ? lo : 0.0f;
    v.inv_w = (std::isfinite(width) && width > 0.0f && lo > 0.0f) ? 1.0f / width : 0.0f;
}

// Secondary index for open search (device_common.cuh: WideIndexView): the sorted fragments as {PeptideIx, m/z} and a per-block u32 m/z LUT.
// `block` = the scorer's count-tile size. Returns a view with frag == nullptr when the index cannot be built (out of memory,
// SAGE_B200_NO_WIDE_INDEX=1): k_prelim_wide then streams the page slices as the reference does. wmu must be held.
static WideIndexView build_wide_index(const sage_b200_db* db, BlockIndexSlot<WideIndexView>& slot, uint32_t block, uint32_t cells) {
    if (slot.v.frag != nullptr && slot.v.block == block) return slot.v;
    if (slot.failed || block == 0 || db->v.n_frag == 0 || db->v.n_pep == 0) return WideIndexView{};
    const uint64_t nf = db->v.n_frag;
    const uint32_t n_block = (db->v.n_pep + block - 1) / block;
    while (cells > 256 && (uint64_t)n_block * (cells + 1) * 4 > (1024ull << 20)) cells >>= 1;   // at most 1 GB of LUT
    // a rebuild with another block size (tests, scorers with very different tolerances): see BlockIndexSlot::retire
    return slot.rebuild([&](DevArena& mem, WideIndexView& w, uint64_t& bytes) -> int {
        DevArena A;
        Stream st;
        CUDA_TRY(st.create());
        uint2* frag = nullptr;
        uint64_t *blk = nullptr, *keys = nullptr;
        uint32_t *lut = nullptr, *peps = nullptr;
        CUDA_TRY(mem.alloc(&frag, nf + 8));
        CUDA_TRY(mem.alloc(&blk, (uint64_t)n_block + 1));
        CUDA_TRY(mem.alloc(&lut, (uint64_t)n_block * (cells + 1)));
        float lo, hi;
        if (int rc = sort_block_major(db, A, st, block, n_block, blk, &keys, &peps, lo, hi)) return rc;
        LAUNCH_N(k_wide_pack, nf, st, nf, keys, peps, frag);
        w.frag = frag; w.blk_off = blk; w.lut = lut;
        w.block = block; w.n_block = n_block;
        set_mz_cells(w, lo, hi, cells);
        const uint64_t total = (uint64_t)n_block * (cells + 1);
        if (w.inv_w > 0.0f) LAUNCH_N(k_wide_lut, total, st, w, lut);
        else CUDA_TRY(cudaMemsetAsync(lut, 0, 4 * total, st));   // degenerate range: every walk starts at the block start
        CUDA_TRY(cudaStreamSynchronize(st));
        bytes = 8 * nf + 8 * ((uint64_t)n_block + 1) + 4ull * n_block * (cells + 1);
        return 0;
    });
}

static WideIndexView db_wide_index(const sage_b200_db* db, uint32_t block) {
    std::lock_guard<std::mutex> lock(db->wmu);
    if (const char* e = getenv("SAGE_B200_NO_WIDE_INDEX")) if (e[0] == '1') return WideIndexView{};   // A/B + tests: stream the page slices instead
    // ~2 M entries per 80 k-peptide block, most of them inside a third of the m/z range: 2^18 cells leave a few dozen entries per cell there,
    // so the conservative (one cell early) start of a walk costs about one extra 32-entry fetch (measured: 2^16 cells -> ~8 extra fetches)
    return build_wide_index(db, db->wide, block, 1u << 18);
}

// Directory cells of the narrow copy: the power of two at or above twice the mean block's entries, 1024..32768 (cfg2: 16384 cells for 6 660
// entries per 256-peptide block; cfg3: 85 k entries per 2048-peptide block, capped at 32768 = 0.5 GB of directory). Measured on cfg2 (H100
// SXM, 700 W; counting kernel, ms): 1 cell per entry 0.638, 2 cells 0.582, 4 cells 0.615 — a start one coarse cell early walks more entries.
// The directory is held to 1 GB (halving the cells), which only small blocks over a large index reach: e.g. cfg3's 678 M fragments in blocks
// of 256 peptides get 8192 cells per block (1.0 GB) instead of 32768 (4.2 GB).
constexpr uint64_t NARROW_CELLS_PER_ENTRY = 2;
static uint32_t narrow_dir_cells(uint64_t n_frag, uint32_t n_block) {
    const uint64_t per_block = n_block ? n_frag / n_block : 0;
    uint32_t cells = 1024;
    while (cells < 32768u && (uint64_t)cells < per_block * NARROW_CELLS_PER_ENTRY) cells <<= 1;
    while (cells > 1024u && 2ull * n_block * cells > (1024ull << 20)) cells >>= 1;
    return cells;
}

// The narrow-search copy (device_common.cuh: NarrowIndexView), blocks of `block` peptides (a +-20 ppm window holds a few hundred). Returns a
// view with mz == nullptr when it cannot be built (out of memory): the narrow kernels then probe the page index. An automatically sized
// request (!exact) accepts an existing copy whose blocks are within a factor of two (scorers with different tolerances sharing one index must
// not rebuild it in turns).
static NarrowIndexView db_narrow_index(const sage_b200_db* db, uint32_t block, bool exact) {
    std::lock_guard<std::mutex> lock(db->wmu);
    BlockIndexSlot<NarrowIndexView>& slot = db->narrow;
    if (slot.v.mz != nullptr && (slot.v.block == block || (!exact && slot.v.block * 2 >= block && slot.v.block <= block * 2))) return slot.v;
    if (slot.failed || block == 0 || block > 65536 || db->v.n_frag == 0 || db->v.n_pep == 0) return NarrowIndexView{};
    const uint64_t nf = db->v.n_frag;
    const uint32_t n_block = (db->v.n_pep + block - 1) / block;
    const uint32_t cells = narrow_dir_cells(nf, n_block), ngrp = cells / NARROW_GROUP;
    return slot.rebuild([&](DevArena& mem, NarrowIndexView& v, uint64_t& bytes) -> int {
        DevArena A;
        Stream st;
        CUDA_TRY(st.create());
        float* mz = nullptr;
        uint16_t *pep = nullptr, *dir = nullptr;
        uint64_t *blk = nullptr, *keys = nullptr;
        uint32_t *grp = nullptr, *peps = nullptr;
        const uint64_t total = (uint64_t)n_block * cells;
        CUDA_TRY(mem.alloc(&mz, nf + 16));
        CUDA_TRY(mem.alloc(&pep, nf + 32));
        CUDA_TRY(mem.alloc(&blk, (uint64_t)n_block + 1));
        CUDA_TRY(mem.alloc(&dir, total));
        CUDA_TRY(mem.alloc(&grp, (uint64_t)n_block * ngrp));
        float lo, hi;
        if (int rc = sort_block_major(db, A, st, block, n_block, blk, &keys, &peps, lo, hi)) return rc;
        LAUNCH_N(k_narrow_pack, nf, st, nf, keys, peps, block, mz, pep);
        v.mz = mz; v.pep = pep; v.blk_off = blk; v.dir = dir;
        v.grp = grp; v.block = block; v.n_block = n_block;
        set_mz_cells(v, lo, hi, cells);
        LAUNCH_N(k_narrow_dir, total, st, v, dir, grp);
        CUDA_TRY(cudaStreamSynchronize(st));
        bytes = mem.bytes;
        return 0;
    });
}

// Dynamic shared-memory opt-in of the kernels that need more than 48 KB: set ONCE per device to the device maximum (the attribute is per-function,
// per-device state; setting it per launch to the launch's own size would let two scorers with different shapes undo each other's setting).
static int ensure_kernel_attributes(int device) {
    static std::mutex mu;
    static bool done[64] = {};
    std::lock_guard<std::mutex> lock(mu);
    if (device >= 0 && device < 64 && done[device]) return 0;
    int optin = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    auto raise = [&](const void* fn) -> cudaError_t {   // dynamic limit = opt-in maximum minus the kernel's static shared memory
        cudaFuncAttributes fa;
        cudaError_t e = cudaFuncGetAttributes(&fa, fn);
        if (e != cudaSuccess) return e;
        return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
    };
    CUDA_TRY(raise((const void*)k_prelim_narrow));
    CUDA_TRY(raise((const void*)k_replay<true>));
    CUDA_TRY(raise((const void*)k_replay<false>));
    CUDA_TRY(raise((const void*)k_prelim_wide));
    CUDA_TRY(raise((const void*)k_score<false>));
    CUDA_TRY(raise((const void*)k_score<true>));
    CUDA_TRY(raise((const void*)k_process_ms2));
    if (device >= 0 && device < 64) done[device] = true;
    return 0;
}

// One step of the xorshift64 generator that draws the inputs of the host libm probes below.
static uint64_t xorshift64(uint64_t& s) {
    s ^= s << 13;
    s ^= s >> 7;
    s ^= s << 17;
    return s;
}

// Which build of glibc's log() is the host libm (glibc_log.cuh)? Both variants are evaluated on the CPU and compared with std::log bit for bit
// on a few thousand inputs of the kinds the path feeds it: hyperscore products, lambda, arguments near 1 (the only region where the two
// variants differ). Returns 0 (FMA-contracted), 1 (plain), or -1 when neither matches (non-glibc libm: the device then uses variant 0 and
// hyperscore / poisson agree with the host to <= 1 ulp instead of bit for bit).
extern "C" int sage_b200_host_log_variant(void) {
    static const int variant = []() {   // initialised once, thread-safe
        uint64_t st = 0x9E3779B97F4A7C15ull;
        bool ok[2] = {true, true};
        for (int i = 0; i < 6000; i++) {
            const uint64_t u = xorshift64(st);
            double x;
            switch (i % 3) {
                case 0: x = (double)((float)(u & 0xffffff) * 0.37f + 1.0f) * (double)((float)((u >> 24) & 0xffffff) * 1.91f + 1.0f); break;
                case 1: x = 0.93 + (double)(u >> 11) * 0x1p-53 * 0.15; break;
                default: x = (double)(u >> 11) * 0x1p-53 * 64.0; break;
            }
            volatile double vx = x;   // keep the compiler from folding std::log
            const double ref = std::log(vx);
            const double a = glog::glibc_log<true>(x), b = glog::glibc_log<false>(x);
            if (memcmp(&a, &ref, 8)) ok[0] = false;
            if (memcmp(&b, &ref, 8)) ok[1] = false;
        }
        return ok[0] ? 0 : (ok[1] ? 1 : -1);
    }();
    return variant;
}

// 1 when the host libm's log1pf (Rust's f32::ln_1p, OpenMS hyperscore) is the fdlibm/glibc function the kernels reproduce (glibc_log.cuh).
extern "C" int sage_b200_host_log1pf_exact(void) {
    static const int exact = []() {   // initialised once, thread-safe
        uint64_t st = 0x2545F4914F6CDD1Dull;
        for (int i = 0; i < 20000; i++) {
            const uint64_t u = xorshift64(st);
            float x;
            switch (i % 3) {
                case 0: x = (float)(u & 0xffffff) * 3.7f; break;                                  // summed intensities
                case 1: x = (float)((double)(u >> 11) * 0x1p-53 * 2.0 - 0.9); break;            // around the branch points
                default: { uint32_t b = (uint32_t)(u >> 33); memcpy(&x, &b, 4); break; }          // any non-negative float
            }
            volatile float vx = x;
            const float ref = log1pf(vx), got = glog::glibc_log1pf(x);
            if (memcmp(&ref, &got, 4) && !(ref != ref && got != got)) return 0;
        }
        return 1;
    }();
    return exact;
}

// ------------------------------------------------------------------------------------------------ scorer
constexpr int MASS_PARTS = 4;   // the masses copy of a chunk is cut into at most this many parts, each followed by its own counting launch

struct ChunkState {
    bool loaded = false;
    uint32_t nparts = 1, part_lo[MASS_PARTS + 1] = {0, 0, 0, 0, 0};   // spectra [part_lo[p], part_lo[p+1]) belong to part p of the masses copy
    uint32_t n = 0, pmax = 2, zmax = 1, base = 0;
    uint64_t npk = 0;
    size_t nitems = 0, smem = 0, small_bytes = 0;
    size_t o_off = 0, o_pmz = 0, o_tic = 0, o_ilo = 0, o_ihi = 0, o_rt = 0, o_ims = 0, o_chg = 0;
    bool timed_upload = false;
    uint64_t hits_cap = 0, force_hits = 0;   // split scoring: entries of the hit arena / exact need of a re-run
    uint64_t nlist_cap = 0, force_nlist = 0, force_wide = 0;   // work-list capacities of the current attempt / exact needs for a re-run
    uint32_t wide_cap = 0;
    double t_issue0 = 0, t_issue1 = 0;   // host time (ms since the call started) when queueing this chunk began / ended (trace only)
};

// One in-flight chunk: its own stream, device buffers, pinned staging and pending-download bookkeeping. score_batch alternates
// between two lanes so that the H2D copy of chunk i+1 and the D2H of chunk i-1 overlap the kernels of chunk i.
struct Lane {
    Stream stream;   // kernels + D2H
    Stream copy;     // H2D: masses first (all the counting kernels need), intensities behind them, overlapping setup + preliminary scoring
    // No work is ever queued on `spare`, but creating it keeps the lane streams' creation order: without it the second lane's streams come
    // one position earlier, and cfg4's score_batch (open search, several chunks over both lanes) measured about 2 % slower end to end on an
    // H100 80GB HBM3 at 700 W, kernels unchanged. The driver hands out hardware work queues to streams in creation order.
    Stream spare;
    // stage boundaries of the chunk in flight: its timings (counters, SAGE_B200_TRACE) and the wait on the other lane's k_score
    Event ev_h2d_begin, ev_h2d_end, ev_run, ev_setup_end, ev_count_end, ev_replay_end, ev_score_end, ev_d2h_begin, ev_d2h_end;
    Event ev_masses, ev_intens, ev_small;
    Event ev_part[MASS_PARTS];   // masses of the spectra [part_lo[p], part_lo[p+1]) are on the device
    DevBuf d_small, d_masses, d_intens, d_queries, d_hits, d_keys, d_features, d_counts, d_counters, d_dbgk, d_dbgm, d_sort, d_sorttmp, d_wlist, d_wslots,
        d_witems, d_citems, d_nlist, d_nslots;
    PinBuf h_small, h_masses, h_intens, h_features, h_counts, h_counters;
    DevBuf d_frags;
    DevBuf d_cand, d_meta, d_recs, d_hkey, d_emit, d_hitk, d_hiti, d_hitt;   // split scoring (k_score<true> -> k_fold -> k_features)
    ChunkState chunk;
    // pending work of the chunk in flight
    bool ran = false, downloading = false, dbg = false;
    uint64_t launches = 0;
    sage_b200_feature* fdst = nullptr;
    uint32_t* cdst = nullptr;
    bool f_pinned = false, c_pinned = false;
    // helper thread staging the intensities of a chunk whose caller arrays are pageable (chunk_upload starts it, chunk_run joins it)
    std::thread stager;
    std::unique_ptr<StagePool> pool{new StagePool};   // copy threads of staged_h2d (started by the first pageable chunk)
    int stager_rc = 0;
    char stager_msg[256] = {0};
    cudaError_t create() {
        for (Stream* s : {&stream, &copy, &spare})
            if (cudaError_t e = s->create()) return e;
        for (Event* ev : {&ev_h2d_begin, &ev_h2d_end, &ev_run, &ev_setup_end, &ev_count_end, &ev_replay_end, &ev_score_end, &ev_d2h_begin, &ev_d2h_end, &ev_masses,
                          &ev_intens, &ev_small})
            if (cudaError_t e = ev->create()) return e;
        for (Event& ev : ev_part)
            if (cudaError_t e = ev.create()) return e;
        return cudaSuccess;
    }
    ~Lane() { if (stager.joinable()) stager.join(); }   // the staging thread uses the stream, the pinned buffers and the pool
};

struct sage_b200_scorer {
    const sage_b200_db* db = nullptr;
    int device = 0;   // copy of db->device: scorer_destroy must not touch a db that was destroyed first
    sage_b200_scorer_params params{};
    ScorerView sv{};
    std::mutex mu;
    Lane lanes[2];
    DevBuf d_lnfact, d_keep;
    uint32_t quick_mode = 0;   // != 0 only inside sage_b200_quick_score
    int sort_spectra = 1;
    // annotate_matches: caller's fragment array for the current call and the running global offset
    sage_b200_fragment* frag_dst = nullptr;
    uint64_t frag_cap = 0, frag_used = 0;
    int pipeline_chunks = 1;   // score_batch cuts a batch into at least this many chunks (tuning / tests; large batches are cut at 65536 spectra anyway)
    // learned work-list sizes (per spectrum of a chunk): narrow key-list arena entries and open-search queries. A chunk that needs more than
    // its capacity is re-run once with the exact sizes it counted, and the estimates grow.
    double nlist_per_spectrum = 512.0, wide_per_spectrum = 0.0;
    // narrow windows are counted against the small-block copy of the index (block_probe) unless narrow_index == 0: then the reference's loop
    // order probes the page index and the page / entry work counters are produced (tests, bench's work_per_step pass)
    int score_split = 1;            // non-chimeric scoring runs as k_score<true> -> k_fold -> k_features -> k_rows (0: the fused kernel; tests compare both)
    double hits_per_spectrum = 0.0; // learned: hit-arena entries (= scoring tasks) a spectrum needs
    int narrow_index = 1;
    uint32_t narrow_block_auto = 0;   // block size narrow_block_for chose for this scorer's precursor tolerance
    int narrow_cta = 1;   // windows of WARPQ_CAP+1..NARROW_CAP peptides (one CTA per query) use the copy too
    uint32_t narrow_block = 0;   // 0 = sized by the average precursor window, see narrow_block_for
    int mass_parts = 2;        // chosen by A/B on cfg2 (e2e) against 1, 3 and 4 parts
    int first_chunk_pct = 0;   // chosen by A/B on cfg2 (e2e) against 10..35 %
    // SAGE_B200_TRACE=1: per-chunk device timeline (ms since the start of the call) on stderr
    bool trace = false;
    Event ev_base;
    std::chrono::steady_clock::time_point t_base;
    sage_b200_counters last{};
};

extern "C" int sage_b200_scorer_create(const sage_b200_db* db, const sage_b200_scorer_params* p, sage_b200_scorer** out) {
    if (!db || !p || !out) return fail(SAGE_B200_EINVAL, "scorer_create: null argument");
    if (p->report_psms == 0) return fail(SAGE_B200_EINVAL, "report_psms must be >= 1");
    if (p->report_psms > K_MAX / 2) return fail(SAGE_B200_ELIMIT, "report_psms %u > %d not supported", p->report_psms, K_MAX / 2);
    if (p->precursor_tol.kind < 0 || p->precursor_tol.kind > 2 || p->fragment_tol.kind < 0 || p->fragment_tol.kind > 2) return fail(SAGE_B200_EINVAL, "bad tolerance kind");
    if (p->score_type > 1) return fail(SAGE_B200_EINVAL, "bad score_type");
    CUDA_TRY(cudaSetDevice(db->device));
    if (int rc = ensure_kernel_attributes(db->device)) return rc;
    Guard<sage_b200_scorer> guard(new sage_b200_scorer(), sage_b200_scorer_destroy);
    sage_b200_scorer* s = guard.get();
    s->db = db;
    s->device = db->device;
    s->params = *p;
    ScorerView& v = s->sv;
    v.precursor_tol = {p->precursor_tol.kind, p->precursor_tol.lo, p->precursor_tol.hi};
    v.fragment_tol = {p->fragment_tol.kind, p->fragment_tol.lo, p->fragment_tol.hi};
    v.min_matched_peaks = p->min_matched_peaks;
    v.min_iso = p->min_isotope_err; v.max_iso = p->max_isotope_err;
    v.min_charge = p->min_precursor_charge; v.max_charge = p->max_precursor_charge;
    v.override_charge = p->override_precursor_charge; v.max_fragment_charge_opt = p->max_fragment_charge;
    v.chimera = p->chimera; v.wide_window = p->wide_window; v.annotate = p->annotate_matches; v.score_type = p->score_type;
    v.report_psms = p->report_psms;
    v.kparam = std::max<uint32_t>(50, 2 * p->report_psms);  // trim_hits (scoring.rs:323-326): k = min(len, max(50, 2*report_psms))
    v.n_iso = (v.min_iso != v.max_iso) ? (uint32_t)std::max(0, v.max_iso - v.min_iso + 1) : 1;
    v.n_ch_max = v.max_charge >= v.min_charge ? v.max_charge - v.min_charge + 1 : 0;
    if (v.n_ch_max < 1) v.n_ch_max = 1;  // known-charge spectra still need one slot
    if (v.n_iso > 32 || v.n_ch_max > 16) return fail(SAGE_B200_ELIMIT, "isotope range > 32 or charge range > 16 not supported");
    v.qmax = std::max<uint32_t>(1, v.n_iso) * v.n_ch_max;
    v.lcap = std::max<uint32_t>(std::max<uint32_t>(v.n_iso, v.n_ch_max), 1) * v.kparam;
    v.wide_tile = WIDE_TILE;
    v.wide_lmax = WIDE_LMAX;
    v.wide_variant = 0;  // float compares measured faster than the unsigned bit-window on cfg4
    if (const char* e = getenv("SAGE_B200_WIDE_VARIANT")) v.wide_variant = (uint32_t)atoi(e);
    v.pep_cap = 0;   // peptide-centric counting of small windows is opt-in: with the dense page grid the index path won on cfg2 at every cap tried
    if (const char* e = getenv("SAGE_B200_PEP_CAP")) v.pep_cap = (uint32_t)std::min<long>(std::max<long>(atol(e), 0), (long)NARROW_CAP);
    for (Lane& L : s->lanes) CUDA_TRY(L.create());
    {   // lnfact table with the host libm (the reference's f64::ln): Stirling form of scoring.rs:170-177
        const uint32_t N = 4096;
        std::vector<double> tab(N);
        tab[0] = 1.0;
        for (uint32_t n = 1; n < N; n++) {
            const double x = (double)n;
            tab[n] = x * std::log(x) - x + 0.5 * std::log(x) + 0.5 * std::log(3.14159265358979323846 * 2.0 * x);
        }
        if (int rc = s->d_lnfact.reserve(8 * N)) return rc;
        CUDA_TRY(cudaMemcpyAsync(s->d_lnfact.p, tab.data(), 8 * N, cudaMemcpyHostToDevice, s->lanes[0].stream));
        CUDA_TRY(cudaStreamSynchronize(s->lanes[0].stream));   // both lanes read the table
        v.lnfact_tab = s->d_lnfact.as<double>();
        v.lnfact_n = N;
    }
    v.log_variant = (uint32_t)std::max(0, sage_b200_host_log_variant());
    v.score_fast = 1;
    if (const char* e = getenv("SAGE_B200_SCORE_FAST")) v.score_fast = atoi(e) != 0;
    if (const char* e = getenv("SAGE_B200_SORT")) s->sort_spectra = atoi(e);
    if (const char* e = getenv("SAGE_B200_PIPELINE_CHUNKS")) s->pipeline_chunks = std::max(1, atoi(e));
    if (const char* e = getenv("SAGE_B200_TRACE")) s->trace = e[0] == '1';
    if (const char* e = getenv("SAGE_B200_SCORE_SPLIT")) s->score_split = atoi(e) != 0;
    if (const char* e = getenv("SAGE_B200_NARROW_INDEX")) s->narrow_index = atoi(e) != 0;
    if (const char* e = getenv("SAGE_B200_NARROW_CTA")) s->narrow_cta = atoi(e) != 0;
    if (const char* e = getenv("SAGE_B200_NARROW_BLOCK")) s->narrow_block = (uint32_t)std::min(65536, std::max(0, atoi(e)));   // 0 or 64..65536 (u16 offsets)
    if (s->narrow_block != 0 && s->narrow_block < 64) s->narrow_block = 64;
    if (const char* e = getenv("SAGE_B200_MASS_PARTS")) s->mass_parts = std::min(MASS_PARTS, std::max(1, atoi(e)));
    if (const char* e = getenv("SAGE_B200_FIRST_CHUNK_PCT")) s->first_chunk_pct = std::min(50, std::max(0, atoi(e)));
    CUDA_TRY(s->ev_base.create());
    *out = guard.release();
    return 0;
}

extern "C" int sage_b200_scorer_set_option(sage_b200_scorer* s, const char* name, int64_t value) {
    if (!s || !name) return fail(SAGE_B200_EINVAL, "scorer_set_option: null argument");
    std::lock_guard<std::mutex> lock(s->mu);
    if (!strcmp(name, "sort_spectra")) { s->sort_spectra = value != 0; return 0; }
    if (!strcmp(name, "pipeline_chunks")) { s->pipeline_chunks = (int)std::max<int64_t>(1, value); return 0; }
    if (!strcmp(name, "score_split")) { s->score_split = value != 0; return 0; }
    if (!strcmp(name, "narrow_index")) { s->narrow_index = value != 0; return 0; }
    if (!strcmp(name, "narrow_block")) {   // test hook: peptides per block of the narrow-search copy (rebuilds it on the next batch)
        if (value != 0 && (value < 64 || value > 65536)) return fail(SAGE_B200_EINVAL, "narrow_block must be 0 (automatic) or 64..65536");
        s->narrow_block = (uint32_t)value;
        return 0;
    }
    if (!strcmp(name, "mass_parts")) {
        if (value < 1 || value > MASS_PARTS) return fail(SAGE_B200_EINVAL, "mass_parts must be 1..%d", MASS_PARTS);
        s->mass_parts = (int)value;
        return 0;
    }
    if (!strcmp(name, "wide_lmax")) {  // test hook: a tiny survivor list forces the overflow -> in-kernel serial replay path
        if (value < (int64_t)K_MAX || value > (int64_t)WIDE_LMAX) return fail(SAGE_B200_EINVAL, "wide_lmax must be in %d..%u", K_MAX, WIDE_LMAX);
        s->sv.wide_lmax = (uint32_t)value;
        return 0;
    }
    if (!strcmp(name, "wide_tile")) {  // test hook: smaller tiles exercise the multi-tile path on small databases
        if (value < 256 || value > (int64_t)WIDE_TILE || (value & 1)) return fail(SAGE_B200_EINVAL, "wide_tile must be even and in 256..%u", WIDE_TILE);
        s->sv.wide_tile = (uint32_t)value;
        return 0;
    }
    if (!strcmp(name, "worklist_reset")) {   // test hook: forget the learned work-list sizes; value = narrow arena entries per spectrum to start from
        if (value < 0) return fail(SAGE_B200_EINVAL, "worklist_reset takes a non-negative entry count");
        s->nlist_per_spectrum = (double)value;
        s->wide_per_spectrum = 0.0;
        s->hits_per_spectrum = value > 0 ? (double)value : 0.0;   // > 0: start the split scorer's hit arena at that many entries per spectrum too
        return 0;
    }
    if (!strcmp(name, "score_fast")) {  // 0: k_score always takes the generic task body (tests compare both)
        s->sv.score_fast = value != 0;
        return 0;
    }
    if (!strcmp(name, "log_variant")) {  // test hook: 0 = glibc log() as built with FMA contraction, 1 = without (default: whichever the host libm is)
        if (value < 0 || value > 1) return fail(SAGE_B200_EINVAL, "log_variant must be 0 or 1");
        s->sv.log_variant = (uint32_t)value;
        return 0;
    }
    if (!strcmp(name, "pep_cap")) {  // 0 (default) = always probe the fragment index (reference loop order)
        if (value < 0 || value > (int64_t)NARROW_CAP) return fail(SAGE_B200_EINVAL, "pep_cap must be 0..%u", NARROW_CAP);
        s->sv.pep_cap = (uint32_t)value;
        return 0;
    }
    return fail(SAGE_B200_EINVAL, "unknown option '%s'", name);
}

extern "C" void sage_b200_scorer_destroy(sage_b200_scorer* s) {
    if (!s) return;
    cudaSetDevice(s->device);
    delete s;
}

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Peptides per block of the narrow-search copy of the index: the power of two at or above the average precursor window of this scorer
// (sampled on the device from the peptide masses themselves), 128..4096. A probe then reads one or two short m/z runs. Chosen by A/B of the
// counting kernels on cfg2 (windows ~180 peptides: 256 best) and cfg3 (windows ~1500: 2048 best), both well ahead of the page index.
// The sample runs on lane 0's kernel stream.
static int narrow_block_for(sage_b200_scorer* S) {
    if (S->narrow_block_auto) return 0;
    const uint32_t samples = 4096;
    cudaStream_t st = S->lanes[0].stream;
    DevArena A;
    unsigned long long* d_sum = nullptr;
    unsigned long long sum = 0;
    CUDA_TRY(A.zeros(&d_sum, 1, st));
    LAUNCH_N(k_window_sample, samples, st, S->db->v, S->sv.precursor_tol, samples, d_sum);
    if (int rc = read_back(st, &sum, d_sum, 8)) return rc;
    const double avg = (double)sum / samples;
    uint32_t block = 128;
    while (block < 4096 && (double)block < avg) block <<= 1;
    S->narrow_block_auto = block;
    return 0;
}

// Waits for the lane's staging thread (if one is running) and reports its error as this thread's.
static int lane_join_stager(Lane& L) {
    if (!L.stager.joinable()) return 0;
    L.stager.join();
    if (L.stager_rc) return fail(L.stager_rc, "%s", L.stager_msg);
    return 0;
}

// ---- one chunk of spectra through the device pipeline, in three phases:
//   chunk_upload   pack + H2D (spectra become device-resident)
//   chunk_run      k_setup_queries -> k_prelim_{narrow,wide} -> k_score (results stay on the device)
//   chunk_download D2H of Feature rows + counts
static int chunk_upload(sage_b200_scorer* S, Lane& L, const sage_b200_spectra* sp, uint64_t c0, uint64_t c1) {
    const ScorerView& sv = S->sv;
    ChunkState& C = L.chunk;
    C.loaded = false;
    const uint32_t n = (uint32_t)(c1 - c0);
    const uint64_t pk0 = sp->peak_offsets[c0], pk1 = sp->peak_offsets[c1];
    const uint64_t npk = pk1 - pk0;
    if (npk > 0xFFFFFFF0ull) return fail(SAGE_B200_ELIMIT, "chunk has too many peaks");
    C.n = n; C.npk = npk; C.base = (uint32_t)c0;
    // small per-spectrum arrays -> one pinned blob -> one H2D
    C.o_off = 0;
    C.o_pmz = align_up(C.o_off + 4 * (size_t)(n + 1), 16);
    C.o_tic = align_up(C.o_pmz + 4 * (size_t)n, 16);
    C.o_ilo = align_up(C.o_tic + 4 * (size_t)n, 16);
    C.o_ihi = align_up(C.o_ilo + 4 * (size_t)n, 16);
    C.o_rt = align_up(C.o_ihi + 4 * (size_t)n, 16);
    C.o_ims = align_up(C.o_rt + 4 * (size_t)n, 16);
    C.o_chg = align_up(C.o_ims + 4 * (size_t)n, 16);
    C.small_bytes = align_up(C.o_chg + n, 16);
    int rc;
    if ((rc = L.h_small.reserve(C.small_bytes))) return rc;
    if ((rc = L.d_small.reserve(C.small_bytes))) return rc;
    if ((rc = L.d_masses.reserve(4 * npk + 16))) return rc;
    if ((rc = L.d_intens.reserve(4 * npk + 16))) return rc;
    // Copy order on the lane's copy stream (one DMA queue, served in issue order):
    //   pinned caller arrays:   first quarter of the peak masses (needs no host preparation; in flight while the per-spectrum arrays are
    //                           validated and packed) -> per-spectrum blob -> rest of the masses -> intensities.  k_setup_queries + the
    //                           precursor sort need only the blob, so they run under the rest of the masses copy instead of after it.
    //   pageable caller arrays: blob first (the host, not the link, is the bottleneck: nothing is lost by packing before the first DMA),
    //                           then the masses through the staging buffer, then the intensities staged by a helper thread while this
    //                           thread already queues the kernels (chunk_run joins it before k_score is queued).
    cudaStream_t cp = L.copy;
    if ((rc = lane_join_stager(L))) return rc;
    CUDA_TRY(cudaEventRecord(L.ev_h2d_begin, cp));
    const float* src_m = sp->masses + pk0;
    const float* src_i = sp->intensities + pk0;
    const bool pin_m = npk == 0 || is_pinned(src_m), pin_i = npk == 0 || is_pinned(src_i);
    // Pinned masses are also cut into `nparts` runs of spectra (caller order), each followed by its own event: the counting kernel is queued
    // once per part and starts on part p while part p + 1 is still in flight (it walks its spectra in precursor order either way).
    C.nparts = (pin_m && npk > (1u << 21) && n >= 4096) ? (uint32_t)S->mass_parts : 1u;
    for (uint32_t q = 0; q <= C.nparts; q++) C.part_lo[q] = (uint32_t)((uint64_t)n * q / C.nparts);
    // (clamped: the offsets are only validated by pack() below, and a copy must never leave the caller's array)
    auto part_off = [&](uint32_t q) -> uint64_t { const uint64_t o = sp->peak_offsets[c0 + C.part_lo[q]]; return o < pk0 ? 0 : std::min(o - pk0, npk); };
    // floats of the masses sent ahead of the blob: half of part 0 (a quarter of everything when there is one part)
    const uint64_t npk_a = !pin_m ? 0 : (npk > (1u << 21) ? (C.nparts > 1 ? part_off(1) / 2 : npk / 4) : npk);
    if (npk_a) CUDA_TRY(cudaMemcpyAsync(L.d_masses.p, src_m, 4 * npk_a, cudaMemcpyHostToDevice, cp));
    unsigned char* hs = (unsigned char*)L.h_small.p;
    auto pack = [&]() -> int {   // small per-spectrum arrays -> one pinned blob -> one H2D
        uint32_t* h_off = (uint32_t*)(hs + C.o_off);
        uint32_t pmax = 2, zmax = sv.max_charge;
        for (uint32_t i = 0; i <= n; i++) h_off[i] = (uint32_t)(sp->peak_offsets[c0 + i] - pk0);
        for (uint32_t i = 0; i < n; i++) {
            zmax = std::max<uint32_t>(zmax, sp->precursor_charge[c0 + i]);
            if (sp->peak_offsets[c0 + i + 1] < sp->peak_offsets[c0 + i]) return fail(SAGE_B200_EINVAL, "peak_offsets not monotone at spectrum %llu", (unsigned long long)(c0 + i));
            pmax = std::max(pmax, h_off[i + 1] - h_off[i]);
            if (sp->level && sp->level[c0 + i] != 2)
                return fail(SAGE_B200_ENOTMS2, "internal bug, trying to score a non-MS2 scan! (spectrum %llu has level %u)", (unsigned long long)(c0 + i), sp->level[c0 + i]);
            if (std::isnan(sp->precursor_mz[c0 + i])) return fail(SAGE_B200_ENOPRECURSOR, "missing MS1 precursor for spectrum %llu", (unsigned long long)(c0 + i));
        }
        C.pmax = (pmax + 3) & ~3u;   // multiple of 4 floats: the staged copies in k_score are 16-byte granular
        C.zmax = zmax;
        memcpy(hs + C.o_pmz, sp->precursor_mz + c0, 4 * (size_t)n);
        memcpy(hs + C.o_tic, sp->total_ion_current + c0, 4 * (size_t)n);
        float* h_ilo = (float*)(hs + C.o_ilo);
        float* h_ihi = (float*)(hs + C.o_ihi);
        float* h_rt = (float*)(hs + C.o_rt);
        float* h_ims = (float*)(hs + C.o_ims);
        for (uint32_t i = 0; i < n; i++) {
            h_ilo[i] = sp->isolation_lo ? sp->isolation_lo[c0 + i] : NAN;
            h_ihi[i] = sp->isolation_hi ? sp->isolation_hi[c0 + i] : NAN;
            h_rt[i] = sp->scan_start_time ? sp->scan_start_time[c0 + i] : 0.0f;
            h_ims[i] = sp->inverse_ion_mobility ? sp->inverse_ion_mobility[c0 + i] : NAN;
        }
        memcpy(hs + C.o_chg, sp->precursor_charge + c0, n);
        C.smem = (size_t)(C.pmax + 4) * 8 + (size_t)sv.lcap * 16 + (size_t)sv.kparam * (sizeof(ScoreRec) + 4) + C.pmax + 32;   // peaks, lists, records, order, marks
        if (C.smem + sizeof(ScoreTile) > 200 * 1024) return fail(SAGE_B200_ELIMIT, "spectrum with %u peaks exceeds the shared-memory budget", C.pmax);
        C.nitems = (size_t)n * sv.qmax;
        if (C.nitems > 0x7FFFFFFFull) return fail(SAGE_B200_ELIMIT, "too many queries in one chunk");
        int r;
        if ((r = L.d_queries.reserve(C.nitems * sizeof(QueryDesc)))) return r;
        if ((r = L.d_hits.reserve(C.nitems * sizeof(QueryHits)))) return r;
        if ((r = L.d_keys.reserve(C.nitems * sv.kparam * 8))) return r;
        if ((r = L.d_features.reserve((size_t)n * sv.report_psms * sizeof(FeatureOut)))) return r;
        if ((r = L.d_counts.reserve(4 * (size_t)n))) return r;
        if ((r = L.d_counters.reserve(8 * (C_COUNT + (size_t)sv.qmax)))) return r;   // + one in-use flag per query slot
        if ((r = L.h_counters.reserve(8 * C_COUNT + 32))) return r;
        return 0;
    };
    if ((rc = pack())) {
        cudaStreamSynchronize(cp);   // the masses copy may still be reading the caller's array
        return rc;
    }
    // The blob travels on the SAME stream as the bulk copies. Measured with SAGE_B200_TRACE: on a second stream it is not served
    // by a second copy engine ahead of the queued bulk copies — it landed after BOTH of them and the whole pipeline started later.
    CUDA_TRY(cudaMemcpyAsync(L.d_small.p, hs, C.small_bytes, cudaMemcpyHostToDevice, cp));
    CUDA_TRY(cudaEventRecord(L.ev_small, cp));
    if (!pin_m) {
        if (npk && (rc = staged_h2d(L.d_masses.p, src_m, 4 * npk, L.h_masses, *L.pool, cp))) { cudaStreamSynchronize(cp); return rc; }   // pageable caller memory: staged + overlapped
        CUDA_TRY(cudaEventRecord(L.ev_part[0], cp));
    } else {
        uint64_t sent = npk_a;
        for (uint32_t q = 0; q < C.nparts; q++) {
            const uint64_t end = q + 1 == C.nparts ? npk : part_off(q + 1);
            if (end > sent) {
                CUDA_TRY(cudaMemcpyAsync(L.d_masses.as<float>() + sent, src_m + sent, 4 * (end - sent), cudaMemcpyHostToDevice, cp));
                sent = end;
            }
            CUDA_TRY(cudaEventRecord(L.ev_part[q], cp));
        }
    }
    CUDA_TRY(cudaEventRecord(L.ev_masses, cp));   // preliminary scoring can start: it never reads intensities
    if (npk && !pin_i) {
        if ((rc = L.h_intens.reserve(4 * npk))) { cudaStreamSynchronize(cp); return rc; }
        L.stager_rc = 0;
        L.stager_msg[0] = 0;
        const int device = S->device;
        void* dst = L.d_intens.p;
        Lane* lane = &L;
        L.stager = std::thread([lane, device, dst, src_i, npk, cp]() {
            cudaSetDevice(device);
            int r = staged_h2d(dst, src_i, 4 * npk, lane->h_intens, *lane->pool, cp);
            if (r == 0 && (cudaEventRecord(lane->ev_intens, cp) != cudaSuccess || cudaEventRecord(lane->ev_h2d_end, cp) != cudaSuccess)) r = fail(SAGE_B200_ECUDA, "event record failed after the staged copy");
            if (r) snprintf(lane->stager_msg, sizeof lane->stager_msg, "%s", g_last_error.c_str());
            lane->stager_rc = r;
        });
    } else {
        if (npk) CUDA_TRY(cudaMemcpyAsync(L.d_intens.p, src_i, 4 * npk, cudaMemcpyHostToDevice, cp));
        CUDA_TRY(cudaEventRecord(L.ev_intens, cp));
        CUDA_TRY(cudaEventRecord(L.ev_h2d_end, cp));
    }
    S->last.h2d_bytes += C.small_bytes + 8 * npk;
    C.loaded = true;
    C.force_nlist = C.force_wide = 0;
    C.force_hits = 0;
    C.timed_upload = true;
    L.ran = false;
    L.downloading = false;
    return 0;
}

static int chunk_run(sage_b200_scorer* S, Lane& L, bool dbg) {
    const sage_b200_db* db = S->db;
    const ScorerView& sv = S->sv;
    cudaStream_t st = L.stream;
    ChunkState& C = L.chunk;
    if (!C.loaded) return fail(SAGE_B200_EINVAL, "no spectra resident on the device (call batch_upload first)");
    cudaGetLastError();   // a stale non-sticky error left by another user of the runtime must not be blamed on the launches below
    const uint32_t n = C.n;
    int rc;
    if (dbg) {
        if ((rc = L.d_dbgk.reserve((size_t)n * sv.kparam * 8))) return rc;
        if ((rc = L.d_dbgm.reserve((size_t)n * 16))) return rc;
    }
    // the small-block copy of the index: built on first use, before this chunk queues
    // anything (narrow_block_for waits for lane 0's kernel stream); never for wide-window (DIA) scorers
    // (nor for open-search tolerances, whose windows exceed the warp kernel's cap: the copy would only cost memory)
    const float ptol_span = std::max(std::fabs(sv.precursor_tol.lo), std::fabs(sv.precursor_tol.hi));
    const bool narrow_tol = ptol_span <= (sv.precursor_tol.kind == 0 ? 2000.0f : sv.precursor_tol.kind == 1 ? 0.2f : 5.0f);   // ppm / percent / Da
    NarrowIndexView nv{};
    if (S->narrow_index && !sv.wide_window && narrow_tol) {
        if (S->narrow_block == 0 && (rc = narrow_block_for(S))) return rc;
        nv = db_narrow_index(db, S->narrow_block ? S->narrow_block : S->narrow_block_auto, S->narrow_block != 0);
    }
    BatchView bv{};
    unsigned char* ds = (unsigned char*)L.d_small.p;
    bv.n = n;
    bv.spectrum_base = C.base;
    bv.peak_off = (const uint32_t*)(ds + C.o_off);
    bv.masses = L.d_masses.as<float>();
    bv.intens = L.d_intens.as<float>();
    bv.prec_mz = (const float*)(ds + C.o_pmz);
    bv.prec_charge = (const uint8_t*)(ds + C.o_chg);
    bv.iso_lo = (const float*)(ds + C.o_ilo);
    bv.iso_hi = (const float*)(ds + C.o_ihi);
    bv.tic = (const float*)(ds + C.o_tic);
    bv.rt = (const float*)(ds + C.o_rt);
    bv.ims = (const float*)(ds + C.o_ims);
    bv.queries = L.d_queries.as<QueryDesc>();
    bv.hits = L.d_hits.as<QueryHits>();
    bv.hit_keys = L.d_keys.as<uint64_t>();
    bv.counters = L.d_counters.as<unsigned long long>();

    // kernels of the two lanes never overlap (measured: k_score of one chunk next to k_prelim_narrow of the other slows both); only
    // copies overlap kernels. Wait for the end of the other lane's k_score (a never-recorded event counts as complete).
    CUDA_TRY(cudaStreamWaitEvent(st, S->lanes[(&L - S->lanes) ^ 1].ev_score_end, 0));
    CUDA_TRY(cudaStreamWaitEvent(st, L.ev_small, 0));
    CUDA_TRY(cudaEventRecord(L.ev_run, st));
    CUDA_TRY(cudaMemsetAsync(L.d_counters.p, 0, 8 * (C_COUNT + (size_t)sv.qmax), st));
    const bool annotate = sv.annotate && S->frag_dst != nullptr;
    if (annotate) {   // fragment offsets are global across the chunks of one call: start this chunk's counter at what was used so far
        if ((rc = L.d_frags.reserve(S->frag_cap * sizeof(sage_b200_fragment) + 64))) return rc;
        unsigned long long* hbase = (unsigned long long*)L.h_counters.p + C_COUNT + 1;
        *hbase = S->frag_used;
        CUDA_TRY(cudaMemcpyAsync(L.d_counters.as<unsigned long long>() + C_FRAGS, hbase, 8, cudaMemcpyHostToDevice, st));
    }
    // ---- setup: resolve precursor windows. Peptide-centric counting needs LO/HI bound arrays of nfc_max * pmax floats in smem.
    ScorerView svq = sv;
    uint32_t mfc = sv.max_fragment_charge_opt >= 0 ? std::min<uint32_t>(C.zmax, (uint32_t)(sv.max_fragment_charge_opt + 1) & 0xFF) : C.zmax;
    if (mfc < 2) mfc = 2;
    size_t pep_smem = (size_t)(mfc - 1) * (2 * (size_t)C.pmax * sizeof(float) + 2 * LUT_CELLS * sizeof(uint16_t));
    if (mfc - 1 > 8) pep_smem = 200 * 1024;
    if (pep_smem > 96 * 1024) { svq.pep_cap = 0; pep_smem = 0; }
    if (svq.pep_cap == 0) pep_smem = 0;
    uint32_t *sk_in = nullptr, *sk_out = nullptr, *sv_in = nullptr, *sv_out = nullptr;
    int sort_bits = 1;   // keys are PeptideIx < n_pep (spectra without a query sort last within those bits: the order only matters for locality)
    while (sort_bits < 32 && (db->v.n_pep >> sort_bits)) sort_bits++;
    // the top 16 bits are enough for that (two 8-bit radix passes instead of three on a 2M-peptide index: windows span hundreds of peptides)
    const int sort_lo = std::max(0, sort_bits - 16);
    size_t sort_tmp = 0;
    if (S->sort_spectra && n > 1) {  // process spectra in ascending precursor-window order: neighbouring CTAs then touch the same index lines
        if ((rc = L.d_sort.reserve(16 * (size_t)n))) return rc;
        sk_in = L.d_sort.as<uint32_t>(); sk_out = sk_in + n; sv_in = sk_out + n; sv_out = sv_in + n;
        CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, sk_in, sk_out, sv_in, sv_out, (int)n, sort_lo, sort_bits, st));
        if ((rc = L.d_sorttmp.reserve(sort_tmp + 16))) return rc;
    }
    // Work-list capacities come from what earlier chunks needed (S->nlist_per_spectrum / wide_per_spectrum) or, on a re-run, from the
    // exact need the failed attempt counted: nothing in a chunk waits for the host, so chunks of both lanes queue back to back.
    C.nlist_cap = std::max<uint64_t>(C.force_nlist, (uint64_t)std::ceil(S->nlist_per_spectrum * (double)n) + 4096);
    C.wide_cap = (uint32_t)std::min<uint64_t>(C.nitems, std::max<uint64_t>(C.force_wide, S->wide_per_spectrum > 0.0
                                                                               ? (uint64_t)std::ceil(S->wide_per_spectrum * 1.1 * (double)n) + 64 : 0));
    if ((rc = L.d_nlist.reserve(8 * (C.nlist_cap + 16)))) return rc;
    if ((rc = L.d_nslots.reserve(C.nitems * sizeof(ReplaySlot)))) return rc;
    if (C.wide_cap) {
        if ((rc = L.d_witems.reserve(4 * (size_t)C.wide_cap))) return rc;
        if ((rc = L.d_wlist.reserve((size_t)C.wide_cap * WIDE_LMAX * 8))) return rc;
        if ((rc = L.d_wslots.reserve((size_t)C.wide_cap * sizeof(WideSlot)))) return rc;
    }
    if ((rc = L.d_citems.reserve(8 * C.nitems))) return rc;
    bv.cta_items = L.d_citems.as<uint32_t>();
    bv.exact_items = bv.cta_items + C.nitems;
    bv.nslots = L.d_nslots.as<ReplaySlot>();
    bv.wide_items = L.d_witems.as<uint32_t>();
    bv.wide_cap = C.wide_cap;
    bv.nlist_cap = C.nlist_cap;
    LAUNCH(k_setup_queries<<<(n + 127) / 128, 128, 0, st>>>(db->v, svq, bv, sk_in, sv_in));
    if (sk_in) {
        CUDA_TRY(cub::DeviceRadixSort::SortPairs(L.d_sorttmp.p, sort_tmp, sk_in, sk_out, sv_in, sv_out, (int)n, sort_lo, sort_bits, st));
        bv.order = sv_out;
    }
    CUDA_TRY(cudaEventRecord(L.ev_setup_end, st));
    if (C.nparts <= 1) CUDA_TRY(cudaStreamWaitEvent(st, L.ev_masses, 0));   // the counting kernels read the peak masses
    uint64_t launches = 1;

    // ---- preliminary scoring. Both kernels are always queued: CTAs whose query belongs to the other kernel (or to nobody) exit at once.
    const size_t rsm = (size_t)sv.kparam * REPLAY_THREADS * 8;
    for (uint32_t q = 0; q < C.nparts; q++) {   // one launch per part of the masses copy (a resident batch has one part)
        if (C.nparts > 1) CUDA_TRY(cudaStreamWaitEvent(st, L.ev_part[q], 0));
        const dim3 wgrid((n + WARPQ_WARPS - 1) / WARPQ_WARPS, sv.qmax);
        if (nv.mz != nullptr) LAUNCH(k_prelim_narrow_warp<true><<<wgrid, WARPQ_WARPS * 32, 0, st>>>(db->v, svq, bv, L.d_nlist.as<uint64_t>(), C.part_lo[q], C.part_lo[q + 1], nv));
        else LAUNCH(k_prelim_narrow_warp<false><<<wgrid, WARPQ_WARPS * 32, 0, st>>>(db->v, svq, bv, L.d_nlist.as<uint64_t>(), C.part_lo[q], C.part_lo[q + 1], nv));
        launches += q > 0;
    }
    if (C.nparts > 1) CUDA_TRY(cudaStreamWaitEvent(st, L.ev_masses, 0));
    LAUNCH(k_prelim_narrow<<<(unsigned)std::min<uint64_t>(C.nitems, (uint64_t)db->sm_count * PRELIM_CTAS), PRELIM_THREADS, pep_smem, st>>>(
        db->v, svq, bv, C.pmax, L.d_nlist.as<uint64_t>(), S->narrow_cta ? nv : NarrowIndexView{}));
    // the rare queries with >= 2^16 matches, listed by both counting kernels: exact wrapped u16 counts (kernels.cuh: EXACT_TRIGGER). Usually
    // there are none, so the grid is small: the launch costs one short kernel, and a listed query is a whole pass over its window anyway
    LAUNCH(k_prelim_exact<<<(unsigned)std::min<uint64_t>(C.nitems, 8), PRELIM_THREADS, 0, st>>>(db->v, svq, bv, L.d_nlist.as<uint64_t>(), nv));
    CUDA_TRY(cudaEventRecord(L.ev_count_end, st));   // narrow counting kernels done (the open-search kernel, when present, is timed with the replays)
    // narrow windows (<= NARROW_CAP peptides): 32-bit heap keys, half the shared memory
    LAUNCH(k_replay<true><<<(unsigned)((C.nitems + REPLAY_THREADS - 1) / REPLAY_THREADS), REPLAY_THREADS, rsm / 2, st>>>(
        sv, bv, L.d_nlist.as<uint64_t>(), L.d_nslots.as<ReplaySlot>(), (uint32_t)C.nitems, nullptr, n));
    launches += 4;
    if (C.wide_cap) {
        const int ctas = (int)std::min<uint64_t>((uint64_t)db->sm_count * WIDE_CTAS, C.wide_cap);
        const WideIndexView wv = db_wide_index(db, sv.wide_tile);   // built on first use (the first open-search chunk of a scorer is a re-run anyway)
        LAUNCH(k_prelim_wide<<<ctas, WIDE_THREADS, sizeof(WideSmem), st>>>(db->v, sv, bv, (uint32_t)C.nitems, L.d_wlist.as<uint64_t>(), L.d_wslots.as<WideSlot>(), wv));
        if (wv.frag != nullptr) {   // reference-terms work counters of the queries the block-index path counted (no index entry is read)
            LAUNCH(k_wide_account<<<(C.wide_cap + 7) / 8, 256, 0, st>>>(db->v, sv, bv));
            launches++;
        }
        LAUNCH(k_replay<false><<<(unsigned)((C.wide_cap + REPLAY_THREADS - 1) / REPLAY_THREADS), REPLAY_THREADS, rsm, st>>>(
            sv, bv, L.d_wlist.as<uint64_t>(), L.d_wslots.as<WideSlot>(), C.wide_cap, L.d_counters.as<unsigned long long>() + C_WIDE, 0u));
        launches += 2;
    }
    CUDA_TRY(cudaEventRecord(L.ev_replay_end, st));

    // ---- candidate scoring + feature assembly (first reader of the intensities)
    if ((rc = lane_join_stager(L))) return rc;   // ev_intens is recorded by the staging thread of a pageable chunk
    CUDA_TRY(cudaStreamWaitEvent(st, L.ev_intens, 0));
    const bool split = S->score_split && !sv.chimera && !annotate && !dbg && S->quick_mode == 0;
    if (split) {
        // hit arena: one entry per scoring task is reserved (sparsely used); sized from what earlier chunks needed, exact on a re-run
        C.hits_cap = std::max<uint64_t>(C.force_hits, (uint64_t)std::ceil((S->hits_per_spectrum > 0.0 ? S->hits_per_spectrum : 4096.0) * (double)n) + 65536);
        if ((rc = L.d_cand.reserve((size_t)n * sv.kparam * sizeof(CandOut)))) return rc;
        if ((rc = L.d_meta.reserve((size_t)n * sizeof(SpecMeta)))) return rc;
        if ((rc = L.d_recs.reserve((size_t)n * sv.kparam * sizeof(ScoreRec)))) return rc;
        if ((rc = L.d_hkey.reserve((size_t)n * sv.kparam * 8))) return rc;
        if ((rc = L.d_emit.reserve((size_t)n * sv.report_psms * 4 + 16))) return rc;
        if ((rc = L.d_hitk.reserve(2 * C.hits_cap + 16))) return rc;
        if ((rc = L.d_hiti.reserve(4 * C.hits_cap + 16))) return rc;
        if ((rc = L.d_hitt.reserve(4 * C.hits_cap + 16))) return rc;
        SplitOut so{};
        so.cand = L.d_cand.as<CandOut>(); so.meta = L.d_meta.as<SpecMeta>(); so.hit_k = L.d_hitk.as<uint16_t>(); so.hit_i = L.d_hiti.as<float>();
        so.hit_t = L.d_hitt.as<float>(); so.hit_cap = C.hits_cap; so.recs = L.d_recs.as<ScoreRec>(); so.hkey = L.d_hkey.as<unsigned long long>(); so.counters = bv.counters;
        // k_score<true> stages the peaks and the hit lists only (no records / order / marks)
        const size_t smem_split = (size_t)(C.pmax + 4) * 8 + (size_t)sv.lcap * 16 + 32;
        LAUNCH(k_score<true><<<n, SCORE_THREADS, smem_split, st>>>(db->v, sv, bv, L.d_features.as<FeatureOut>(), L.d_counts.as<uint32_t>(), C.pmax, nullptr, nullptr, nullptr,
                                                                   0ull, 0u, nullptr, so));
        const uint64_t nthr = (uint64_t)n * sv.kparam, nrow = (uint64_t)n * sv.report_psms;
        CUDA_TRY(cudaMemsetAsync(L.d_emit.p, 0xFF, 4 * nrow, st));   // rank slots: RANK_EMPTY
        LAUNCH(k_fold<<<(unsigned)((nthr + 127) / 128), 128, 0, st>>>(db->v, sv, so, n));
        LAUNCH(k_features<<<(unsigned)((nthr + 127) / 128), 128, 0, st>>>(sv, n, so, L.d_emit.as<uint32_t>()));
        LAUNCH(k_rows<<<(unsigned)((nrow + 127) / 128), 128, 0, st>>>(db->v, sv, bv, so, L.d_emit.as<uint32_t>(), L.d_counts.as<uint32_t>(), L.d_features.as<FeatureOut>()));
        launches += 4;
    } else {
        C.hits_cap = 0;
        LAUNCH(k_score<false><<<n, SCORE_THREADS, C.smem, st>>>(db->v, sv, bv, L.d_features.as<FeatureOut>(), L.d_counts.as<uint32_t>(), C.pmax,
                                                               dbg ? L.d_dbgk.as<uint64_t>() : nullptr, dbg ? L.d_dbgm.as<uint32_t>() : nullptr,
                                                               annotate ? L.d_frags.as<FragmentOut>() : nullptr, (unsigned long long)S->frag_cap, S->quick_mode,
                                                               S->d_keep.as<uint8_t>(), SplitOut{}));
        launches++;
    }
    CUDA_TRY(cudaEventRecord(L.ev_score_end, st));
    CUDA_TRY(cudaMemcpyAsync(L.h_counters.p, L.d_counters.p, 8 * C_COUNT, cudaMemcpyDeviceToHost, st));
    L.launches = launches;
    L.dbg = dbg;
    L.ran = true;
    return 0;
}

static int chunk_download(sage_b200_scorer* S, Lane& L, sage_b200_feature* fdst, uint32_t* cdst) {
    const ScorerView& sv = S->sv;
    cudaStream_t st = L.stream;
    ChunkState& C = L.chunk;
    if (!C.loaded) return fail(SAGE_B200_EINVAL, "no results on the device");
    const uint32_t n = C.n;
    int rc;
    const size_t fbytes = (size_t)n * sv.report_psms * sizeof(sage_b200_feature);
    const bool f_pinned = is_pinned(fdst), c_pinned = is_pinned(cdst);
    if (!f_pinned && (rc = L.h_features.reserve(fbytes))) return rc;
    if (!c_pinned && (rc = L.h_counts.reserve(4 * (size_t)n))) return rc;
    CUDA_TRY(cudaEventRecord(L.ev_d2h_begin, st));
    CUDA_TRY(cudaMemcpyAsync(f_pinned ? (void*)fdst : L.h_features.p, L.d_features.p, fbytes, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(c_pinned ? (void*)cdst : L.h_counts.p, L.d_counts.p, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaEventRecord(L.ev_d2h_end, st));
    L.fdst = fdst; L.cdst = cdst; L.f_pinned = f_pinned; L.c_pinned = c_pinned;
    L.downloading = true;
    S->last.d2h_bytes += fbytes + 4 * (size_t)n;
    return 0;
}

// Open search keeps one survivor list (WIDE_LMAX keys, 96 KiB) per wide query and lane. The arena is bounded by a memory budget: a chunk whose
// wide queries would need more is not re-run at its size — the call restarts with chunks small enough for the budget (internal code ERECHUNK).
constexpr int SAGE_B200_ERECHUNK = -100;   // never returned to callers
static uint64_t wide_arena_budget() {
    if (const char* e = getenv("SAGE_B200_WIDE_ARENA_MB")) return std::max<uint64_t>(1, (uint64_t)atoll(e)) << 20;   // (tests use a tiny budget)
    return 8ull << 30;
}
static uint64_t wide_max_chunk(double wide_per_spectrum, uint64_t otherwise) {
    if (!(wide_per_spectrum > 0.0)) return otherwise;
    const double per_spectrum = wide_per_spectrum * 1.1 * (double)WIDE_LMAX * 8.0;
    const uint64_t fit = (uint64_t)std::max(1.0, (double)wide_arena_budget() / per_spectrum);
    return std::min<uint64_t>(32768, std::max<uint64_t>(64, fit));   // open search: at most 32768 spectra per chunk
}

// Waits for everything queued on the lane and folds its counters / timings into S->last.
static int lane_finish(sage_b200_scorer* S, Lane& L) {
    ChunkState& C = L.chunk;
    if (!C.loaded) return 0;
    { const int jrc = lane_join_stager(L); if (jrc) return jrc; }
    CUDA_TRY(cudaStreamSynchronize(L.copy));
    for (int attempt = 0;; attempt++) {
        CUDA_TRY(cudaStreamSynchronize(L.stream));
        if (!L.ran) break;
        const unsigned long long* hc = (const unsigned long long*)L.h_counters.p;
        const uint64_t need = hc[C_NLIST_NEED], nw = hc[C_WIDE], nh = C.hits_cap ? hc[C_HITS] : 0;
        if (nh) S->hits_per_spectrum = std::max(S->hits_per_spectrum, 1.25 * (double)nh / (double)C.n);
        if (need <= C.nlist_cap && nw <= C.wide_cap && nh <= C.hits_cap) {   // the chunk fitted its work lists: remember what it needed
            S->nlist_per_spectrum = std::max(S->nlist_per_spectrum, 1.25 * (double)need / (double)C.n);
            S->wide_per_spectrum = std::max(S->wide_per_spectrum, (double)nw / (double)C.n);
            break;
        }
        if (attempt >= 2) return fail(SAGE_B200_ECUDA, "internal error: chunk re-run with exact work-list sizes did not fit");
        S->nlist_per_spectrum = std::max(S->nlist_per_spectrum, 1.25 * (double)need / (double)C.n);
        S->wide_per_spectrum = std::max(S->wide_per_spectrum, (double)nw / (double)C.n);
        if (nw > C.wide_cap && nw * (uint64_t)WIDE_LMAX * 8 > wide_arena_budget() && C.n > wide_max_chunk(S->wide_per_spectrum, 65536))
            return fail(SAGE_B200_ERECHUNK, "open-search chunk of %u spectra needs %llu survivor lists: restarting with smaller chunks", C.n, (unsigned long long)nw);
        // a work list was too small: the queries it could not hold reported no hits. Re-run the chunk with the sizes just counted.
        C.force_nlist = need;
        C.force_wide = nw;
        C.force_hits = nh;
        S->last.chunk_retries++;
        int rc;
        if ((rc = chunk_run(S, L, L.dbg))) return rc;
        if (L.downloading) {
            S->last.d2h_bytes -= (uint64_t)C.n * S->sv.report_psms * sizeof(sage_b200_feature) + 4 * (uint64_t)C.n;
            if ((rc = chunk_download(S, L, L.fdst, L.cdst))) return rc;
        }
    }
    if (S->trace && L.ran && L.downloading) {
        float t[8];
        const cudaEvent_t marks[8] = {L.ev_h2d_begin, L.ev_h2d_end, L.ev_run, L.ev_setup_end, L.ev_replay_end, L.ev_score_end, L.ev_d2h_begin, L.ev_d2h_end};
        for (int i = 0; i < 8; i++) cudaEventElapsedTime(&t[i], S->ev_base, marks[i]);
        const double now = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - S->t_base).count();
        float tm = 0;
        cudaEventElapsedTime(&tm, S->ev_base, L.ev_masses);
        fprintf(stderr, "[sage_b200 trace] chunk base=%u n=%u | host issue %.3f..%.3f, finished %.3f | dev h2d %.3f..(masses %.3f)..%.3f run %.3f setup-end %.3f prelim-end %.3f score-end %.3f d2h %.3f..%.3f\n",
                C.base, C.n, C.t_issue0, C.t_issue1, now, t[0], tm, t[1], t[2], t[3], t[4], t[5], t[6], t[7]);
    }
    sage_b200_counters& T = S->last;
    float ms;
    if (C.timed_upload) { cudaEventElapsedTime(&ms, L.ev_h2d_begin, L.ev_h2d_end); T.ms_h2d += ms; T.ms_total += ms; C.timed_upload = false; }
    if (L.ran) {
        const unsigned long long* hc = (const unsigned long long*)L.h_counters.p;
        cudaEventElapsedTime(&ms, L.ev_run, L.ev_setup_end); T.ms_setup += ms;
        cudaEventElapsedTime(&ms, L.ev_setup_end, L.ev_replay_end); T.ms_prelim += ms;
        cudaEventElapsedTime(&ms, L.ev_setup_end, L.ev_count_end); T.ms_prelim_count += ms;
        cudaEventElapsedTime(&ms, L.ev_replay_end, L.ev_score_end); T.ms_score += ms;
        cudaEventElapsedTime(&ms, L.ev_run, L.ev_score_end); T.ms_total += ms;
        T.spectra += C.n; T.peaks += C.npk; T.queries += hc[C_QUERIES]; T.tasks += hc[C_TASKS]; T.pages += hc[C_PAGES]; T.entries_scanned += hc[C_ENTRIES];
        T.matched_fragments += hc[C_MATCHED]; T.candidates_scored += hc[C_CANDS]; T.peptide_record_floats += hc[C_PEPFLOATS]; T.psms += hc[C_PSMS];
        T.wide_queries += hc[C_WIDE]; T.pep_queries += hc[C_PEPQ]; T.pep_fallbacks += hc[C_PEPFALLBACK]; T.wide_overflows += hc[C_WOVERFLOW];
        T.d2h_bytes += 2 * 8 * C_COUNT;
        T.kernel_launches += L.launches;
        if (S->sv.annotate && S->frag_dst != nullptr) {
            const uint64_t end = hc[C_FRAGS], begin = S->frag_used;
            const uint64_t lim = std::min<uint64_t>(end, S->frag_cap);
            if (lim > begin) {
                if (int rc = read_back(L.stream, S->frag_dst + begin, L.d_frags.as<sage_b200_fragment>() + begin, (lim - begin) * sizeof(sage_b200_fragment))) return rc;
                T.d2h_bytes += (lim - begin) * sizeof(sage_b200_fragment);
            }
            S->frag_used = end;
        }
        L.ran = false;
    }
    if (L.downloading) {
        const size_t fbytes = (size_t)C.n * S->sv.report_psms * sizeof(sage_b200_feature);
        if (!L.f_pinned) memcpy(L.fdst, L.h_features.p, fbytes);
        if (!L.c_pinned) memcpy(L.cdst, L.h_counts.p, 4 * (size_t)C.n);
        cudaEventElapsedTime(&ms, L.ev_d2h_begin, L.ev_d2h_end); T.ms_d2h += ms; T.ms_total += ms;
        L.downloading = false;
    }
    return 0;
}

static void finish_counters(sage_b200_scorer* S) {
    // SURVEY.md §8(d): B = 8*P + sum_q[8*ceil(log2 N_pep)] + sum_tasks[8*ceil(log2 N_bucket)] + sum_pages[8*ceil(log2 bucket_size) + 8*entries]
    //                    + sum_candidates 4*(2L+2) + 64*n_psm
    sage_b200_counters& L = S->last;
    const DbView& v = S->db->v;
    const uint64_t lp = ceil_log2_u64(v.n_pep), lb = ceil_log2_u64(v.n_bucket), ls = ceil_log2_u64(v.bucket_size);
    L.prelim_bytes = 4 * L.peaks + 8 * lb * L.tasks + 8 * ls * L.pages + 8 * L.entries_scanned;
    L.score_bytes = 4 * L.peaks + 4 * L.peptide_record_floats + 64 * L.psms;
    L.algorithmic_bytes = 8 * L.peaks + 8 * lp * L.queries + 8 * lb * L.tasks + 8 * ls * L.pages + 8 * L.entries_scanned + 4 * L.peptide_record_floats + 64 * L.psms;
}

static int check_spectra(const sage_b200_spectra* sp) {
    if (!sp) return fail(SAGE_B200_EINVAL, "spectra: null");
    if (sp->n && (!sp->peak_offsets || !sp->precursor_mz || !sp->precursor_charge || !sp->total_ion_current)) return fail(SAGE_B200_EINVAL, "spectra: null array");
    if (sp->n && sp->peak_offsets[sp->n] > sp->peak_offsets[0] && (!sp->masses || !sp->intensities)) return fail(SAGE_B200_EINVAL, "spectra: null peak arrays");
    return 0;
}

// Waits for everything queued on both lanes and marks them empty. Returns the first synchronisation error.
static cudaError_t idle_lanes(sage_b200_scorer* S) {
    cudaError_t first = cudaSuccess;
    for (Lane& L : S->lanes) {
        const cudaError_t a = cudaStreamSynchronize(L.copy), b = cudaStreamSynchronize(L.stream);
        if (first == cudaSuccess) first = a != cudaSuccess ? a : b;
        L.chunk.loaded = false; L.ran = false; L.downloading = false;
    }
    return first;
}

// Error exit of a batch call: the other lane may still have an H2D reading the caller's arrays or a D2H writing into them. Drain both lanes
// before the error is returned, so the caller may free or reuse its buffers at once; the error message of the failure is preserved.
static int drain_lanes(sage_b200_scorer* S, int rc) {
    const std::string msg = g_last_error;
    for (Lane& L : S->lanes)
        if (L.stager.joinable()) L.stager.join();   // it reads the caller's arrays
    idle_lanes(S);
    cudaGetLastError();
    S->frag_dst = nullptr;
    g_last_error = msg;
    return rc;
}

static int score_batch_chunks(sage_b200_scorer* S, const sage_b200_spectra* sp, sage_b200_feature* features, uint32_t* counts, bool annotate);

extern "C" int sage_b200_score_batch(sage_b200_scorer* S, const sage_b200_spectra* sp, sage_b200_feature* features, uint32_t* counts,
                                     sage_b200_fragment* fragments, uint64_t fragment_capacity, uint64_t* fragments_used) {
    if (!S) return fail(SAGE_B200_EINVAL, "score_batch: null scorer");
    const auto t_call = std::chrono::steady_clock::now();
    int rc = check_spectra(sp);
    if (rc) return rc;
    if (sp->n && (!features || !counts)) return fail(SAGE_B200_EINVAL, "score_batch: null output");
    std::lock_guard<std::mutex> lock(S->mu);
    CUDA_TRY(cudaSetDevice(S->db->device));
    S->last = sage_b200_counters{};
    if (fragments_used) *fragments_used = 0;
    const bool annotate = S->sv.annotate != 0;
    if (annotate && (!fragments || !fragments_used)) return fail(SAGE_B200_EINVAL, "annotate_matches needs a fragments array and fragments_used");
    S->frag_dst = annotate ? fragments : nullptr;
    S->frag_cap = annotate ? fragment_capacity : 0;
    S->frag_used = 0;
    CUDA_TRY(idle_lanes(S));   // a previous call may have failed half-way: make sure nothing is still queued on the lanes
    if (S->trace) { S->t_base = std::chrono::steady_clock::now(); CUDA_TRY(cudaEventRecord(S->ev_base, S->lanes[0].stream)); }
    for (int restart = 0;; restart++) {
        rc = score_batch_chunks(S, sp, features, counts, annotate);
        if (rc != SAGE_B200_ERECHUNK) break;
        drain_lanes(S, rc);   // nothing of this call is kept: the first chunk that needs the re-chunking is the first open-search chunk of the handle
        if (restart >= 3) return fail(SAGE_B200_ELIMIT, "open search: survivor lists do not fit the arena budget even with the smallest chunks");
        const uint64_t retries = S->last.chunk_retries;
        S->last = sage_b200_counters{};
        S->last.chunk_retries = retries + 1;
        S->frag_dst = annotate ? fragments : nullptr;
        S->frag_used = 0;
    }
    if (rc) return drain_lanes(S, rc);
    finish_counters(S);
    S->last.ms_wall = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_call).count();
    if (annotate) {
        *fragments_used = S->frag_used;
        S->frag_dst = nullptr;
        if (S->frag_used > fragment_capacity)
            return fail(SAGE_B200_ELIMIT, "fragment_capacity %llu too small: %llu fragments matched (features are complete; re-run with a larger array)",
                        (unsigned long long)fragment_capacity, (unsigned long long)S->frag_used);
    }
    return 0;
}

// The end of the chunk of at most `len` spectra that starts at c0: halved until its peaks fit the lane's staging bound (one spectrum always fits).
static uint64_t chunk_end(const sage_b200_spectra* sp, uint64_t c0, uint64_t len) {
    const uint64_t max_peaks = 1ull << 25;
    uint64_t c1 = std::min<uint64_t>(sp->n, c0 + len);
    while (c1 > c0 + 1 && sp->peak_offsets[c1] - sp->peak_offsets[c0] > max_peaks) c1 = c0 + (c1 - c0) / 2;
    return c1;
}

// The chunk loop of score_batch (two pipelined lanes). Returns SAGE_B200_ERECHUNK when an open-search chunk must be cut smaller.
static int score_batch_chunks(sage_b200_scorer* S, const sage_b200_spectra* sp, sage_b200_feature* features, uint32_t* counts, bool annotate) {
    int rc = 0;
    // Chunks are as large as the staging bounds allow: on cfg2 one 50k chunk computes faster than two 25k chunks (the kernels process
    // spectra in precursor order, so a denser chunk shares more index lines). Inside a chunk the intensities copy overlaps setup + preliminary
    // scoring; across chunks (two lanes) the whole H2D of chunk i+1 and the D2H of chunk i-1 overlap the kernels of chunk i.
    const uint64_t max_chunk = wide_max_chunk(S->wide_per_spectrum, 65536);   // open search: one ~100 KB survivor list per query, bounded by the arena budget
    // A short first chunk (first_chunk_pct of the batch, at most 16384 spectra) lets the kernels start while most of the H2D is still in flight.
    uint64_t first = 0, rest = sp->n;
    if (S->pipeline_chunks <= 1 && sp->n >= 16384) { first = std::min<uint64_t>(sp->n * (uint64_t)S->first_chunk_pct / 100, 16384); rest = sp->n - first; }
    const uint64_t nchunks = std::max<uint64_t>((uint64_t)S->pipeline_chunks, (rest + max_chunk - 1) / max_chunk);
    uint64_t target = (rest + nchunks - 1) / nchunks;
    target = std::min<uint64_t>(std::max<uint64_t>(target, 1), max_chunk);
    uint64_t c0 = 0;
    int li = 0;
    while (c0 < sp->n) {
        const uint64_t c1 = chunk_end(sp, c0, c0 == 0 && first ? first : target);
        Lane& L = S->lanes[li];
        if ((rc = lane_finish(S, L))) return rc;   // the chunk that used this lane two iterations ago
        const double ti0 = S->trace ? std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - S->t_base).count() : 0.0;
        if ((rc = chunk_upload(S, L, sp, c0, c1))) return rc;
        if ((rc = chunk_run(S, L, false))) return rc;
        if ((rc = chunk_download(S, L, features + c0 * S->sv.report_psms, counts + c0))) return rc;
        if (S->trace) { L.chunk.t_issue0 = ti0; L.chunk.t_issue1 = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - S->t_base).count(); }
        if (annotate && (rc = lane_finish(S, L))) return rc;   // fragment offsets are global: chunks run one after another
        c0 = c1;
        if (!annotate) li ^= 1;
    }
    for (Lane& L : S->lanes) {
        if ((rc = lane_finish(S, L))) return rc;
        L.chunk.loaded = false;
    }
    return 0;
}

// Pins the calling host thread to the CPUs of the NUMA node the GPU hangs off (sysfs: PCI device -> numa_node -> cpulist), so that the thread's
// pinned staging buffers (first touch) and its cudaMemcpyAsync submissions stay on the socket next to the GPU. Returns the node (>= 0), or -1
// when the topology cannot be read (single-node hosts, containers without sysfs): the thread is left alone.
static int device_numa_cpus(int device, cpu_set_t* want_out);

extern "C" int sage_b200_bind_thread_to_device(int device) {
    // topology lookups (sysfs) are cached per device: score_batch_multi binds its worker threads on every call
    static std::mutex mu;
    static int node_of[64];
    static cpu_set_t cpus_of[64];
    static bool known[64] = {};
    cpu_set_t want;
    int node;
    {
        std::lock_guard<std::mutex> lock(mu);
        if (device >= 0 && device < 64 && known[device]) { node = node_of[device]; want = cpus_of[device]; }
        else {
            node = device_numa_cpus(device, &want);
            if (device >= 0 && device < 64) { known[device] = true; node_of[device] = node; cpus_of[device] = want; }
        }
    }
    if (node < 0) return -1;
    if (pthread_setaffinity_np(pthread_self(), sizeof want, &want) != 0) return -1;
    return node;
}

// NUMA node of the GPU and the CPUs of that node this process may run on (-1: unknown).
static int device_numa_cpus(int device, cpu_set_t* want_out) {
    char bus[64] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char* c = bus; *c; c++) *c = (char)tolower(*c);
    char path[256];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    if (node < 0) return -1;
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r");
    if (!f) return -1;
    char list[4096] = {0};
    const size_t got = fread(list, 1, sizeof list - 1, f);
    fclose(f);
    if (got == 0) return -1;
    // CPUs the process was given when the library was loaded (before any thread was bound by us): never widen that set
    static const cpu_set_t initial = []() { cpu_set_t c; CPU_ZERO(&c); sched_getaffinity(0, sizeof c, &c); return c; }();
    cpu_set_t cur = initial, want;
    CPU_ZERO(&want);
    if (CPU_COUNT(&cur) == 0) return -1;
    int n_set = 0;
    for (char* tok = strtok(list, ",\n"); tok; tok = strtok(nullptr, ",\n")) {   // "0-31,64-95"
        int a = 0, b = 0;
        const int k = sscanf(tok, "%d-%d", &a, &b);
        if (k == 1) b = a;
        if (k < 1) continue;
        for (int c = a; c <= b && c < CPU_SETSIZE; c++)
            if (CPU_ISSET(c, &cur)) { CPU_SET(c, &want); n_set++; }   // never widen the affinity the process was given
    }
    if (n_set == 0) return -1;
    *want_out = want;
    return node;
}

// One process, several GPUs (SURVEY.md §8e): spectra are independent, so the batch is cut into contiguous blocks, block g goes to
// scorers[g] (each bound to its own device and index replica) on its own host thread; Feature.spectrum stays batch-relative.
// No collective and no peer traffic: results land directly in the caller's arrays.
extern "C" int sage_b200_score_batch_multi(sage_b200_scorer* const* scorers, int n_scorers, const sage_b200_spectra* sp, sage_b200_feature* features,
                                           uint32_t* counts) {
    if (!scorers || n_scorers <= 0) return fail(SAGE_B200_EINVAL, "score_batch_multi: no scorers");
    int rc = check_spectra(sp);
    if (rc) return rc;
    if (sp->n && (!features || !counts)) return fail(SAGE_B200_EINVAL, "score_batch_multi: null output");
    for (int g = 0; g < n_scorers; g++) {
        if (!scorers[g]) return fail(SAGE_B200_EINVAL, "score_batch_multi: null scorer %d", g);
        if (scorers[g]->sv.report_psms != scorers[0]->sv.report_psms || scorers[g]->sv.annotate)
            return fail(SAGE_B200_EINVAL, "score_batch_multi: scorers must share report_psms and not annotate matches");
    }
    const uint32_t r = scorers[0]->sv.report_psms;
    std::vector<int> rcs(n_scorers, 0);
    std::vector<std::string> msgs(n_scorers);
    std::vector<std::thread> th;
    for (int g = 0; g < n_scorers; g++) {
        const uint64_t a = sp->n * (uint64_t)g / (uint64_t)n_scorers, b = sp->n * (uint64_t)(g + 1) / (uint64_t)n_scorers;
        th.emplace_back([&, g, a, b]() {
            if (a == b) return;
            sage_b200_bind_thread_to_device(scorers[g]->db->device);   // worker + its staging copies on the GPU's NUMA node
            sage_b200_spectra sub = *sp;   // a view: same arrays, shifted per-spectrum pointers (peak_offsets stay absolute)
            sub.n = b - a;
            sub.peak_offsets = sp->peak_offsets + a;
            sub.precursor_mz = sp->precursor_mz + a;
            sub.precursor_charge = sp->precursor_charge + a;
            sub.isolation_lo = sp->isolation_lo ? sp->isolation_lo + a : nullptr;
            sub.isolation_hi = sp->isolation_hi ? sp->isolation_hi + a : nullptr;
            sub.total_ion_current = sp->total_ion_current + a;
            sub.level = sp->level ? sp->level + a : nullptr;
            sub.scan_start_time = sp->scan_start_time ? sp->scan_start_time + a : nullptr;
            sub.inverse_ion_mobility = sp->inverse_ion_mobility ? sp->inverse_ion_mobility + a : nullptr;
            rcs[g] = sage_b200_score_batch(scorers[g], &sub, features + a * r, counts + a, nullptr, 0, nullptr);
            if (rcs[g]) msgs[g] = g_last_error;
            else
                for (uint64_t i = a; i < b; i++)
                    for (uint32_t k = 0; k < counts[i]; k++) features[i * r + k].spectrum += (uint32_t)a;
        });
    }
    for (auto& x : th) x.join();
    for (int g = 0; g < n_scorers; g++)
        if (rcs[g]) return fail(rcs[g], "scorer %d (device %d): %s", g, scorers[g]->db->device, msgs[g].c_str());
    return 0;
}

// Scorer::quick_score over a batch (scoring.rs:255-298), the prefilter used by runner.rs:143-278: keep[PeptideIx] |= peptide identified.
// prefilter_low_memory != 0: peptides of the report_psms "largest" scored candidates per spectrum (see k_score); == 0: every preliminary hit.
// quick_score over a batch with the marks left on the device: S->d_keep holds one byte per PeptideIx (nonzero = kept) and every lane is idle
// on return. The caller holds S->mu and has selected the device.
static int quick_score_device(sage_b200_scorer* S, const sage_b200_spectra* sp, int prefilter_low_memory) {
    int rc = 0;
    const size_t npep = S->db->v.n_pep;
    if ((rc = S->d_keep.reserve(npep + 16))) return rc;
    S->last = sage_b200_counters{};
    S->frag_dst = nullptr;
    CUDA_TRY(idle_lanes(S));
    S->quick_mode = prefilter_low_memory ? 2u : 1u;
    Lane& L = S->lanes[0];   // every chunk runs on lane 0, behind the zeroing of the marks
    CUDA_TRY(cudaMemsetAsync(S->d_keep.p, 0, npep + 16, L.stream));
    for (int restart = 0; restart < 4; restart++) {
        uint64_t c0 = 0;
        rc = 0;
        const uint64_t max_chunk = wide_max_chunk(S->wide_per_spectrum, 32768);
        while (c0 < sp->n && rc == 0) {
            const uint64_t c1 = chunk_end(sp, c0, max_chunk);
            if ((rc = chunk_upload(S, L, sp, c0, c1)) == 0 && (rc = chunk_run(S, L, false)) == 0) rc = lane_finish(S, L);
            c0 = c1;
        }
        if (rc != SAGE_B200_ERECHUNK) break;
        drain_lanes(S, rc);   // overflowed attempts leave no keep[] marks (k_score), so the marks of the finished chunks stay valid
        S->quick_mode = prefilter_low_memory ? 2u : 1u;
        CUDA_TRY(cudaMemsetAsync(S->d_keep.p, 0, npep + 16, L.stream));
    }
    if (rc == SAGE_B200_ERECHUNK) rc = fail(SAGE_B200_ELIMIT, "open search: survivor lists do not fit the arena budget even with the smallest chunks");
    S->quick_mode = 0;
    L.chunk.loaded = false;
    if (rc) return drain_lanes(S, rc);
    CUDA_TRY(cudaStreamSynchronize(L.stream));   // the marks are complete (also when no chunk ran)
    finish_counters(S);
    return 0;
}

// Scorer::quick_score over a batch (scoring.rs:255-298), the prefilter used by runner.rs:143-278: keep[PeptideIx] |= peptide identified.
// prefilter_low_memory != 0: peptides of the report_psms "largest" scored candidates per spectrum (see k_score); == 0: every preliminary hit.
extern "C" int sage_b200_quick_score(sage_b200_scorer* S, const sage_b200_spectra* sp, int prefilter_low_memory, uint8_t* keep) {
    if (!S || !keep) return fail(SAGE_B200_EINVAL, "quick_score: null argument");
    int rc = check_spectra(sp);
    if (rc) return rc;
    std::lock_guard<std::mutex> lock(S->mu);
    CUDA_TRY(cudaSetDevice(S->db->device));
    if ((rc = quick_score_device(S, sp, prefilter_low_memory))) return rc;
    const size_t npep = S->db->v.n_pep;
    std::vector<uint8_t> h(npep);
    if ((rc = read_back(S->lanes[0].stream, h.data(), S->d_keep.p, npep))) return rc;
    for (size_t i = 0; i < npep; i++) keep[i] |= h[i];
    return 0;
}

// Device-resident variant of score_batch, split in phases (single chunk, lane 0): upload once, run the kernels any number of
// times (bench.py times this with the inputs already in HBM), download the Feature rows.
extern "C" int sage_b200_batch_upload(sage_b200_scorer* S, const sage_b200_spectra* sp) {
    if (!S) return fail(SAGE_B200_EINVAL, "batch_upload: null scorer");
    int rc = check_spectra(sp);
    if (rc) return rc;
    if (sp->n == 0 || sp->n > (1u << 18) || sp->peak_offsets[sp->n] - sp->peak_offsets[0] > (1ull << 26))
        return fail(SAGE_B200_ELIMIT, "batch_upload takes 1..262144 spectra and at most 2^26 peaks (use score_batch for larger batches)");
    std::lock_guard<std::mutex> lock(S->mu);
    CUDA_TRY(cudaSetDevice(S->db->device));
    S->last = sage_b200_counters{};
    Lane& L = S->lanes[0];
    if ((rc = chunk_upload(S, L, sp, 0, sp->n))) return rc;
    if ((rc = lane_finish(S, L))) return rc;
    L.chunk.nparts = 1;   // everything is resident: batch_run queues one counting launch
    L.chunk.part_lo[1] = L.chunk.n;
    return 0;
}
extern "C" int sage_b200_batch_run(sage_b200_scorer* S) {
    if (!S) return fail(SAGE_B200_EINVAL, "batch_run: null scorer");
    std::lock_guard<std::mutex> lock(S->mu);
    CUDA_TRY(cudaSetDevice(S->db->device));
    const uint64_t h2d = S->last.h2d_bytes;
    S->last = sage_b200_counters{};
    S->last.h2d_bytes = h2d;
    Lane& L = S->lanes[0];
    int rc = chunk_run(S, L, false);
    if (rc) return rc;
    if ((rc = lane_finish(S, L))) {
        if (rc == SAGE_B200_ERECHUNK) rc = fail(SAGE_B200_ELIMIT, "batch_run: the resident batch needs more open-search survivor lists than the arena budget allows; use score_batch");
        return rc;
    }
    finish_counters(S);
    return 0;
}
extern "C" int sage_b200_batch_download(sage_b200_scorer* S, sage_b200_feature* features, uint32_t* counts) {
    if (!S || !features || !counts) return fail(SAGE_B200_EINVAL, "batch_download: null argument");
    std::lock_guard<std::mutex> lock(S->mu);
    CUDA_TRY(cudaSetDevice(S->db->device));
    Lane& L = S->lanes[0];
    int rc = chunk_download(S, L, features, counts);
    if (rc) return rc;
    return lane_finish(S, L);
}

extern "C" int64_t sage_b200_initial_hits(sage_b200_scorer* S, const sage_b200_spectra* sp, uint16_t* matched, uint32_t* peptide, uint8_t* charge,
                                          int8_t* isotope_error, uint64_t cap, uint64_t* matched_peaks, uint64_t* scored_candidates) {
    if (!S) return fail(SAGE_B200_EINVAL, "initial_hits: null scorer");
    int rc = check_spectra(sp);
    if (rc) return rc;
    if (sp->n != 1) return fail(SAGE_B200_EINVAL, "initial_hits takes exactly one spectrum");
    std::lock_guard<std::mutex> lock(S->mu);
    CUDA_TRY(cudaSetDevice(S->db->device));
    S->last = sage_b200_counters{};
    std::vector<sage_b200_feature> f(S->sv.report_psms);
    uint32_t cnt = 0;
    Lane& L = S->lanes[0];
    if ((rc = chunk_upload(S, L, sp, 0, 1))) return rc;
    if ((rc = chunk_run(S, L, true))) return rc;
    if ((rc = chunk_download(S, L, f.data(), &cnt))) return rc;
    if ((rc = lane_finish(S, L))) return rc;
    L.chunk.loaded = false;
    std::vector<uint64_t> keys(S->sv.kparam);
    uint32_t meta[4] = {0, 0, 0, 0};
    CUDA_TRY(cudaMemcpyAsync(keys.data(), L.d_dbgk.p, 8 * (size_t)S->sv.kparam, cudaMemcpyDeviceToHost, L.stream));
    if ((rc = read_back(L.stream, meta, L.d_dbgm.p, 16))) return rc;
    const uint32_t nk = meta[0];
    for (uint32_t i = 0; i < nk && i < cap; i++) {
        const uint64_t k = keys[i];
        if (matched) matched[i] = (uint16_t)(k >> 48);
        if (peptide) peptide[i] = (uint32_t)(k >> 16);
        if (charge) charge[i] = (uint8_t)(k >> 8);
        if (isotope_error) isotope_error[i] = (int8_t)((int)(k & 0xFF) - 128);
    }
    if (matched_peaks) *matched_peaks = meta[1];
    if (scored_candidates) *scored_candidates = meta[2];
    return (int64_t)nk;
}

// k_process_ms2's shared memory for spectra of at most pmax raw peaks (p2: pmax rounded up to a power of two), or ELIMIT past its budget.
static int ms2_smem(uint32_t pmax, uint32_t& p2, size_t& smem) {
    p2 = 1;
    while (p2 < pmax) p2 <<= 1;
    smem = (size_t)p2 * 12 + (size_t)pmax * (5 * 4 + 2) + 32;
    if (smem > 200 * 1024) return fail(SAGE_B200_ELIMIT, "spectrum with %u raw peaks exceeds the shared-memory budget of the preprocessing kernel", pmax);
    return 0;
}

// SpectrumProcessor::new(take_top_n, deisotope, min_deisotope_mz).process(..) for a batch of centroided MS2 RawSpectrum (spectrum.rs:271-412).
extern "C" int sage_b200_process_spectra(int device, const sage_b200_processor_params* pr, const sage_b200_raw_spectra* raw, uint64_t* out_peak_offsets,
                                         float* out_masses, float* out_intensities, float* out_tic) {
    if (!pr || !raw || !out_peak_offsets || !out_tic) return fail(SAGE_B200_EINVAL, "process_spectra: null argument");
    if (int rc = select_device(device)) return rc;
    cudaGetLastError();   // a stale non-sticky error left by another user of the runtime must not be blamed on the launches below
    const uint64_t n = raw->n;
    out_peak_offsets[0] = 0;
    if (n == 0) return 0;
    if (!raw->peak_offsets || !raw->precursor_charge) return fail(SAGE_B200_EINVAL, "process_spectra: null array");
    const uint64_t pk0 = raw->peak_offsets[0], npk = raw->peak_offsets[n] - pk0;
    if (npk && (!raw->mz || !raw->intensity || !out_masses || !out_intensities)) return fail(SAGE_B200_EINVAL, "process_spectra: null peak arrays");
    if (n > 0x7FFFFFFFull || npk > 0xFFFFFFF0ull) return fail(SAGE_B200_ELIMIT, "process_spectra: batch too large");
    std::vector<uint32_t> off(n + 1);
    uint32_t pmax = 1;
    for (uint64_t i = 0; i <= n; i++) off[i] = (uint32_t)(raw->peak_offsets[i] - pk0);
    for (uint64_t i = 0; i < n; i++) {
        if (raw->level && raw->level[i] != 2) return fail(SAGE_B200_ENOTMS2, "process_spectra handles MS2 spectra only (spectrum %llu has level %u)", (unsigned long long)i, raw->level[i]);
        pmax = std::max(pmax, off[i + 1] - off[i]);
    }
    uint32_t p2 = 1;
    size_t smem = 0;
    if (int rc = ms2_smem(pmax, p2, smem)) return rc;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    uint32_t *d_off = nullptr, *d_cnt = nullptr;
    float *d_mz = nullptr, *d_int = nullptr, *d_om = nullptr, *d_oi = nullptr, *d_tic = nullptr;
    uint8_t* d_chg = nullptr;
    CUDA_TRY(A.upload(&d_off, off.data(), n + 1, st));
    CUDA_TRY(A.upload(&d_mz, raw->mz + pk0, npk, st, 4));
    CUDA_TRY(A.upload(&d_int, raw->intensity + pk0, npk, st, 4));
    CUDA_TRY(A.upload(&d_chg, raw->precursor_charge, n, st));
    CUDA_TRY(A.alloc(&d_om, npk + 4));
    CUDA_TRY(A.alloc(&d_oi, npk + 4));
    CUDA_TRY(A.alloc(&d_cnt, n));
    CUDA_TRY(A.alloc(&d_tic, n));
    ProcParams pp{(uint32_t)std::min<uint64_t>(pr->take_top_n, 0xFFFFFFFFull), pr->deisotope ? 1u : 0u, pr->min_deisotope_mz};
    if (int rc = ensure_kernel_attributes(device)) return rc;
    LAUNCH(k_process_ms2<<<(unsigned)n, 32, smem, st>>>(pp, (uint32_t)n, d_off, d_mz, d_int, d_chg, pmax, p2, d_om, d_oi, d_cnt, d_tic));
    std::vector<uint32_t> cnt(n);
    std::vector<float> om(npk), oi(npk);
    CUDA_TRY(cudaMemcpyAsync(cnt.data(), d_cnt, 4 * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out_tic, d_tic, 4 * n, cudaMemcpyDeviceToHost, st));
    if (npk) {
        CUDA_TRY(cudaMemcpyAsync(om.data(), d_om, 4 * npk, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(oi.data(), d_oi, 4 * npk, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    uint64_t w = 0;   // compact: spectrum i keeps cnt[i] <= raw count peaks
    for (uint64_t i = 0; i < n; i++) {
        memcpy(out_masses + w, om.data() + off[i], 4 * (size_t)cnt[i]);
        memcpy(out_intensities + w, oi.data() + off[i], 4 * (size_t)cnt[i]);
        w += cnt[i];
        out_peak_offsets[i + 1] = w;
    }
    return 0;
}

// Launches the processing of the batch's spectra that are not MS2 (spectra.cuh) on st. `a` points at device arrays; off and level are the
// host's copies of a.in_off and a.level (level NULL: every spectrum is MS1). Temporaries of the large size class come from A.
static int raw_launch(cudaStream_t st, DevArena& A, RawArgs a, const uint64_t* off, const uint8_t* level) {
    std::vector<uint32_t> slot(a.n, 0), large;
    uint32_t pmax = 0;
    bool any = false;
    for (uint32_t s = 0; s < a.n; s++) {
        if (level && level[s] == 2) continue;
        any = true;
        const uint64_t np = off[s + 1] - off[s];
        if (np > RAW_SMEM_PEAKS) {
            slot[s] = (uint32_t)large.size();
            large.push_back(s);
        } else pmax = std::max(pmax, (uint32_t)np);
    }
    if (!any) return 0;
    uint32_t p2 = 1;
    while (p2 < pmax) p2 <<= 1;
    const uint64_t npk = off[a.n] - off[0];
    const int nl = (int)large.size();
    uint32_t *d_ids = nullptr, *key_out = nullptr, *val_out = nullptr;
    if (nl) {
        uint32_t* d_slot = nullptr;
        CUDA_TRY(A.upload(&d_slot, slot.data(), a.n, st));
        CUDA_TRY(A.upload(&d_ids, large.data(), large.size(), st));
        CUDA_TRY(A.alloc(&a.seg_begin, large.size()));
        CUDA_TRY(A.alloc(&a.seg_end, large.size()));
        CUDA_TRY(A.alloc(&a.sort_key, npk));
        CUDA_TRY(A.alloc(&a.sort_val, npk));
        CUDA_TRY(A.alloc(&key_out, npk));
        CUDA_TRY(A.alloc(&val_out, npk));
        a.large_slot = d_slot;
    }
    LAUNCH(k_raw_process<<<a.n, RAW_THREADS, (size_t)p2 * 12, st>>>(a));
    if (nl) {
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) {
            return cub::DeviceSegmentedSort::StableSortPairs(t, b, a.sort_key, key_out, a.sort_val, val_out, (int)npk, nl, a.seg_begin, a.seg_end, st);
        }));
        a.sort_key = key_out;
        a.sort_val = val_out;
        LAUNCH(k_raw_gather_large<<<nl, RAW_THREADS, 0, st>>>(a, d_ids));
    }
    return 0;
}

// SpectrumProcessor::process (spectrum.rs:338-412) for a batch of any MS levels: level 2 through k_process_ms2, the others through spectra.cuh.
extern "C" int sage_b200_process_raw(int device, const sage_b200_processor_params* pr, const sage_b200_raw_batch* raw, uint64_t* out_peak_offsets,
                                     float* out_masses, float* out_intensities, float* out_mobilities, float* out_tic) {
    if (!pr || !raw || !out_peak_offsets || !out_tic) return fail(SAGE_B200_EINVAL, "process_raw: null argument");
    const uint64_t n = raw->n;
    if (n && (!raw->peak_offsets || !raw->level)) return fail(SAGE_B200_EINVAL, "process_raw: null array");
    const uint64_t pk0 = n ? raw->peak_offsets[0] : 0, npk = n ? raw->peak_offsets[n] - pk0 : 0;
    if (npk && (!raw->mz || !raw->intensity || !out_masses || !out_intensities || !out_mobilities))
        return fail(SAGE_B200_EINVAL, "process_raw: null peak arrays");
    if (n > 0x7FFFFFFEull || npk > 0x7FFFFFFFull) return fail(SAGE_B200_ELIMIT, "process_raw: more than 2^31 - 2 spectra or 2^31 - 1 peaks");
    std::vector<uint64_t> off(n + 1);
    std::vector<uint32_t> ms2_ids, ms2_off(1, 0), ms2_pos(n, 0);
    std::vector<uint8_t> ms2_chg;
    uint32_t pmax2 = 1;
    for (uint64_t i = 0; i <= n; i++) {
        if (i < n && raw->peak_offsets[i + 1] < raw->peak_offsets[i])
            return fail(SAGE_B200_EINVAL, "process_raw: peak_offsets not monotone at spectrum %llu", (unsigned long long)i);
        off[i] = raw->peak_offsets[i] - pk0;
    }
    for (uint64_t i = 0; i < n; i++) {
        if (raw->level[i] != 2) continue;
        if (!raw->precursor_charge) return fail(SAGE_B200_EINVAL, "process_raw: spectrum %llu is MS2 and precursor_charge is NULL", (unsigned long long)i);
        const uint32_t np = (uint32_t)(off[i + 1] - off[i]);
        ms2_pos[i] = (uint32_t)ms2_ids.size();
        ms2_ids.push_back((uint32_t)i);
        ms2_off.push_back(ms2_off.back() + np);
        ms2_chg.push_back(raw->precursor_charge[i]);
        pmax2 = std::max(pmax2, np);
    }
    uint32_t p2 = 1;
    size_t smem = 0;
    if (!ms2_ids.empty()) {
        if (int rc = ms2_smem(pmax2, p2, smem)) return rc;
    }
    out_peak_offsets[0] = 0;
    if (n == 0) return 0;
    if (int rc = select_device(device)) return rc;
    cudaGetLastError();   // a stale non-sticky error left by another user of the runtime must not be blamed on the launches below
    {
        // inputs and outputs (28 B per peak), the level-2 copies (16 B per level-2 peak), and the large class's sort (16 B per peak)
        size_t free_b = 0, total_b = 0;
        CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
        const uint64_t need = npk * 44 + (uint64_t)ms2_off.back() * 16 + n * 64 + (64ull << 20);
        if (need > free_b) return fail(SAGE_B200_ELIMIT, "process_raw: %llu peaks need about %llu bytes of device memory, %llu free", (unsigned long long)npk,
                                       (unsigned long long)need, (unsigned long long)free_b);
    }
    const uint32_t n2 = (uint32_t)ms2_ids.size();
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    RawArgs a{};
    a.n = (uint32_t)n;
    uint64_t *d_in_off = nullptr, *d_count = nullptr, *d_out_off = nullptr;
    float *d_mz = nullptr, *d_int = nullptr, *d_mob = nullptr;
    uint8_t* d_level = nullptr;
    CUDA_TRY(A.upload(&d_in_off, off.data(), n + 1, st));
    CUDA_TRY(A.upload(&d_mz, raw->mz + pk0, npk, st));
    CUDA_TRY(A.upload(&d_int, raw->intensity + pk0, npk, st));
    if (raw->mobility) CUDA_TRY(A.upload(&d_mob, raw->mobility + pk0, npk, st));
    CUDA_TRY(A.upload(&d_level, raw->level, n, st));
    CUDA_TRY(A.alloc(&d_count, n + 1));
    CUDA_TRY(A.alloc(&d_out_off, n + 1));
    CUDA_TRY(A.alloc(&a.out_mass, npk));
    CUDA_TRY(A.alloc(&a.out_int, npk));
    CUDA_TRY(A.alloc(&a.out_mob, npk));
    CUDA_TRY(A.alloc(&a.out_tic, n));
    uint32_t *d_ms2_ids = nullptr, *d_ms2_off = nullptr, *d_ms2_pos = nullptr, *d_ms2_cnt = nullptr;
    float *d_ms2_mz = nullptr, *d_ms2_in = nullptr, *d_ms2_om = nullptr, *d_ms2_oi = nullptr, *d_ms2_tic = nullptr;
    if (n2) {
        const uint64_t q = ms2_off.back();
        uint8_t* d_chg = nullptr;
        CUDA_TRY(A.upload(&d_ms2_ids, ms2_ids.data(), n2, st));
        CUDA_TRY(A.upload(&d_ms2_off, ms2_off.data(), n2 + 1, st));
        CUDA_TRY(A.upload(&d_ms2_pos, ms2_pos.data(), n, st));
        CUDA_TRY(A.upload(&d_chg, ms2_chg.data(), n2, st));
        CUDA_TRY(A.alloc(&d_ms2_mz, q + 4));
        CUDA_TRY(A.alloc(&d_ms2_in, q + 4));
        CUDA_TRY(A.alloc(&d_ms2_om, q + 4));
        CUDA_TRY(A.alloc(&d_ms2_oi, q + 4));
        CUDA_TRY(A.alloc(&d_ms2_cnt, n2));
        CUDA_TRY(A.alloc(&d_ms2_tic, n2));
        LAUNCH(k_raw_gather_ms2<<<n2, RAW_THREADS, 0, st>>>(n2, d_ms2_ids, d_ms2_off, d_in_off, d_mz, d_int, d_ms2_mz, d_ms2_in));
        ProcParams pp{(uint32_t)std::min<uint64_t>(pr->take_top_n, 0xFFFFFFFFull), pr->deisotope ? 1u : 0u, pr->min_deisotope_mz};
        if (int rc = ensure_kernel_attributes(device)) return rc;
        LAUNCH(k_process_ms2<<<n2, 32, smem, st>>>(pp, n2, d_ms2_off, d_ms2_mz, d_ms2_in, d_chg, pmax2, p2, d_ms2_om, d_ms2_oi, d_ms2_cnt, d_ms2_tic));
    }
    LAUNCH_N(k_raw_counts, n + 1, st, (uint32_t)n, d_in_off, d_level, d_ms2_pos, d_ms2_cnt, d_count);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_count, d_out_off, (int)(n + 1), st); }));
    if (n2)
        LAUNCH(k_raw_compact_ms2<<<n2, RAW_THREADS, 0, st>>>(n2, d_ms2_ids, d_ms2_off, d_ms2_cnt, d_ms2_om, d_ms2_oi, d_ms2_tic, d_out_off, a.out_mass,
                                                               a.out_int, a.out_mob, a.out_tic));
    a.in_off = d_in_off;
    a.mz = d_mz;
    a.intensity = d_int;
    a.mobility = d_mob;
    a.level = d_level;
    a.out_off = d_out_off;
    if (int rc = raw_launch(st, A, a, off.data(), raw->level)) return rc;
    if (int rc = read_back(st, out_peak_offsets, d_out_off, 8 * (n + 1))) return rc;
    const uint64_t kept = out_peak_offsets[n];
    CUDA_TRY(cudaMemcpyAsync(out_tic, a.out_tic, 4 * n, cudaMemcpyDeviceToHost, st));
    if (kept) {
        CUDA_TRY(cudaMemcpyAsync(out_masses, a.out_mass, 4 * kept, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(out_intensities, a.out_int, 4 * kept, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(out_mobilities, a.out_mob, 4 * kept, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

// tmt::find_reporter_ions over a batch of ProcessedSpectrum (tmt.rs:193-211, called from tmt::quantify tmt.rs:322-333).
extern "C" int sage_b200_find_reporter_ions(int device, uint64_t n, const uint64_t* peak_offsets, const float* masses, const float* intensities, const float* labels,
                                            uint64_t n_labels, sage_b200_tolerance label_tolerance, float* out) {
    if (n == 0 || n_labels == 0) return 0;
    if (!peak_offsets || !labels || !out) return fail(SAGE_B200_EINVAL, "find_reporter_ions: null argument");
    if (int rc = select_device(device)) return rc;
    if (label_tolerance.kind < 0 || label_tolerance.kind > 2) return fail(SAGE_B200_EINVAL, "bad tolerance kind");
    const uint64_t pk0 = peak_offsets[0], npk = peak_offsets[n] - pk0;
    if (npk && (!masses || !intensities)) return fail(SAGE_B200_EINVAL, "find_reporter_ions: null peak arrays");
    if (n > 0x7FFFFFFFull || npk > 0xFFFFFFF0ull || n_labels > 4096) return fail(SAGE_B200_ELIMIT, "find_reporter_ions: batch too large");
    std::vector<uint32_t> off(n + 1);
    for (uint64_t i = 0; i <= n; i++) off[i] = (uint32_t)(peak_offsets[i] - pk0);
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    uint32_t* d_off = nullptr;
    float *d_m = nullptr, *d_i = nullptr, *d_l = nullptr, *d_o = nullptr;
    const uint64_t total = n * n_labels;
    CUDA_TRY(A.upload(&d_off, off.data(), n + 1, st));
    CUDA_TRY(A.upload(&d_m, masses + pk0, npk, st, 4));
    CUDA_TRY(A.upload(&d_i, intensities + pk0, npk, st, 4));
    CUDA_TRY(A.upload(&d_l, labels, n_labels, st));
    CUDA_TRY(A.alloc(&d_o, total));
    LAUNCH_N(k_find_reporter_ions, total, st, (uint32_t)n, (uint32_t)n_labels, d_off, d_m, d_i, d_l,
             Tol{label_tolerance.kind, label_tolerance.lo, label_tolerance.hi}, d_o);
    return read_back(st, out, d_o, 4 * total);
}

__global__ void k_device_log(int variant, const double* x, uint64_t n, double* out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = variant == 2 ? (double)glog::glibc_log1pf((float)x[i]) : glog::glibc_log_v(x[i], variant);
}
extern "C" int sage_b200_device_log(int device, int variant, const double* x, uint64_t n, double* out) {
    if (n == 0) return 0;
    if (!x || !out || variant < 0 || variant > 2) return fail(SAGE_B200_EINVAL, "device_log: bad argument");
    if (int rc = select_device(device)) return rc;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    double *dx = nullptr, *dy = nullptr;
    CUDA_TRY(A.upload(&dx, x, n, st));
    CUDA_TRY(A.alloc(&dy, n));
    LAUNCH_N(k_device_log, n, st, variant, dx, n, dy);
    return read_back(st, out, dy, 8 * n);
}

extern "C" int sage_b200_counters_get(const sage_b200_scorer* S, sage_b200_counters* out) {
    if (!S || !out) return fail(SAGE_B200_EINVAL, "counters_get: null argument");
    *out = S->last;
    return 0;
}

// Page-locked buffer for a batch that sage_b200_score_batch_multi will cut into n contiguous blocks: block i is first-touched by a thread bound to
// the NUMA node of devices[i] and then the whole region is registered with CUDA, so every GPU DMA-reads its block from the memory next to it
// (one buffer allocated by one thread would sit on a single node and half of the GPUs of a two-socket box would pull across the socket link).
static std::mutex g_blocks_mu;
static std::vector<std::pair<void*, size_t>> g_blocks;
extern "C" void* sage_b200_host_alloc_blocks(size_t bytes, const int* devices, int n_devices) {
    if (bytes == 0) bytes = 16;
    const size_t page = 4096, total = (bytes + page - 1) / page * page;
    void* p = aligned_alloc(page, total);
    if (!p) { fail(SAGE_B200_ECUDA, "host_alloc_blocks: out of memory (%zu bytes)", total); return nullptr; }
    const int n = (devices && n_devices > 0) ? n_devices : 1;
    std::vector<std::thread> th;
    for (int g = 0; g < n; g++) {
        const size_t a = (total / page) * (size_t)g / (size_t)n * page, b = (total / page) * (size_t)(g + 1) / (size_t)n * page;
        th.emplace_back([=]() {
            if (devices) sage_b200_bind_thread_to_device(devices[g]);
            memset((char*)p + a, 0, b - a);   // first touch places the pages
        });
    }
    for (auto& t : th) t.join();
    if (cudaHostRegister(p, total, cudaHostRegisterPortable) != cudaSuccess) {
        cudaGetLastError();
        free(p);
        fail(SAGE_B200_ECUDA, "host_alloc_blocks: cudaHostRegister(%zu) failed", total);
        return nullptr;
    }
    std::lock_guard<std::mutex> lock(g_blocks_mu);
    g_blocks.emplace_back(p, total);
    return p;
}

extern "C" void* sage_b200_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 16, cudaHostAllocPortable) != cudaSuccess) {
        fail(SAGE_B200_ECUDA, "cudaHostAlloc(%zu) failed", bytes);
        cudaGetLastError();
        return nullptr;
    }
    return p;
}
extern "C" void sage_b200_host_free(void* p) {
    if (!p) return;
    {
        std::lock_guard<std::mutex> lock(g_blocks_mu);
        for (size_t i = 0; i < g_blocks.size(); i++)
            if (g_blocks[i].first == p) {
                cudaHostUnregister(p);
                free(p);
                g_blocks.erase(g_blocks.begin() + i);
                return;
            }
    }
    cudaFreeHost(p);
}

extern "C" size_t sage_b200_last_error(char* buf, size_t cap) {
    if (buf && cap) {
        snprintf(buf, cap, "%s", g_last_error.c_str());
    }
    return g_last_error.size();
}

// ================================================================================== label-free quantification (lfq.rs, kernels in lfq.cuh)
// The feature map (sorted PrecursorRange pages) and one dense f64 grid per possible (PrecursorId, decoy) key stay on the device; a key's grid
// is "touched" once a contribution reached it, which is when the reference's DashMap would have created it (lfq.rs:250-262).
static constexpr uint32_t LFQ_MAX_FILES = 128;              // k_lfq_integrate keeps 2 x 100 f64 per file in shared memory
static constexpr uint64_t LFQ_CHUNK_PEAKS = 1ull << 24;     // add_ms1 traces at most this many peaks per pass (results do not depend on it)

struct sage_b200_lfq {
    std::mutex mu;
    int device = 0;
    sage_b200_lfq_params p{};
    uint32_t n_files = 0, n_charges = 0;
    uint64_t n_slots = 0, n_ranges = 0, n_pages = 0, n_grids = 0;
    DevArena fixed;   // the arrays below, exact-size
    sage_b200_lfq_range* d_ranges = nullptr;
    uint32_t *d_grid_of = nullptr, *d_slot_file = nullptr;
    float *d_min_rts = nullptr, *d_slot_dist = nullptr;
    double *d_grids = nullptr, *d_consts = nullptr;
    uint8_t* d_touched = nullptr;
    sage_b200_alignment* d_align = nullptr;
    std::vector<uint32_t> slot_pep;   // slot -> PeptideIx, ascending
    DevBuf sp_off, sp_mass, sp_int, sp_mob, raw_mz, raw_int, raw_mob, sp_file, sp_sst, counts, offsets, cell[2], value[2], tmp, ids, o_present, o_rt, o_sa, o_score, o_areas;
    Stream st;
    Event ev[2];
    sage_b200_lfq_info info{};
    uint64_t scratch_bytes() const {
        uint64_t b = 0;
        for (const DevBuf* d : {&sp_off, &sp_mass, &sp_int, &sp_mob, &raw_mz, &raw_int, &raw_mob, &sp_file, &sp_sst, &counts, &offsets, &cell[0], &cell[1], &value[0], &value[1], &tmp, &ids,
                                &o_present, &o_rt, &o_sa, &o_score, &o_areas})
            b += d->cap;
        return b;
    }
};

// composition (mass.rs:78-116): carbon and sulfur count of one residue
static void residue_composition(uint8_t aa, uint16_t& c, uint16_t& s) {
    static const uint8_t carbon[26] = {3, 0, 3, 4, 5, 9, 2, 6, 6, 0, 6, 6, 5, 4, 12, 5, 5, 6, 3, 4, 3, 5, 11, 0, 9, 0};   // A..Z (B J X Z: 0)
    c = 0;
    s = 0;
    if (aa < 'A' || aa > 'Z') return;
    c = carbon[aa - 'A'];
    s = (aa == 'C' || aa == 'M') ? 1 : 0;
}

// the event-timed span of one stage: ms += elapsed(ev0, ev1) after a synchronize
static int lfq_elapsed(sage_b200_lfq* L, float& ms) {
    CUDA_TRY(cudaEventRecord(L->ev[1], L->st));
    CUDA_TRY(cudaEventSynchronize(L->ev[1]));
    float t = 0.0f;
    CUDA_TRY(cudaEventElapsedTime(&t, L->ev[0], L->ev[1]));
    ms += t;
    return 0;
}

extern "C" void sage_b200_lfq_destroy(sage_b200_lfq* L) {
    if (!L) return;
    cudaSetDevice(L->device);
    delete L;
}

static int lfq_build(sage_b200_lfq* L, const sage_b200_db* db, const sage_b200_peptides* P, const sage_b200_lfq_features* F, const sage_b200_alignment* align) {
    const uint64_t n = F->n, n_pep = db->v.n_pep;
    cudaStream_t st = L->st;
    CUDA_TRY(cudaEventRecord(L->ev[0], st));
    // per-peptide first kept row (lfq.rs:100-131)
    DevArena A;
    uint32_t *d_rows[7] = {}, *d_first = nullptr, *d_slots = nullptr, *d_nsel = nullptr;   // d_rows: the feature columns, 4 bytes per row each
    uint8_t* d_flag = nullptr;
    const void* src[7] = {F->peptide_idx, F->peptide_q, F->label, F->aligned_rt, F->calcmass, F->file_id, F->ims};
    for (int k = 0; k < 7; k++) CUDA_TRY(A.upload(&d_rows[k], (const uint32_t*)src[k], n, st, 4));
    CUDA_TRY(A.alloc(&d_first, n_pep + 4));
    CUDA_TRY(A.alloc(&d_flag, n_pep + 16));
    CUDA_TRY(A.alloc(&d_slots, n_pep + 4));
    CUDA_TRY(A.alloc(&d_nsel, 4));
    CUDA_TRY(cudaMemsetAsync(d_first, 0xFF, 4 * n_pep, st));
    LAUNCH_N(k_lfq_first_row, n, st, n, d_rows[0], (const float*)d_rows[1], (const int32_t*)d_rows[2], L->p.peptide_q_value, d_first);
    LAUNCH_N(k_lfq_flag, n_pep, st, n_pep, d_first, d_flag);
    thrust::counting_iterator<uint32_t> it(0);
    CUDA_TRY(L->tmp.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, it, d_flag, d_slots, d_nsel, (int)n_pep, st); }));
    uint32_t n_slots = 0;
    if (int rc = read_back(st, &n_slots, d_nsel, 4)) return rc;
    std::vector<uint32_t> slot_pep(n_slots);
    if (n_slots)
        if (int rc = read_back(st, slot_pep.data(), d_slots, 4ull * n_slots)) return rc;

    L->n_slots = n_slots;
    L->slot_pep = slot_pep;
    L->n_ranges = (uint64_t)n_slots * L->n_charges * LFQ_ISO * 2;
    L->n_pages = (L->n_ranges + LFQ_PAGE - 1) / LFQ_PAGE;
    L->n_grids = (uint64_t)n_slots * (L->p.combine_charge_states ? 1 : L->n_charges) * 2;
    if (L->n_ranges > 0x7FFFFFFFull) return fail(SAGE_B200_ELIMIT, "%llu precursor ranges exceed 2^31", (unsigned long long)L->n_ranges);
    const uint64_t cells = L->n_grids * L->n_files * LFQ_ISO * LFQ_GRID, grid_bytes = 8 * cells;
    {
        size_t free_b = 0, total_b = 0;
        CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
        // the grids plus the map, leaving room for the tracing and integration scratch
        const uint64_t need = grid_bytes + L->n_grids + 40 * L->n_ranges + (1ull << 28);
        if (need > (uint64_t)free_b)
            return fail(SAGE_B200_ELIMIT, "LFQ grids need %llu bytes of device memory (%llu grids x %u files x 300 f64) but %llu are free",
                        (unsigned long long)need, (unsigned long long)L->n_grids, L->n_files, (unsigned long long)free_b);
    }

    // isotope distributions: composition on the host, peptide_isotopes on the device with host-libm exp tables
    std::vector<uint16_t> carbon(n_slots), sulfur(n_slots);
    uint16_t max_c = 0, max_s = 0;
    for (uint32_t s = 0; s < n_slots; s++) {
        uint32_t c = 0, su = 0;
        for (uint32_t r = P->residue_offsets[slot_pep[s]]; r < P->residue_offsets[slot_pep[s] + 1]; r++) {
            uint16_t rc_, rs_;
            residue_composition(P->sequence[r], rc_, rs_);
            c += rc_;
            su += rs_;
        }
        carbon[s] = (uint16_t)c;
        sulfur[s] = (uint16_t)su;
        max_c = std::max(max_c, carbon[s]);
        max_s = std::max(max_s, sulfur[s]);
    }
    std::vector<float> expt((size_t)max_c + 1 + 2 * ((size_t)max_s + 1));
    float* exp_c = expt.data();
    float* exp_s33 = exp_c + max_c + 1;
    float* exp_s35 = exp_s33 + max_s + 1;
    for (uint32_t c = 0; c <= max_c; c++) exp_c[c] = std::exp(-((float)c * 0.011f));
    for (uint32_t s = 0; s <= max_s; s++) {
        exp_s33[s] = std::exp(-((float)s * 0.0076f));
        exp_s35[s] = std::exp(-((float)s * 0.044f));
    }
    // gaussian_kernel(0.5, 10) (lfq.rs:614-628) and the RT factor of scores (lfq.rs:425, 430-431)
    double consts[LFQ_K_WIDTH + LFQ_GRID];
    {
        const double sigma = 0.5, step = 2.0 / (double)(LFQ_K_WIDTH - 1), constant = 1.0 / (sigma * std::sqrt(2.0 * 3.141592653589793));
        double sum = 0.0;
        for (int i = 0; i < LFQ_K_WIDTH; i++) {
            const double x = (double)i * step - 1.0, xs = x / sigma;
            consts[i] = constant * std::exp(-0.5 * (xs * xs));
            sum = sum + consts[i];
        }
        for (int i = 0; i < LFQ_K_WIDTH; i++) consts[i] = consts[i] / sum;
        const int center = LFQ_GRID / 2;
        for (int rt = 0; rt < LFQ_GRID; rt++) consts[LFQ_K_WIDTH + rt] = std::pow(1.0 - ((double)std::abs(rt - center) / (double)center), 0.33);
    }

    CUDA_TRY(L->fixed.alloc(&L->d_ranges, L->n_ranges));
    CUDA_TRY(L->fixed.alloc(&L->d_grid_of, L->n_ranges));
    CUDA_TRY(L->fixed.alloc(&L->d_min_rts, L->n_pages));
    CUDA_TRY(L->fixed.alloc(&L->d_slot_dist, 3ull * n_slots));
    CUDA_TRY(L->fixed.alloc(&L->d_slot_file, n_slots));
    CUDA_TRY(L->fixed.zeros(&L->d_touched, L->n_grids, st));
    CUDA_TRY(L->fixed.upload(&L->d_align, align, L->n_files, st));
    CUDA_TRY(L->fixed.upload(&L->d_consts, consts, LFQ_K_WIDTH + LFQ_GRID, st));
    CUDA_TRY(L->fixed.zeros(&L->d_grids, cells, st));
    if (n_slots) {
        uint16_t *d_c = nullptr, *d_s = nullptr;
        float* d_exp = nullptr;
        CUDA_TRY(A.upload(&d_c, carbon.data(), n_slots, st));
        CUDA_TRY(A.upload(&d_s, sulfur.data(), n_slots, st));
        CUDA_TRY(A.upload(&d_exp, expt.data(), expt.size(), st));
        LAUNCH_N(k_lfq_isotopes, n_slots, st, n_slots, d_c, d_s, d_exp, d_exp + max_c + 1, d_exp + max_c + 1 + max_s + 1, L->d_slot_dist);

        // expansion, stable RT sort, stable per-page mass_lo sort (lfq.rs:134-184)
        const uint32_t nr = (uint32_t)L->n_ranges, nt = (uint32_t)(n_slots * L->n_charges * LFQ_ISO);
        DevArena B;   // freed before the call returns
        sage_b200_lfq_range* pre = nullptr;
        uint32_t *k32[2] = {}, *v32[2] = {};
        uint64_t *k64 = nullptr, *k64o = nullptr;
        CUDA_TRY(B.alloc(&pre, nr));
        for (int k = 0; k < 2; k++) {
            CUDA_TRY(B.alloc(&k32[k], nr));
            CUDA_TRY(B.alloc(&v32[k], nr));
        }
        CUDA_TRY(B.alloc(&k64, nr));
        LAUNCH_N(k_lfq_expand, nt, st, n_slots, L->n_charges, L->p.min_precursor_charge, L->p.ppm_tolerance, L->p.mobility_pct_tolerance, d_slots, d_first,
                 (const float*)d_rows[3], (const float*)d_rows[4], d_rows[5], (const float*)d_rows[6], pre, k32[0], v32[0], L->d_slot_file);
        size_t tb = 0, tb2 = 0;
        CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, k32[0], k32[1], v32[0], v32[1], (int)nr, 0, 32, st));
        CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb2, k64, k64, v32[1], v32[0], (int)nr, 0, 64, st));
        if (int rc = L->tmp.reserve(std::max(tb, tb2))) return rc;
        CUDA_TRY(cub::DeviceRadixSort::SortPairs(L->tmp.p, tb, k32[0], k32[1], v32[0], v32[1], (int)nr, 0, 32, st));
        LAUNCH_N(k_lfq_page_keys, nr, st, nr, v32[1], pre, k64, L->d_min_rts);
        CUDA_TRY(B.alloc(&k64o, nr));
        const int end_bit = 32 + (int)ceil_log2_u64(L->n_pages + 1);
        CUDA_TRY(cub::DeviceRadixSort::SortPairs(L->tmp.p, tb2, k64, k64o, v32[1], v32[0], (int)nr, 0, end_bit, st));
        LAUNCH_N(k_lfq_gather, nr, st, nr, L->n_charges, L->p.combine_charge_states, v32[0], pre, L->d_ranges, L->d_grid_of);
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    return lfq_elapsed(L, L->info.ms_build);
}

extern "C" int sage_b200_lfq_create(const sage_b200_db* db, const sage_b200_peptides* peptides, const sage_b200_lfq_params* params,
                                    const sage_b200_lfq_features* features, uint64_t n_files, const sage_b200_alignment* alignments, sage_b200_lfq** out) {
    if (int rc = select_device(db ? db->device : 0)) return rc;
    if (!db || !peptides || !params || !features || !out || !alignments) return fail(SAGE_B200_EINVAL, "lfq_create: null argument");
    if (peptides->n_peptides != db->v.n_pep || (peptides->n_peptides && (!peptides->residue_offsets || !peptides->sequence)))
        return fail(SAGE_B200_EINVAL, "lfq_create: peptides is not the table the db was built from");
    if (n_files == 0) return fail(SAGE_B200_EINVAL, "lfq_create: n_files must be >= 1");
    if (n_files > LFQ_MAX_FILES) return fail(SAGE_B200_ELIMIT, "lfq_create: %llu files (at most %u supported)", (unsigned long long)n_files, LFQ_MAX_FILES);
    if (params->peak_scoring < 0 || params->peak_scoring > 3 || params->integration < 0 || params->integration > 1)
        return fail(SAGE_B200_EINVAL, "lfq_create: bad peak_scoring / integration");
    if (params->min_precursor_charge == 0 || params->min_precursor_charge > params->max_precursor_charge)
        return fail(SAGE_B200_EINVAL, "lfq_create: precursor_charge must be (min, max) with 1 <= min <= max");
    const sage_b200_lfq_features* F = features;
    if (F->n && (!F->peptide_idx || !F->peptide_q || !F->label || !F->aligned_rt || !F->calcmass || !F->file_id || !F->ims))
        return fail(SAGE_B200_EINVAL, "lfq_create: null feature array");
    if (F->n > 0xFFFFFFFEull) return fail(SAGE_B200_ELIMIT, "lfq_create: more than 2^32 - 2 features");
    for (uint64_t i = 0; i < F->n; i++) {
        if (!(F->peptide_q[i] <= params->peptide_q_value && F->label[i] == 1)) continue;
        if (F->peptide_idx[i] >= db->v.n_pep)
            return fail(SAGE_B200_EINVAL, "lfq_create: feature %llu has peptide_idx %u outside the db", (unsigned long long)i, F->peptide_idx[i]);
        if (F->file_id[i] >= n_files)
            return fail(SAGE_B200_EINVAL, "lfq_create: feature %llu has file_id %u >= n_files %llu", (unsigned long long)i, F->file_id[i], (unsigned long long)n_files);
    }
    Guard<sage_b200_lfq> guard(new sage_b200_lfq(), sage_b200_lfq_destroy);
    sage_b200_lfq* L = guard.get();
    L->device = db->device;
    L->p = *params;
    L->n_files = (uint32_t)n_files;
    L->n_charges = (uint32_t)params->max_precursor_charge - params->min_precursor_charge + 1;
    CUDA_TRY(L->st.create());
    for (Event& e : L->ev) CUDA_TRY(e.create());
    if (int rc = lfq_build(L, db, peptides, F, alignments)) return rc;
    L->info.n_peptides = L->n_slots;
    L->info.n_ranges = L->n_ranges;
    L->info.n_pages = L->n_pages;
    L->info.n_grids = L->n_grids;
    L->info.n_files = L->n_files;
    *out = guard.release();
    return 0;
}

// One pass of the tracing loop over spectra [a, b) of the batch (peaks already counted to fit LFQ_CHUNK_PEAKS unless a single spectrum is larger).
// raw: m holds raw MS1 spectra (masses are m/z, in any order), uploaded to the raw_* buffers and processed into the sp_* ones first.
static int lfq_trace_chunk(sage_b200_lfq* L, const sage_b200_ms1* m, uint64_t a, uint64_t b, bool raw) {
    cudaStream_t st = L->st;
    const uint64_t ns = b - a, p0 = m->peak_offsets[a], np = m->peak_offsets[b] - p0;
    std::vector<uint64_t> off(ns + 1);
    for (uint64_t i = 0; i <= ns; i++) off[i] = m->peak_offsets[a + i] - p0;
    int rc;
    if ((rc = L->sp_off.reserve(8 * (ns + 1))) || (rc = L->sp_mass.reserve(4 * np + 16)) || (rc = L->sp_int.reserve(4 * np + 16)) ||
        (rc = L->sp_file.reserve(4 * ns)) || (rc = L->sp_sst.reserve(4 * ns)) || (rc = L->counts.reserve(8 * np + 16)) || (rc = L->offsets.reserve(8 * np + 16)) ||
        (m->mobilities && (rc = L->sp_mob.reserve(4 * np + 16))))
        return rc;
    if (raw && ((rc = L->raw_mz.reserve(4 * np + 16)) || (rc = L->raw_int.reserve(4 * np + 16)) || (m->mobilities && (rc = L->raw_mob.reserve(4 * np + 16)))))
        return rc;
    DevBuf &up_mass = raw ? L->raw_mz : L->sp_mass, &up_int = raw ? L->raw_int : L->sp_int, &up_mob = raw ? L->raw_mob : L->sp_mob;
    CUDA_TRY(cudaMemcpyAsync(L->sp_off.p, off.data(), 8 * (ns + 1), cudaMemcpyHostToDevice, st));
    if (np) {
        CUDA_TRY(cudaMemcpyAsync(up_mass.p, m->masses + p0, 4 * np, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(up_int.p, m->intensities + p0, 4 * np, cudaMemcpyHostToDevice, st));
        if (m->mobilities) CUDA_TRY(cudaMemcpyAsync(up_mob.p, m->mobilities + p0, 4 * np, cudaMemcpyHostToDevice, st));
    }
    CUDA_TRY(cudaMemcpyAsync(L->sp_file.p, m->file_id + a, 4 * ns, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(L->sp_sst.p, m->scan_start_time + a, 4 * ns, cudaMemcpyHostToDevice, st));
    if (np == 0 || L->n_ranges == 0) return 0;
    if (raw) {   // SpectrumProcessor::process of level 1: every peak is kept, so the processed batch has the raw offsets
        RawArgs r{};
        r.n = (uint32_t)ns;
        r.in_off = r.out_off = L->sp_off.as<uint64_t>();
        r.mz = L->raw_mz.as<float>();
        r.intensity = L->raw_int.as<float>();
        r.mobility = m->mobilities ? L->raw_mob.as<float>() : nullptr;
        r.out_mass = L->sp_mass.as<float>();
        r.out_int = L->sp_int.as<float>();
        r.out_mob = m->mobilities ? L->sp_mob.as<float>() : nullptr;
        DevArena A;   // the large size class's temporaries
        if ((rc = raw_launch(st, A, r, off.data(), nullptr))) return rc;
        if (A.bytes) CUDA_TRY(cudaStreamSynchronize(st));
    }

    LfqTraceArgs t{};
    t.n_spectra = (uint32_t)ns;
    t.peak_off = L->sp_off.as<uint64_t>();
    t.masses = L->sp_mass.as<float>();
    t.intensities = L->sp_int.as<float>();
    t.mobilities = m->mobilities ? L->sp_mob.as<float>() : nullptr;
    t.file_id = L->sp_file.as<uint32_t>();
    t.sst = L->sp_sst.as<float>();
    t.align = (const sage_b200_alignment*)L->d_align;
    t.ranges = (const sage_b200_lfq_range*)L->d_ranges;
    t.grid_of = (const uint32_t*)L->d_grid_of;
    t.n_ranges = (uint32_t)L->n_ranges;
    t.n_pages = (uint32_t)L->n_pages;
    t.n_files = L->n_files;
    t.min_rts = (const float*)L->d_min_rts;
    t.counts = L->counts.as<uint64_t>();
    const unsigned blocks = (unsigned)((ns * 32 + LFQ_THREADS - 1) / LFQ_THREADS);
    LAUNCH(k_lfq_trace<false><<<blocks, LFQ_THREADS, 0, st>>>(t));
    CUDA_TRY(L->tmp.two_phase([&](void* tmp, size_t& b) { return cub::DeviceScan::ExclusiveSum(tmp, b, L->counts.as<uint64_t>(), L->offsets.as<uint64_t>(), (int)np, st); }));
    uint64_t last[2] = {0, 0};
    CUDA_TRY(cudaMemcpyAsync(&last[0], L->offsets.as<uint64_t>() + np - 1, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&last[1], L->counts.as<uint64_t>() + np - 1, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    const uint64_t matches = last[0] + last[1], nc = 2 * matches;
    if (nc == 0) return 0;
    if (nc > 0x7FFFFFFFull) return fail(SAGE_B200_ELIMIT, "one tracing pass produced %llu contributions (> 2^31): pass fewer spectra per add_ms1", (unsigned long long)nc);
    for (int k = 0; k < 2; k++)
        if ((rc = L->cell[k].reserve(8 * nc)) || (rc = L->value[k].reserve(8 * nc))) return rc;
    t.offsets = L->offsets.as<uint64_t>();
    t.cell = L->cell[0].as<uint64_t>();
    t.value = L->value[0].as<double>();
    LAUNCH(k_lfq_trace<true><<<blocks, LFQ_THREADS, 0, st>>>(t));
    const uint64_t cells = L->n_grids * L->n_files * LFQ_ISO * LFQ_GRID;
    const int end_bit = std::max(1, (int)ceil_log2_u64(cells));
    CUDA_TRY(L->tmp.two_phase([&](void* tmp, size_t& b) {
        return cub::DeviceRadixSort::SortPairs(tmp, b, L->cell[0].as<uint64_t>(), L->cell[1].as<uint64_t>(), L->value[0].as<double>(), L->value[1].as<double>(),
                                               (int)nc, 0, end_bit, st);
    }));
    LAUNCH_N(k_lfq_fold, nc, st, nc, L->cell[1].as<uint64_t>(), L->value[1].as<double>(), (double*)L->d_grids, (uint8_t*)L->d_touched,
             (uint64_t)L->n_files * LFQ_ISO * LFQ_GRID);
    L->info.contributions += nc;
    return 0;
}

// add_ms1 and add_raw_ms1 (raw: masses are raw m/z, processed on the device first). `what` names the entry point in errors.
static int lfq_add(sage_b200_lfq* L, const sage_b200_ms1* m, bool raw, const char* what) {
    std::lock_guard<std::mutex> lock(L->mu);
    if (m->n == 0) return 0;
    if (!m->peak_offsets || !m->file_id || !m->scan_start_time) return fail(SAGE_B200_EINVAL, "%s: null array", what);
    if (m->peak_offsets[m->n] > m->peak_offsets[0] && (!m->masses || !m->intensities)) return fail(SAGE_B200_EINVAL, "%s: null peak arrays", what);
    for (uint64_t i = 0; i < m->n; i++) {
        if (m->file_id[i] >= L->n_files)
            return fail(SAGE_B200_EINVAL, "%s: spectrum %llu has file_id %u >= n_files %u", what, (unsigned long long)i, m->file_id[i], L->n_files);
        if (m->peak_offsets[i + 1] < m->peak_offsets[i]) return fail(SAGE_B200_EINVAL, "%s: peak_offsets not monotone at spectrum %llu", what, (unsigned long long)i);
    }
    CUDA_TRY(cudaSetDevice(L->device));
    CUDA_TRY(cudaEventRecord(L->ev[0], L->st));
    for (uint64_t a = 0; a < m->n;) {
        uint64_t b = a + 1;
        while (b < m->n && b - a < 0x7FFFFFull && m->peak_offsets[b + 1] - m->peak_offsets[a] <= LFQ_CHUNK_PEAKS) b++;
        const int rc = lfq_trace_chunk(L, m, a, b, raw);
        if (rc) return rc;
        a = b;
    }
    L->info.ms1_spectra += m->n;
    L->info.ms1_peaks += m->peak_offsets[m->n] - m->peak_offsets[0];
    return lfq_elapsed(L, L->info.ms_trace);
}

extern "C" int sage_b200_lfq_add_ms1(sage_b200_lfq* L, const sage_b200_ms1* m) {
    if (!L || !m) return fail(SAGE_B200_EINVAL, "lfq_add_ms1: null argument");
    return lfq_add(L, m, false, "lfq_add_ms1");
}

extern "C" int sage_b200_lfq_add_raw_ms1(sage_b200_lfq* L, const sage_b200_raw_ms1* r) {
    if (!L || !r) return fail(SAGE_B200_EINVAL, "lfq_add_raw_ms1: null argument");
    const sage_b200_ms1 m{r->n, r->peak_offsets, r->mz, r->intensity, r->file_id, r->scan_start_time, r->mobility};
    return lfq_add(L, &m, true, "lfq_add_raw_ms1");
}

extern "C" int sage_b200_lfq_integrate(sage_b200_lfq* L, sage_b200_lfq_row* rows, double* areas, uint64_t capacity, uint64_t* n_rows) {
    if (!L || !n_rows) return fail(SAGE_B200_EINVAL, "lfq_integrate: null argument");
    std::lock_guard<std::mutex> lock(L->mu);
    CUDA_TRY(cudaSetDevice(L->device));
    cudaStream_t st = L->st;
    const uint32_t F = L->n_files;
    *n_rows = 0;
    if (L->n_grids == 0) return 0;
    int rc;
    CUDA_TRY(cudaEventRecord(L->ev[0], st));
    if ((rc = L->ids.reserve(4 * L->n_grids + 16)) || (rc = L->o_present.reserve(4 * L->n_grids + 16))) return rc;
    thrust::counting_iterator<uint32_t> it(0);
    uint32_t* d_n = L->o_present.as<uint32_t>() + L->n_grids;   // the selected count lives behind the present flags' room
    CUDA_TRY(L->tmp.two_phase([&](void* t, size_t& b) {
        return cub::DeviceSelect::Flagged(t, b, it, (const uint8_t*)L->d_touched, L->ids.as<uint32_t>(), d_n, (int)L->n_grids, st);
    }));
    uint32_t nt = 0;
    if ((rc = read_back(st, &nt, d_n, 4))) return rc;
    L->info.grids_touched = nt;
    if (nt == 0) { L->info.ms_integrate = 0.0f; return lfq_elapsed(L, L->info.ms_integrate); }
    if ((rc = L->o_rt.reserve(4ull * nt)) || (rc = L->o_sa.reserve(8ull * nt)) || (rc = L->o_score.reserve(8ull * nt)) || (rc = L->o_areas.reserve(8ull * nt * F)))
        return rc;
    const size_t smem = lfq_integrate_smem(F);
    CUDA_TRY(cudaFuncSetAttribute(k_lfq_integrate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    LfqIntegrateArgs a{};
    a.n = nt;
    a.grid_ids = L->ids.as<uint32_t>();
    a.grids = (const double*)L->d_grids;
    a.slot_dist = (const float*)L->d_slot_dist;
    a.slot_file = (const uint32_t*)L->d_slot_file;
    a.consts = (const double*)L->d_consts;
    a.n_files = F;
    a.n_charges = L->n_charges;
    a.combine = L->p.combine_charge_states;
    a.peak_scoring = L->p.peak_scoring;
    a.integration = L->p.integration;
    a.spectral_angle = L->p.spectral_angle;
    a.present = L->o_present.as<uint8_t>();
    a.rt = L->o_rt.as<uint32_t>();
    a.sa = L->o_sa.as<double>();
    a.score = L->o_score.as<double>();
    a.areas = L->o_areas.as<double>();
    LAUNCH(k_lfq_integrate<<<nt, LFQ_THREADS, smem, st>>>(a));
    L->info.ms_integrate = 0.0f;
    if ((rc = lfq_elapsed(L, L->info.ms_integrate))) return rc;

    // copy back and keep the grids that produced a peak, in grid order == (PrecursorId, decoy) order
    CUDA_TRY(cudaEventRecord(L->ev[0], st));
    std::vector<uint32_t> ids(nt), rt(nt);
    std::vector<uint8_t> present(nt);
    std::vector<double> sa(nt), score(nt), ar((size_t)nt * F);
    CUDA_TRY(cudaMemcpyAsync(ids.data(), L->ids.p, 4ull * nt, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(present.data(), L->o_present.p, nt, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(rt.data(), L->o_rt.p, 4ull * nt, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(sa.data(), L->o_sa.p, 8ull * nt, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(score.data(), L->o_score.p, 8ull * nt, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(ar.data(), L->o_areas.p, 8ull * nt * F, cudaMemcpyDeviceToHost, st));
    L->info.ms_download = 0.0f;
    if ((rc = lfq_elapsed(L, L->info.ms_download))) return rc;
    uint64_t k = 0;
    for (uint32_t i = 0; i < nt; i++) {
        if (!present[i]) continue;
        if (k >= capacity) return fail(SAGE_B200_ELIMIT, "lfq_integrate: capacity %llu too small (at most n_grids = %llu rows)", (unsigned long long)capacity,
                                       (unsigned long long)L->n_grids);
        const uint32_t g = ids[i], slot = L->p.combine_charge_states ? g / 2 : g / 2 / L->n_charges;
        sage_b200_lfq_row r{};
        r.peptide = L->slot_pep[slot];
        r.charge = L->p.combine_charge_states ? 0 : (uint8_t)(L->p.min_precursor_charge + (g / 2) % L->n_charges);
        r.decoy = (uint8_t)(g & 1);
        r.rt = rt[i];
        r.spectral_angle = sa[i];
        r.score = score[i];
        if (rows) rows[k] = r;
        if (areas) memcpy(areas + k * F, ar.data() + (size_t)i * F, 8ull * F);
        k++;
    }
    *n_rows = k;
    return 0;
}

extern "C" int sage_b200_lfq_get_info(sage_b200_lfq* L, sage_b200_lfq_info* info) {
    if (!L || !info) return fail(SAGE_B200_EINVAL, "lfq_get_info: null argument");
    std::lock_guard<std::mutex> lock(L->mu);
    *info = L->info;
    info->device_bytes = L->fixed.bytes + L->scratch_bytes();
    return 0;
}

extern "C" int sage_b200_lfq_export(sage_b200_lfq* L, sage_b200_lfq_range* ranges, float* min_rts, double* grids, uint8_t* touched) {
    if (!L) return fail(SAGE_B200_EINVAL, "lfq_export: null handle");
    std::lock_guard<std::mutex> lock(L->mu);
    CUDA_TRY(cudaSetDevice(L->device));
    cudaStream_t st = L->st;
    if (ranges && L->n_ranges) CUDA_TRY(cudaMemcpyAsync(ranges, L->d_ranges, sizeof(sage_b200_lfq_range) * L->n_ranges, cudaMemcpyDeviceToHost, st));
    if (min_rts && L->n_pages) CUDA_TRY(cudaMemcpyAsync(min_rts, L->d_min_rts, 4 * L->n_pages, cudaMemcpyDeviceToHost, st));
    if (grids && L->n_grids) CUDA_TRY(cudaMemcpyAsync(grids, L->d_grids, 8 * L->n_grids * L->n_files * LFQ_ISO * LFQ_GRID, cudaMemcpyDeviceToHost, st));
    if (touched && L->n_grids) CUDA_TRY(cudaMemcpyAsync(touched, L->d_touched, L->n_grids, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

// ================================================================================== rescoring (linear_discriminant.rs, kde.rs, qvalue.rs; kernels in fdr.cuh)
// Which build of glibc's exp / log1p / log10 is the host libm (glibc_math.cuh)? Both variants are compared with the host functions bit for bit on
// a few thousand inputs each, of the kinds rescoring feeds them. 0 = the FMA builds, 1 = the uncontracted ones, -1 = neither matched (the device
// then uses variant 0 and agrees with the host to about 1e-12 relative).
static int host_math_variant() {
    static const int variant = []() {   // initialised once, thread-safe
        uint64_t st = 0x853C49E6748FEA9Bull;
        bool ok[2] = {true, true};
        for (int i = 0; i < 9000; i++) {
            const uint64_t u = xorshift64(st);
            const double unit = (double)(u >> 11) * 0x1p-53;
            const int f = i % 3;
            const double x = f == 0 ? -0.5 * (unit * 40.0) * (unit * 40.0) : f == 1 ? unit * 200.0 - 0.5 : unit * (1.0 + (double)(u & 7));
            volatile double vx = x;
            const double ref = f == 0 ? std::exp(vx) : f == 1 ? std::log1p(vx) : std::log10(vx);
            for (int v = 0; v < 2; v++) {
                const double got = gmath::eval(f, v, x);
                if (memcmp(&got, &ref, 8)) ok[v] = false;
            }
        }
        return ok[0] ? 0 : (ok[1] ? 1 : -1);
    }();
    return variant;
}

// gauss.rs + the matrix.rs subset it uses, on the host (20 x 20). Row-major.
struct HostMat {
    int rows = 0, cols = 0;
    std::vector<double> a;
    HostMat(int r, int c) : rows(r), cols(c), a((size_t)r * c, 0.0) {}
    double& operator()(int i, int j) { return a[(size_t)i * cols + j]; }
    void swap_rows(int i, int j) { for (int k = 0; k < cols; k++) std::swap((*this)(i, k), (*this)(j, k)); }
};
static bool gauss_solve_inner(HostMat left, HostMat right, double eps, std::vector<double>* x) {
    const int m = left.rows, n = left.cols;
    for (int i = 0; i < n; i++) left(i, i) += eps;   // fill_zero
    for (int h = 0, k = 0; h < m && k < n;) {        // echelon
        int imax = 0;
        double vmax = -1.7976931348623157e308;
        for (int i = h; i < m; i++)
            if (left(i, k) >= vmax) { imax = i; vmax = left(i, k); }
        if (left(imax, k) == 0.0) { k++; continue; }
        if (h != imax) { left.swap_rows(h, imax); right.swap_rows(h, imax); }
        for (int i = h + 1; i < m; i++) {
            const double factor = left(i, k) / left(h, k);
            left(i, k) = 0.0;
            for (int j = k + 1; j < n; j++) left(i, j) -= left(h, j) * factor;
            for (int j = 0; j < right.cols; j++) right(i, j) -= right(h, j) * factor;
        }
        h++;
        k++;
    }
    for (int i = left.rows - 1; i >= 0; i--)          // reduce
        for (int j = 0; j < left.cols; j++) {
            const double v = left(i, j);
            if (v == 0.0) continue;
            for (int k = j; k < left.cols; k++) left(i, k) /= v;
            for (int k = 0; k < right.cols; k++) right(i, k) /= v;
            break;
        }
    for (int i = left.rows - 1; i >= 0; i--)          // backfill
        for (int j = 0; j < left.cols; j++) {
            if (left(i, j) == 0.0) continue;
            for (int k = 0; k < i; k++) {
                const double factor = left(k, j) / left(i, j);
                for (int h = 0; h < left.cols; h++) left(k, h) -= left(i, h) * factor;
                for (int h = 0; h < right.cols; h++) right(k, h) -= right(i, h) * factor;
            }
            break;
        }
    for (int i = 0; i < n; i++)                       // left_solved
        for (int j = 0; j < n; j++) {
            const double v = left(i, j);
            if (i == j ? (v != 1.0 && v != 0.0) : v > 1e-8) return false;
        }
    *x = right.a;
    return true;
}
static bool gauss_solve(const HostMat& left, const HostMat& right, std::vector<double>* x, double* eps_used) {
    for (double eps = 1e-8; eps <= 1.0; eps *= 10.0)
        if (gauss_solve_inner(left, right, eps, x)) { *eps_used = eps; return true; }
    return false;
}

// kde::Builder::build (kde.rs:83-136) with bw_adjust = x * bw_factor, on device scores; d_out_bins[bins], d_moments[4] = std_d, std_t, min, max.
static int fdr_kde(cudaStream_t st, DevArena& A, const double* d_scores, const uint8_t* d_decoy, const uint8_t* d_target, uint64_t n, uint32_t bins,
                   bool monotonic, double bw_factor, bool fma, double* d_out_bins, double* d_moments) {
    double *d_sel = nullptr, *part[2] = {nullptr, nullptr};
    uint64_t* d_nsel = nullptr;
    CUDA_TRY(A.alloc(&d_sel, 2 * n));
    CUDA_TRY(A.alloc(&d_nsel, 2));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, d_scores, d_decoy, d_sel, d_nsel, (int64_t)n, st); }));   // decoys in row order
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, d_scores, d_target, d_sel + n, d_nsel + 1, (int64_t)n, st); }));   // targets in row order
    uint64_t m[2];
    if (int rc = read_back(st, m, d_nsel, 16)) return rc;
    LAUNCH(k_fdr_kde_moments<<<1, 256, 0, st>>>(d_sel, m[0], d_sel + n, m[1], d_scores, n, d_moments));
    double mom[2];
    if (int rc = read_back(st, mom, d_moments, 16)) return rc;
    double cst[2];
    uint32_t chunks[2];
    for (int c = 0; c < 2; c++) {   // Kde::new (kde.rs:21-32): the bandwidth and normalising constant, host libm pow / sqrt
        const double bw = (mom[c] * std::pow((4.0 / 3.0) / (double)m[c], 1.0 / 5.0)) * bw_factor;
        cst[c] = std::sqrt(2.0 * M_PI) * bw * (double)m[c];
        chunks[c] = (uint32_t)((m[c] + KDE_CHUNK - 1) / KDE_CHUNK);
        if (chunks[c] > 65535) return fail(SAGE_B200_ELIMIT, "kde: %llu samples exceed the %d-chunk grid", (unsigned long long)m[c], 65535);
        CUDA_TRY(A.alloc(&part[c], (size_t)bins * chunks[c]));
        if (chunks[c]) {
            const dim3 grid((bins + 127) / 128, chunks[c]);
            if (fma) LAUNCH(k_fdr_kde_bins<true><<<grid, 128, 0, st>>>(d_sel + c * n, m[c], bins, chunks[c], d_moments, bw, part[c]));
            else LAUNCH(k_fdr_kde_bins<false><<<grid, 128, 0, st>>>(d_sel + c * n, m[c], bins, chunks[c], d_moments, bw, part[c]));
        }
    }
    const double pi = (double)m[0] / (double)n;
    LAUNCH(k_fdr_kde_pep<<<(bins + 127) / 128, 128, 0, st>>>(part[0], chunks[0], part[1], chunks[1], bins, cst[0], cst[1], pi, monotonic, d_out_bins));
    if (monotonic) LAUNCH(k_fdr_kde_monotone<<<1, 1, 0, st>>>(d_out_bins, bins));
    return 0;
}

extern "C" int sage_b200_kde_build(int device, const double* scores, const uint8_t* decoy, uint64_t n, uint64_t bins, int monotonic, double bw_factor,
                                   double* out_bins, double* min_score, double* score_step) {
    if (n == 0 || !scores || !decoy || !out_bins || !min_score || !score_step || bins < 2) return fail(SAGE_B200_EINVAL, "kde_build: bad argument");
    if (n > (uint64_t)INT32_MAX || bins > (1u << 24)) return fail(SAGE_B200_ELIMIT, "kde_build: n or bins too large");
    if (int rc = select_device(device)) return rc;
    std::vector<uint8_t> flags(2 * n);
    for (uint64_t i = 0; i < n; i++) { flags[i] = decoy[i] != 0; flags[n + i] = decoy[i] == 0; }
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    double *d_s = nullptr, *d_bins = nullptr, *d_mom = nullptr;
    uint8_t* d_flags = nullptr;
    CUDA_TRY(A.upload(&d_s, scores, n, st));
    CUDA_TRY(A.upload(&d_flags, flags.data(), 2 * n, st));
    CUDA_TRY(A.alloc(&d_bins, bins));
    CUDA_TRY(A.alloc(&d_mom, 4));
    const int v = host_math_variant();
    if (int rc = fdr_kde(st, A, d_s, d_flags, d_flags + n, n, (uint32_t)bins, monotonic != 0, bw_factor, v != 1, d_bins, d_mom)) return rc;
    double mom[4];
    CUDA_TRY(cudaMemcpyAsync(out_bins, d_bins, 8 * bins, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(mom, d_mom, 32, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    *min_score = mom[2];
    *score_step = (mom[3] - mom[2]) / (double)(bins - 1);
    return 0;
}

extern "C" int sage_b200_device_math(int device, int function, int variant, const double* x, uint64_t n, double* out) {
    if (function < 0 || function > 2 || variant < -1 || variant > 1 || (n && (!x || !out))) return fail(SAGE_B200_EINVAL, "device_math: bad argument");
    if (n == 0) return 0;
    if (int rc = select_device(device)) return rc;
    if (variant == -1) variant = host_math_variant() == 1 ? 1 : 0;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    double *dx = nullptr, *dy = nullptr;
    CUDA_TRY(A.upload(&dx, x, n, st));
    CUDA_TRY(A.alloc(&dy, n));
    if (variant == 0) LAUNCH_N(k_device_math<true>, n, st, function, dx, n, dy);
    else LAUNCH_N(k_device_math<false>, n, st, function, dx, n, dy);
    return read_back(st, out, dy, 8 * n);
}

struct MinF {
    __device__ float operator()(float a, float b) const { return fminf(a, b); }
};

// qvalue::spectrum_q_value over the rows in ascending (key, row) order: d_key / d_idx hold each row's sort key and index. d_key_sorted,
// d_isdec, d_dscan, d_rq and d_rqmin are n-element work columns (allocated by the caller with its other arrays: an allocation here would
// stall the stage). Returns the row at each sorted position (d_order), each row's q-value (d_q) and the count at q <= 0.01 (d_passing).
template <class Key>
static int spectrum_q_values(cudaStream_t st, DevArena& A, const sage_b200_feature* d_rows, uint64_t n, const Key* d_key, Key* d_key_sorted,
                             const uint32_t* d_idx, uint32_t* d_isdec, uint32_t* d_dscan, float* d_rq, float* d_rqmin, uint32_t* d_order, float* d_q,
                             unsigned long long* d_passing) {
    size_t tb = 0, tb2 = 0, tb3 = 0;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, d_key, d_key_sorted, d_idx, d_order, (int)n, 0, 8 * (int)sizeof(Key), st));
    CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, tb2, d_isdec, d_dscan, (int)n, st));
    CUDA_TRY(cub::DeviceScan::InclusiveScan(nullptr, tb3, d_rq, d_rqmin, MinF(), (int)n, st));
    CUDA_TRY(A.reserve_tmp(std::max(tb, std::max(tb2, tb3))));
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(A.tmp, tb, d_key, d_key_sorted, d_idx, d_order, (int)n, 0, 8 * (int)sizeof(Key), st));
    LAUNCH_N(k_fdr_sorted_decoy, n, st, d_rows, d_order, n, d_isdec);
    CUDA_TRY(cub::DeviceScan::InclusiveSum(A.tmp, tb2, d_isdec, d_dscan, (int)n, st));
    LAUNCH_N(k_fdr_q_raw, n, st, d_dscan, n, d_rq);
    CUDA_TRY(cub::DeviceScan::InclusiveScan(A.tmp, tb3, d_rq, d_rqmin, MinF(), (int)n, st));
    CUDA_TRY(cudaMemsetAsync(d_passing, 0, 8, st));
    LAUNCH_N(k_fdr_q_out, n, st, d_rqmin, d_order, n, d_q, d_passing);
    return 0;
}

// spectrum_fdr (runner.rs:280-291): score_psms, the heuristic fallback when it returns None, the descending sort and spectrum_q_value.
extern "C" int sage_b200_spectrum_fdr(int device, const sage_b200_fdr_params* p, const sage_b200_feature* rows, uint64_t n, const float* aligned_rt,
                                      const float* delta_rt_model, const float* delta_ims_model, sage_b200_fdr_out* out) {
    if (!p || !out || (n && (!rows || !out->discriminant_score || !out->posterior_error || !out->spectrum_q || !out->order)))
        return fail(SAGE_B200_EINVAL, "spectrum_fdr: null argument");
    const int kind = p->precursor_tol.kind;
    if (kind == SAGE_B200_TOL_PCT) return fail(SAGE_B200_EINVAL, "spectrum_fdr: Pct tolerance is never used on precursor m/z (linear_discriminant.rs:142)");
    if (kind != SAGE_B200_TOL_PPM && kind != SAGE_B200_TOL_DA) return fail(SAGE_B200_EINVAL, "spectrum_fdr: unknown tolerance kind %d", kind);
    if (n > (uint64_t)INT32_MAX) return fail(SAGE_B200_ELIMIT, "spectrum_fdr: more than 2^31 - 1 rows (qvalue.rs counts in i32)");
    out->passing = 0;
    out->lda_fitted = 0;
    memset(out->coef, 0, sizeof out->coef);
    out->eps = 0.0;
    out->ms_mass_kde = out->ms_features = out->ms_lda = out->ms_discriminant_kde = out->ms_sort_q = out->ms_total = 0.0f;
    if (n == 0) return 0;
    if (int rc = select_device(device)) return rc;
    if (n > (uint64_t)65535 * KDE_CHUNK) return fail(SAGE_B200_ELIMIT, "spectrum_fdr: more than 65535 KDE chunks of %d rows", KDE_CHUNK);
    const int variant = host_math_variant();
    const bool fma = variant != 1;
    // linear_discriminant.rs:146-150: bandwidth factor and bin count of the mass-error KDE, in the tolerance's f32
    const float lo = p->precursor_tol.lo, hi = p->precursor_tol.hi;
    const float span = std::ceil(std::fmax(hi - lo, kind == SAGE_B200_TOL_PPM ? 100.0f : 1000.0f));
    const double bw_factor = kind == SAGE_B200_TOL_PPM ? 2.0 : 0.1;
    const float span_abs = std::fabs(span);
    if (!(span_abs < 16777216.0f)) return fail(SAGE_B200_ELIMIT, "spectrum_fdr: tolerance span gives too many mass-error bins");
    const uint32_t mbins = (uint32_t)span_abs;
    {   // everything below stays allocated until the call returns: fail with ELIMIT before allocating when it cannot fit
        size_t free_b = 0, total_b = 0;
        CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
        // per row: the rows, mass errors, flags, feature matrix, f64 discriminants, five f32 and six u32 work columns, the three optional
        // columns, the class-compacted samples of both KDEs (16 bytes each) and the radix sort's temporary storage; then both KDEs' partial sums
        const uint64_t per_row = sizeof(sage_b200_feature) + 8 + 2 + 8 * FDR_FEATURES + 8 + 4 * 5 + 4 * 6 + 4 * 3 + 16 * 2 + 16;
        const uint64_t partial = 8ull * ((uint64_t)mbins + 1000) * (n / KDE_CHUNK + 2);
        const uint64_t need = n * per_row + partial + (64ull << 20);
        if (need > free_b) return fail(SAGE_B200_ELIMIT, "spectrum_fdr: %llu rows need about %llu bytes of device memory, %llu free", (unsigned long long)n,
                                       (unsigned long long)need, (unsigned long long)free_b);
    }

    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    Event ev[6];
    for (Event& e : ev) CUDA_TRY(e.create());
    sage_b200_feature* d_rows = nullptr;
    double *d_mass = nullptr, *d_mbins = nullptr, *d_mmom = nullptr, *d_X = nullptr, *d_means = nullptr, *d_scatter = nullptr, *d_coef = nullptr,
           *d_disc = nullptr, *d_dbins = nullptr, *d_dmom = nullptr;
    uint8_t* d_flags = nullptr;
    uint64_t* d_counts = nullptr;
    float *d_disc32 = nullptr, *d_pep = nullptr, *d_q = nullptr, *d_rq = nullptr, *d_rqmin = nullptr, *d_cols[3] = {nullptr, nullptr, nullptr};
    uint32_t *d_key = nullptr, *d_key2 = nullptr, *d_idx = nullptr, *d_order = nullptr, *d_isdec = nullptr, *d_dscan = nullptr;
    unsigned long long* d_passing = nullptr;
    CUDA_TRY(A.upload(&d_rows, rows, n, st));
    CUDA_TRY(A.alloc(&d_mass, n));
    CUDA_TRY(A.alloc(&d_flags, 2 * n));
    CUDA_TRY(A.alloc(&d_mbins, mbins));
    CUDA_TRY(A.alloc(&d_mmom, 4));
    CUDA_TRY(A.alloc(&d_X, n * FDR_FEATURES));
    CUDA_TRY(A.alloc(&d_means, 2 * FDR_FEATURES));
    CUDA_TRY(A.alloc(&d_scatter, 2 * FDR_FEATURES * FDR_FEATURES));
    CUDA_TRY(A.alloc(&d_counts, 2));
    CUDA_TRY(A.alloc(&d_coef, FDR_FEATURES));
    CUDA_TRY(A.alloc(&d_disc, n));
    CUDA_TRY(A.alloc(&d_dbins, 1000));
    CUDA_TRY(A.alloc(&d_dmom, 4));
    CUDA_TRY(A.alloc(&d_disc32, n));
    CUDA_TRY(A.alloc(&d_pep, n));
    CUDA_TRY(A.alloc(&d_q, n));
    CUDA_TRY(A.alloc(&d_rq, n));
    CUDA_TRY(A.alloc(&d_rqmin, n));
    CUDA_TRY(A.alloc(&d_key, n));
    CUDA_TRY(A.alloc(&d_key2, n));
    CUDA_TRY(A.alloc(&d_idx, n));
    CUDA_TRY(A.alloc(&d_order, n));
    CUDA_TRY(A.alloc(&d_isdec, n));
    CUDA_TRY(A.alloc(&d_dscan, n));
    CUDA_TRY(A.alloc(&d_passing, 1));
    const float* cols_h[3] = {aligned_rt, delta_rt_model, delta_ims_model};
    for (int c = 0; c < 3; c++)
        if (cols_h[c]) CUDA_TRY(A.upload(&d_cols[c], cols_h[c], n, st));

    // 1. mass-error KDE (linear_discriminant.rs:140-158)
    CUDA_TRY(cudaEventRecord(ev[0], st));
    LAUNCH_N(k_fdr_mass, n, st, d_rows, n, kind, d_mass, d_flags, d_flags + n);
    if (int rc = fdr_kde(st, A, d_mass, d_flags, d_flags + n, n, mbins, false, bw_factor, fma, d_mbins, d_mmom)) return rc;
    CUDA_TRY(cudaEventRecord(ev[1], st));
    // 2. feature rows (linear_discriminant.rs:162-193)
    const FdrColumns cols{d_cols[0], d_cols[1], d_cols[2]};
    if (fma) LAUNCH_N(k_fdr_features<true>, n, st, d_rows, n, cols, d_mass, d_mbins, mbins, d_mmom, d_X);
    else LAUNCH_N(k_fdr_features<false>, n, st, d_rows, n, cols, d_mass, d_mbins, mbins, d_mmom, d_X);
    CUDA_TRY(cudaEventRecord(ev[2], st));
    // 3. LDA class sums and scatter on the device, Gauss::solve on the host (linear_discriminant.rs:63-124, 195-208)
    LAUNCH(k_fdr_lda<<<2, 256, 0, st>>>(d_X, d_flags, n, d_means, d_scatter, d_counts));
    std::vector<double> means(2 * FDR_FEATURES), scatter(2 * FDR_FEATURES * FDR_FEATURES);
    uint64_t counts[2];
    CUDA_TRY(cudaMemcpyAsync(means.data(), d_means, 8 * means.size(), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(scatter.data(), d_scatter, 8 * scatter.size(), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(counts, d_counts, 16, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    bool fitted = false;
    if (counts[0] != 0 && counts[1] != 0) {
        HostMat sw(FDR_FEATURES, FDR_FEATURES), rhs(FDR_FEATURES, 1);
        for (int c = 0; c < 2; c++)   // scatter_within = (0 + S_decoy / n_decoy) + S_target / n_target
            for (int e = 0; e < FDR_FEATURES * FDR_FEATURES; e++) sw.a[e] += scatter[(size_t)c * FDR_FEATURES * FDR_FEATURES + e] / (double)counts[c];
        for (int j = 0; j < FDR_FEATURES; j++) rhs.a[j] = means[FDR_FEATURES + j] - means[j];
        std::vector<double> coef;
        double eps = 0.0;
        if (gauss_solve(sw, rhs, &coef, &eps)) {
            for (int j = 0; j < FDR_FEATURES; j++) out->coef[j] = coef[j];
            out->eps = eps;
            fitted = true;
            for (double w : coef) fitted = fitted && std::isfinite(w);   // linear_discriminant.rs:196-208
        }
    }
    CUDA_TRY(cudaEventRecord(ev[3], st));
    // 4. projection, discriminant KDE and posterior errors (linear_discriminant.rs:209-228), or the fallback (runner.rs:284-287)
    if (fitted) {
        CUDA_TRY(cudaMemcpyAsync(d_coef, out->coef, 8 * FDR_FEATURES, cudaMemcpyHostToDevice, st));
        LAUNCH_N(k_fdr_project, n, st, d_X, n, d_coef, d_disc, d_disc32);
        if (int rc = fdr_kde(st, A, d_disc, d_flags, d_flags + n, n, 1000, true, 1.0, fma, d_dbins, d_dmom)) return rc;
        if (fma) LAUNCH_N(k_fdr_pep<true>, n, st, d_disc, n, d_dbins, 1000, d_dmom, d_pep);
        else LAUNCH_N(k_fdr_pep<false>, n, st, d_disc, n, d_dbins, 1000, d_dmom, d_pep);
    } else {
        LAUNCH_N(k_fdr_fallback, n, st, d_rows, n, d_disc32, d_pep);
    }
    CUDA_TRY(cudaEventRecord(ev[4], st));
    // 5. stable descending sort (ties by input row) and spectrum_q_value (qvalue.rs)
    LAUNCH_N(k_fdr_sort_key, n, st, d_disc32, n, d_key, d_idx);
    if (int rc = spectrum_q_values(st, A, d_rows, n, d_key, d_key2, d_idx, d_isdec, d_dscan, d_rq, d_rqmin, d_order, d_q, d_passing)) return rc;
    CUDA_TRY(cudaEventRecord(ev[5], st));
    unsigned long long passing = 0;
    CUDA_TRY(cudaMemcpyAsync(out->discriminant_score, d_disc32, 4 * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out->posterior_error, d_pep, 4 * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out->spectrum_q, d_q, 4 * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out->order, d_order, 4 * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&passing, d_passing, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    out->passing = passing;
    out->lda_fitted = fitted ? 1 : 0;
    float* ms[5] = {&out->ms_mass_kde, &out->ms_features, &out->ms_lda, &out->ms_discriminant_kde, &out->ms_sort_q};
    for (int i = 0; i < 5; i++) CUDA_TRY(cudaEventElapsedTime(ms[i], ev[i], ev[i + 1]));
    CUDA_TRY(cudaEventElapsedTime(&out->ms_total, ev[0], ev[5]));
    return 0;
}

// ================================================================================== predict_rt (runner.rs:513-531; kernels in rt.cuh)
// LinearRegression::fit (regression.rs:72-117) for one model over the training list: chunk accumulators on the device, merged in chunk order,
// Gauss::solve on the host, the SSE pass chunked the same way; then predict for every row (or the Feature defaults when the fit is None).
template <int MODEL>
static int rt_model(cudaStream_t st, DevArena& A, bool fma, const RtPeptides& P, const sage_b200_feature* d_rows, uint64_t n, const uint32_t* d_train,
                    uint64_t n_train, const float* d_ycol, const float* d_aligned, float* d_pred, float* d_delta, int32_t* fitted, double* r2, double* eps,
                    double* beta_out) {
    using Dm = RtDims<MODEL>;
    constexpr int D = Dm::D;
    *fitted = 0;
    *r2 = 0.0;
    *eps = 0.0;
    std::fill(beta_out, beta_out + D, 0.0);
    std::vector<double> beta;
    if (n_train) {
        const uint64_t n_chunks = (n_train + RT_CHUNK - 1) / RT_CHUNK;
        double *d_part = nullptr, *d_acc = nullptr, *d_sse = nullptr, *d_beta = nullptr;
        CUDA_TRY(A.alloc(&d_part, n_chunks * Dm::NACC));
        CUDA_TRY(A.alloc(&d_acc, Dm::NACC));
        const dim3 grid((unsigned)n_chunks, grid256(Dm::NACC));
        if (fma) LAUNCH(k_rt_accumulate<MODEL, true><<<grid, 256, 0, st>>>(P, d_rows, d_train, n_train, d_ycol, d_part));
        else LAUNCH(k_rt_accumulate<MODEL, false><<<grid, 256, 0, st>>>(P, d_rows, d_train, n_train, d_ycol, d_part));
        LAUNCH_N(k_rt_merge, Dm::NACC, st, d_part, n_chunks, Dm::NACC, d_acc);
        std::vector<double> acc(Dm::NACC);
        if (int rc = read_back(st, acc.data(), d_acc, 8 * Dm::NACC)) return rc;
        HostMat cov(D, D), b(D, 1);
        for (int j = 0, a = 0; j < D; j++)
            for (int k = j; k < D; k++, a++) cov(j, k) = cov(k, j) = acc[a];
        for (int j = 0; j < D; j++) b.a[j] = acc[Dm::NCOV + j];
        const double sum_y = acc[Dm::NCOV + D], sum_y2 = acc[Dm::NCOV + D + 1];
        const double nf = (double)n_train, y_mean = sum_y / nf, y_var = sum_y2 - nf * y_mean * y_mean;
        if (gauss_solve(cov, b, &beta, eps)) {
            CUDA_TRY(A.upload(&d_beta, beta.data(), D, st));
            CUDA_TRY(A.alloc(&d_sse, n_chunks));
            if (fma) LAUNCH(k_rt_sse<MODEL, true><<<(unsigned)n_chunks, 32, 0, st>>>(P, d_rows, d_train, n_train, d_ycol, d_beta, d_sse));
            else LAUNCH(k_rt_sse<MODEL, false><<<(unsigned)n_chunks, 32, 0, st>>>(P, d_rows, d_train, n_train, d_ycol, d_beta, d_sse));
            std::vector<double> chunk_sse(n_chunks);
            if (int rc = read_back(st, chunk_sse.data(), d_sse, 8 * n_chunks)) return rc;
            double sse = -0.0;   // f64 Sum of the chunk sums, in chunk order
            for (double s : chunk_sse) sse = sse + s;
            *r2 = 1.0 - sse / y_var;
            *fitted = 1;
            std::copy(beta.begin(), beta.end(), beta_out);
            const unsigned g = (unsigned)((n + RT_TILE - 1) / RT_TILE);
            if (fma) LAUNCH(k_rt_predict<MODEL, true><<<g, 32, 0, st>>>(P, d_rows, n, d_beta, d_aligned, d_pred, d_delta));
            else LAUNCH(k_rt_predict<MODEL, false><<<g, 32, 0, st>>>(P, d_rows, n, d_beta, d_aligned, d_pred, d_delta));
            return 0;
        }
        *eps = 0.0;
    }
    LAUNCH_N(k_rt_defaults, n, st, n, d_pred, d_delta);
    return 0;
}

extern "C" int sage_b200_predict_rt(const sage_b200_db* db, const sage_b200_peptides* P, const sage_b200_feature* rows, const uint32_t* file_id, uint64_t n,
                                    uint64_t n_files, sage_b200_rt_out* out) {
    if (!db || !P || !out || (n_files && !out->alignments) ||
        (n && (!rows || !file_id || !out->aligned_rt || !out->predicted_rt || !out->delta_rt_model || !out->predicted_ims || !out->delta_ims_model)))
        return fail(SAGE_B200_EINVAL, "predict_rt: null argument");
    if (P->n_peptides != db->v.n_pep) return fail(SAGE_B200_EINVAL, "predict_rt: the peptide table has %llu peptides, the db %u",
                                                  (unsigned long long)P->n_peptides, db->v.n_pep);
    const uint64_t n_pep = P->n_peptides;
    if (n_pep && (!P->residue_offsets || !P->sequence || !P->monoisotopic)) return fail(SAGE_B200_EINVAL, "predict_rt: null peptide array");
    if (n && n_files == 0) return fail(SAGE_B200_EINVAL, "predict_rt: rows but no files");
    if (n > (uint64_t)INT32_MAX) return fail(SAGE_B200_ELIMIT, "predict_rt: more than 2^31 - 1 rows (qvalue.rs counts in i32)");
    out->training_rows = out->aligned_peptides = 0;
    out->rt_fitted = out->ims_fitted = 0;
    out->rt_r2 = out->rt_eps = out->ims_r2 = out->ims_eps = 0.0;
    memset(out->rt_beta, 0, sizeof out->rt_beta);
    memset(out->ims_beta, 0, sizeof out->ims_beta);
    out->ms_sort_q = out->ms_alignment = out->ms_rt_model = out->ms_ims_model = out->ms_total = 0.0f;
    // argument checks: the reference indexes out of bounds (file_id, peptide_idx) or panics (residue - b'A') on these
    std::vector<uint8_t> referenced(n_pep, 0);
    for (uint64_t i = 0; i < n; i++) {
        if (file_id[i] >= n_files) return fail(SAGE_B200_EINVAL, "predict_rt: row %llu has file_id %u >= n_files %llu", (unsigned long long)i, file_id[i],
                                               (unsigned long long)n_files);
        if (rows[i].peptide_idx >= n_pep) return fail(SAGE_B200_EINVAL, "predict_rt: row %llu has peptide_idx %u outside the db (%llu peptides)",
                                                      (unsigned long long)i, rows[i].peptide_idx, (unsigned long long)n_pep);
        referenced[rows[i].peptide_idx] = 1;
    }
    for (uint64_t p = 0; p < n_pep; p++)
        if (referenced[p])
            for (uint64_t r = P->residue_offsets[p]; r < P->residue_offsets[p + 1]; r++)
                if (P->sequence[r] < 'A' || P->sequence[r] > 'Z')
                    return fail(SAGE_B200_EINVAL, "predict_rt: peptide %llu has residue byte 0x%02x outside 'A'..'Z'", (unsigned long long)p, P->sequence[r]);
    if (n == 0) {
        for (uint64_t f = 0; f < n_files; f++) out->alignments[f] = sage_b200_alignment{0.0f, 1.0f, 0.0f};
        return 0;
    }
    CUDA_TRY(cudaSetDevice(db->device));
    const uint64_t nres = P->residue_offsets[n_pep];
    const uint64_t n_chunks = (n + RT_CHUNK - 1) / RT_CHUNK + 1;
    {   // everything below stays allocated until the call returns: fail with ELIMIT before allocating when it cannot fit
        size_t free_b = 0, total_b = 0;
        CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
        // per row: the rows, file ids, sort keys / values / order, the q-value work columns, flags, training list, (peptide, file) keys and
        // values, segment arrays, the five outputs and the sort's temporary storage; the peptide table; per file the maxima and alignments;
        // both models' chunk partials; and the peptide x file matrix, at most one row per referenced peptide
        const double per_row = sizeof(sage_b200_feature) + 4 + 8 * 2 + 4 * 2 + 4 * 5 + 1 + 4 + 8 * 2 + 4 * 2 + 1 + 4 + 8 + 1 + 4 + 4 + 4 + 4 * 5 + 48;
        uint64_t n_ref = 0;
        for (uint8_t r : referenced) n_ref += r;
        const double need = (double)n * per_row + (double)nres + 8.0 * (double)n_pep + 24.0 * (double)n_files +
                            8.0 * (double)n_chunks * (RtDims<0>::NACC + RtDims<1>::NACC + 2) + 8.0 * (double)n_ref * ((double)n_files + 1) + (double)(64ull << 20);
        if (need > (double)free_b)
            return fail(SAGE_B200_ELIMIT, "predict_rt: %llu rows over %llu files need about %.0f bytes of device memory, %llu free", (unsigned long long)n,
                        (unsigned long long)n_files, need, (unsigned long long)free_b);
    }
    const bool fma = host_math_variant() != 1;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    Event ev[5];
    for (Event& e : ev) CUDA_TRY(e.create());
    sage_b200_feature* d_rows = nullptr;
    uint32_t *d_file = nullptr, *d_off = nullptr, *d_idx = nullptr, *d_order = nullptr, *d_isdec = nullptr, *d_dscan = nullptr, *d_train = nullptr,
             *d_val = nullptr, *d_val2 = nullptr, *d_seg = nullptr, *d_prow = nullptr, *d_keep = nullptr, *d_mrow = nullptr, *d_count = nullptr;
    uint8_t *d_seq = nullptr, *d_flag = nullptr;
    float *d_mono = nullptr, *d_q = nullptr, *d_rq = nullptr, *d_rqmin = nullptr, *d_out[5] = {};
    uint64_t *d_key = nullptr, *d_key2 = nullptr;
    unsigned* d_maxrt = nullptr;
    unsigned long long* d_passing = nullptr;
    double *d_segmin = nullptr, *d_mat = nullptr, *d_mean = nullptr;
    sage_b200_alignment* d_align = nullptr;
    CUDA_TRY(A.upload(&d_rows, rows, n, st));
    CUDA_TRY(A.upload(&d_file, file_id, n, st));
    CUDA_TRY(A.upload(&d_off, P->residue_offsets, n_pep + 1, st));
    CUDA_TRY(A.upload(&d_seq, P->sequence, nres, st));
    CUDA_TRY(A.upload(&d_mono, P->monoisotopic, n_pep, st));
    CUDA_TRY(A.alloc(&d_key, n));
    CUDA_TRY(A.alloc(&d_key2, n));
    CUDA_TRY(A.alloc(&d_idx, n));
    CUDA_TRY(A.alloc(&d_order, n));
    CUDA_TRY(A.alloc(&d_isdec, n));
    CUDA_TRY(A.alloc(&d_dscan, n));
    CUDA_TRY(A.alloc(&d_q, n));
    CUDA_TRY(A.alloc(&d_rq, n));
    CUDA_TRY(A.alloc(&d_rqmin, n));
    CUDA_TRY(A.alloc(&d_flag, n));
    CUDA_TRY(A.alloc(&d_train, n));
    CUDA_TRY(A.alloc(&d_val, n));
    CUDA_TRY(A.alloc(&d_val2, n));
    CUDA_TRY(A.alloc(&d_seg, n));
    CUDA_TRY(A.alloc(&d_segmin, n));
    CUDA_TRY(A.alloc(&d_prow, n));
    CUDA_TRY(A.alloc(&d_keep, n));
    CUDA_TRY(A.alloc(&d_mrow, n));
    CUDA_TRY(A.alloc(&d_count, 4));
    CUDA_TRY(A.alloc(&d_passing, 1));
    CUDA_TRY(A.alloc(&d_maxrt, n_files));
    CUDA_TRY(A.alloc(&d_align, n_files));
    for (auto& o : d_out) CUDA_TRY(A.alloc(&o, n));
    const RtPeptides pk{d_off, d_seq, d_mono};
    thrust::counting_iterator<uint32_t> count_it(0);

    // 1. par_sort_unstable_by(poisson.total_cmp), ties by input row, then spectrum_q_value (runner.rs:517-520)
    CUDA_TRY(cudaEventRecord(ev[0], st));
    LAUNCH_N(k_rt_poisson_key, n, st, d_rows, n, d_key, d_idx);
    if (int rc = spectrum_q_values(st, A, d_rows, n, d_key, d_key2, d_idx, d_isdec, d_dscan, d_rq, d_rqmin, d_order, d_q, d_passing)) return rc;
    // the training rows (label == 1 && spectrum_q <= 0.01) in poisson order
    LAUNCH_N(k_rt_train_flag, n, st, d_rows, d_order, d_q, n, d_flag);
    uint32_t n_train = 0;
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, d_order, d_flag, d_train, d_count, (int)n, st); }));
    if (int rc = read_back(st, &n_train, d_count, 4)) return rc;
    CUDA_TRY(cudaEventRecord(ev[1], st));

    // 2. global_alignment (retention_alignment.rs:95-173)
    CUDA_TRY(cudaMemsetAsync(d_maxrt, 0, 4 * n_files, st));
    LAUNCH_N(k_rt_max_rt, n, st, d_rows, d_file, n, d_maxrt);
    uint32_t n_seg = 0, n_pr = 0;
    uint64_t n_rows = 0;
    if (n_train) {
        LAUNCH_N(k_rt_pf_key, n_train, st, d_rows, d_file, d_train, n_train, d_key);
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) {   // stable: poisson order kept
            return cub::DeviceRadixSort::SortPairs(t, b, d_key, d_key2, d_train, d_val, (int)n_train, 0, 64, st);
        }));
        LAUNCH_N(k_rt_heads, n_train, st, d_key2, n_train, d_flag);
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, count_it, d_flag, d_seg, d_count, (int)n_train, st); }));
        if (int rc = read_back(st, &n_seg, d_count, 4)) return rc;
        LAUNCH_N(k_rt_seg_min, n_seg, st, d_rows, d_key2, d_val, d_seg, n_seg, n_train, d_segmin, d_flag);
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, count_it, d_flag, d_prow, d_count, (int)n_seg, st); }));
        if (int rc = read_back(st, &n_pr, d_count, 4)) return rc;
        LAUNCH_N(k_rt_row_mean, n_pr, st, d_key2, d_seg, d_segmin, d_prow, n_pr, n_seg, d_maxrt, d_keep);
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_keep, d_mrow, (int)n_pr, st); }));
        uint32_t last[2] = {0, 0};
        CUDA_TRY(cudaMemcpyAsync(&last[0], d_mrow + n_pr - 1, 4, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(&last[1], d_keep + n_pr - 1, 4, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        n_rows = (uint64_t)last[0] + last[1];
        CUDA_TRY(A.alloc(&d_mat, n_rows * n_files));
        CUDA_TRY(A.alloc(&d_mean, n_rows));
        CUDA_TRY(cudaMemsetAsync(d_mat, 0xFF, 8 * n_rows * n_files, st));   // NaN where a peptide was not seen in a file
        LAUNCH_N(k_rt_fill, n_pr, st, d_key2, d_seg, d_segmin, d_prow, n_pr, n_seg, d_maxrt, d_keep, d_mrow, n_files, d_mat, d_mean);
    }
    LAUNCH(k_rt_align<<<(unsigned)((n_files + 127) / 128), 128, 0, st>>>(d_mat, d_mean, n_rows, n_files, d_maxrt, d_align));
    float* d_aligned = d_out[0];
    LAUNCH_N(k_rt_aligned, n, st, d_rows, d_file, n, d_align, d_aligned);
    CUDA_TRY(cudaEventRecord(ev[2], st));

    // 3. retention_model::predict, 4. mobility_model::predict
    if (int rc = rt_model<0>(st, A, fma, pk, d_rows, n, d_train, n_train, d_aligned, d_aligned, d_out[1], d_out[2], &out->rt_fitted, &out->rt_r2,
                             &out->rt_eps, out->rt_beta))
        return rc;
    CUDA_TRY(cudaEventRecord(ev[3], st));
    if (int rc = rt_model<1>(st, A, fma, pk, d_rows, n, d_train, n_train, nullptr, d_aligned, d_out[3], d_out[4], &out->ims_fitted, &out->ims_r2,
                             &out->ims_eps, out->ims_beta))
        return rc;
    CUDA_TRY(cudaEventRecord(ev[4], st));

    float* dst[5] = {out->aligned_rt, out->predicted_rt, out->delta_rt_model, out->predicted_ims, out->delta_ims_model};
    for (int c = 0; c < 5; c++) CUDA_TRY(cudaMemcpyAsync(dst[c], d_out[c], 4 * n, cudaMemcpyDeviceToHost, st));
    if (out->spectrum_q) CUDA_TRY(cudaMemcpyAsync(out->spectrum_q, d_q, 4 * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out->alignments, d_align, sizeof(sage_b200_alignment) * n_files, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    out->training_rows = n_train;
    out->aligned_peptides = n_rows;
    float* ms[4] = {&out->ms_sort_q, &out->ms_alignment, &out->ms_rt_model, &out->ms_ims_model};
    for (int i = 0; i < 4; i++) CUDA_TRY(cudaEventElapsedTime(ms[i], ev[i], ev[i + 1]));
    CUDA_TRY(cudaEventElapsedTime(&out->ms_total, ev[0], ev[4]));
    return 0;
}

// ================================================================================== picked FDR (fdr.rs; kernels in picked.cuh)
static constexpr uint32_t PICKED_HOOK_MAX_ROWS = 1u << 16;   // competition_keys with hash_bits < 64

// Checks run before the device is looked at, and the capacity check before anything is allocated. Per competing row: keys, indices, sorted
// copies, ranks, scores, flags, the q-value tail's columns and the sorts' temporary storage; per row of the call also the key material.
static int picked_limits(const char* what, uint64_t n) {
    if (n > (uint64_t)INT32_MAX) return fail(SAGE_B200_ELIMIT, "%s: more than 2^31 - 1 rows", what);
    if (n > (uint64_t)65535 * KDE_CHUNK) return fail(SAGE_B200_ELIMIT, "%s: more than 65535 KDE chunks of %d rows", what, KDE_CHUNK);
    return 0;
}
static int picked_memory(const char* what, uint64_t n, uint64_t extra) {
    size_t free_b = 0, total_b = 0;
    CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
    const uint64_t need = n * 256 + extra + 2 * 8000ull * (n / KDE_CHUNK + 2) + (64ull << 20);
    if (need > free_b) return fail(SAGE_B200_ELIMIT, "%s: %llu rows need about %llu bytes of device memory, %llu free", what, (unsigned long long)n,
                                   (unsigned long long)need, (unsigned long long)free_b);
    return 0;
}

// The q-value tail shared by assign_q_value (fdr.rs:87-119) and picked_precursor (fdr.rs:255-286), over R rows in their pre-sort order:
// the stable descending sort, the PEPs (from the KDE's bins, or 1 / 0 by decoy flag when bins == NULL), the sequential running sum, q, the
// suffix minimum, passing, and the q of each of the n_ix ixs (the latest sorted row that carries it wins).
static int picked_tail(cudaStream_t st, DevArena& A, uint32_t R, const float* q_score, const uint8_t* q_decoy, const uint32_t* q_ix,
                       const uint32_t* q_key, const uint32_t* q_idx, const double* bins, const double* moments, float threshold, uint32_t n_ix,
                       float* q_ix_val, unsigned long long* d_passing) {
    CUDA_TRY(cudaMemsetAsync(d_passing, 0, 8, st));
    if (R == 0) return 0;
    uint32_t *key_s = nullptr, *order = nullptr, *is_t = nullptr, *tinc = nullptr, *win = nullptr;
    float *pep = nullptr, *sum = nullptr, *rq = nullptr, *rqmin = nullptr, *q = nullptr;
    CUDA_TRY(A.alloc(&key_s, R));
    CUDA_TRY(A.alloc(&order, R));
    CUDA_TRY(A.alloc(&is_t, R));
    CUDA_TRY(A.alloc(&tinc, R));
    CUDA_TRY(A.alloc(&win, n_ix));
    CUDA_TRY(A.alloc(&pep, R));
    CUDA_TRY(A.alloc(&sum, R));
    CUDA_TRY(A.alloc(&rq, R));
    CUDA_TRY(A.alloc(&rqmin, R));
    CUDA_TRY(A.alloc(&q, R));
    size_t tb = 0, tb2 = 0, tb3 = 0;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, q_key, key_s, q_idx, order, (int)R, 0, 32, st));
    CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, tb2, is_t, tinc, (int)R, st));
    CUDA_TRY(cub::DeviceScan::InclusiveScan(nullptr, tb3, rq, rqmin, PickedMin(), (int)R, st));
    CUDA_TRY(A.reserve_tmp(std::max(tb, std::max(tb2, tb3))));
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(A.tmp, tb, q_key, key_s, q_idx, order, (int)R, 0, 32, st));   // stable: pre-sort order on ties
    LAUNCH_N(k_picked_pep, R, st, order, q_score, q_decoy, R, bins, moments, pep, is_t);
    LAUNCH(k_picked_running_sum<<<1, 32, 0, st>>>(pep, R, sum));
    CUDA_TRY(cub::DeviceScan::InclusiveSum(A.tmp, tb2, is_t, tinc, (int)R, st));
    LAUNCH_N(k_picked_q_raw, R, st, sum, tinc, R, rq);
    CUDA_TRY(cub::DeviceScan::InclusiveScan(A.tmp, tb3, rq, rqmin, PickedMin(), (int)R, st));
    CUDA_TRY(cudaMemsetAsync(win, 0, 4ull * n_ix, st));
    LAUNCH_N(k_picked_q_min, R, st, rqmin, q_decoy, order, q_ix, R, threshold, q, win, d_passing);
    LAUNCH_N(k_picked_q_ix, R, st, q, order, q_ix, win, R, q_ix_val);
    return 0;
}

// Competition::assign_q_value (fdr.rs:59-120) over m competing rows: d_key groups them into entries (equal key = one entry), d_decoy picks the
// side, d_score is the discriminant. d_pep (peptide level) holds each row's PeptideIx for the same-side check. d_rank[m] receives each row's
// entry rank (first-appearance order); with d_out == NULL the call stops there. Otherwise d_out[m] receives each row's q.
static int picked_competition(cudaStream_t st, DevArena& A, bool fma, uint32_t m, const uint32_t* d_key, const uint8_t* d_decoy, const float* d_score,
                              const uint32_t* d_pep, bool ix_has_side, uint32_t* d_rank, float* d_out, uint64_t* entries, uint64_t* passing) {
    *entries = *passing = 0;
    if (m == 0) return 0;
    thrust::counting_iterator<uint32_t> count_it(0);
    uint32_t *idx = nullptr, *key_s = nullptr, *row_s = nullptr, *head = nullptr, *ginc = nullptr, *first = nullptr, *first_s = nullptr, *gidx = nullptr,
             *g_sorted = nullptr, *rank_of_group = nullptr, *cnt = nullptr;
    CUDA_TRY(A.alloc(&idx, m));
    CUDA_TRY(A.alloc(&key_s, m));
    CUDA_TRY(A.alloc(&row_s, m));
    CUDA_TRY(A.alloc(&head, m));
    CUDA_TRY(A.alloc(&ginc, m));
    CUDA_TRY(A.alloc(&cnt, 4));
    // 1. entries: sort (key, row); a run's head row is the first row that reaches the entry; rank the entries by it
    LAUNCH_N(k_picked_iota, m, st, m, idx);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, d_key, key_s, idx, row_s, (int)m, 0, 32, st); }));
    LAUNCH_N(k_picked_heads, m, st, key_s, m, head);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, head, ginc, (int)m, st); }));
    uint32_t G = 0;
    if (int rc = read_back(st, &G, ginc + m - 1, 4)) return rc;
    CUDA_TRY(A.alloc(&first, G));
    CUDA_TRY(A.alloc(&first_s, G));
    CUDA_TRY(A.alloc(&gidx, G));
    CUDA_TRY(A.alloc(&g_sorted, G));
    CUDA_TRY(A.alloc(&rank_of_group, G));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, row_s, head, first, cnt, (int)m, st); }));
    LAUNCH_N(k_picked_iota, G, st, G, gidx);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, first, first_s, gidx, g_sorted, (int)G, 0, 32, st); }));
    LAUNCH_N(k_picked_scatter_rank, G, st, g_sorted, G, rank_of_group);
    uint32_t *side_key = nullptr, *sk_s = nullptr, *row2_s = nullptr, *seg = nullptr;
    CUDA_TRY(A.alloc(&side_key, m));
    LAUNCH_N(k_picked_row_rank, m, st, row_s, ginc, rank_of_group, d_decoy, m, d_rank, side_key, idx);
    *entries = G;
    if (!d_out) return 0;

    // 2. fold each (entry, side) in row order (fdr.rs:125-144 / 160-177)
    CUDA_TRY(A.alloc(&sk_s, m));
    CUDA_TRY(A.alloc(&row2_s, m));
    CUDA_TRY(A.alloc(&seg, m));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) {   // stable: row order within a side
        return cub::DeviceRadixSort::SortPairs(t, b, side_key, sk_s, idx, row2_s, (int)m, 0, 32, st);
    }));
    LAUNCH_N(k_picked_heads, m, st, sk_s, m, head);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, count_it, head, seg, cnt, (int)m, st); }));
    uint32_t S = 0;
    if (int rc = read_back(st, &S, cnt, 4)) return rc;
    float* side_score = nullptr;
    uint8_t *side_has = nullptr, *kde_flags = nullptr;
    uint32_t *clash = nullptr, *n_rows = nullptr, *row_off = nullptr;
    CUDA_TRY(A.alloc(&side_score, 2ull * G));
    CUDA_TRY(A.zeros(&side_has, 2ull * G, st));
    CUDA_TRY(A.zeros(&clash, 3, st));
    LAUNCH_N(k_picked_fold, S, st, sk_s, row2_s, seg, S, m, d_score, d_pep, side_score, side_has, clash);
    if (d_pep) {
        uint32_t c[3];
        if (int rc = read_back(st, c, clash, 12)) return rc;
        if (c[2]) return fail(SAGE_B200_EINVAL, "picked_fdr: peptides %u and %u are distinct on one side with one key (the reference panics)", c[0], c[1]);
    }

    // 3. the KDE over the entries in rank order (fdr.rs:51-57), the rows (fdr.rs:69-85), the q-value tail
    double *kde_score = nullptr, *bins = nullptr, *moments = nullptr;
    CUDA_TRY(A.alloc(&kde_score, G));
    CUDA_TRY(A.alloc(&kde_flags, 2ull * G));
    CUDA_TRY(A.alloc(&n_rows, G));
    CUDA_TRY(A.alloc(&row_off, G));
    CUDA_TRY(A.alloc(&bins, 1000));
    CUDA_TRY(A.alloc(&moments, 4));
    LAUNCH_N(k_picked_entries, G, st, side_score, side_has, G, kde_score, kde_flags, n_rows);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, n_rows, row_off, (int)G, st); }));
    if (int rc = fdr_kde(st, A, kde_score, kde_flags, kde_flags + G, G, 1000, true, 1.0, fma, bins, moments)) return rc;
    float *q_score = nullptr, *q_ix_val = nullptr;
    uint8_t* q_decoy = nullptr;
    uint32_t *q_ix = nullptr, *q_key = nullptr, *q_idx = nullptr;
    unsigned long long* d_passing = nullptr;
    CUDA_TRY(A.alloc(&q_score, S));
    CUDA_TRY(A.alloc(&q_decoy, S));
    CUDA_TRY(A.alloc(&q_ix, S));
    CUDA_TRY(A.alloc(&q_key, S));
    CUDA_TRY(A.alloc(&q_idx, S));
    CUDA_TRY(A.alloc(&q_ix_val, 2ull * G));
    CUDA_TRY(A.alloc(&d_passing, 1));
    LAUNCH_N(k_picked_rows, G, st, side_score, side_has, row_off, G, ix_has_side, q_score, q_decoy, q_ix, q_key, q_idx);
    if (int rc = picked_tail(st, A, S, q_score, q_decoy, q_ix, q_key, q_idx, bins, moments, 0.01f, 2 * G, q_ix_val, d_passing)) return rc;
    LAUNCH_N(k_picked_gather, m, st, d_rank, d_decoy, m, ix_has_side, q_ix_val, d_out);
    unsigned long long pass = 0;
    if (int rc = read_back(st, &pass, d_passing, 8)) return rc;
    *passing = pass;
    return 0;
}

static int picked_check_peptides(const char* what, const sage_b200_peptides* P, const sage_b200_picked_params* p, bool proteins) {
    if (!P || !p || (proteins && (!p->n_proteins || !p->protein))) return fail(SAGE_B200_EINVAL, "%s: null argument", what);
    if (P->n_peptides && (!P->residue_offsets || !P->sequence || !P->modifications || !P->nterm || !P->decoy))
        return fail(SAGE_B200_EINVAL, "%s: null peptide array", what);
    if (P->n_peptides >= 0xFFFFFFFFull) return fail(SAGE_B200_ELIMIT, "%s: too many peptides for u32 PeptideIx", what);
    return 0;
}

// The peptide keys of the rows (fdr.rs:126-131): the referenced peptides' key material goes to the device compacted, each is hashed and
// grouped exactly; d_key[i] = the group of row i's peptide. Also each row's decoy flag and PeptideIx.
static int picked_peptide_keys(cudaStream_t st, DevArena& A, const sage_b200_peptides* P, const sage_b200_picked_params* p, const uint32_t* pep_idx,
                               uint32_t n, uint32_t hash_bits, uint32_t* d_key, uint8_t* d_decoy, uint32_t* d_pep) {
    const uint64_t n_pep = P->n_peptides;
    std::vector<uint32_t> slot_of(n_pep, ~0u), row_slot(n), off(1, 0);
    std::vector<uint8_t> row_decoy(n), seq, rev;
    std::vector<float> mods, nterm, cterm;
    for (uint32_t i = 0; i < n; i++) slot_of[pep_idx[i]] = 0;
    for (uint64_t q = 0; q < n_pep; q++) {
        if (slot_of[q]) continue;
        slot_of[q] = (uint32_t)nterm.size();
        const uint32_t a = P->residue_offsets[q], b = P->residue_offsets[q + 1];
        seq.insert(seq.end(), P->sequence + a, P->sequence + b);
        mods.insert(mods.end(), P->modifications + a, P->modifications + b);
        off.push_back((uint32_t)seq.size());
        nterm.push_back(P->nterm[q]);
        cterm.push_back(p->cterm ? p->cterm[q] : std::numeric_limits<float>::quiet_NaN());
        rev.push_back(p->generate_decoys && P->decoy[q] ? 1 : 0);
    }
    for (uint32_t i = 0; i < n; i++) {
        row_slot[i] = slot_of[pep_idx[i]];
        row_decoy[i] = P->decoy[pep_idx[i]] ? 1 : 0;
    }
    const uint32_t U = (uint32_t)nterm.size();
    uint32_t *d_off = nullptr, *d_row_slot = nullptr, *d_u = nullptr, *d_u_s = nullptr, *d_group = nullptr;
    uint8_t *d_seq = nullptr, *d_rev = nullptr;
    float *d_mods = nullptr, *d_nterm = nullptr, *d_cterm = nullptr;
    uint64_t *d_hash = nullptr, *d_hash_s = nullptr;
    CUDA_TRY(A.upload(&d_off, off.data(), U + 1, st));
    CUDA_TRY(A.upload(&d_seq, seq.data(), seq.size(), st));
    CUDA_TRY(A.upload(&d_mods, mods.data(), mods.size(), st));
    CUDA_TRY(A.upload(&d_nterm, nterm.data(), U, st));
    CUDA_TRY(A.upload(&d_cterm, cterm.data(), U, st));
    CUDA_TRY(A.upload(&d_rev, rev.data(), U, st));
    CUDA_TRY(A.upload(&d_row_slot, row_slot.data(), n, st));
    CUDA_TRY(A.alloc(&d_u, U));
    CUDA_TRY(A.alloc(&d_u_s, U));
    CUDA_TRY(A.alloc(&d_group, U));
    CUDA_TRY(A.alloc(&d_hash, U));
    CUDA_TRY(A.alloc(&d_hash_s, U));
    CUDA_TRY(cudaMemcpyAsync(d_decoy, row_decoy.data(), n, cudaMemcpyHostToDevice, st));
    if (d_pep) CUDA_TRY(cudaMemcpyAsync(d_pep, pep_idx, 4ull * n, cudaMemcpyHostToDevice, st));
    const PickedPeptides pk{d_off, d_seq, d_mods, d_nterm, d_cterm, d_rev};
    const uint64_t mask = hash_bits >= 64 ? ~0ull : ((1ull << hash_bits) - 1);
    LAUNCH_N(k_picked_hash, U, st, pk, U, mask, d_hash, d_u);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, d_hash, d_hash_s, d_u, d_u_s, (int)U, 0, 64, st); }));
    LAUNCH_N(k_picked_group, U, st, pk, d_hash_s, d_u_s, U, d_group);
    LAUNCH_N(k_picked_peptide_keys, n, st, d_row_slot, d_group, n, d_key);
    return 0;
}

extern "C" int sage_b200_picked_fdr(int device, const sage_b200_peptides* P, const sage_b200_picked_params* p, const sage_b200_feature* rows,
                                    const float* discriminant_score, uint64_t n, sage_b200_picked_out* out) {
    if (!out || (n && (!rows || !discriminant_score || !out->peptide_q || !out->protein_q))) return fail(SAGE_B200_EINVAL, "picked_fdr: null argument");
    if (int rc = picked_check_peptides("picked_fdr", P, p, true)) return rc;
    if (int rc = picked_limits("picked_fdr", n)) return rc;
    out->peptide_passing = out->protein_passing = out->peptide_entries = out->protein_entries = 0;
    out->ms_keys = out->ms_peptide = out->ms_protein = out->ms_total = 0.0f;
    std::vector<uint32_t> pep_idx(n);
    for (uint64_t i = 0; i < n; i++) {
        pep_idx[i] = rows[i].peptide_idx;
        if (pep_idx[i] >= P->n_peptides)
            return fail(SAGE_B200_EINVAL, "picked_fdr: row %llu has peptide_idx %u outside the peptide table (%llu peptides)", (unsigned long long)i,
                        pep_idx[i], (unsigned long long)P->n_peptides);
    }
    if (n == 0) return 0;
    if (int rc = select_device(device)) return rc;
    const uint64_t nres = P->residue_offsets[P->n_peptides];
    if (int rc = picked_memory("picked_fdr", 2 * n, 16 * nres + 32 * P->n_peptides)) return rc;
    // picked_protein's rows: those whose peptide has exactly one protein (fdr.rs:160-162), keyed by that protein's id
    std::vector<uint32_t> prot_row, prot_key;
    std::vector<uint8_t> prot_decoy;
    std::vector<float> prot_score;
    for (uint64_t i = 0; i < n; i++) {
        const uint32_t q = pep_idx[i];
        if (p->n_proteins[q] != 1) continue;
        prot_row.push_back((uint32_t)i);
        prot_key.push_back(p->protein[q]);
        prot_decoy.push_back(P->decoy[q] ? 1 : 0);
        prot_score.push_back(discriminant_score[i]);
    }
    const uint32_t m = (uint32_t)prot_row.size();
    const bool fma = host_math_variant() != 1;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    Event ev[4];
    for (Event& e : ev) CUDA_TRY(e.create());
    uint32_t *d_key = nullptr, *d_pep = nullptr, *d_rank = nullptr, *d_pkey = nullptr, *d_prank = nullptr;
    uint8_t *d_decoy = nullptr, *d_pdecoy = nullptr;
    float *d_score = nullptr, *d_q = nullptr, *d_pscore = nullptr, *d_pq = nullptr;
    CUDA_TRY(A.alloc(&d_key, n));
    CUDA_TRY(A.alloc(&d_pep, n));
    CUDA_TRY(A.alloc(&d_rank, n));
    CUDA_TRY(A.alloc(&d_decoy, n));
    CUDA_TRY(A.upload(&d_score, discriminant_score, n, st));
    CUDA_TRY(A.alloc(&d_q, n));
    CUDA_TRY(A.upload(&d_pkey, prot_key.data(), m, st));
    CUDA_TRY(A.alloc(&d_prank, m));
    CUDA_TRY(A.upload(&d_pdecoy, prot_decoy.data(), m, st));
    CUDA_TRY(A.upload(&d_pscore, prot_score.data(), m, st));
    CUDA_TRY(A.alloc(&d_pq, m));
    CUDA_TRY(cudaEventRecord(ev[0], st));
    if (int rc = picked_peptide_keys(st, A, P, p, pep_idx.data(), (uint32_t)n, 64, d_key, d_decoy, d_pep)) return rc;
    CUDA_TRY(cudaEventRecord(ev[1], st));
    if (int rc = picked_competition(st, A, fma, (uint32_t)n, d_key, d_decoy, d_score, d_pep, true, d_rank, d_q, &out->peptide_entries, &out->peptide_passing))
        return rc;
    CUDA_TRY(cudaEventRecord(ev[2], st));
    // Ix of picked_protein is proteins(decoy_tag, generate_decoys): the tagged name per side with generate_decoys, else the name alone
    if (int rc = picked_competition(st, A, fma, m, d_pkey, d_pdecoy, d_pscore, nullptr, p->generate_decoys != 0, d_prank, d_pq, &out->protein_entries,
                                    &out->protein_passing))
        return rc;
    CUDA_TRY(cudaEventRecord(ev[3], st));
    std::vector<float> pq(m);
    CUDA_TRY(cudaMemcpyAsync(out->peptide_q, d_q, 4 * n, cudaMemcpyDeviceToHost, st));
    if (m) CUDA_TRY(cudaMemcpyAsync(pq.data(), d_pq, 4ull * m, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    for (uint64_t i = 0; i < n; i++) out->protein_q[i] = 1.0f;
    for (uint32_t c = 0; c < m; c++) out->protein_q[prot_row[c]] = pq[c];
    CUDA_TRY(cudaEventElapsedTime(&out->ms_keys, ev[0], ev[1]));
    CUDA_TRY(cudaEventElapsedTime(&out->ms_peptide, ev[1], ev[2]));
    CUDA_TRY(cudaEventElapsedTime(&out->ms_protein, ev[2], ev[3]));
    CUDA_TRY(cudaEventElapsedTime(&out->ms_total, ev[0], ev[3]));
    return 0;
}

extern "C" int sage_b200_picked_precursor(int device, const double* score, const uint8_t* decoy, uint64_t n, float* q_value, uint64_t* passing) {
    if (!passing || (n && (!score || !decoy || !q_value))) return fail(SAGE_B200_EINVAL, "picked_precursor: null argument");
    if (n > (uint64_t)INT32_MAX) return fail(SAGE_B200_ELIMIT, "picked_precursor: more than 2^31 - 1 rows");
    *passing = 0;
    if (n == 0) return 0;
    if (int rc = select_device(device)) return rc;
    if (int rc = picked_memory("picked_precursor", n, 0)) return rc;
    std::vector<uint8_t> flags(n);
    for (uint64_t i = 0; i < n; i++) flags[i] = decoy[i] ? 1 : 0;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    const uint32_t R = (uint32_t)n;
    double* d_in = nullptr;
    float *d_score = nullptr, *d_q = nullptr;
    uint8_t* d_decoy = nullptr;
    uint32_t *d_ix = nullptr, *d_key = nullptr, *d_idx = nullptr;
    unsigned long long* d_passing = nullptr;
    CUDA_TRY(A.upload(&d_in, score, n, st));
    CUDA_TRY(A.alloc(&d_score, n));
    CUDA_TRY(A.alloc(&d_q, n));
    CUDA_TRY(A.upload(&d_decoy, flags.data(), n, st));
    CUDA_TRY(A.alloc(&d_ix, n));
    CUDA_TRY(A.alloc(&d_key, n));
    CUDA_TRY(A.alloc(&d_idx, n));
    CUDA_TRY(A.alloc(&d_passing, 1));
    LAUNCH_N(k_picked_precursor_rows, n, st, d_in, R, d_score, d_ix, d_key, d_idx);
    if (int rc = picked_tail(st, A, R, d_score, d_decoy, d_ix, d_key, d_idx, nullptr, nullptr, 0.05f, R, d_q, d_passing)) return rc;
    unsigned long long pass = 0;
    CUDA_TRY(cudaMemcpyAsync(q_value, d_q, 4 * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&pass, d_passing, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    *passing = pass;
    return 0;
}

extern "C" int sage_b200_competition_keys(int device, const sage_b200_peptides* P, const sage_b200_picked_params* p, const uint32_t* peptide_idx, uint64_t n,
                                          uint32_t hash_bits, uint32_t* entry_rank) {
    if (n && (!peptide_idx || !entry_rank)) return fail(SAGE_B200_EINVAL, "competition_keys: null argument");
    if (hash_bits < 3 || hash_bits > 64) return fail(SAGE_B200_EINVAL, "competition_keys: hash_bits %u outside 3..64", hash_bits);
    // a truncated hash makes equal-hash runs of about n / 2^hash_bits peptides, compared pairwise: bound that work
    if (hash_bits < 64 && n > PICKED_HOOK_MAX_ROWS)
        return fail(SAGE_B200_ELIMIT, "competition_keys: more than %u rows with a truncated hash", PICKED_HOOK_MAX_ROWS);
    if (int rc = picked_check_peptides("competition_keys", P, p, false)) return rc;
    if (int rc = picked_limits("competition_keys", n)) return rc;
    for (uint64_t i = 0; i < n; i++)
        if (peptide_idx[i] >= P->n_peptides)
            return fail(SAGE_B200_EINVAL, "competition_keys: row %llu has peptide_idx %u outside the peptide table (%llu peptides)", (unsigned long long)i,
                        peptide_idx[i], (unsigned long long)P->n_peptides);
    if (n == 0) return 0;
    if (int rc = select_device(device)) return rc;
    const uint64_t nres = P->residue_offsets[P->n_peptides];
    if (int rc = picked_memory("competition_keys", n, 16 * nres + 32 * P->n_peptides)) return rc;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    uint32_t *d_key = nullptr, *d_rank = nullptr;
    uint8_t* d_decoy = nullptr;
    CUDA_TRY(A.alloc(&d_key, n));
    CUDA_TRY(A.alloc(&d_rank, n));
    CUDA_TRY(A.alloc(&d_decoy, n));
    if (int rc = picked_peptide_keys(st, A, P, p, peptide_idx, (uint32_t)n, hash_bits, d_key, d_decoy, nullptr)) return rc;
    uint64_t entries = 0, passing = 0;
    if (int rc = picked_competition(st, A, true, (uint32_t)n, d_key, d_decoy, nullptr, nullptr, true, d_rank, nullptr, &entries, &passing)) return rc;
    return read_back(st, entry_rank, d_rank, 4 * n);
}

// ================================================================================== protein grouping (protein_grouping.rs; kernels in protein_groups.cuh)
// out[0..n] = exclusive prefix sum of in[0..n) (in[n] must be 0); returns out[n] in *total.
static int pg_offsets(cudaStream_t st, DevArena& A, const uint32_t* in, uint32_t* out, uint32_t n, uint32_t* total) {
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, in, out, (int)n + 1, st); }));
    return read_back(st, total, out + n, 4);
}

struct PgCoverStats {
    uint64_t forced = 0, greedy = 0, components = 0, largest = 0, covered = 0;
};

// BipartiteGraph::into_cover (protein_grouping.rs) over E edges (el[k], er[k]) between G left and M right nodes; lcov[G] receives the cover.
// Phase 1 is the first trim's forced picks; phase 2 the greedy of each connected component of what remains (DESIGN.md §13).
static int pg_cover(cudaStream_t st, DevArena& A, uint32_t E, uint32_t G, uint32_t M, const uint32_t* el, const uint32_t* er, uint8_t* lcov,
                    PgCoverStats* s) {
    *s = {};
    if (G) CUDA_TRY(cudaMemsetAsync(lcov, 0, G, st));
    if (E == 0) return 0;
    uint32_t *ldeg, *rdeg, *loff, *roff, *key_s, *ladj, *radj, *rcov, *rem, *parent, tot = 0;
    uint8_t* active;
    unsigned long long* cnt;
    CUDA_TRY(A.zeros(&ldeg, G + 1, st));
    CUDA_TRY(A.zeros(&rdeg, M + 1, st));
    CUDA_TRY(A.alloc(&loff, G + 1));
    CUDA_TRY(A.alloc(&roff, M + 1));
    CUDA_TRY(A.alloc(&key_s, E));
    CUDA_TRY(A.alloc(&ladj, E));
    CUDA_TRY(A.alloc(&radj, E));
    CUDA_TRY(A.zeros(&rcov, M, st));
    CUDA_TRY(A.alloc(&rem, G));
    CUDA_TRY(A.alloc(&parent, G + M));
    CUDA_TRY(A.alloc(&active, G));
    CUDA_TRY(A.zeros(&cnt, 3, st));   // forced, greedy picks, covered
    LAUNCH_N(k_pg_degrees, E, st, el, er, E, ldeg, rdeg);
    if (int rc = pg_offsets(st, A, ldeg, loff, G, &tot)) return rc;
    if (int rc = pg_offsets(st, A, rdeg, roff, M, &tot)) return rc;
    // adjacency of each left node (by a sort on the left end) and of each right node
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, el, key_s, er, ladj, (int)E, 0, 32, st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, er, key_s, el, radj, (int)E, 0, 32, st); }));
    LAUNCH_N(k_pg_forced, E, st, el, er, rdeg, E, lcov);
    LAUNCH_N(k_pg_count, G, st, lcov, G, cnt);
    LAUNCH_N(k_pg_cover_rights, E, st, el, er, lcov, E, rcov);
    LAUNCH_N(k_pg_remaining, G, st, ladj, loff, lcov, rcov, G, rem, active);
    LAUNCH_N(k_picked_iota, G + M, st, G + M, parent);
    LAUNCH_N(k_pg_union, E, st, el, er, lcov, rcov, E, G, parent);
    // the groups left with edges, by component (ascending group index within one)
    thrust::counting_iterator<uint32_t> it(0);
    uint32_t *act, *comp, *lefts, *uniq, *clen, *coff, *large, *nsel, n_act = 0, n_comp = 0, n_large = 0;
    uint8_t* lflag;
    CUDA_TRY(A.alloc(&act, G));
    CUDA_TRY(A.alloc(&nsel, 1));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, it, active, act, nsel, (int)G, st); }));
    if (int rc = read_back(st, &n_act, nsel, 4)) return rc;
    if (n_act) {
        CUDA_TRY(A.alloc(&comp, n_act));
        CUDA_TRY(A.alloc(&lefts, n_act));
        CUDA_TRY(A.alloc(&uniq, n_act));
        CUDA_TRY(A.alloc(&clen, n_act + 1));
        CUDA_TRY(A.alloc(&coff, n_act + 1));
        LAUNCH_N(k_pg_comp_of, n_act, st, parent, act, n_act, comp);
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, comp, key_s, act, lefts, (int)n_act, 0, 32, st); }));
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRunLengthEncode::Encode(t, b, key_s, uniq, clen, nsel, (int)n_act, st); }));
        if (int rc = read_back(st, &n_comp, nsel, 4)) return rc;
        CUDA_TRY(cudaMemsetAsync(clen + n_comp, 0, 4, st));
        if (int rc = pg_offsets(st, A, clen, coff, n_comp, &tot)) return rc;
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceReduce::Max(t, b, clen, uniq, (int)n_comp, st); }));
        uint32_t largest = 0;
        if (int rc = read_back(st, &largest, uniq, 4)) return rc;
        CUDA_TRY(A.alloc(&lflag, n_comp));
        CUDA_TRY(A.alloc(&large, n_comp));
        LAUNCH_N(k_pg_large_flag, n_comp, st, clen, n_comp, lflag);
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, it, lflag, large, nsel, (int)n_comp, st); }));
        if (int rc = read_back(st, &n_large, nsel, 4)) return rc;
        LAUNCH_N(k_pg_greedy_warp, 32ull * n_comp, st, coff, clen, n_comp, lefts, ldeg, ladj, loff, radj, roff, rem, rcov, lcov, cnt + 1);
        if (n_large) LAUNCH(k_pg_greedy_cta<<<n_large, PG_CTA, 0, st>>>(large, coff, clen, lefts, ldeg, ladj, loff, radj, roff, rem, rcov, lcov, cnt + 1));
        s->components = n_comp;
        s->largest = largest;
    }
    LAUNCH_N(k_pg_count, G, st, lcov, G, cnt + 2);
    unsigned long long c[3];
    if (int rc = read_back(st, c, cnt, 24)) return rc;
    s->forced = c[0];
    s->greedy = c[1];
    s->covered = c[2];
    return 0;
}

// The inputs of the call on the device.
struct PgInputs {
    uint32_t n, n_pep, n_names;
    const uint32_t *pep, *poff, *pids;
    const uint8_t *label_ok, *pdecoy;
    const float* q;
    const uint64_t* cap_off;
};

// One pass's group table on the device: group g has members[goff[g] .. goff[g+1]) (name ids, ascending), gdecoy[g], lcov[g].
struct PgTable {
    uint32_t G = 0, P = 0;
    uint32_t *goff = nullptr, *members = nullptr;
    uint8_t *gdecoy = nullptr, *lcov = nullptr;
};

// annotate_features (protein_grouping.rs) at one threshold: ProteinGrouper::build, into_group_map's cover, and the lookup of every row still
// unannotated (pass[i] == 0), whose distinct covered groups (numbered from `base`) go to the row's slot of `scratch`.
static int pg_pass(cudaStream_t st, DevArena& A, const PgInputs& in, float threshold, uint8_t pass_no, uint32_t base, uint8_t* pass, uint32_t* count,
                   uint32_t* scratch, PgTable* T, sage_b200_protein_group_out* out, cudaEvent_t ev_built, cudaEvent_t ev_covered) {
    const int k = pass_no - 1;
    const uint32_t NK = 2 * in.n_names;
    thrust::counting_iterator<uint32_t> it(0);
    uint32_t *nsel, U = 0;
    uint8_t* mark;
    CUDA_TRY(A.alloc(&nsel, 1));
    // 1. the peptide set, ascending PeptideIx
    CUDA_TRY(A.zeros(&mark, in.n_pep, st));
    LAUNCH_N(k_pg_mark, in.n, st, in.pep, in.label_ok, in.q, in.n, threshold, mark);
    uint32_t* set;
    CUDA_TRY(A.alloc(&set, in.n_pep));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, it, mark, set, nsel, (int)in.n_pep, st); }));
    if (int rc = read_back(st, &U, nsel, 4)) return rc;
    out->peptides[k] = U;
    uint32_t M = 0, P = 0, G = 0, E = 0, T_pairs = 0, tot = 0;
    uint32_t *pix_of_key = nullptr, *group_of = nullptr, *el = nullptr, *er = nullptr;
    CUDA_TRY(A.alloc(&pix_of_key, NK));
    CUDA_TRY(cudaMemsetAsync(pix_of_key, 0xFF, 4ull * NK, st));
    if (U) {
        // 2. the (peptide, protein) pairs; ProteinIx by first encounter
        uint32_t *len, *soff, *pair_key, *first, *present, *first_p, *first_s, *key_by_pix;
        uint8_t* flag;
        CUDA_TRY(A.alloc(&len, U + 1));
        CUDA_TRY(A.alloc(&soff, U + 1));
        CUDA_TRY(cudaMemsetAsync(len + U, 0, 4, st));
        LAUNCH_N(k_pg_set_len, U, st, set, in.poff, U, len);
        if (int rc = pg_offsets(st, A, len, soff, U, &T_pairs)) return rc;
        CUDA_TRY(A.alloc(&pair_key, T_pairs));
        CUDA_TRY(A.alloc(&first, NK));
        CUDA_TRY(A.alloc(&flag, NK));
        CUDA_TRY(cudaMemsetAsync(first, 0xFF, 4ull * NK, st));
        LAUNCH_N(k_pg_flatten, U, st, set, soff, in.poff, in.pids, in.pdecoy, U, pair_key, first);
        LAUNCH_N(k_pg_key_present, NK, st, first, NK, flag);
        CUDA_TRY(A.alloc(&present, NK));
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, it, flag, present, nsel, (int)NK, st); }));
        if (int rc = read_back(st, &P, nsel, 4)) return rc;
        CUDA_TRY(A.alloc(&first_p, P));
        CUDA_TRY(A.alloc(&first_s, P));
        CUDA_TRY(A.alloc(&key_by_pix, P));
        LAUNCH_N(k_pg_gather_u32, P, st, first, present, P, first_p);
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, first_p, first_s, present, key_by_pix, (int)P, 0, 32, st); }));
        LAUNCH_N(k_pg_scatter_rank, P, st, key_by_pix, P, pix_of_key);
        // 3. each peptide's sorted ProteinIx list; meta-peptides = the distinct lists, ranked lexicographically
        uint32_t *pix, *pix_s, *idx, *head, *incl, *mrep;
        CUDA_TRY(A.alloc(&pix, T_pairs));
        CUDA_TRY(A.alloc(&pix_s, T_pairs));
        CUDA_TRY(A.alloc(&idx, U));
        CUDA_TRY(A.alloc(&head, U));
        CUDA_TRY(A.alloc(&incl, U));
        CUDA_TRY(A.alloc(&mrep, U));
        LAUNCH_N(k_pg_pair_pix, T_pairs, st, pair_key, pix_of_key, T_pairs, pix);
        if (T_pairs)
            CUDA_TRY(A.two_phase([&](void* t, size_t& b) {
                return cub::DeviceSegmentedSort::SortKeys(t, b, pix, pix_s, (int)T_pairs, (int)U, soff, soff + 1, st);
            }));
        LAUNCH_N(k_picked_iota, U, st, U, idx);
        const PgLexLess meta_less{pix_s, soff};
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceMergeSort::StableSortKeys(t, b, idx, (int)U, meta_less, st); }));
        LAUNCH_N(k_pg_lex_heads, U, st, idx, pix_s, soff, U, head);
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, head, incl, (int)U, st); }));
        if (int rc = read_back(st, &M, incl + U - 1, 4)) return rc;
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, idx, head, mrep, nsel, (int)U, st); }));
        if (P) {
            // 4. each protein's evidence: the meta-peptides that hold it, ascending, with multiplicity
            uint32_t *mlen, *moff, *pdeg, *ev, *ev_off, TM = 0;
            uint64_t *pairs, *pairs_s;
            CUDA_TRY(A.alloc(&mlen, M + 1));
            CUDA_TRY(A.alloc(&moff, M + 1));
            CUDA_TRY(cudaMemsetAsync(mlen + M, 0, 4, st));
            LAUNCH_N(k_pg_csr_len, M, st, mrep, soff, M, mlen);
            if (int rc = pg_offsets(st, A, mlen, moff, M, &TM)) return rc;
            CUDA_TRY(A.zeros(&pdeg, P + 1, st));
            CUDA_TRY(A.alloc(&ev_off, P + 1));
            CUDA_TRY(A.alloc(&pairs, TM));
            CUDA_TRY(A.alloc(&pairs_s, TM));
            CUDA_TRY(A.alloc(&ev, TM));
            LAUNCH_N(k_pg_meta_pairs, M, st, mrep, pix_s, soff, moff, M, pairs, pdeg);
            CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortKeys(t, b, pairs, pairs_s, (int)TM, 0, 64, st); }));
            LAUNCH_N(k_pg_low32, TM, st, pairs_s, TM, ev);
            if (int rc = pg_offsets(st, A, pdeg, ev_off, P, &tot)) return rc;
            // 5. groups: proteins of equal evidence, ranked by it; members in ascending id; edges (group, each evidence entry)
            uint32_t *pidx, *phead, *pincl, *grep, *gsize, *elen, *eoff;
            uint64_t *mem, *mem_s;
            CUDA_TRY(A.alloc(&pidx, P));
            CUDA_TRY(A.alloc(&phead, P));
            CUDA_TRY(A.alloc(&pincl, P));
            CUDA_TRY(A.alloc(&grep, P));
            CUDA_TRY(A.alloc(&group_of, P));
            LAUNCH_N(k_picked_iota, P, st, P, pidx);
            const PgLexLess group_less{ev, ev_off};
            CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceMergeSort::StableSortKeys(t, b, pidx, (int)P, group_less, st); }));
            LAUNCH_N(k_pg_lex_heads, P, st, pidx, ev, ev_off, P, phead);
            CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, phead, pincl, (int)P, st); }));
            if (int rc = read_back(st, &G, pincl + P - 1, 4)) return rc;
            LAUNCH_N(k_pg_rank_of, P, st, pidx, pincl, P, group_of);
            CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, pidx, phead, grep, nsel, (int)P, st); }));
            CUDA_TRY(A.zeros(&gsize, G + 1, st));
            CUDA_TRY(A.alloc(&T->goff, G + 1));
            CUDA_TRY(A.alloc(&T->members, P));
            CUDA_TRY(A.alloc(&T->gdecoy, G));
            CUDA_TRY(A.alloc(&mem, P));
            CUDA_TRY(A.alloc(&mem_s, P));
            LAUNCH_N(k_pg_members, P, st, group_of, key_by_pix, P, mem, gsize, T->gdecoy);
            CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortKeys(t, b, mem, mem_s, (int)P, 0, 64, st); }));
            LAUNCH_N(k_pg_low32, P, st, mem_s, P, T->members);
            if (int rc = pg_offsets(st, A, gsize, T->goff, G, &tot)) return rc;
            CUDA_TRY(A.alloc(&elen, G + 1));
            CUDA_TRY(A.alloc(&eoff, G + 1));
            CUDA_TRY(cudaMemsetAsync(elen + G, 0, 4, st));
            LAUNCH_N(k_pg_csr_len, G, st, grep, ev_off, G, elen);
            if (int rc = pg_offsets(st, A, elen, eoff, G, &E)) return rc;
            CUDA_TRY(A.alloc(&el, E));
            CUDA_TRY(A.alloc(&er, E));
            LAUNCH_N(k_pg_edges, G, st, grep, ev, ev_off, eoff, G, el, er);
        }
    }
    T->G = G;
    T->P = P;
    out->proteins[k] = P;
    out->meta_peptides[k] = M;
    out->groups[k] = G;
    out->edges[k] = E;
    CUDA_TRY(cudaEventRecord(ev_built, st));
    // 6. the cover
    CUDA_TRY(A.alloc(&T->lcov, G));
    PgCoverStats cs;
    if (int rc = pg_cover(st, A, E, G, M, el, er, T->lcov, &cs)) return rc;
    out->covered[k] = cs.covered;
    out->forced[k] = cs.forced;
    out->greedy_picks[k] = cs.greedy;
    out->components[k] = cs.components;
    out->largest_component[k] = cs.largest;
    CUDA_TRY(cudaEventRecord(ev_covered, st));
    // 7. the rows still unannotated
    if (G) {
        unsigned long long* d_ann;
        CUDA_TRY(A.zeros(&d_ann, 1, st));
        LAUNCH_N(k_pg_lookup, in.n, st, in.pep, in.n, in.poff, in.pids, in.pdecoy, in.cap_off, pix_of_key, group_of, T->lcov, base, pass_no, pass, count,
                 scratch, d_ann);
        unsigned long long ann = 0;
        if (int rc = read_back(st, &ann, d_ann, 8)) return rc;
        out->annotated[k] = ann;
    }
    return 0;
}

extern "C" int sage_b200_protein_groups(int device, const sage_b200_peptides* P, const sage_b200_protein_group_params* p, const sage_b200_feature* rows,
                                        const float* peptide_q, const float* discriminant_score, uint64_t n, sage_b200_protein_group_out* out) {
    if (!out || !P || !p) return fail(SAGE_B200_EINVAL, "protein_groups: null argument");
    if (n && (!rows || !peptide_q || !discriminant_score || !out->num_protein_groups || !out->protein_group_q || !out->pass || !out->row_group_offsets ||
              !out->row_groups || !out->group_offsets || !out->group_members || !out->group_covered || !out->group_decoy))
        return fail(SAGE_B200_EINVAL, "protein_groups: null argument");
    if (!p->protein_offsets || (P->n_peptides && !P->decoy)) return fail(SAGE_B200_EINVAL, "protein_groups: null peptide array");
    if (P->n_peptides >= 0xFFFFFFFFull) return fail(SAGE_B200_ELIMIT, "protein_groups: too many peptides for u32 PeptideIx");
    if (int rc = picked_limits("protein_groups", n)) return rc;
    if (p->n_names >= (1ull << 30)) return fail(SAGE_B200_ELIMIT, "protein_groups: 2^30 or more protein names");
    const uint64_t n_pep = P->n_peptides;
    if (p->protein_offsets[0] != 0) return fail(SAGE_B200_EINVAL, "protein_groups: protein_offsets[0] is %u, not 0", p->protein_offsets[0]);
    for (uint64_t q = 0; q < n_pep; q++)
        if (p->protein_offsets[q + 1] < p->protein_offsets[q])
            return fail(SAGE_B200_EINVAL, "protein_groups: protein_offsets decreases at peptide %llu", (unsigned long long)q);
    const uint64_t NP = p->protein_offsets[n_pep];
    if (NP >= (uint64_t)INT32_MAX) return fail(SAGE_B200_ELIMIT, "protein_groups: 2^31 - 1 or more protein entries");
    if (NP && !p->protein_ids) return fail(SAGE_B200_EINVAL, "protein_groups: null protein_ids");
    for (uint64_t j = 0; j < NP; j++)
        if (p->protein_ids[j] >= p->n_names)
            return fail(SAGE_B200_EINVAL, "protein_groups: protein id %u at entry %llu is not below n_names (%llu)", p->protein_ids[j], (unsigned long long)j,
                        (unsigned long long)p->n_names);
    std::vector<uint32_t> pep_idx(n);
    std::vector<uint8_t> label_ok(n);
    std::vector<uint64_t> cap_off(n + 1, 0);
    for (uint64_t i = 0; i < n; i++) {
        pep_idx[i] = rows[i].peptide_idx;
        if (pep_idx[i] >= n_pep)
            return fail(SAGE_B200_EINVAL, "protein_groups: row %llu has peptide_idx %u outside the peptide table (%llu peptides)", (unsigned long long)i,
                        pep_idx[i], (unsigned long long)n_pep);
        label_ok[i] = rows[i].label != -1;
        cap_off[i + 1] = cap_off[i] + (p->protein_offsets[pep_idx[i] + 1] - p->protein_offsets[pep_idx[i]]);
    }
    for (int k = 0; k < 2; k++)
        out->peptides[k] = out->proteins[k] = out->meta_peptides[k] = out->groups[k] = out->edges[k] = out->covered[k] = out->forced[k] =
            out->greedy_picks[k] = out->components[k] = out->largest_component[k] = out->annotated[k] = 0;
    out->passing = out->entries = 0;
    out->ms_build[0] = out->ms_build[1] = out->ms_cover[0] = out->ms_cover[1] = out->ms_lookup[0] = out->ms_lookup[1] = out->ms_picked = out->ms_total = 0.0f;
    if (n == 0) {
        out->row_group_offsets[0] = 0;
        return 0;
    }
    if (int rc = select_device(device)) return rc;
    const uint64_t cap = cap_off[n];
    if (int rc = picked_memory("protein_groups", n, 96 * NP + 48 * p->n_names + 8 * cap + 16 * n_pep)) return rc;
    const uint32_t N = (uint32_t)n;
    const bool gen = p->generate_decoys != 0, fma = host_math_variant() != 1;
    std::vector<uint8_t> pdecoy(n_pep);
    for (uint64_t q = 0; q < n_pep; q++) pdecoy[q] = P->decoy[q] ? 1 : 0;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    Event ev[9];
    for (Event& e : ev) CUDA_TRY(e.create());
    uint32_t *d_pep, *d_poff, *d_pids, *d_count, *d_scratch, *d_csr_len, *d_rows_out;
    uint8_t *d_label, *d_pdecoy, *d_pass;
    float *d_q, *d_score;
    uint64_t *d_cap, *d_out_off;
    CUDA_TRY(A.upload(&d_pep, pep_idx.data(), N, st));
    CUDA_TRY(A.upload(&d_poff, p->protein_offsets, n_pep + 1, st));
    CUDA_TRY(A.upload(&d_pids, p->protein_ids, NP, st));
    CUDA_TRY(A.upload(&d_label, label_ok.data(), N, st));
    CUDA_TRY(A.upload(&d_pdecoy, pdecoy.data(), n_pep, st));
    CUDA_TRY(A.upload(&d_q, peptide_q, N, st));
    CUDA_TRY(A.upload(&d_score, discriminant_score, N, st));
    CUDA_TRY(A.upload(&d_cap, cap_off.data(), N + 1, st));
    CUDA_TRY(A.zeros(&d_pass, N, st));
    CUDA_TRY(A.zeros(&d_count, N, st));
    CUDA_TRY(A.alloc(&d_scratch, cap));
    CUDA_TRY(cudaEventRecord(ev[0], st));
    const PgInputs in{N, (uint32_t)n_pep, (uint32_t)p->n_names, d_pep, d_poff, d_pids, d_label, d_pdecoy, d_q, d_cap};

    // generate_protein_groups: pass 1 at threshold.clamp(0, 1) (NaN stays NaN), pass 2 at 1.0; then the fallback
    PgTable T[2];
    for (int k = 0; k < 2; k++) {
        cudaEvent_t e0 = ev[3 * k], e1 = ev[3 * k + 1], e2 = ev[3 * k + 2], e3 = ev[3 * k + 3];
        if (k == 0) CUDA_TRY(cudaEventRecord(e0, st));
        const bool run = p->protein_grouping && (k == 1 || p->has_threshold);
        if (run) {
            float t = 1.0f;
            if (k == 0) {
                t = p->threshold;
                if (t < 0.0f) t = 0.0f;
                if (t > 1.0f) t = 1.0f;
            }
            if (int rc = pg_pass(st, A, in, t, (uint8_t)(k + 1), T[0].G, d_pass, d_count, d_scratch, &T[k], out, e1, e2)) return rc;
        } else {
            CUDA_TRY(cudaEventRecord(e1, st));
            CUDA_TRY(cudaEventRecord(e2, st));
        }
        CUDA_TRY(cudaEventRecord(e3, st));
    }
    CUDA_TRY(A.alloc(&d_csr_len, N + 1));
    CUDA_TRY(A.alloc(&d_out_off, N + 1));
    CUDA_TRY(cudaMemsetAsync(d_csr_len + N, 0, 4, st));
    LAUNCH_N(k_pg_fallback, N, st, d_pep, N, d_poff, d_pass, d_count, d_csr_len);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) {
        return cub::DeviceScan::ExclusiveSum(t, b, d_csr_len, d_out_off, (int)N + 1, st);
    }));
    uint64_t n_out = 0;
    if (int rc = read_back(st, &n_out, d_out_off + N, 8)) return rc;
    CUDA_TRY(A.alloc(&d_rows_out, n_out));
    LAUNCH_N(k_pg_compact_rows, N, st, d_cap, d_out_off, d_scratch, d_csr_len, N, d_rows_out);

    // the group tables of both passes, concatenated
    const uint32_t Gt = T[0].G + T[1].G, Pt = T[0].P + T[1].P;
    if (2ull * p->n_names + Gt >= 0xFFFFFFFFull) return fail(SAGE_B200_ELIMIT, "protein_groups: 2 * n_names + groups reach 2^32");
    uint32_t *goff, *members;
    uint8_t *gdecoy, *gcov;
    CUDA_TRY(A.alloc(&goff, Gt + 1));
    CUDA_TRY(A.alloc(&members, Pt));
    CUDA_TRY(A.alloc(&gdecoy, Gt));
    CUDA_TRY(A.alloc(&gcov, Gt));
    CUDA_TRY(cudaMemsetAsync(goff, 0, 4, st));
    for (int k = 0, g0 = 0, p0 = 0; k < 2; g0 += T[k].G, p0 += T[k].P, k++) {
        if (!T[k].G) continue;
        CUDA_TRY(cudaMemcpyAsync(goff + g0 + 1, T[k].goff + 1, 4ull * T[k].G, cudaMemcpyDeviceToDevice, st));
        LAUNCH_N(k_pg_add, T[k].G, st, goff + g0 + 1, T[k].G, (uint32_t)p0);
        CUDA_TRY(cudaMemcpyAsync(members + p0, T[k].members, 4ull * T[k].P, cudaMemcpyDeviceToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(gdecoy + g0, T[k].gdecoy, T[k].G, cudaMemcpyDeviceToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(gcov + g0, T[k].lcov, T[k].G, cudaMemcpyDeviceToDevice, st));
    }

    // picked_protein_group (fdr.rs:192-226): rows with one group string, keyed by it, side Peptide::decoy, Ix = the key
    uint32_t *rep, *gidx, *gidx_s, *key, *crow, *ckey, *crank, *nsel, m = 0;
    uint64_t *hash, *hash_s;
    uint8_t *side, *competes, *cside;
    float *cscore, *cq, *d_pgq;
    CUDA_TRY(A.alloc(&rep, Gt));
    CUDA_TRY(A.alloc(&gidx, Gt));
    CUDA_TRY(A.alloc(&gidx_s, Gt));
    CUDA_TRY(A.alloc(&hash, Gt));
    CUDA_TRY(A.alloc(&hash_s, Gt));
    LAUNCH_N(k_pg_group_hash, Gt, st, goff, members, gdecoy, Gt, gen, hash, gidx);
    if (Gt) CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, hash, hash_s, gidx, gidx_s, (int)Gt, 0, 64, st); }));
    LAUNCH_N(k_pg_group_rep, Gt, st, goff, members, gdecoy, gen, hash_s, gidx_s, Gt, rep);
    CUDA_TRY(A.alloc(&key, N));
    CUDA_TRY(A.alloc(&side, N));
    CUDA_TRY(A.alloc(&competes, N));
    CUDA_TRY(A.alloc(&crow, N));
    CUDA_TRY(A.alloc(&ckey, N));
    CUDA_TRY(A.alloc(&cside, N));
    CUDA_TRY(A.alloc(&cscore, N));
    CUDA_TRY(A.alloc(&crank, N));
    CUDA_TRY(A.alloc(&cq, N));
    CUDA_TRY(A.alloc(&d_pgq, N));
    CUDA_TRY(A.alloc(&nsel, 1));
    LAUNCH_N(k_pg_row_keys, N, st, d_pep, N, d_pass, d_count, d_out_off, d_rows_out, goff, members, gdecoy, rep, d_poff, d_pids, d_pdecoy, gen,
             (uint32_t)p->n_names, key, side, competes);
    thrust::counting_iterator<uint32_t> it(0);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, it, competes, crow, nsel, (int)N, st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, key, competes, ckey, nsel, (int)N, st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, side, competes, cside, nsel, (int)N, st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, d_score, competes, cscore, nsel, (int)N, st); }));
    if (int rc = read_back(st, &m, nsel, 4)) return rc;
    if (int rc = picked_competition(st, A, fma, m, ckey, cside, cscore, nullptr, false, crank, cq, &out->entries, &out->passing)) return rc;
    LAUNCH_N(k_pg_fill, N, st, d_pgq, N, 1.0f);
    LAUNCH_N(k_pg_scatter_q, m, st, crow, cq, m, d_pgq);
    CUDA_TRY(cudaEventRecord(ev[7], st));

    // outputs
    std::vector<uint32_t> h_goff(Gt + 1);
    CUDA_TRY(cudaMemcpyAsync(out->num_protein_groups, d_count, 4ull * N, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out->protein_group_q, d_pgq, 4ull * N, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out->pass, d_pass, N, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out->row_group_offsets, d_out_off, 8ull * (N + 1), cudaMemcpyDeviceToHost, st));
    if (n_out) CUDA_TRY(cudaMemcpyAsync(out->row_groups, d_rows_out, 4 * n_out, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(h_goff.data(), goff, 4ull * (Gt + 1), cudaMemcpyDeviceToHost, st));
    if (Pt) CUDA_TRY(cudaMemcpyAsync(out->group_members, members, 4ull * Pt, cudaMemcpyDeviceToHost, st));
    if (Gt) {
        CUDA_TRY(cudaMemcpyAsync(out->group_covered, gcov, Gt, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(out->group_decoy, gdecoy, Gt, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    for (uint32_t g = 0; g <= Gt; g++) out->group_offsets[g] = h_goff[g];
    for (int k = 0; k < 2; k++) {
        CUDA_TRY(cudaEventElapsedTime(&out->ms_build[k], ev[3 * k], ev[3 * k + 1]));
        CUDA_TRY(cudaEventElapsedTime(&out->ms_cover[k], ev[3 * k + 1], ev[3 * k + 2]));
        CUDA_TRY(cudaEventElapsedTime(&out->ms_lookup[k], ev[3 * k + 2], ev[3 * k + 3]));
    }
    CUDA_TRY(cudaEventElapsedTime(&out->ms_picked, ev[6], ev[7]));
    CUDA_TRY(cudaEventElapsedTime(&out->ms_total, ev[0], ev[7]));
    return 0;
}

extern "C" int sage_b200_bipartite_cover(int device, const uint32_t* left, const uint32_t* right, uint64_t n_edges, uint64_t n_left, uint64_t n_right,
                                         uint8_t* cover) {
    if ((n_edges && (!left || !right)) || (n_left && !cover)) return fail(SAGE_B200_EINVAL, "bipartite_cover: null argument");
    if (n_edges > (uint64_t)INT32_MAX || n_left + n_right > (uint64_t)INT32_MAX) return fail(SAGE_B200_ELIMIT, "bipartite_cover: 2^31 - 1 or more edges or nodes");
    for (uint64_t k = 0; k < n_edges; k++)
        if (left[k] >= n_left || right[k] >= n_right)
            return fail(SAGE_B200_EINVAL, "bipartite_cover: edge %llu (%u, %u) is out of range", (unsigned long long)k, left[k], right[k]);
    if (n_left == 0) return 0;
    if (int rc = select_device(device)) return rc;
    if (int rc = picked_memory("bipartite_cover", n_edges, 64 * (n_left + n_right))) return rc;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    const uint32_t E = (uint32_t)n_edges, G = (uint32_t)n_left, M = (uint32_t)n_right;
    uint32_t *el, *er;
    uint8_t* lcov;
    CUDA_TRY(A.upload(&el, left, E, st));
    CUDA_TRY(A.upload(&er, right, E, st));
    CUDA_TRY(A.alloc(&lcov, G));
    PgCoverStats cs;
    if (int rc = pg_cover(st, A, E, G, M, el, er, lcov, &cs)) return rc;
    return read_back(st, cover, lcov, G);
}

#if SAGE_B200_PHASE_CLOCKS
// variant builds only (not declared in the header): cycles per k_score phase summed over CTAs since the last reset
extern "C" int sage_b200_debug_phase_cycles(unsigned long long* out16, int reset) {
    const unsigned long long z[16] = {0};
    Stream st;
    CUDA_TRY(st.create());
    if (out16) CUDA_TRY(cudaMemcpyFromSymbolAsync(out16, g_phase, sizeof z, 0, cudaMemcpyDeviceToHost, st));
    if (reset) CUDA_TRY(cudaMemcpyToSymbolAsync(g_phase, z, sizeof z, 0, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}
#endif

// ================================================================================== digest (database.rs:162-258; kernels in digest.cuh)
struct sage_b200_digest {
    int device = 0;
    DevArena out;   // the output table, exact-size
    uint32_t *d_res_off = nullptr, *d_ref_off = nullptr, *d_ids = nullptr;
    uint8_t *d_seq = nullptr, *d_decoy = nullptr, *d_missed = nullptr, *d_semi = nullptr;
    float *d_mods = nullptr, *d_nterm = nullptr, *d_cterm = nullptr, *d_mono = nullptr;
    std::vector<uint64_t> name_off;
    std::string names;
    sage_b200_digest_info info{};
};

extern "C" void sage_b200_digest_destroy(sage_b200_digest* d) {
    if (!d) return;
    cudaSetDevice(d->device);
    delete d;
}

// ModificationSpecificity::from_str (modification.rs:63-100): "^", "$", "[", "]" with an optional residue, or one residue of mass.rs's
// VALID_AA (a second character after a residue is ignored); anything else is invalid and skipped by the Builder.
static bool dg_parse_spec(const char* s, DgSpec& out) {
    const size_t n = strlen(s);
    if (n == 0 || n > 2) return false;
    const int rest = n > 1 ? (int)(uint8_t)s[1] : -1;
    switch (s[0]) {
        case '^': out.kind = DG_SPEC_PEP_N; out.residue = rest; return true;
        case '$': out.kind = DG_SPEC_PEP_C; out.residue = rest; return true;
        case '[': out.kind = DG_SPEC_PROT_N; out.residue = rest; return true;
        case ']': out.kind = DG_SPEC_PROT_C; out.residue = rest; return true;
        default:
            if (!strchr("ACDEFGHIKLMNPQRSTVWYUO", s[0])) return false;
            out.kind = DG_SPEC_RESIDUE;
            out.residue = (uint8_t)s[0];
            return true;
    }
}

struct DgFasta {
    std::vector<uint8_t> res;
    std::vector<uint32_t> off{0};
    std::vector<std::string> acc;
    std::vector<uint8_t> decoy;
};

// u8::is_ascii_whitespace, the separator of split_ascii_whitespace: no '\v'.
static bool dg_ascii_space(uint8_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\f' || c == '\r'; }

// char::is_whitespace (Unicode White_Space), which str::trim strips: the byte length of the whitespace character s[0..n) encodes in UTF-8,
// or 0 when s[0..n) is not one.
static size_t dg_utf8_space(const uint8_t* s, size_t n) {
    if (n == 1) return ((s[0] >= 0x09 && s[0] <= 0x0D) || s[0] == 0x20) ? 1 : 0;
    if (n == 2) return (s[0] == 0xC2 && (s[1] == 0x85 || s[1] == 0xA0)) ? 2 : 0;   // U+0085, U+00A0
    if (n != 3) return 0;
    const uint32_t c = (uint32_t)s[0] << 16 | (uint32_t)s[1] << 8 | s[2];
    return (c == 0xE19A80 || (c >= 0xE28080 && c <= 0xE2808A) || c == 0xE280A8 || c == 0xE280A9 || c == 0xE280AF || c == 0xE2819F || c == 0xE38080)
               ? 3 : 0;   // U+1680, U+2000..U+200A, U+2028, U+2029, U+202F, U+205F, U+3000
}

// Fasta::parse (fasta.rs:14-56): lines split on '\n' with a trailing '\r' dropped, empty lines skipped, then trimmed of Unicode whitespace
// (str::trim); '>' starts a header whose first token split at ASCII whitespace is the accession. A protein is kept when it has residues,
// and with generate_decoys only when its accession does not contain the decoy tag; without generate_decoys a tagged protein is kept as a
// decoy.
static int dg_parse_fasta(const char* text, uint64_t len, const std::string& tag, bool generate_decoys, DgFasta& F) {
    std::string last_id;
    auto flush = [&]() -> int {
        size_t a = 0;
        while (a < last_id.size() && dg_ascii_space((uint8_t)last_id[a])) a++;
        size_t b = a;
        while (b < last_id.size() && !dg_ascii_space((uint8_t)last_id[b])) b++;
        std::string acc = last_id.substr(a, b - a);
        const bool tagged = acc.find(tag) != std::string::npos;
        if (tagged && generate_decoys) {
            F.res.resize(F.off.back());
            return 0;
        }
        if (F.res.size() >= 0xFFFFFFFFull) return fail(SAGE_B200_ELIMIT, "digest: 2^32 or more residues");
        F.off.push_back((uint32_t)F.res.size());
        F.acc.push_back(std::move(acc));
        F.decoy.push_back(tagged ? 1 : 0);
        return 0;
    };
    uint64_t pos = 0;
    while (pos <= len) {
        const char* nl = pos < len ? (const char*)memchr(text + pos, '\n', len - pos) : nullptr;
        uint64_t a = pos, b = nl ? (uint64_t)(nl - text) : len;
        pos = nl ? b + 1 : len + 1;
        if (b > a && text[b - 1] == '\r') b--;
        if (b == a) continue;
        const uint8_t* u = (const uint8_t*)text;
        for (bool more = true; more;) {
            more = false;
            for (size_t k = 1; k <= 3 && !more; k++)
                if (a + k <= b && dg_utf8_space(u + a, k)) a += k, more = true;
        }
        for (bool more = true; more;) {
            more = false;
            for (size_t k = 1; k <= 3 && !more; k++)
                if (b >= a + k && dg_utf8_space(u + b - k, k)) b -= k, more = true;
        }
        if (b > a && text[a] == '>') {
            if (F.res.size() > F.off.back())
                if (int rc = flush()) return rc;
            last_id.assign(text + a + 1, b - a - 1);
        } else {
            F.res.insert(F.res.end(), (const uint8_t*)text + a, (const uint8_t*)text + b);
        }
    }
    if (F.res.size() > F.off.back())
        if (int rc = flush()) return rc;
    if (F.res.size() >= 0xFFFFFFFFull) return fail(SAGE_B200_ELIMIT, "digest: 2^32 or more residues");
    return 0;
}

struct DgMax {
    __device__ uint32_t operator()(uint32_t a, uint32_t b) const { return a > b ? a : b; }
};

static int dg_memory(const char* stage, uint64_t bytes) {
    size_t free_b = 0, total_b = 0;
    CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
    if (bytes + (64ull << 20) > free_b)
        return fail(SAGE_B200_ELIMIT, "digest: the %s stage needs about %llu bytes of device memory, %llu free", stage, (unsigned long long)bytes,
                    (unsigned long long)free_b);
    return 0;
}

// Digests proteins [p0, p1) of the parsed FASTA as a FASTA of their own (its `targets` set, database.rs:186-200, is local to the range) into
// D's table. prot_name maps each protein of F to its id in the names table. With `seen`, the call stops after the per-protein `seen` stage
// and writes the number of windows it keeps: fasta.digest(&enzyme).len() of the range (enzyme.rs:310-330, fasta.rs:58-79).
static int dg_run(sage_b200_digest* D, const DgFasta& F, uint32_t p0, uint32_t p1, const DgParams& hp, const std::vector<DgSpec>& statics,
                  const std::vector<DgSpec>& vars, const std::vector<uint32_t>& prot_name, uint64_t* seen = nullptr) {
    sage_b200_digest_info& I = D->info;
    if (seen) *seen = 0;
    const uint32_t P = p1 - p0;
    const uint64_t R = F.off[p1] - F.off[p0];
    std::vector<uint32_t> off(F.off.begin() + p0, F.off.begin() + p1 + 1);
    for (uint32_t& o : off) o -= F.off[p0];
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    Event ev[8];
    for (Event& e : ev) CUDA_TRY(e.create());
    auto done = [&]() { I.peak_device_bytes = A.bytes + D->out.bytes; I.device_bytes = D->out.bytes; };
    thrust::counting_iterator<uint32_t> count_it(0);
    uint32_t* d_cnt = nullptr;
    CUDA_TRY(A.alloc(&d_cnt, 1));

    // upload
    if (int rc = dg_memory("upload", R + 16ull * P + 64)) return rc;
    CUDA_TRY(cudaEventRecord(ev[0], st));
    uint8_t *d_res = nullptr, *d_pdecoy = nullptr;
    uint32_t *d_poff = nullptr, *d_pname = nullptr;
    DgSpec *d_statics = nullptr, *d_vars = nullptr;
    CUDA_TRY(A.upload(&d_res, F.res.data() + F.off[p0], R, st));
    CUDA_TRY(A.upload(&d_poff, off.data(), P + 1, st));
    CUDA_TRY(A.upload(&d_pdecoy, F.decoy.data() + p0, P, st));
    CUDA_TRY(A.upload(&d_pname, prot_name.data() + p0, P, st));
    CUDA_TRY(A.upload(&d_statics, statics.data(), statics.size(), st));
    CUDA_TRY(A.upload(&d_vars, vars.data(), vars.size(), st));
    DgParams p = hp;
    p.statics = d_statics;
    p.vars = d_vars;
    CUDA_TRY(cudaEventRecord(ev[1], st));

    // 1. cleavage sites: count, scan, write
    uint32_t *d_ncut = nullptr, *d_cut_off = nullptr, *d_cuts = nullptr;
    CUDA_TRY(A.zeros(&d_ncut, P + 1, st));
    CUDA_TRY(A.alloc(&d_cut_off, P + 1));
    LAUNCH_N(k_dg_sites, 32ull * P, st, d_res, d_poff, P, p, d_ncut, nullptr, nullptr);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_ncut, d_cut_off, (int)(P + 1), st); }));
    uint32_t n_cuts = 0;
    if (int rc = read_back(st, &n_cuts, d_cut_off + P, 4)) return rc;
    CUDA_TRY(A.alloc(&d_cuts, n_cuts));
    LAUNCH_N(k_dg_sites, 32ull * P, st, d_res, d_poff, P, p, nullptr, d_cut_off, d_cuts);
    CUDA_TRY(cudaEventRecord(ev[2], st));

    // 2. windows: count, scan, write
    uint64_t *d_nwin = nullptr, *d_win_off = nullptr;
    CUDA_TRY(A.zeros(&d_nwin, P + 1, st));
    CUDA_TRY(A.alloc(&d_win_off, P + 1));
    LAUNCH_N(k_dg_windows, P, st, d_res, d_poff, d_cut_off, d_cuts, P, p, d_nwin, nullptr, nullptr);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_nwin, d_win_off, (int)(P + 1), st); }));
    uint64_t W64 = 0;
    if (int rc = read_back(st, &W64, d_win_off + P, 8)) return rc;
    if (W64 >= 0xFFFFFFFEull) return fail(SAGE_B200_ELIMIT, "digest: %llu windows (2^32 - 2 or more)", (unsigned long long)W64);
    const uint32_t W = (uint32_t)W64;
    I.n_windows = W;
    if (W == 0) return done(), 0;
    // windows, hashes and indices twice each, classes, keys twice, flags and the sorts' temporary storage
    if (int rc = dg_memory("window", 100ull * W)) return rc;
    DgWin* d_win = nullptr;
    CUDA_TRY(A.alloc(&d_win, W));
    LAUNCH_N(k_dg_windows, P, st, d_res, d_poff, d_cut_off, d_cuts, P, p, nullptr, d_win_off, d_win);
    CUDA_TRY(cudaEventRecord(ev[3], st));

    // 3. per-protein `seen` and group_digests: sort by hash, exact classes, stable sort by class, keep each protein's first window of a class,
    // stable sort by (class, Position, decoy): a group is a run, its first window the lowest protein's
    uint64_t *d_hash = nullptr, *d_hash_s = nullptr, *d_key = nullptr, *d_key_k = nullptr, *d_key3 = nullptr;
    uint32_t *d_idx = nullptr, *d_idx_s = nullptr, *d_rs = nullptr, *d_cls = nullptr, *d_cls_s = nullptr, *d_idx2 = nullptr, *d_idx_k = nullptr, *d_idx3 = nullptr,
             *d_head = nullptr;
    uint8_t* d_keep = nullptr;
    CUDA_TRY(A.alloc(&d_hash, W));
    CUDA_TRY(A.alloc(&d_hash_s, W));
    CUDA_TRY(A.alloc(&d_idx, W));
    CUDA_TRY(A.alloc(&d_idx_s, W));
    CUDA_TRY(A.alloc(&d_rs, W));
    CUDA_TRY(A.alloc(&d_cls, W));
    LAUNCH_N(k_dg_hash, W, st, d_res, d_win, W, d_hash, d_idx);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, d_hash, d_hash_s, d_idx, d_idx_s, (int)W, 0, 64, st); }));
    LAUNCH_N(k_dg_run_start, W, st, d_hash_s, W, d_rs);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::InclusiveScan(t, b, d_rs, d_rs, DgMax(), (int)W, st); }));
    LAUNCH_N(k_dg_class, W, st, d_res, d_win, d_idx_s, d_rs, W, d_cls);
    const int cbits = (int)std::max<uint32_t>(1, ceil_log2_u64(W));
    CUDA_TRY(A.alloc(&d_cls_s, W));
    CUDA_TRY(A.alloc(&d_idx2, W));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, d_cls, d_cls_s, d_idx_s, d_idx2, (int)W, 0, cbits, st); }));
    CUDA_TRY(A.alloc(&d_keep, W));
    CUDA_TRY(A.alloc(&d_key, W));
    LAUNCH_N(k_dg_seen, W, st, d_win, d_cls_s, d_idx2, d_pdecoy, W, d_keep, d_key);
    CUDA_TRY(A.alloc(&d_key_k, W));
    CUDA_TRY(A.alloc(&d_idx_k, W));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, d_key, d_keep, d_key_k, d_cnt, (int)W, st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, d_idx2, d_keep, d_idx_k, d_cnt, (int)W, st); }));
    uint32_t Kc = 0;
    if (int rc = read_back(st, &Kc, d_cnt, 4)) return rc;
    if (seen) {
        *seen = Kc;
        return done(), 0;
    }
    CUDA_TRY(A.alloc(&d_key3, Kc));
    CUDA_TRY(A.alloc(&d_idx3, Kc));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, d_key_k, d_key3, d_idx_k, d_idx3, (int)Kc, 0, cbits + 3, st); }));
    CUDA_TRY(A.alloc(&d_head, Kc));
    LAUNCH_N(k_dg_heads64, Kc, st, d_key3, Kc, d_head);
    uint32_t* d_gstart = nullptr;
    CUDA_TRY(A.alloc(&d_gstart, Kc + 1));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, count_it, d_head, d_gstart, d_cnt, (int)Kc, st); }));
    uint32_t G = 0;
    if (int rc = read_back(st, &G, d_cnt, 4)) return rc;
    I.n_groups = G;
    CUDA_TRY(cudaMemcpyAsync(d_gstart + G, &Kc, 4, cudaMemcpyHostToDevice, st));
    uint32_t *d_gwin = nullptr, *d_gcls = nullptr;
    uint8_t *d_gmeta = nullptr, *d_cls_target = nullptr;
    CUDA_TRY(A.alloc(&d_gwin, G));
    CUDA_TRY(A.alloc(&d_gcls, G));
    CUDA_TRY(A.alloc(&d_gmeta, G));
    CUDA_TRY(A.zeros(&d_cls_target, W, st));
    LAUNCH_N(k_dg_groups, G, st, d_key3, d_idx3, d_gstart, G, d_gwin, d_gmeta, d_gcls, d_cls_target);
    CUDA_TRY(cudaEventRecord(ev[4], st));

    // 4. Peptide::try_from, the variable-mod sites, the forms (apply, the mass filter, reverse and the targets filter)
    float* d_gbase = nullptr;
    uint32_t *d_nsite = nullptr, *d_site_off = nullptr, *d_overflow = nullptr;
    uint64_t *d_nform = nullptr, *d_form_off = nullptr;
    uint8_t* d_revt = nullptr;
    CUDA_TRY(A.alloc(&d_gbase, G));
    CUDA_TRY(A.alloc(&d_nsite, G + 1));
    CUDA_TRY(A.alloc(&d_site_off, G + 1));
    CUDA_TRY(A.alloc(&d_nform, G + 1));
    CUDA_TRY(A.alloc(&d_form_off, G + 1));
    CUDA_TRY(A.alloc(&d_revt, G));
    CUDA_TRY(A.zeros(&d_overflow, 1, st));
    CUDA_TRY(cudaMemsetAsync(d_nsite + G, 0, 4, st));
    CUDA_TRY(cudaMemsetAsync(d_nform + G, 0, 8, st));
    LAUNCH_N(k_dg_group_info, G, st, d_res, d_win, d_gwin, d_gmeta, G, p, d_hash_s, d_idx_s, W, d_gbase, d_nsite, d_nform, d_revt, d_overflow);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_nsite, d_site_off, (int)(G + 1), st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_nform, d_form_off, (int)(G + 1), st); }));
    uint32_t n_sites = 0, overflow = 0;
    uint64_t T64 = 0;
    if (int rc = read_back(st, &n_sites, d_site_off + G, 4)) return rc;
    if (int rc = read_back(st, &T64, d_form_off + G, 8)) return rc;
    if (int rc = read_back(st, &overflow, d_overflow, 4)) return rc;
    if (overflow) return fail(SAGE_B200_ELIMIT, "digest: a peptide has more than 65535 variable-modification sites");
    if (T64 >= (1ull << 31)) return fail(SAGE_B200_ELIMIT, "digest: %llu (peptide, modification combination) candidates (2^31 or more)", (unsigned long long)T64);
    const uint32_t T = (uint32_t)T64;
    I.n_candidates = T;
    if (T == 0) return done(), 0;
    if (int rc = dg_memory("expansion", 8ull * n_sites + 12ull * T)) return rc;
    uint32_t *d_site_code = nullptr, *d_rows = nullptr, *d_row_off = nullptr;
    float* d_site_mass = nullptr;
    CUDA_TRY(A.alloc(&d_site_code, n_sites));
    CUDA_TRY(A.alloc(&d_site_mass, n_sites));
    LAUNCH_N(k_dg_site_fill, G, st, d_res, d_win, d_gwin, d_gmeta, d_site_off, G, p, d_site_code, d_site_mass);
    DgView V{d_res, d_poff, d_win, d_gwin, d_gmeta, d_site_off, d_site_code, d_site_mass, nullptr, nullptr, p};
    CUDA_TRY(A.alloc(&d_rows, T + 1));
    CUDA_TRY(A.alloc(&d_row_off, T + 1));
    CUDA_TRY(cudaMemsetAsync(d_rows + T, 0, 4, st));
    LAUNCH_N(k_dg_expand, T, st, V, d_form_off, G, T, d_gbase, d_gcls, d_cls_target, d_revt, d_rows, nullptr, nullptr, nullptr);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_rows, d_row_off, (int)(T + 1), st); }));
    uint32_t N = 0;
    if (int rc = read_back(st, &N, d_row_off + T, 4)) return rc;
    if (N >= 0xFFFFFFFEu) return fail(SAGE_B200_ELIMIT, "digest: 2^32 - 2 or more peptide rows");
    I.n_rows = N;
    if (N == 0) return done(), 0;
    // forms and masses, keys and indices twice, run flags and positions, merge heads, and the merge sort's buffers
    if (int rc = dg_memory("sort", 64ull * N)) return rc;
    DgForm* d_forms = nullptr;
    float* d_fmono = nullptr;
    CUDA_TRY(A.alloc(&d_forms, N));
    CUDA_TRY(A.alloc(&d_fmono, N));
    LAUNCH_N(k_dg_expand, T, st, V, d_form_off, G, T, d_gbase, d_gcls, d_cls_target, d_revt, d_rows, d_row_off, d_forms, d_fmono);
    V.forms = d_forms;
    V.form_mono = d_fmono;
    CUDA_TRY(cudaEventRecord(ev[5], st));

    // 5. reorder_peptides' sort: stable radix sort by total_cmp(mono), then a stable merge sort of the equal-mono runs by initial_sort
    uint32_t *d_mkey = nullptr, *d_mkey_s = nullptr, *d_fidx = nullptr, *d_order = nullptr, *d_rpos = nullptr, *d_rval = nullptr;
    uint8_t* d_inrun = nullptr;
    CUDA_TRY(A.alloc(&d_mkey, N));
    CUDA_TRY(A.alloc(&d_mkey_s, N));
    CUDA_TRY(A.alloc(&d_fidx, N));
    CUDA_TRY(A.alloc(&d_order, N));
    CUDA_TRY(A.alloc(&d_inrun, N));
    LAUNCH_N(k_dg_mono_key, N, st, d_fmono, N, d_mkey, d_fidx);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, d_mkey, d_mkey_s, d_fidx, d_order, (int)N, 0, 32, st); }));
    LAUNCH_N(k_dg_in_run, N, st, d_mkey_s, N, d_inrun);
    CUDA_TRY(A.alloc(&d_rpos, N));
    CUDA_TRY(A.alloc(&d_rval, N));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, count_it, d_inrun, d_rpos, d_cnt, (int)N, st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, d_order, d_inrun, d_rval, d_cnt, (int)N, st); }));
    uint32_t M = 0;
    if (int rc = read_back(st, &M, d_cnt, 4)) return rc;
    if (M) {
        const DgRowLess less{V};
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceMergeSort::StableSortKeys(t, b, d_rval, (int)M, less, st); }));
        LAUNCH_N(k_dg_scatter, M, st, d_rpos, d_rval, M, d_order);
    }
    CUDA_TRY(cudaEventRecord(ev[6], st));

    // 6. reorder_peptides' merge and the output table
    uint32_t *d_mhead = nullptr, *d_first = nullptr;
    CUDA_TRY(A.alloc(&d_mhead, N));
    CUDA_TRY(A.alloc(&d_first, N + 1));
    LAUNCH_N(k_dg_merge_heads, N, st, V, d_order, N, d_mhead);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, count_it, d_mhead, d_first, d_cnt, (int)N, st); }));
    uint32_t n_pep = 0;
    if (int rc = read_back(st, &n_pep, d_cnt, 4)) return rc;
    CUDA_TRY(cudaMemcpyAsync(d_first + n_pep, &N, 4, cudaMemcpyHostToDevice, st));
    // offsets in 64 bits, so that a table of 2^32 residues or protein references or more is reported rather than wrapped
    uint64_t *d_nres = nullptr, *d_nref = nullptr, *d_res_off64 = nullptr, *d_ref_off64 = nullptr;
    CUDA_TRY(A.alloc(&d_nres, n_pep + 1));
    CUDA_TRY(A.alloc(&d_nref, n_pep + 1));
    CUDA_TRY(A.alloc(&d_res_off64, n_pep + 1));
    CUDA_TRY(A.alloc(&d_ref_off64, n_pep + 1));
    CUDA_TRY(cudaMemsetAsync(d_nres + n_pep, 0, 8, st));
    CUDA_TRY(cudaMemsetAsync(d_nref + n_pep, 0, 8, st));
    LAUNCH_N(k_dg_pep_counts, n_pep, st, V, d_order, d_first, n_pep, d_gstart, d_nres, d_nref);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_nres, d_res_off64, (int)(n_pep + 1), st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_nref, d_ref_off64, (int)(n_pep + 1), st); }));
    uint64_t n_res = 0, n_ref = 0;
    if (int rc = read_back(st, &n_res, d_res_off64 + n_pep, 8)) return rc;
    if (int rc = read_back(st, &n_ref, d_ref_off64 + n_pep, 8)) return rc;
    if (n_res > 0xFFFFFFFFull || n_ref >= 0x7FFFFFFFull)
        return fail(SAGE_B200_ELIMIT, "digest: %llu residues / %llu protein references in the table (u32 offsets)", (unsigned long long)n_res,
                    (unsigned long long)n_ref);
    if (int rc = dg_memory("output", 5ull * n_res + 30ull * n_pep + 8ull * n_ref)) return rc;
    DevArena& O = D->out;
    uint32_t* d_ids_raw = nullptr;
    CUDA_TRY(O.alloc(&D->d_res_off, n_pep + 1));
    CUDA_TRY(O.alloc(&D->d_ref_off, n_pep + 1));
    CUDA_TRY(O.alloc(&D->d_ids, n_ref));
    CUDA_TRY(O.alloc(&D->d_seq, n_res));
    CUDA_TRY(O.alloc(&D->d_mods, n_res));
    CUDA_TRY(O.alloc(&D->d_nterm, n_pep));
    CUDA_TRY(O.alloc(&D->d_cterm, n_pep));
    CUDA_TRY(O.alloc(&D->d_mono, n_pep));
    CUDA_TRY(O.alloc(&D->d_decoy, n_pep));
    CUDA_TRY(O.alloc(&D->d_missed, n_pep));
    CUDA_TRY(O.alloc(&D->d_semi, n_pep));
    CUDA_TRY(A.alloc(&d_ids_raw, n_ref));
    LAUNCH_N(k_dg_u64_to_u32, n_pep + 1, st, d_res_off64, n_pep + 1, D->d_res_off);
    LAUNCH_N(k_dg_u64_to_u32, n_pep + 1, st, d_ref_off64, n_pep + 1, D->d_ref_off);
    LAUNCH_N(k_dg_export, n_pep, st, V, d_order, d_first, n_pep, d_gstart, d_idx3, d_pname, D->d_res_off, D->d_ref_off, D->d_seq, D->d_mods,
             D->d_nterm, D->d_cterm, D->d_mono, D->d_decoy, D->d_missed, D->d_semi, d_ids_raw);
    // proteins.sort_unstable() (database.rs:250): ids are name ranks, so an ascending sort of the ids is the sort of the names
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) {
        return cub::DeviceSegmentedSort::SortKeys(t, b, d_ids_raw, D->d_ids, (int)n_ref, (int)n_pep, D->d_ref_off, D->d_ref_off + 1, st);
    }));
    CUDA_TRY(cudaEventRecord(ev[7], st));
    CUDA_TRY(cudaStreamSynchronize(st));
    I.n_peptides = n_pep;
    I.n_residues = n_res;
    I.n_protein_refs = n_ref;
    float* ms[7] = {&I.ms_upload, &I.ms_sites, &I.ms_windows, &I.ms_group, &I.ms_expand, &I.ms_sort, &I.ms_merge};
    for (int i = 0; i < 7; i++) CUDA_TRY(cudaEventElapsedTime(ms[i], ev[i], ev[i + 1]));
    CUDA_TRY(cudaEventElapsedTime(&I.ms_total, ev[0], ev[7]));
    done();
    return 0;
}

// Builder::make_parameters and Enzyme::new (database.rs:96-115, enzyme.rs:145-184) of the digest parameters, with their argument checks.
struct DgSetup {
    DgParams hp{};
    std::vector<DgSpec> statics, vars;
    uint64_t n_var_specs = 0;   // distinct valid variable specs: Parameters::variable_mods.len()
};

static int dg_setup(const sage_b200_digest_params* p, DgSetup& S) {
    if ((p->n_static && (!p->static_specs || !p->static_masses)) || (p->n_variable && (!p->variable_specs || !p->variable_masses)))
        return fail(SAGE_B200_EINVAL, "digest_create: null modification array");
    if (p->max_len > 255) return fail(SAGE_B200_ELIMIT, "digest: max_len %llu > 255 (the library's peptide-length limit)", (unsigned long long)p->max_len);
    if (p->max_variable_mods > DG_KMAX) return fail(SAGE_B200_ELIMIT, "digest: max_variable_mods %llu > %u", (unsigned long long)p->max_variable_mods, DG_KMAX);
    for (uint64_t i = 0; i < p->n_static; i++)
        if (!p->static_specs[i] || !std::isfinite(p->static_masses[i])) return fail(SAGE_B200_EINVAL, "digest: static mod %llu: null spec or non-finite mass", (unsigned long long)i);
    for (uint64_t i = 0; i < p->n_variable; i++)
        if (!p->variable_specs[i] || !std::isfinite(p->variable_masses[i]))
            return fail(SAGE_B200_EINVAL, "digest: variable mod %llu: null spec or non-finite mass", (unsigned long long)i);
    DgParams& hp = S.hp;
    const std::string cleave_at = p->cleave_at ? p->cleave_at : "", restrict_ = p->restrict_ ? p->restrict_ : "";
    hp.min_len = (uint32_t)std::min<uint64_t>(p->min_len, 256);
    hp.max_len = (uint32_t)p->max_len;
    hp.missed = p->missed_cleavages;
    hp.c_terminal = p->c_terminal ? 1 : 0;
    hp.has_enzyme = !cleave_at.empty();
    if (!hp.has_enzyme) {
        hp.missed = 0;
    } else if (cleave_at == "$") {
        hp.dollar = 1;
        hp.c_terminal = 1;
    } else {
        for (char c : cleave_at) if (c >= 'A' && c <= 'Z') hp.cleave |= 1u << (c - 'A');
        for (char c : restrict_) if (c >= 'A' && c <= 'Z') hp.restrict_ |= 1u << (c - 'A');
        hp.semi = p->semi_enzymatic ? 1 : 0;
    }
    hp.generate_decoys = p->generate_decoys ? 1 : 0;
    hp.kmax = (uint32_t)std::max<uint64_t>(p->max_variable_mods, 1);
    hp.min_mass = p->peptide_min_mass;
    hp.max_mass = p->peptide_max_mass;
    auto spec_less = [](const DgSpec& a, const DgSpec& b) { return a.kind != b.kind ? a.kind < b.kind : a.residue < b.residue; };
    for (uint64_t i = 0; i < p->n_static; i++) {   // a map keyed by spec: ordered, the last mass of a repeated spec wins
        DgSpec s{};
        if (!dg_parse_spec(p->static_specs[i], s)) continue;
        s.mass = p->static_masses[i];
        auto it = std::lower_bound(S.statics.begin(), S.statics.end(), s, spec_less);
        if (it != S.statics.end() && !spec_less(s, *it)) it->mass = s.mass;
        else S.statics.insert(it, s);
    }
    // validate_var_mods inserts each spec string's masses into a map keyed by spec (modification.rs:129-155): a later spec string naming the
    // same spec replaces the masses of the earlier one. Entries with equal spec strings are one string's list.
    std::vector<const char*> var_str;
    for (uint64_t i = 0; i < p->n_variable; i++) {
        DgSpec s{};
        if (!dg_parse_spec(p->variable_specs[i], s)) continue;
        s.mass = p->variable_masses[i];
        for (size_t j = 0; j < S.vars.size();)
            if (!spec_less(S.vars[j], s) && !spec_less(s, S.vars[j]) && strcmp(var_str[j], p->variable_specs[i]) != 0) {
                S.vars.erase(S.vars.begin() + j);
                var_str.erase(var_str.begin() + j);
            } else {
                j++;
            }
        S.vars.push_back(s);
        var_str.push_back(p->variable_specs[i]);
    }
    std::stable_sort(S.vars.begin(), S.vars.end(), spec_less);
    for (size_t i = 0; i < S.vars.size(); i++)
        if (i == 0 || spec_less(S.vars[i - 1], S.vars[i])) S.n_var_specs++;
    hp.n_static = (uint32_t)S.statics.size();
    hp.n_var = (uint32_t)S.vars.size();
    return 0;
}

// The names table: distinct accessions in byte order; a protein's id is its accession's rank.
static void dg_names(const DgFasta& F, sage_b200_digest* D, std::vector<uint32_t>& prot_name) {
    std::vector<uint32_t> order(F.acc.size());
    prot_name.assign(F.acc.size(), 0);
    for (uint32_t i = 0; i < order.size(); i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return F.acc[a] < F.acc[b]; });
    D->name_off.push_back(0);
    for (size_t k = 0; k < order.size(); k++) {
        if (k == 0 || F.acc[order[k]] != F.acc[order[k - 1]]) {
            D->names += F.acc[order[k]];
            D->name_off.push_back(D->names.size());
        }
        prot_name[order[k]] = (uint32_t)(D->name_off.size() - 2);
    }
    sage_b200_digest_info& I = D->info;
    I.n_proteins = F.acc.size();
    I.n_names = D->name_off.size() - 1;
    I.name_bytes = D->names.size();
}

extern "C" int sage_b200_digest_create(int device, const char* fasta, uint64_t fasta_len, const sage_b200_digest_params* p, sage_b200_digest** out) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!out || !p || (fasta_len && !fasta)) return fail(SAGE_B200_EINVAL, "digest_create: null argument");
    *out = nullptr;
    DgSetup S;
    if (int rc = dg_setup(p, S)) return rc;
    Guard<sage_b200_digest> guard(new sage_b200_digest(), sage_b200_digest_destroy);
    sage_b200_digest* D = guard.get();
    D->device = device;
    DgFasta F;
    if (int rc = dg_parse_fasta(fasta, fasta_len, p->decoy_tag ? p->decoy_tag : "rev_", p->generate_decoys != 0, F)) return rc;
    std::vector<uint32_t> prot_name;
    dg_names(F, D, prot_name);
    sage_b200_digest_info& I = D->info;
    I.ms_parse = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (int rc = select_device(device)) return rc;
    if (!F.acc.empty())
        if (int rc = dg_run(D, F, 0, (uint32_t)F.acc.size(), S.hp, S.statics, S.vars, prot_name)) return rc;
    I.ms_wall = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    *out = guard.release();
    return 0;
}

extern "C" int sage_b200_digest_get_info(const sage_b200_digest* D, sage_b200_digest_info* info) {
    if (!D || !info) return fail(SAGE_B200_EINVAL, "digest_get_info: null argument");
    *info = D->info;
    return 0;
}

extern "C" int sage_b200_digest_export(const sage_b200_digest* D, uint32_t* residue_offsets, uint8_t* sequence, float* modifications, float* nterm,
                                       float* cterm, float* monoisotopic, uint8_t* decoy, uint8_t* missed_cleavages, uint8_t* semi_enzymatic,
                                       uint32_t* protein_offsets, uint32_t* protein_ids, uint64_t* name_offsets, char* name_bytes) {
    if (!D) return fail(SAGE_B200_EINVAL, "digest_export: null handle");
    const sage_b200_digest_info& I = D->info;
    if (name_offsets) memcpy(name_offsets, D->name_off.data(), 8 * D->name_off.size());
    if (name_bytes && !D->names.empty()) memcpy(name_bytes, D->names.data(), D->names.size());
    const uint64_t n = I.n_peptides;
    if (n == 0) {
        if (residue_offsets) residue_offsets[0] = 0;
        if (protein_offsets) protein_offsets[0] = 0;
        return 0;
    }
    CUDA_TRY(cudaSetDevice(D->device));
    Stream st;
    CUDA_TRY(st.create());
    struct Copy { void* dst; const void* src; uint64_t bytes; };
    const Copy copies[] = {{residue_offsets, D->d_res_off, 4 * (n + 1)}, {sequence, D->d_seq, I.n_residues}, {modifications, D->d_mods, 4 * I.n_residues},
                           {nterm, D->d_nterm, 4 * n}, {cterm, D->d_cterm, 4 * n}, {monoisotopic, D->d_mono, 4 * n}, {decoy, D->d_decoy, n},
                           {missed_cleavages, D->d_missed, n}, {semi_enzymatic, D->d_semi, n}, {protein_offsets, D->d_ref_off, 4 * (n + 1)},
                           {protein_ids, D->d_ids, 4 * I.n_protein_refs}};
    for (const Copy& c : copies)
        if (c.dst && c.bytes) CUDA_TRY(cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

// ================================================================================== prefilter (runner.rs:104-128, 161-238; kernels in prefilter.cuh)
struct sage_b200_prefilter {
    int device = 0;
    sage_b200_digest table;               // the final peptide table and the whole FASTA's names table
    sage_b200_db* db = nullptr;           // the index over the final table, until the caller takes it
    std::vector<uint64_t> chunk_rows, chunk_kept;
    sage_b200_prefilter_info info{};
};

extern "C" void sage_b200_prefilter_destroy(sage_b200_prefilter* f) {
    if (!f) return;
    cudaSetDevice(f->device);
    sage_b200_db_destroy(f->db);
    delete f;
}

// The kept rows of the chunks so far, in chunk order, in the digest's export layout. Rows, residues and protein references each grow
// geometrically; a growth copies the rows already held.
struct PfTable {
    static constexpr int NA = 11;   // res_off, ref_off, nterm, cterm, mono, decoy, missed, semi | seq, mods | ids
    static constexpr size_t SZ[NA] = {4, 4, 4, 4, 4, 1, 1, 1, 1, 4, 4};
    void* p[NA] = {};
    uint64_t n = 0, n_res = 0, n_ref = 0, cap[3] = {0, 0, 0};
    PfTable() = default;
    PfTable(const PfTable&) = delete;
    PfTable& operator=(const PfTable&) = delete;
    ~PfTable() { for (void* q : p) if (q) cudaFree(q); }
    static int group(int a) { return a < 8 ? 0 : (a < 10 ? 1 : 2); }
    uint64_t bytes() const { return (cap[0] + 1) * 23 + cap[1] * 5 + cap[2] * 4; }
    // Room for `rows` rows, `res` residues and `refs` references in all; the arrays are copied on st.
    cudaError_t reserve(uint64_t rows, uint64_t res, uint64_t refs, cudaStream_t st) {
        const uint64_t need[3] = {rows, res, refs}, used[3] = {n, n_res, n_ref};
        for (int g = 0; g < 3; g++) {
            if (need[g] <= cap[g] && p[g == 0 ? 0 : (g == 1 ? 8 : 10)]) continue;
            const uint64_t c = std::max<uint64_t>(std::max<uint64_t>(need[g], 2 * cap[g]), 1024);
            for (int a = 0; a < NA; a++) {
                if (group(a) != g) continue;
                void* q = nullptr;
                const uint64_t count = g == 0 ? c + 1 : c, keep = g == 0 && a < 2 ? used[0] + 1 : used[g];
                if (cudaError_t e = cudaMalloc(&q, count * SZ[a])) return e;
                if (p[a]) {
                    if (cudaError_t e = cudaMemcpyAsync(q, p[a], keep * SZ[a], cudaMemcpyDeviceToDevice, st)) { cudaFree(q); return e; }
                    if (cudaError_t e = cudaStreamSynchronize(st)) { cudaFree(q); return e; }
                    cudaFree(p[a]);
                }
                p[a] = q;
            }
            cap[g] = c;
        }
        return cudaSuccess;
    }
    DevTable view() const {
        DevTable t;
        t.n = n; t.n_res = n_res; t.n_ref = n_ref;
        t.res_off = (const uint32_t*)p[0]; t.ref_off = (const uint32_t*)p[1]; t.nterm = (const float*)p[2]; t.cterm = (const float*)p[3];
        t.mono = (const float*)p[4]; t.decoy = (const uint8_t*)p[5]; t.missed = (const uint8_t*)p[6]; t.semi = (const uint8_t*)p[7];
        t.seq = (const uint8_t*)p[8]; t.mods = (const float*)p[9]; t.ids = (const uint32_t*)p[10];
        return t;
    }
};

static DevTable dg_table(const sage_b200_digest& D) {
    DevTable t;
    t.n = D.info.n_peptides; t.n_res = D.info.n_residues; t.n_ref = D.info.n_protein_refs;
    t.res_off = D.d_res_off; t.ref_off = D.d_ref_off; t.ids = D.d_ids; t.seq = D.d_seq; t.decoy = D.d_decoy; t.missed = D.d_missed; t.semi = D.d_semi;
    t.mods = D.d_mods; t.nterm = D.d_nterm; t.cterm = D.d_cterm; t.mono = D.d_mono;
    return t;
}

// Appends the rows of chunk table C whose keep byte is set to T (the protein ids are already global), on st. Returns the kept count in *kept.
static int pf_compact(const DevTable& C, const uint8_t* d_keep, PfTable& T, cudaStream_t st, uint64_t* kept, uint64_t* peak, uint64_t held) {
    *kept = 0;
    const uint32_t n = (uint32_t)C.n;
    if (n == 0) return 0;
    if (int rc = dg_memory("prefilter compaction", 44ull * (n + 1))) return rc;
    DevArena A;
    uint32_t *d_kept = nullptr, *d_row_at = nullptr;
    uint64_t *d_nres = nullptr, *d_nref = nullptr, *d_res_at = nullptr, *d_ref_at = nullptr;
    CUDA_TRY(A.zeros(&d_kept, n + 1, st));
    CUDA_TRY(A.zeros(&d_nres, n + 1, st));
    CUDA_TRY(A.zeros(&d_nref, n + 1, st));
    CUDA_TRY(A.alloc(&d_row_at, n + 1));
    CUDA_TRY(A.alloc(&d_res_at, n + 1));
    CUDA_TRY(A.alloc(&d_ref_at, n + 1));
    LAUNCH_N(k_pf_keep_counts, n, st, d_keep, C.res_off, C.ref_off, n, d_kept, d_nres, d_nref);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_kept, d_row_at, (int)(n + 1), st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_nres, d_res_at, (int)(n + 1), st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_nref, d_ref_at, (int)(n + 1), st); }));
    uint32_t k = 0;
    uint64_t tot[2] = {0, 0};
    CUDA_TRY(cudaMemcpyAsync(&k, d_row_at + n, 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&tot[0], d_res_at + n, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&tot[1], d_ref_at + n, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    const uint64_t rows = T.n + k, res = T.n_res + tot[0], refs = T.n_ref + tot[1];
    if (rows >= 0xFFFFFFFEull || res > 0xFFFFFFFFull || refs >= 0x7FFFFFFFull)
        return fail(SAGE_B200_ELIMIT, "prefilter: %llu kept rows / %llu residues / %llu protein references (u32 offsets)", (unsigned long long)rows,
                    (unsigned long long)res, (unsigned long long)refs);
    if (k == 0) return 0;
    if (rows > T.cap[0] || res > T.cap[1] || refs > T.cap[2])
        if (int rc = dg_memory("prefilter table", 2 * (23ull * rows + 5ull * res + 4ull * refs))) return rc;
    CUDA_TRY(T.reserve(rows, res, refs, st));
    *peak = std::max<uint64_t>(*peak, held + T.bytes() + A.bytes);
    uint32_t *res_off = (uint32_t*)T.p[0], *ref_off = (uint32_t*)T.p[1];
    LAUNCH_N(k_pf_gather, n, st, C.rows(), n, d_keep, d_row_at, d_res_at, d_ref_at, (uint32_t)T.n, T.n_res, T.n_ref, res_off, ref_off, (uint8_t*)T.p[8],
             (float*)T.p[9], (float*)T.p[2], (float*)T.p[3], (float*)T.p[4], (uint8_t*)T.p[5], (uint8_t*)T.p[6], (uint8_t*)T.p[7], (uint32_t*)T.p[10]);
    const uint32_t tail[2] = {(uint32_t)res, (uint32_t)refs};
    CUDA_TRY(cudaMemcpyAsync(res_off + rows, &tail[0], 4, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(ref_off + rows, &tail[1], 4, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    T.n = rows;
    T.n_res = res;
    T.n_ref = refs;
    *kept = k;
    return 0;
}

// reorder_peptides (database.rs:221-258) over the stored rows of T into D's output table: a stable radix sort by total_cmp(mono), a stable
// merge sort of the equal-mono runs by initial_sort, the adjacent merge, and a segmented sort of each peptide's protein ids.
static int pf_merge(const PfTable& T, sage_b200_digest* D, cudaStream_t st, uint64_t* peak, uint64_t held) {
    sage_b200_digest_info& I = D->info;
    const uint32_t N = (uint32_t)T.n;
    if (N == 0) return 0;
    const PfRows rows = T.view().rows();
    if (int rc = dg_memory("prefilter merge", 64ull * N)) return rc;
    DevArena A;
    thrust::counting_iterator<uint32_t> count_it(0);
    uint32_t *d_cnt = nullptr, *d_mkey = nullptr, *d_mkey_s = nullptr, *d_idx = nullptr, *d_order = nullptr, *d_rpos = nullptr, *d_rval = nullptr;
    uint8_t* d_inrun = nullptr;
    CUDA_TRY(A.alloc(&d_cnt, 1));
    CUDA_TRY(A.alloc(&d_mkey, N));
    CUDA_TRY(A.alloc(&d_mkey_s, N));
    CUDA_TRY(A.alloc(&d_idx, N));
    CUDA_TRY(A.alloc(&d_order, N));
    CUDA_TRY(A.alloc(&d_inrun, N));
    LAUNCH_N(k_dg_mono_key, N, st, rows.mono, N, d_mkey, d_idx);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, d_mkey, d_mkey_s, d_idx, d_order, (int)N, 0, 32, st); }));
    LAUNCH_N(k_dg_in_run, N, st, d_mkey_s, N, d_inrun);
    CUDA_TRY(A.alloc(&d_rpos, N));
    CUDA_TRY(A.alloc(&d_rval, N));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, count_it, d_inrun, d_rpos, d_cnt, (int)N, st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, d_order, d_inrun, d_rval, d_cnt, (int)N, st); }));
    uint32_t M = 0;
    if (int rc = read_back(st, &M, d_cnt, 4)) return rc;
    if (M) {
        const PfRowLess less{rows};
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceMergeSort::StableSortKeys(t, b, d_rval, (int)M, less, st); }));
        LAUNCH_N(k_dg_scatter, M, st, d_rpos, d_rval, M, d_order);
    }
    uint32_t *d_mhead = nullptr, *d_first = nullptr;
    CUDA_TRY(A.alloc(&d_mhead, N));
    CUDA_TRY(A.alloc(&d_first, N + 1));
    LAUNCH_N(k_pf_merge_heads, N, st, rows, d_order, N, d_mhead);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, count_it, d_mhead, d_first, d_cnt, (int)N, st); }));
    uint32_t n_pep = 0;
    if (int rc = read_back(st, &n_pep, d_cnt, 4)) return rc;
    CUDA_TRY(cudaMemcpyAsync(d_first + n_pep, &N, 4, cudaMemcpyHostToDevice, st));
    uint64_t *d_nres = nullptr, *d_nref = nullptr, *d_res_off64 = nullptr, *d_ref_off64 = nullptr;
    CUDA_TRY(A.zeros(&d_nres, n_pep + 1, st));
    CUDA_TRY(A.zeros(&d_nref, n_pep + 1, st));
    CUDA_TRY(A.alloc(&d_res_off64, n_pep + 1));
    CUDA_TRY(A.alloc(&d_ref_off64, n_pep + 1));
    LAUNCH_N(k_pf_pep_counts, n_pep, st, rows, d_order, d_first, n_pep, d_nres, d_nref);
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_nres, d_res_off64, (int)(n_pep + 1), st); }));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, d_nref, d_ref_off64, (int)(n_pep + 1), st); }));
    uint64_t n_res = 0, n_ref = 0;
    CUDA_TRY(cudaMemcpyAsync(&n_res, d_res_off64 + n_pep, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&n_ref, d_ref_off64 + n_pep, 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (n_res > 0xFFFFFFFFull || n_ref >= 0x7FFFFFFFull)
        return fail(SAGE_B200_ELIMIT, "prefilter: %llu residues / %llu protein references in the table (u32 offsets)", (unsigned long long)n_res,
                    (unsigned long long)n_ref);
    if (int rc = dg_memory("prefilter output", 5ull * n_res + 30ull * n_pep + 8ull * n_ref)) return rc;
    DevArena& O = D->out;
    uint32_t* d_ids_raw = nullptr;
    CUDA_TRY(O.alloc(&D->d_res_off, n_pep + 1));
    CUDA_TRY(O.alloc(&D->d_ref_off, n_pep + 1));
    CUDA_TRY(O.alloc(&D->d_ids, n_ref));
    CUDA_TRY(O.alloc(&D->d_seq, n_res));
    CUDA_TRY(O.alloc(&D->d_mods, n_res));
    CUDA_TRY(O.alloc(&D->d_nterm, n_pep));
    CUDA_TRY(O.alloc(&D->d_cterm, n_pep));
    CUDA_TRY(O.alloc(&D->d_mono, n_pep));
    CUDA_TRY(O.alloc(&D->d_decoy, n_pep));
    CUDA_TRY(O.alloc(&D->d_missed, n_pep));
    CUDA_TRY(O.alloc(&D->d_semi, n_pep));
    CUDA_TRY(A.alloc(&d_ids_raw, n_ref));
    LAUNCH_N(k_dg_u64_to_u32, n_pep + 1, st, d_res_off64, n_pep + 1, D->d_res_off);
    LAUNCH_N(k_dg_u64_to_u32, n_pep + 1, st, d_ref_off64, n_pep + 1, D->d_ref_off);
    LAUNCH_N(k_pf_export, n_pep, st, rows, d_order, d_first, n_pep, D->d_res_off, D->d_ref_off, D->d_seq, D->d_mods, D->d_nterm, D->d_cterm, D->d_mono,
             D->d_decoy, D->d_missed, D->d_semi, d_ids_raw);
    // proteins.sort_unstable() (database.rs:250): ids are ranks in the whole FASTA's names table, so an ascending sort of the ids is the sort of
    // the names across chunks
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) {
        return cub::DeviceSegmentedSort::SortKeys(t, b, d_ids_raw, D->d_ids, (int)n_ref, (int)n_pep, D->d_ref_off, D->d_ref_off + 1, st);
    }));
    CUDA_TRY(cudaStreamSynchronize(st));
    *peak = std::max<uint64_t>(*peak, held + A.bytes + O.bytes);
    I.n_peptides = n_pep;
    I.n_residues = n_res;
    I.n_protein_refs = n_ref;
    return 0;
}

// The spectra runner.rs:252-268 passes to quick_score: masses.len() >= min_peaks && level == 2, gathered into `out`'s arrays.
struct PfSpectra {
    std::vector<uint64_t> off{0};
    std::vector<float> masses, intens, mz, iso_lo, iso_hi, tic;
    std::vector<uint8_t> charge;
    sage_b200_spectra s{};
};

static void pf_filter_spectra(const sage_b200_spectra* sp, uint64_t min_peaks, PfSpectra& F) {
    for (uint64_t i = 0; i < sp->n; i++) {
        const uint64_t a = sp->peak_offsets[i], b = sp->peak_offsets[i + 1];
        if (b - a < min_peaks || (sp->level && sp->level[i] != 2)) continue;
        F.masses.insert(F.masses.end(), sp->masses + a, sp->masses + b);
        F.intens.insert(F.intens.end(), sp->intensities + a, sp->intensities + b);
        F.off.push_back(F.masses.size());
        F.mz.push_back(sp->precursor_mz[i]);
        F.charge.push_back(sp->precursor_charge[i]);
        F.iso_lo.push_back(sp->isolation_lo ? sp->isolation_lo[i] : NAN);
        F.iso_hi.push_back(sp->isolation_hi ? sp->isolation_hi[i] : NAN);
        F.tic.push_back(sp->total_ion_current[i]);
    }
    F.s.n = F.mz.size();
    F.s.peak_offsets = F.off.data();
    F.s.masses = F.masses.data();
    F.s.intensities = F.intens.data();
    F.s.precursor_mz = F.mz.data();
    F.s.precursor_charge = F.charge.data();
    F.s.isolation_lo = F.iso_lo.data();
    F.s.isolation_hi = F.iso_hi.data();
    F.s.total_ion_current = F.tic.data();
}

static float ms_since(std::chrono::steady_clock::time_point t) { return std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t).count(); }

extern "C" int sage_b200_prefilter_create(int device, const char* fasta, uint64_t fasta_len, const sage_b200_digest_params* dp, const sage_b200_scorer_params* sp,
                                          const sage_b200_prefilter_params* pp, const sage_b200_spectra* spectra, uint64_t bucket_size, const uint8_t* ion_kinds,
                                          uint64_t n_ion_kinds, uint64_t min_ion_index, sage_b200_prefilter** out) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!out || !dp || !sp || !pp || !ion_kinds || (fasta_len && !fasta)) return fail(SAGE_B200_EINVAL, "prefilter_create: null argument");
    *out = nullptr;
    if (int rc = check_spectra(spectra)) return rc;
    DgSetup S;
    if (int rc = dg_setup(dp, S)) return rc;
    if (int rc = db_check_bucket_size(bucket_size)) return rc;
    if (n_ion_kinds == 0 || n_ion_kinds > MAX_KINDS) return fail(SAGE_B200_EINVAL, "ion_kinds: need 1..%d kinds", MAX_KINDS);
    for (uint64_t k = 0; k < n_ion_kinds; k++)
        if (ion_kinds[k] > 5) return fail(SAGE_B200_EINVAL, "ion kind %u out of range", ion_kinds[k]);
    if (sp->report_psms == 0) return fail(SAGE_B200_EINVAL, "report_psms must be >= 1");
    if (sp->report_psms + 1ull > (uint64_t)K_MAX / 2)
        return fail(SAGE_B200_ELIMIT, "prefilter: report_psms + 1 = %llu > %d not supported", sp->report_psms + 1ull, K_MAX / 2);
    if (sp->precursor_tol.kind < 0 || sp->precursor_tol.kind > 2 || sp->fragment_tol.kind < 0 || sp->fragment_tol.kind > 2)
        return fail(SAGE_B200_EINVAL, "bad tolerance kind");
    if (sp->score_type > 1) return fail(SAGE_B200_EINVAL, "bad score_type");
    Guard<sage_b200_prefilter> guard(new sage_b200_prefilter(), sage_b200_prefilter_destroy);
    sage_b200_prefilter* PF = guard.get();
    PF->device = device;
    PF->table.device = device;
    sage_b200_prefilter_info& I = PF->info;
    DgFasta F;
    if (int rc = dg_parse_fasta(fasta, fasta_len, dp->decoy_tag ? dp->decoy_tag : "rev_", dp->generate_decoys != 0, F)) return rc;
    std::vector<uint32_t> prot_name;
    dg_names(F, &PF->table, prot_name);
    const uint64_t targets = F.acc.size();
    I.n_proteins = targets;
    I.ms_parse = ms_since(t0);
    if (int rc = select_device(device)) return rc;

    // auto_calculate_prefilter_chunk_size (database.rs:142-160)
    uint64_t chunk = pp->chunk_size;
    if (chunk == 0) {
        const auto tc = std::chrono::steady_clock::now();
        uint64_t total = 0;
        if (targets) {
            sage_b200_digest counter;
            counter.device = device;
            if (int rc = dg_run(&counter, F, 0, (uint32_t)targets, S.hp, S.statics, S.vars, prot_name, &total)) return rc;
            I.peak_device_bytes = std::max<uint64_t>(I.peak_device_bytes, counter.info.peak_device_bytes);
        }
        I.unmodified_peptides = total;
        const uint64_t chunk_count = (S.n_var_specs + 1) * (1ull << S.hp.kmax) * total / (1ull << 23);
        chunk = chunk_count == 0 ? targets : targets / chunk_count;
        I.ms_count = ms_since(tc);
        if (chunk == 0 && targets)
            return fail(SAGE_B200_EINVAL, "prefilter: the automatic chunk size is 0 (%llu proteins, %llu estimated chunks): set a chunk size",
                        (unsigned long long)targets, (unsigned long long)chunk_count);
    }
    I.chunk_size = chunk;
    if (chunk >= targets) {   // runner.rs:110: the plain build, no quick_score
        I.plain_build = 1;
        const auto td = std::chrono::steady_clock::now();
        if (targets)
            if (int rc = dg_run(&PF->table, F, 0, (uint32_t)targets, S.hp, S.statics, S.vars, prot_name)) return rc;
        I.ms_digest = ms_since(td);
        I.rows_digested = I.rows_kept = PF->table.info.n_peptides;
        I.peak_device_bytes = std::max<uint64_t>(I.peak_device_bytes, PF->table.info.peak_device_bytes);
    } else {
        I.n_chunks = (targets + chunk - 1) / chunk;
        PfSpectra Q;
        pf_filter_spectra(spectra, pp->min_peaks, Q);
        I.n_spectra = Q.s.n;
        sage_b200_scorer_params qp = *sp;
        qp.report_psms = sp->report_psms + 1;   // runner.rs:191
        PfTable T;
        Stream st;
        CUDA_TRY(st.create());
        for (uint64_t c = 0; c < I.n_chunks; c++) {
            const uint32_t p0 = (uint32_t)(c * chunk), p1 = (uint32_t)std::min<uint64_t>(targets, (c + 1) * chunk);
            auto t = std::chrono::steady_clock::now();
            sage_b200_digest D;
            D.device = device;
            if (int rc = dg_run(&D, F, p0, p1, S.hp, S.statics, S.vars, prot_name)) return rc;
            I.ms_digest += ms_since(t);
            I.peak_device_bytes = std::max<uint64_t>(I.peak_device_bytes, T.bytes() + D.info.peak_device_bytes);
            const DevTable C = dg_table(D);
            PF->chunk_rows.push_back(C.n);
            PF->chunk_kept.push_back(0);
            I.rows_digested += C.n;
            if (C.n == 0) continue;
            t = std::chrono::steady_clock::now();
            sage_b200_db* cdb = nullptr;
            if (int rc = db_build_device(C, bucket_size, ion_kinds, n_ion_kinds, min_ion_index, device, &cdb)) return rc;
            Guard<sage_b200_db> cdb_guard(cdb, sage_b200_db_destroy);
            I.ms_index += ms_since(t);
            const uint64_t held = T.bytes() + D.out.bytes + cdb->mem.bytes;
            I.peak_device_bytes = std::max<uint64_t>(I.peak_device_bytes, held);
            t = std::chrono::steady_clock::now();
            sage_b200_scorer* sc = nullptr;
            if (int rc = sage_b200_scorer_create(cdb, &qp, &sc)) return rc;
            Guard<sage_b200_scorer> sc_guard(sc, sage_b200_scorer_destroy);
            {
                std::lock_guard<std::mutex> lock(sc->mu);
                if (int rc = quick_score_device(sc, &Q.s, pp->low_memory)) return rc;
            }
            I.ms_quick_score += ms_since(t);
            I.ms_spectra_upload += sc->last.ms_h2d;
            t = std::chrono::steady_clock::now();
            uint64_t kept = 0;
            if (int rc = pf_compact(C, sc->d_keep.as<uint8_t>(), T, st, &kept, &I.peak_device_bytes, D.out.bytes + cdb->mem.bytes)) return rc;
            I.ms_compact += ms_since(t);
            PF->chunk_kept.back() = kept;
            I.rows_kept += kept;
        }   // the chunk's digest, index and scorer are freed here
        const auto tm = std::chrono::steady_clock::now();
        if (int rc = pf_merge(T, &PF->table, st, &I.peak_device_bytes, T.bytes())) return rc;
        I.ms_merge = ms_since(tm);
    }
    const auto tf = std::chrono::steady_clock::now();
    if (int rc = db_build_device(dg_table(PF->table), bucket_size, ion_kinds, n_ion_kinds, min_ion_index, device, &PF->db)) return rc;
    I.ms_final_index = ms_since(tf);
    const sage_b200_digest_info& O = PF->table.info;
    I.n_peptides = O.n_peptides;
    I.n_residues = O.n_residues;
    I.n_protein_refs = O.n_protein_refs;
    I.n_names = O.n_names;
    I.name_bytes = O.name_bytes;
    I.n_fragments = PF->db->v.n_frag;
    I.device_bytes = PF->table.out.bytes + PF->db->mem.bytes;
    I.peak_device_bytes = std::max<uint64_t>(I.peak_device_bytes, I.device_bytes);
    I.ms_wall = ms_since(t0);
    *out = guard.release();
    return 0;
}

extern "C" int sage_b200_prefilter_get_info(const sage_b200_prefilter* f, sage_b200_prefilter_info* info) {
    if (!f || !info) return fail(SAGE_B200_EINVAL, "prefilter_get_info: null argument");
    *info = f->info;
    return 0;
}

extern "C" int sage_b200_prefilter_chunk_counts(const sage_b200_prefilter* f, uint64_t* rows_digested, uint64_t* rows_kept) {
    if (!f) return fail(SAGE_B200_EINVAL, "prefilter_chunk_counts: null handle");
    if (rows_digested && !f->chunk_rows.empty()) memcpy(rows_digested, f->chunk_rows.data(), 8 * f->chunk_rows.size());
    if (rows_kept && !f->chunk_kept.empty()) memcpy(rows_kept, f->chunk_kept.data(), 8 * f->chunk_kept.size());
    return 0;
}

extern "C" int sage_b200_prefilter_export(const sage_b200_prefilter* f, uint32_t* residue_offsets, uint8_t* sequence, float* modifications, float* nterm,
                                          float* cterm, float* monoisotopic, uint8_t* decoy, uint8_t* missed_cleavages, uint8_t* semi_enzymatic,
                                          uint32_t* protein_offsets, uint32_t* protein_ids, uint64_t* name_offsets, char* name_bytes) {
    if (!f) return fail(SAGE_B200_EINVAL, "prefilter_export: null handle");
    return sage_b200_digest_export(&f->table, residue_offsets, sequence, modifications, nterm, cterm, monoisotopic, decoy, missed_cleavages, semi_enzymatic,
                                   protein_offsets, protein_ids, name_offsets, name_bytes);
}

extern "C" int sage_b200_prefilter_take_db(sage_b200_prefilter* f, sage_b200_db** out) {
    if (!f || !out) return fail(SAGE_B200_EINVAL, "prefilter_take_db: null argument");
    if (!f->db) return fail(SAGE_B200_EINVAL, "prefilter_take_db: the db was already taken");
    *out = f->db;
    f->db = nullptr;
    return 0;
}

// ------------------------------------------------------------------------------------------------ result files (DESIGN.md §17)
static constexpr uint64_t WRITE_CUT = 4096;                  // records per block: chunks are cut at block boundaries
static constexpr uint64_t WRITE_BUDGET = 256ull << 20;      // default device text per chunk

static int write_check_strings(const char* what, const uint64_t* off, const char* bytes, uint64_t n) {
    if (!off || (!bytes && off[n] > off[0])) return fail(SAGE_B200_EINVAL, "write_tsv: null %s table", what);
    for (uint64_t i = 0; i < n; i++)
        if (off[i + 1] < off[i]) return fail(SAGE_B200_EINVAL, "write_tsv: %s offsets decrease at %llu", what, (unsigned long long)i);
    return 0;
}
template <class T>
static int write_check_ids(const char* what, const T* ids, uint64_t n, uint64_t bound, const char* of) {
    for (uint64_t i = 0; i < n; i++)
        if ((uint64_t)ids[i] >= bound)
            return fail(SAGE_B200_EINVAL, "write_tsv: %s %llu is %llu, %llu %s", what, (unsigned long long)i, (unsigned long long)ids[i], (unsigned long long)bound, of);
    return 0;
}

// The peptide table and its protein names (results, pin, lfq).
static int write_check_peptides(const sage_b200_write_inputs* in) {
    const sage_b200_peptides* P = in->peptides;
    if (!P || !P->residue_offsets || !P->nterm || !P->decoy || !in->protein_offsets || (P->n_peptides && (!P->sequence || !P->modifications)))
        return fail(SAGE_B200_EINVAL, "write_tsv: null peptide table");
    if (P->n_peptides > (uint64_t)UINT32_MAX) return fail(SAGE_B200_ELIMIT, "write_tsv: more than 2^32 - 1 peptides");
    for (uint64_t p = 0; p < P->n_peptides; p++)
        if (P->residue_offsets[p + 1] < P->residue_offsets[p] || in->protein_offsets[p + 1] < in->protein_offsets[p])
            return fail(SAGE_B200_EINVAL, "write_tsv: peptide offsets decrease at %llu", (unsigned long long)p);
    const uint64_t n_refs = in->protein_offsets[P->n_peptides] - in->protein_offsets[0];
    if (in->protein_offsets[0] != 0 || (n_refs && !in->protein_ids)) return fail(SAGE_B200_EINVAL, "write_tsv: bad protein lists");
    if (int rc = write_check_strings("protein name", in->name_offsets, in->name_bytes, in->n_names)) return rc;
    return write_check_ids("protein id", in->protein_ids, n_refs, in->n_names, "names");
}

// Argument checks of one file (no device); n_rec = its records, h2d = the bytes its inputs take on the device.
static int write_check(int file, const sage_b200_write_inputs* in, uint64_t& n_rec, uint64_t& h2d) {
    const uint64_t n = in->n_rows;
    const bool by_row = file == SAGE_B200_FILE_RESULTS || file == SAGE_B200_FILE_PIN || file == SAGE_B200_FILE_FRAGMENTS;
    if (by_row && n && (!in->rows || !in->psm_id)) return fail(SAGE_B200_EINVAL, "write_tsv: null rows or psm_id");
    if (n > (uint64_t)UINT32_MAX) return fail(SAGE_B200_ELIMIT, "write_tsv: more than 2^32 - 1 rows");
    if (file != SAGE_B200_FILE_FRAGMENTS) {
        if (int rc = write_check_strings("filename", in->filename_offsets, in->filename_bytes, in->n_files)) return rc;
        h2d += 8 * (in->n_files + 1) + in->filename_offsets[in->n_files] - in->filename_offsets[0];
    }
    if (file == SAGE_B200_FILE_RESULTS || file == SAGE_B200_FILE_PIN || file == SAGE_B200_FILE_TMT) {
        if (int rc = write_check_strings("spectrum id", in->spec_id_offsets, in->spec_id_bytes, in->n_spec_ids)) return rc;
        h2d += 8 * (in->n_spec_ids + 1) + in->spec_id_offsets[in->n_spec_ids] - in->spec_id_offsets[0];
    }
    if (file == SAGE_B200_FILE_RESULTS || file == SAGE_B200_FILE_PIN || file == SAGE_B200_FILE_LFQ) {
        if (int rc = write_check_peptides(in)) return rc;
        const sage_b200_peptides* P = in->peptides;
        h2d += P->n_peptides * 16 + (uint64_t)P->residue_offsets[P->n_peptides] * 5 + 4 * (uint64_t)in->protein_offsets[P->n_peptides] +
               8 * (in->n_names + 1) + in->name_offsets[in->n_names] - in->name_offsets[0];
    }
    if (file == SAGE_B200_FILE_FRAGMENTS) {
        if (in->n_fragments && !in->fragments) return fail(SAGE_B200_EINVAL, "write_tsv: null fragments");
        n_rec = 0;
        for (uint64_t i = 0; i < n; i++) {
            const sage_b200_feature& r = in->rows[i];
            if ((uint64_t)r.fragment_offset + r.fragment_count > in->n_fragments)
                return fail(SAGE_B200_EINVAL, "write_tsv: row %llu's fragments [%u, +%u) lie outside the %llu fragments", (unsigned long long)i, r.fragment_offset,
                            r.fragment_count, (unsigned long long)in->n_fragments);
            n_rec += r.fragment_count;
        }
        for (uint64_t k = 0; k < in->n_fragments; k++)
            if ((uint32_t)in->fragments[k].kind > 5) return fail(SAGE_B200_EINVAL, "write_tsv: fragment %llu has kind %d outside 0..5", (unsigned long long)k, in->fragments[k].kind);
        h2d += n * (sizeof(sage_b200_feature) + 8) + in->n_fragments * sizeof(sage_b200_fragment);
    } else if (file == SAGE_B200_FILE_TMT) {
        n_rec = in->n_quant;
        if (n_rec && (!in->quant_file_id || !in->quant_spec_id || !in->ion_injection_time || (in->n_channels && !in->peaks)))
            return fail(SAGE_B200_EINVAL, "write_tsv: null TMT input");
        if (in->n_channels > (uint64_t)UINT32_MAX / 64) return fail(SAGE_B200_ELIMIT, "write_tsv: %llu channels", (unsigned long long)in->n_channels);
        if (int rc = write_check_ids("record", in->quant_file_id, n_rec, in->n_files, "files")) return rc;
        if (int rc = write_check_ids("record", in->quant_spec_id, n_rec, in->n_spec_ids, "spectrum ids")) return rc;
        h2d += n_rec * (12 + 4 * in->n_channels);
    } else if (file == SAGE_B200_FILE_LFQ) {
        n_rec = in->n_lfq;
        if (n_rec && (!in->lfq_rows || !in->lfq_q || (in->n_files && !in->lfq_areas))) return fail(SAGE_B200_EINVAL, "write_tsv: null LFQ input");
        for (uint64_t i = 0; i < n_rec; i++)
            if (in->lfq_rows[i].peptide >= in->peptides->n_peptides)
                return fail(SAGE_B200_EINVAL, "write_tsv: LFQ row %llu has peptide %u outside the table (%llu peptides)", (unsigned long long)i,
                            in->lfq_rows[i].peptide, (unsigned long long)in->peptides->n_peptides);
        h2d += n_rec * (sizeof(sage_b200_lfq_row) + 4 + 8 * in->n_files);
    } else {   // results, pin
        n_rec = n;
        if (n && (!in->file_id || !in->spec_index)) return fail(SAGE_B200_EINVAL, "write_tsv: null file_id or spec_index");
        for (uint64_t i = 0; i < n; i++)
            if (in->rows[i].peptide_idx >= in->peptides->n_peptides)
                return fail(SAGE_B200_EINVAL, "write_tsv: row %llu has peptide_idx %u outside the table (%llu peptides)", (unsigned long long)i,
                            in->rows[i].peptide_idx, (unsigned long long)in->peptides->n_peptides);
        if (int rc = write_check_ids("row", in->file_id, n, in->n_files, "files")) return rc;
        if (int rc = write_check_ids("row", in->spec_index, n, in->n_spec_ids, "spectrum ids")) return rc;
        h2d += n * (sizeof(sage_b200_feature) + 8 + 8 + 4 * 12 + 1);
        if (file == SAGE_B200_FILE_RESULTS && in->group_pass) {
            if (!in->row_group_offsets || !in->group_offsets || !in->group_decoy || (n && in->row_group_offsets[n] > in->row_group_offsets[0] && !in->row_groups))
                return fail(SAGE_B200_EINVAL, "write_tsv: null protein group table");
            for (uint64_t i = 0; i < n; i++)
                if (in->row_group_offsets[i + 1] < in->row_group_offsets[i]) return fail(SAGE_B200_EINVAL, "write_tsv: row group offsets decrease at %llu", (unsigned long long)i);
            for (uint64_t g = 0; g < in->n_groups; g++)
                if (in->group_offsets[g + 1] < in->group_offsets[g]) return fail(SAGE_B200_EINVAL, "write_tsv: group offsets decrease at %llu", (unsigned long long)g);
            const uint64_t rg0 = in->row_group_offsets[0], nrg = in->row_group_offsets[n] - rg0;
            const uint64_t gm0 = in->group_offsets[0], ngm = in->group_offsets[in->n_groups] - gm0;
            if (rg0 != 0 || gm0 != 0) return fail(SAGE_B200_EINVAL, "write_tsv: group offsets must start at 0");
            if (ngm && !in->group_members) return fail(SAGE_B200_EINVAL, "write_tsv: null group members");
            if (int rc = write_check_ids("row group", in->row_groups, nrg, in->n_groups, "groups")) return rc;
            if (int rc = write_check_ids("group member", in->group_members, ngm, in->n_names, "names")) return rc;
            h2d += 8 * (n + 1) + 4 * nrg + 9 * (in->n_groups + 1) + 4 * ngm;
        }
    }
    return 0;
}

// The header record, formatted on the host with the device's field rule.
static std::string write_header(int file, const sage_b200_write_inputs* in) {
    std::vector<std::string> f;
    if (file == SAGE_B200_FILE_RESULTS) {
        f = {"psm_id", "peptide", "proteins", "protein_groups", "num_proteins", "num_protein_groups", "filename", "scannr", "rank", "label", "expmass",
             "calcmass", "charge", "peptide_len", "missed_cleavages", "semi_enzymatic", "isotope_error", "precursor_ppm", "fragment_ppm", "hyperscore",
             "delta_next", "delta_best", "rt", "aligned_rt", "predicted_rt", "delta_rt_model", "ion_mobility", "predicted_mobility", "delta_mobility",
             "matched_peaks", "longest_b", "longest_y", "longest_y_pct", "matched_intensity_pct", "scored_candidates", "poisson",
             "sage_discriminant_score", "posterior_error", "spectrum_q", "peptide_q", "protein_q", "protein_group_q", "ms2_intensity"};
    } else if (file == SAGE_B200_FILE_PIN) {
        f = {"SpecId", "Label", "ScanNr", "ExpMass", "CalcMass", "FileName", "retentiontime", "ion_mobility", "rank", "z=2", "z=3", "z=4", "z=5", "z=6",
             "z=other", "peptide_len", "missed_cleavages", "semi_enzymatic", "isotope_error", "ln(precursor_ppm)", "fragment_ppm", "ln(hyperscore)",
             "ln(delta_next)", "ln(delta_best)", "aligned_rt", "predicted_rt", "sqrt(delta_rt_model)", "predicted_mobility", "sqrt(delta_mobility)",
             "matched_peaks", "longest_b", "longest_y", "longest_y_pct", "ln(matched_intensity_pct)", "scored_candidates", "ln(-poisson)",
             "posterior_error", "Peptide", "Proteins"};
    } else if (file == SAGE_B200_FILE_FRAGMENTS) {
        f = {"psm_id", "fragment_type", "fragment_ordinals", "fragment_charge", "fragment_mz_calculated", "fragment_mz_experimental", "fragment_intensity"};
    } else if (file == SAGE_B200_FILE_LFQ) {
        f = {"peptide", "charge", "proteins", "q_value", "score", "spectral_angle"};
        for (uint64_t k = 0; k < in->n_files; k++)
            f.emplace_back(in->filename_bytes + in->filename_offsets[k], in->filename_offsets[k + 1] - in->filename_offsets[k]);
    } else {
        f = {"filename", "scannr", "ion_injection_time"};
        for (uint64_t c = 0; c < in->n_channels; c++) f.push_back((in->user_labels ? "user_" : "tmt_") + std::to_string(c + 1));
    }
    std::string out;
    for (size_t i = 0; i < f.size(); i++) {
        if (i) out += '\t';
        wr::Out cnt{nullptr, 0};
        wr::put_field(cnt, f[i].data(), f[i].size());
        std::string s(cnt.n, '\0');
        wr::Out o{&s[0], 0};
        wr::put_field(o, f[i].data(), f[i].size());
        out += s;
    }
    return out + '\n';
}

template <int FILE>
static int write_launch_measure(const wr::WriteArgs& a, uint64_t n, uint64_t* len, cudaStream_t st) {
    LAUNCH_N(wr::k_write_measure<FILE>, n, st, a, n, len);
    return 0;
}
template <int FILE>
static int write_launch_text(const wr::WriteArgs& a, uint64_t j0, uint64_t j1, const uint64_t* off, char* text, cudaStream_t st) {
    LAUNCH_N(wr::k_write_text<FILE>, j1 - j0, st, a, j0, j1, off, text);
    return 0;
}
static int write_measure(int file, const wr::WriteArgs& a, uint64_t n, uint64_t* len, cudaStream_t st) {
    switch (file) {
        case SAGE_B200_FILE_RESULTS: return write_launch_measure<SAGE_B200_FILE_RESULTS>(a, n, len, st);
        case SAGE_B200_FILE_PIN: return write_launch_measure<SAGE_B200_FILE_PIN>(a, n, len, st);
        case SAGE_B200_FILE_FRAGMENTS: return write_launch_measure<SAGE_B200_FILE_FRAGMENTS>(a, n, len, st);
        case SAGE_B200_FILE_LFQ: return write_launch_measure<SAGE_B200_FILE_LFQ>(a, n, len, st);
        default: return write_launch_measure<SAGE_B200_FILE_TMT>(a, n, len, st);
    }
}
static int write_text(int file, const wr::WriteArgs& a, uint64_t j0, uint64_t j1, const uint64_t* off, char* text, cudaStream_t st) {
    switch (file) {
        case SAGE_B200_FILE_RESULTS: return write_launch_text<SAGE_B200_FILE_RESULTS>(a, j0, j1, off, text, st);
        case SAGE_B200_FILE_PIN: return write_launch_text<SAGE_B200_FILE_PIN>(a, j0, j1, off, text, st);
        case SAGE_B200_FILE_FRAGMENTS: return write_launch_text<SAGE_B200_FILE_FRAGMENTS>(a, j0, j1, off, text, st);
        case SAGE_B200_FILE_LFQ: return write_launch_text<SAGE_B200_FILE_LFQ>(a, j0, j1, off, text, st);
        default: return write_launch_text<SAGE_B200_FILE_TMT>(a, j0, j1, off, text, st);
    }
}

// A CSR string table on the device with its offsets rebased to 0.
static int write_upload_strings(DevArena& A, cudaStream_t st, const uint64_t* off, const char* bytes, uint64_t n, uint64_t** d_off, char** d_bytes,
                                std::vector<uint64_t>& keep) {
    keep.assign(off, off + n + 1);
    for (uint64_t& v : keep) v -= off[0];
    CUDA_TRY(A.upload(d_off, keep.data(), keep.size(), st));
    CUDA_TRY(A.upload(d_bytes, bytes + off[0], keep.back(), st));
    return 0;
}
// An optional per-row column: NULL stays NULL.
template <class T>
static cudaError_t write_upload_opt(DevArena& A, cudaStream_t st, T** d, const T* h, uint64_t n) {
    if (!h) return cudaSuccess;
    return A.upload(d, h, n, st);
}

extern "C" int sage_b200_write_tsv(int device, int file, const sage_b200_write_inputs* in, char* out, uint64_t capacity, uint64_t* bytes) {
    const auto t_wall = std::chrono::steady_clock::now();
    if (!in || !bytes) return fail(SAGE_B200_EINVAL, "write_tsv: null argument");
    if (file < SAGE_B200_FILE_RESULTS || file > SAGE_B200_FILE_TMT) return fail(SAGE_B200_EINVAL, "write_tsv: unknown file %d", file);
    uint64_t n_rec = 0, h2d = 0;
    if (int rc = write_check(file, in, n_rec, h2d)) return rc;
    if (n_rec > (uint64_t)UINT32_MAX) return fail(SAGE_B200_ELIMIT, "write_tsv: %llu records, more than 2^32 - 1", (unsigned long long)n_rec);
    const std::string header = write_header(file, in);
    sage_b200_write_stats stats{};
    stats.records = n_rec;
    auto finish = [&](uint64_t total) {
        *bytes = total;
        stats.ms_total = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_wall).count();
        if (in->stats) *in->stats = stats;
        return 0;
    };
    if (n_rec == 0) {
        if (out && capacity < header.size()) {
            *bytes = header.size();
            return fail(SAGE_B200_ELIMIT, "write_tsv: the file is %zu bytes, capacity %llu", header.size(), (unsigned long long)capacity);
        }
        if (out) memcpy(out, header.data(), header.size());
        return finish(header.size());
    }

    if (int rc = select_device(device)) return rc;
    const uint64_t budget = in->text_budget ? in->text_budget : WRITE_BUDGET;
    const uint64_t n_cut = (n_rec + WRITE_CUT - 1) / WRITE_CUT;
    {   // inputs; the fragment file's per-row counts and their scan (16 B per row); lengths and offsets (16 B per record); the cut table; the
        // scan's storage. The text buffer is checked again once its size is known.
        size_t free_b = 0, total_b = 0;
        CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
        const uint64_t row_scan = file == SAGE_B200_FILE_FRAGMENTS ? 16 * in->n_rows : 0;
        const uint64_t need = h2d + row_scan + 16 * (n_rec + 1) + 8 * (n_cut + 1) + (32ull << 20);
        if (need > free_b) return fail(SAGE_B200_ELIMIT, "write_tsv: %llu records need about %llu bytes of device memory, %llu free", (unsigned long long)n_rec,
                                       (unsigned long long)need, (unsigned long long)free_b);
    }
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    Event e0, e1, e2, e3;
    CUDA_TRY(e0.create());
    CUDA_TRY(e1.create());
    CUDA_TRY(e2.create());
    CUDA_TRY(e3.create());
    CUDA_TRY(cudaEventRecord(e0, st));
    wr::WriteArgs a{};
    std::vector<uint64_t> foff, soff, noff;   // rebased offsets: alive until the copies that read them are done
    const uint64_t n = in->n_rows;
    if (file != SAGE_B200_FILE_FRAGMENTS)
        if (int rc = write_upload_strings(A, st, in->filename_offsets, in->filename_bytes, in->n_files, &a.file_off, &a.file_bytes, foff)) return rc;
    if (file == SAGE_B200_FILE_RESULTS || file == SAGE_B200_FILE_PIN || file == SAGE_B200_FILE_TMT)
        if (int rc = write_upload_strings(A, st, in->spec_id_offsets, in->spec_id_bytes, in->n_spec_ids, &a.spec_off, &a.spec_bytes, soff)) return rc;
    if (file == SAGE_B200_FILE_RESULTS || file == SAGE_B200_FILE_PIN || file == SAGE_B200_FILE_LFQ) {
        const sage_b200_peptides* P = in->peptides;
        const uint64_t np = P->n_peptides, nres = P->residue_offsets[np], nref = in->protein_offsets[np];
        CUDA_TRY(A.upload(&a.res_off, P->residue_offsets, np + 1, st));
        CUDA_TRY(A.upload(&a.seq, (const char*)P->sequence, nres, st));
        CUDA_TRY(A.upload(&a.mods, P->modifications, nres, st));
        CUDA_TRY(A.upload(&a.nterm, P->nterm, np, st));
        CUDA_TRY(A.upload(&a.decoy, P->decoy, np, st));
        CUDA_TRY(write_upload_opt(A, st, &a.cterm, in->cterm, np));
        CUDA_TRY(write_upload_opt(A, st, &a.semi, in->semi_enzymatic, np));
        CUDA_TRY(A.upload(&a.prot_off, in->protein_offsets, np + 1, st));
        CUDA_TRY(A.upload(&a.prot_ids, in->protein_ids, nref, st));
        if (int rc = write_upload_strings(A, st, in->name_offsets, in->name_bytes, in->n_names, &a.name_off, &a.name_bytes, noff)) return rc;
        const char* tag = in->decoy_tag ? in->decoy_tag : "rev_";
        a.tag_len = (uint32_t)strlen(tag);
        CUDA_TRY(A.upload(&a.tag, tag, a.tag_len, st));
        a.generate_decoys = in->generate_decoys != 0;
    }
    if (file == SAGE_B200_FILE_RESULTS || file == SAGE_B200_FILE_PIN || file == SAGE_B200_FILE_FRAGMENTS) {
        CUDA_TRY(A.upload(&a.rows, in->rows, n, st));
        CUDA_TRY(A.upload(&a.psm_id, in->psm_id, n, st));
    }
    if (file == SAGE_B200_FILE_RESULTS || file == SAGE_B200_FILE_PIN) {
        CUDA_TRY(A.upload(&a.file_id, in->file_id, n, st));
        CUDA_TRY(A.upload(&a.spec_index, in->spec_index, n, st));
        CUDA_TRY(write_upload_opt(A, st, &a.discriminant, in->discriminant_score, n));
        CUDA_TRY(write_upload_opt(A, st, &a.posterior, in->posterior_error, n));
        CUDA_TRY(write_upload_opt(A, st, &a.spectrum_q, in->spectrum_q, n));
        CUDA_TRY(write_upload_opt(A, st, &a.peptide_q, in->peptide_q, n));
        CUDA_TRY(write_upload_opt(A, st, &a.protein_q, in->protein_q, n));
        CUDA_TRY(write_upload_opt(A, st, &a.aligned_rt, in->aligned_rt, n));
        CUDA_TRY(write_upload_opt(A, st, &a.predicted_rt, in->predicted_rt, n));
        CUDA_TRY(write_upload_opt(A, st, &a.delta_rt, in->delta_rt_model, n));
        CUDA_TRY(write_upload_opt(A, st, &a.predicted_ims, in->predicted_ims, n));
        CUDA_TRY(write_upload_opt(A, st, &a.delta_ims, in->delta_ims_model, n));
        a.fma = host_math_variant() != 1;
    }
    if (file == SAGE_B200_FILE_RESULTS) {
        CUDA_TRY(write_upload_opt(A, st, &a.num_groups, in->num_protein_groups, n));
        CUDA_TRY(write_upload_opt(A, st, &a.protein_group_q, in->protein_group_q, n));
        if (in->group_pass) {
            CUDA_TRY(A.upload(&a.group_pass, in->group_pass, n, st));
            CUDA_TRY(A.upload(&a.row_group_off, in->row_group_offsets, n + 1, st));
            CUDA_TRY(A.upload(&a.row_groups, in->row_groups, in->row_group_offsets[n], st));
            CUDA_TRY(A.upload(&a.group_off, in->group_offsets, in->n_groups + 1, st));
            CUDA_TRY(A.upload(&a.group_members, in->group_members, in->group_offsets[in->n_groups], st));
            CUDA_TRY(A.upload(&a.group_decoy, in->group_decoy, in->n_groups, st));
        }
    }
    if (file == SAGE_B200_FILE_FRAGMENTS) {
        uint64_t *counts = nullptr, *row_end = nullptr;
        CUDA_TRY(A.upload(&a.fragments, in->fragments, in->n_fragments, st));
        CUDA_TRY(A.alloc(&counts, n));
        CUDA_TRY(A.alloc(&row_end, n));
        LAUNCH_N(wr::k_write_fragment_counts, n, st, a.rows, n, counts);
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, counts, row_end, n, st); }));
        a.row_end = row_end;
        a.n_rows = (uint32_t)n;
    }
    if (file == SAGE_B200_FILE_TMT) {
        CUDA_TRY(A.upload(&a.quant_file, in->quant_file_id, n_rec, st));
        CUDA_TRY(A.upload(&a.quant_spec, in->quant_spec_id, n_rec, st));
        CUDA_TRY(A.upload(&a.injection, in->ion_injection_time, n_rec, st));
        CUDA_TRY(A.upload(&a.peaks, in->peaks, n_rec * in->n_channels, st));
        a.n_channels = (uint32_t)in->n_channels;
    }
    if (file == SAGE_B200_FILE_LFQ) {
        CUDA_TRY(A.upload(&a.lfq, in->lfq_rows, n_rec, st));
        CUDA_TRY(A.upload(&a.lfq_q, in->lfq_q, n_rec, st));
        CUDA_TRY(A.upload(&a.lfq_areas, in->lfq_areas, n_rec * in->n_files, st));
        a.n_files = (uint32_t)in->n_files;
    }
    CUDA_TRY(cudaEventRecord(e1, st));
    uint64_t *len = nullptr, *off = nullptr, *d_cuts = nullptr;
    CUDA_TRY(A.alloc(&len, n_rec));
    CUDA_TRY(A.alloc(&off, n_rec + 1));
    CUDA_TRY(A.alloc(&d_cuts, n_cut + 1));
    if (int rc = write_measure(file, a, n_rec, len, st)) return rc;
    CUDA_TRY(cudaEventRecord(e2, st));
    CUDA_TRY(cudaMemsetAsync(off, 0, 8, st));
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, len, off + 1, n_rec, st); }));
    LAUNCH_N(wr::k_write_cuts, n_cut, st, off, n_rec, WRITE_CUT, n_cut, d_cuts);
    std::vector<uint64_t> cuts(n_cut + 1);
    CUDA_TRY(cudaMemcpyAsync(cuts.data(), d_cuts, 8 * (n_cut + 1), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaEventRecord(e3, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaEventElapsedTime(&stats.ms_upload, e0, e1));
    CUDA_TRY(cudaEventElapsedTime(&stats.ms_measure, e1, e2));
    CUDA_TRY(cudaEventElapsedTime(&stats.ms_scan, e2, e3));
    stats.h2d_bytes = h2d;
    stats.d2h_bytes = 8 * (n_cut + 1);
    const uint64_t text = cuts[n_cut], total = header.size() + text;
    if (!out) return finish(total);
    if (capacity < total) {
        *bytes = total;
        return fail(SAGE_B200_ELIMIT, "write_tsv: the file is %llu bytes, capacity %llu", (unsigned long long)total, (unsigned long long)capacity);
    }

    // chunks: consecutive blocks of WRITE_CUT records while their text fits the budget (a larger block is a chunk of its own)
    std::vector<uint64_t> chunk_at{0};   // block indices
    for (uint64_t b = 1; b <= n_cut; b++)
        if (b == n_cut || cuts[b + 1] - cuts[chunk_at.back()] > budget) chunk_at.push_back(b);
    uint64_t text_cap = 0;
    for (size_t c = 0; c + 1 < chunk_at.size(); c++) text_cap = std::max(text_cap, cuts[chunk_at[c + 1]] - cuts[chunk_at[c]]);
    {
        size_t free_b = 0, total_b = 0;
        CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
        if (text_cap + (16ull << 20) > free_b)
            return fail(SAGE_B200_ELIMIT, "write_tsv: a chunk of %llu bytes of text does not fit the %llu bytes of free device memory", (unsigned long long)text_cap,
                        (unsigned long long)free_b);
    }
    char* d_text = nullptr;
    CUDA_TRY(A.alloc(&d_text, text_cap));
    memcpy(out, header.data(), header.size());
    for (size_t c = 0; c + 1 < chunk_at.size(); c++) {
        const uint64_t j0 = chunk_at[c] * WRITE_CUT, j1 = std::min(n_rec, chunk_at[c + 1] * WRITE_CUT);
        const uint64_t t0 = cuts[chunk_at[c]], t1 = cuts[chunk_at[c + 1]];
        CUDA_TRY(cudaEventRecord(e0, st));
        if (int rc = write_text(file, a, j0, j1, off, d_text, st)) return rc;
        CUDA_TRY(cudaEventRecord(e1, st));
        CUDA_TRY(cudaMemcpyAsync(out + header.size() + t0, d_text, t1 - t0, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaEventRecord(e2, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        float ms_w = 0, ms_c = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms_w, e0, e1));
        CUDA_TRY(cudaEventElapsedTime(&ms_c, e1, e2));
        stats.ms_write += ms_w;
        stats.ms_d2h += ms_c;
        stats.d2h_bytes += t1 - t0;
        stats.chunks++;
    }
    return finish(total);
}

extern "C" int sage_b200_format_hashes(int device, int format, uint64_t first, const double* values, uint64_t n, uint64_t block, uint64_t* hashes) {
    if (format < 0 || format > 2 || !hashes || block == 0 || n % block || (format == 2 && n && !values))
        return fail(SAGE_B200_EINVAL, "format_hashes: bad argument");
    if (format < 2 && first + n > (1ull << 32)) return fail(SAGE_B200_EINVAL, "format_hashes: f32 bit patterns beyond 2^32");
    const uint64_t nb = n / block;
    if (nb == 0) return 0;
    if (int rc = select_device(device)) return rc;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    double* d_v = nullptr;
    uint64_t* d_h = nullptr;
    if (format == 2) CUDA_TRY(A.upload(&d_v, values, n, st));
    CUDA_TRY(A.alloc(&d_h, nb));
    LAUNCH(wr::k_format_hashes<<<(unsigned)((nb + 7) / 8), 256, 0, st>>>(format, first, d_v, block, nb, d_h));
    return read_back(st, hashes, d_h, 8 * nb);
}

// ================================================================================== MGF reader (mgf.rs:324-370; kernels in mgf.cuh)
struct sage_b200_mgf {
    int device = 0;
    DevArena out;   // the spectra, exact-size; the text and the line table go with the create call
    uint64_t *d_peak_off = nullptr, *d_prec_off = nullptr, *d_id_off = nullptr;
    float *d_mz = nullptr, *d_int = nullptr, *d_rt = nullptr, *d_tic = nullptr;
    float *d_p_mz = nullptr, *d_p_int = nullptr, *d_p_lo = nullptr, *d_p_hi = nullptr;
    uint8_t *d_p_int_some = nullptr, *d_p_charge = nullptr, *d_p_charge_some = nullptr, *d_p_iso = nullptr, *d_id = nullptr;
    sage_b200_mgf_info info{};
};

extern "C" void sage_b200_mgf_destroy(sage_b200_mgf* m) {
    if (!m) return;
    cudaSetDevice(m->device);
    delete m;
}

static constexpr uint64_t MGF_SELECT_CHUNK = 1ull << 30;   // items per cub::DeviceSelect call (its item count is an int)

static int mgf_memory(const char* stage, uint64_t bytes) {
    size_t free_b = 0, total_b = 0;
    CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
    if (bytes + (64ull << 20) > free_b)
        return fail(SAGE_B200_ELIMIT, "mgf_create: the %s stage needs about %llu bytes of device memory, %llu free", stage, (unsigned long long)bytes,
                    (unsigned long long)free_b);
    return 0;
}

static unsigned mgf_grid(uint64_t n) { return (unsigned)std::min<uint64_t>(std::max<uint64_t>(grid256(n), 1), 1u << 20); }

struct MgfIsNewline {
    const uint8_t* t;
    __device__ bool operator()(uint64_t i) const { return t[i] == '\n'; }
};
struct MgfIsEnd {
    const MgfLine* L;
    __device__ bool operator()(uint64_t i) const { return L[i].kind == MGF_END; }
};

// The indices i in [base, base + n) with pred(i), in order, into out (expect of them).
template <class Pred>
static int mgf_select(DevArena& A, cudaStream_t st, uint64_t base, uint64_t n, Pred pred, uint64_t* out, uint64_t expect) {
    unsigned long long* d_cnt = nullptr;
    CUDA_TRY(A.alloc(&d_cnt, 1));
    uint64_t done = 0;
    for (uint64_t c0 = 0; c0 < n; c0 += MGF_SELECT_CHUNK) {
        const int m = (int)std::min<uint64_t>(MGF_SELECT_CHUNK, n - c0);
        thrust::counting_iterator<uint64_t> it(base + c0);
        CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceSelect::If(t, b, it, out + done, d_cnt, m, pred, st); }));
        unsigned long long got = 0;
        if (int rc = read_back(st, &got, d_cnt, 8)) return rc;
        done += got;
    }
    if (done != expect) return fail(SAGE_B200_ECUDA, "mgf_create: selected %llu items, counted %llu", (unsigned long long)done, (unsigned long long)expect);
    return 0;
}

static int mgf_scan(DevArena& A, cudaStream_t st, const uint64_t* in, uint64_t* out, uint64_t n) {
    CUDA_TRY(A.two_phase([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, in, out, (int)n, st); }));
    return 0;
}

extern "C" int sage_b200_mgf_create(int device, const char* text, uint64_t len, uint64_t file_id, sage_b200_mgf** out) {
    if (!out || (len && !text)) return fail(SAGE_B200_EINVAL, "mgf_create: null argument");
    *out = nullptr;
    if (len == 0) return fail(SAGE_B200_EINVAL, "mgf_create: no BEGIN IONS line (the file is empty)");
    if (int rc = select_device(device)) return rc;
    cudaGetLastError();   // a stale non-sticky error left by another user of the runtime must not be blamed on the launches below
    Guard<sage_b200_mgf> guard(new sage_b200_mgf(), sage_b200_mgf_destroy);
    sage_b200_mgf* M = guard.get();
    M->device = device;
    sage_b200_mgf_info& I = M->info;
    I.n_bytes = len;
    I.file_id = file_id;
    if (int rc = mgf_memory("text", len + 64)) return rc;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    Event e0, e1, e2;
    CUDA_TRY(e0.create());
    CUDA_TRY(e1.create());
    CUDA_TRY(e2.create());
    uint8_t* d_text = nullptr;
    MgfHeader* d_h = nullptr;
    MgfHeader h{~0ull, 0, 0, 0, 0, 0, ~0ull, 0};
    CUDA_TRY(A.upload(&d_h, &h, 1, st));
    CUDA_TRY(cudaEventRecord(e0, st));
    CUDA_TRY(A.upload(&d_text, (const uint8_t*)text, len, st));
    CUDA_TRY(cudaEventRecord(e1, st));
    LAUNCH(k_mgf_bytes<<<mgf_grid(len), 256, 0, st>>>(d_text, len, d_h));
    if (int rc = read_back(st, &h, d_h, sizeof h)) return rc;
    if (h.bad_utf8 != ~0ull) return fail(SAGE_B200_EINVAL, "mgf_create: invalid UTF-8 at byte offset %llu", h.bad_utf8);
    // str::lines: a line per '\n', and one more for text after the last '\n'
    const uint64_t n_nl = h.n_newline;
    if (int rc = mgf_memory("line", n_nl * 8 + (n_nl + 1) * sizeof(MgfLine))) return rc;
    uint64_t* d_nl = nullptr;
    CUDA_TRY(A.alloc(&d_nl, n_nl));
    if (int rc = mgf_select(A, st, 0, len, MgfIsNewline{d_text}, d_nl, n_nl)) return rc;
    uint64_t last_nl = 0;
    if (n_nl) {
        if (int rc = read_back(st, &last_nl, d_nl + n_nl - 1, 8)) return rc;
    }
    const uint64_t n_lines = n_nl + ((n_nl == 0 || last_nl + 1 < len) ? 1 : 0);
    I.n_lines = n_lines;
    MgfLine* d_lines = nullptr;
    CUDA_TRY(A.alloc(&d_lines, n_lines));
    LAUNCH(k_mgf_lines<<<mgf_grid(n_lines), 256, 0, st>>>(d_text, len, d_nl, n_nl, n_lines, d_lines, d_h));
    LAUNCH(k_mgf_scan_lines<<<mgf_grid(n_lines), 256, 0, st>>>(d_lines, n_lines, d_h));
    if (int rc = read_back(st, &h, d_h, sizeof h)) return rc;
    if (h.begin_line == ~0ull) return fail(SAGE_B200_EINVAL, "mgf_create: no BEGIN IONS line (mgf.rs panics at lines.next().unwrap())");
    I.malformed_lines = h.malformed;
    const uint64_t n_rec = h.n_end;
    I.n_records = n_rec;
    if (n_rec > 0x7FFFFFF0ull) return fail(SAGE_B200_ELIMIT, "mgf_create: %llu records, more than 2^31 - 16", (unsigned long long)n_rec);
    uint64_t counts[4] = {0, 0, 0, 0};   // spectra, peaks, precursors, id bytes
    uint64_t* at[4] = {nullptr, nullptr, nullptr, nullptr};
    MgfOut o{};
    uint64_t* d_end = nullptr;
    if (n_rec) {
        if (int rc = mgf_memory("record", n_rec * 8 * 9)) return rc;
        CUDA_TRY(A.alloc(&d_end, n_rec));
        if (int rc = mgf_select(A, st, h.begin_line + 1, n_lines - h.begin_line - 1, MgfIsEnd{d_lines}, d_end, n_rec)) return rc;
        uint64_t* cnt[4];
        for (int k = 0; k < 4; k++) {
            CUDA_TRY(A.alloc(&cnt[k], n_rec + 1));
            CUDA_TRY(A.alloc(&at[k], n_rec + 1));
        }
        o.kept = cnt[0];
        o.n_peaks = cnt[1];
        o.n_prec = cnt[2];
        o.id_len = cnt[3];
        LAUNCH(k_mgf_records<0><<<mgf_grid(n_rec), 256, 0, st>>>(d_text, d_lines, d_end, n_rec, d_h, o));
        for (int k = 0; k < 4; k++) {
            if (int rc = mgf_scan(A, st, cnt[k], at[k], n_rec + 1)) return rc;
            CUDA_TRY(cudaMemcpyAsync(&counts[k], at[k] + n_rec, 8, cudaMemcpyDeviceToHost, st));
        }
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    const uint64_t n = counts[0], npk = counts[1], npr = counts[2], nid = counts[3];
    I.n_spectra = n;
    I.n_peaks = npk;
    I.n_precursors = npr;
    I.id_bytes = nid;
    I.dropped_records = n_rec - n;
    if (int rc = mgf_memory("output", (npk + 4) * 8 + npr * 24 + nid + (n + 1) * 32)) return rc;
    CUDA_TRY(M->out.alloc(&M->d_peak_off, n + 1));
    CUDA_TRY(M->out.alloc(&M->d_prec_off, n + 1));
    CUDA_TRY(M->out.alloc(&M->d_id_off, n + 1));
    CUDA_TRY(M->out.alloc(&M->d_mz, npk + 4));
    CUDA_TRY(M->out.alloc(&M->d_int, npk + 4));
    CUDA_TRY(M->out.alloc(&M->d_rt, n));
    CUDA_TRY(M->out.alloc(&M->d_tic, n));
    CUDA_TRY(M->out.alloc(&M->d_p_mz, npr));
    CUDA_TRY(M->out.alloc(&M->d_p_int, npr));
    CUDA_TRY(M->out.alloc(&M->d_p_lo, npr));
    CUDA_TRY(M->out.alloc(&M->d_p_hi, npr));
    CUDA_TRY(M->out.alloc(&M->d_p_int_some, npr));
    CUDA_TRY(M->out.alloc(&M->d_p_charge, npr));
    CUDA_TRY(M->out.alloc(&M->d_p_charge_some, npr));
    CUDA_TRY(M->out.alloc(&M->d_p_iso, npr));
    CUDA_TRY(M->out.alloc(&M->d_id, nid));
    const uint64_t last[3] = {npk, npr, nid};
    CUDA_TRY(cudaMemcpyAsync(M->d_peak_off + n, &last[0], 8, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(M->d_prec_off + n, &last[1], 8, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(M->d_id_off + n, &last[2], 8, cudaMemcpyHostToDevice, st));
    if (n) {
        o.kept = at[0];
        o.n_peaks = at[1];
        o.n_prec = at[2];
        o.id_len = at[3];
        o.peak_off = M->d_peak_off;
        o.prec_off = M->d_prec_off;
        o.id_off = M->d_id_off;
        o.mz = M->d_mz;
        o.intensity = M->d_int;
        o.rt = M->d_rt;
        o.tic = M->d_tic;
        o.p_mz = M->d_p_mz;
        o.p_int = M->d_p_int;
        o.p_lo = M->d_p_lo;
        o.p_hi = M->d_p_hi;
        o.p_int_some = M->d_p_int_some;
        o.p_charge = M->d_p_charge;
        o.p_charge_some = M->d_p_charge_some;
        o.p_iso = M->d_p_iso;
        o.id_bytes = M->d_id;
        LAUNCH(k_mgf_records<1><<<mgf_grid(n_rec), 256, 0, st>>>(d_text, d_lines, d_end, n_rec, d_h, o));
    }
    CUDA_TRY(cudaEventRecord(e2, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaEventElapsedTime(&I.ms_h2d, e0, e1));
    CUDA_TRY(cudaEventElapsedTime(&I.ms_read, e1, e2));
    I.device_bytes = M->out.bytes;
    I.peak_device_bytes = M->out.bytes + A.bytes;
    *out = guard.release();
    return 0;
}

extern "C" int sage_b200_mgf_get_info(const sage_b200_mgf* m, sage_b200_mgf_info* info) {
    if (!m || !info) return fail(SAGE_B200_EINVAL, "mgf_get_info: null argument");
    *info = m->info;
    return 0;
}

extern "C" int sage_b200_mgf_export(const sage_b200_mgf* M, uint64_t* peak_offsets, float* mz, float* intensity, float* scan_start_time, float* tic,
                                    uint64_t* precursor_offsets, float* precursor_mz, float* precursor_intensity, uint8_t* precursor_intensity_some,
                                    uint8_t* precursor_charge, uint8_t* precursor_charge_some, uint8_t* isolation_kind, float* isolation_lo,
                                    float* isolation_hi, uint64_t* id_offsets, char* id_bytes) {
    if (!M) return fail(SAGE_B200_EINVAL, "mgf_export: null handle");
    const sage_b200_mgf_info& I = M->info;
    const uint64_t n = I.n_spectra, npk = I.n_peaks, npr = I.n_precursors;
    CUDA_TRY(cudaSetDevice(M->device));
    Stream st;
    CUDA_TRY(st.create());
    struct Copy { void* dst; const void* src; uint64_t bytes; };
    const Copy copies[] = {{peak_offsets, M->d_peak_off, 8 * (n + 1)}, {mz, M->d_mz, 4 * npk}, {intensity, M->d_int, 4 * npk},
                           {scan_start_time, M->d_rt, 4 * n}, {tic, M->d_tic, 4 * n}, {precursor_offsets, M->d_prec_off, 8 * (n + 1)},
                           {precursor_mz, M->d_p_mz, 4 * npr}, {precursor_intensity, M->d_p_int, 4 * npr}, {precursor_intensity_some, M->d_p_int_some, npr},
                           {precursor_charge, M->d_p_charge, npr}, {precursor_charge_some, M->d_p_charge_some, npr}, {isolation_kind, M->d_p_iso, npr},
                           {isolation_lo, M->d_p_lo, 4 * npr}, {isolation_hi, M->d_p_hi, 4 * npr}, {id_offsets, M->d_id_off, 8 * (n + 1)},
                           {id_bytes, M->d_id, I.id_bytes}};
    for (const Copy& c : copies)
        if (c.dst && c.bytes) CUDA_TRY(cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int sage_b200_mgf_process(const sage_b200_mgf* M, const sage_b200_processor_params* pr, uint64_t* out_offsets, float* out_masses,
                                     float* out_intensities, float* out_tic) {
    if (!M || !pr || !out_offsets || !out_tic) return fail(SAGE_B200_EINVAL, "mgf_process: null argument");
    const uint64_t n = M->info.n_spectra, npk = M->info.n_peaks;
    if (npk && (!out_masses || !out_intensities)) return fail(SAGE_B200_EINVAL, "mgf_process: null peak arrays");
    out_offsets[0] = 0;
    if (n == 0) return 0;
    if (n > 0x7FFFFFFFull || npk > 0xFFFFFFF0ull) return fail(SAGE_B200_ELIMIT, "mgf_process: more than 2^31 - 1 spectra or 2^32 - 16 peaks");
    CUDA_TRY(cudaSetDevice(M->device));
    cudaGetLastError();
    if (int rc = mgf_memory("process", npk * 16 + n * 24)) return rc;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    uint32_t *d_off = nullptr, *d_cnt = nullptr;
    uint8_t* d_chg = nullptr;
    unsigned int* d_pmax = nullptr;
    unsigned long long* d_zero = nullptr;
    float *d_om = nullptr, *d_oi = nullptr, *d_tic = nullptr, *d_cm = nullptr, *d_ci = nullptr;
    uint64_t *d_cnt64 = nullptr, *d_out_off = nullptr;
    const unsigned int pmax0 = 1;
    const unsigned long long zero0 = ~0ull;
    CUDA_TRY(A.alloc(&d_off, n + 1));
    CUDA_TRY(A.alloc(&d_chg, n));
    CUDA_TRY(A.upload(&d_pmax, &pmax0, 1, st));
    CUDA_TRY(A.upload(&d_zero, &zero0, 1, st));
    LAUNCH(k_mgf_process_inputs<<<mgf_grid(n + 1), 256, 0, st>>>(n, M->d_peak_off, M->d_prec_off, M->d_p_charge, M->d_p_charge_some, d_off, d_chg, d_pmax,
                                                                  d_zero));
    unsigned int pmax = 0;
    unsigned long long zero = 0;
    CUDA_TRY(cudaMemcpyAsync(&pmax, d_pmax, 4, cudaMemcpyDeviceToHost, st));
    if (int rc = read_back(st, &zero, d_zero, 8)) return rc;
    if (zero != ~0ull) {
        uint64_t io[2];
        if (int rc = read_back(st, io, M->d_id_off + zero, 16)) return rc;
        std::string id(std::min<uint64_t>(io[1] - io[0], 200), '\0');
        if (int rc = read_back(st, &id[0], M->d_id + io[0], id.size())) return rc;
        return fail(SAGE_B200_ELIMIT, "mgf_process: spectrum %llu (\"%s\") has first precursor charge Some(0), which the processor's u8 charge (0 = None) cannot carry",
                    zero, id.c_str());
    }
    uint32_t p2 = 1;
    size_t smem = 0;
    if (int rc = ms2_smem(pmax, p2, smem)) return rc;
    CUDA_TRY(A.alloc(&d_om, npk + 4));
    CUDA_TRY(A.alloc(&d_oi, npk + 4));
    CUDA_TRY(A.alloc(&d_cm, npk + 4));
    CUDA_TRY(A.alloc(&d_ci, npk + 4));
    CUDA_TRY(A.alloc(&d_cnt, n));
    CUDA_TRY(A.alloc(&d_tic, n));
    CUDA_TRY(A.alloc(&d_cnt64, n + 1));
    CUDA_TRY(A.alloc(&d_out_off, n + 1));
    ProcParams pp{(uint32_t)std::min<uint64_t>(pr->take_top_n, 0xFFFFFFFFull), pr->deisotope ? 1u : 0u, pr->min_deisotope_mz};
    if (int rc = ensure_kernel_attributes(M->device)) return rc;
    LAUNCH(k_process_ms2<<<(unsigned)n, 32, smem, st>>>(pp, (uint32_t)n, d_off, M->d_mz, M->d_int, d_chg, pmax, p2, d_om, d_oi, d_cnt, d_tic));
    LAUNCH_N(k_mgf_counts64, n + 1, st, n, d_cnt, d_cnt64);
    if (int rc = mgf_scan(A, st, d_cnt64, d_out_off, n + 1)) return rc;
    LAUNCH(k_mgf_compact<<<(unsigned)std::min<uint64_t>(n, 1u << 20), 128, 0, st>>>(n, d_off, d_cnt, d_om, d_oi, d_out_off, d_cm, d_ci));
    if (int rc = read_back(st, out_offsets, d_out_off, 8 * (n + 1))) return rc;
    const uint64_t kept = out_offsets[n];
    CUDA_TRY(cudaMemcpyAsync(out_tic, d_tic, 4 * n, cudaMemcpyDeviceToHost, st));
    if (kept) {
        CUDA_TRY(cudaMemcpyAsync(out_masses, d_cm, 4 * kept, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(out_intensities, d_ci, 4 * kept, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int sage_b200_parse_f32(int device, const char* bytes, const uint64_t* offsets, uint64_t n, float* out, uint8_t* ok) {
    if (n == 0) return 0;
    if (!offsets || !out || !ok) return fail(SAGE_B200_EINVAL, "parse_f32: null argument");
    for (uint64_t i = 0; i < n; i++)
        if (offsets[i + 1] < offsets[i]) return fail(SAGE_B200_EINVAL, "parse_f32: offsets decrease at token %llu", (unsigned long long)i);
    const uint64_t nb = offsets[n] - offsets[0];
    if (nb && !bytes) return fail(SAGE_B200_EINVAL, "parse_f32: null bytes");
    if (int rc = select_device(device)) return rc;
    cudaGetLastError();
    if (int rc = mgf_memory("parse_f32", nb + n * 13)) return rc;
    DevArena A;
    Stream st;
    CUDA_TRY(st.create());
    std::vector<uint64_t> off(n + 1);
    for (uint64_t i = 0; i <= n; i++) off[i] = offsets[i] - offsets[0];
    uint8_t *d_b = nullptr, *d_ok = nullptr;
    uint64_t* d_off = nullptr;
    float* d_out = nullptr;
    CUDA_TRY(A.upload(&d_b, (const uint8_t*)bytes + offsets[0], nb, st));
    CUDA_TRY(A.upload(&d_off, off.data(), n + 1, st));
    CUDA_TRY(A.alloc(&d_out, n));
    CUDA_TRY(A.alloc(&d_ok, n));
    LAUNCH(k_mgf_parse_tokens<<<mgf_grid(n), 256, 0, st>>>(d_b, d_off, n, d_out, d_ok));
    CUDA_TRY(cudaMemcpyAsync(out, d_out, 4 * n, cudaMemcpyDeviceToHost, st));
    return read_back(st, ok, d_ok, n);
}

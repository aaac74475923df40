// Guard-band CUDA allocator for the test suite, loaded into torch as a CUDAPluggableAllocator.
//
// Every block is [front guard 4 KiB | payload (size bytes) | tail guard >= 64 KiB], the tail starting at exactly
// payload + size, so a write one byte past a tensor's end lands in the tail.  The whole block, payload included, is
// filled with the 16-bit pattern 0xFFA5 at allocation: every aligned word of it is a NaN in fp32, fp16 and bf16, a
// large negative int32 / int64 and neither 0 nor 1 as a byte, so an output element a kernel never writes shows up in the
// value comparisons the tests already make.
//
// free() does not release a block: it goes to a quarantine, and nothing is reused before guard_check() has looked at
// its guards.  guard_check() synchronises the device, scans the front and tail guards of every live and quarantined
// block in one kernel, records and restores each guard that changed, and then returns the quarantine to a pool of blocks that
// later allocations of the same rounded size reuse.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

namespace {

constexpr int64_t kFront = 4096;                 // keeps the payload 512-byte aligned
constexpr int64_t kTailMin = 64 << 10;           // wide enough for a stray whole tile
constexpr int64_t kRound = 64 << 10;             // block sizes are multiples of this, so that freed blocks are reusable
constexpr int64_t kAlign = 512;
constexpr uint32_t kPattern = 0xFFA5FFA5u;       // 0xFFA5 in every 16-bit half, little-endian bytes A5 FF
constexpr int64_t kQuarantineCap = int64_t(4) << 30;
constexpr int64_t kPoolCap = int64_t(8) << 30;

struct Block {
    char* raw;          // what cudaMalloc returned
    char* base;         // raw rounded up to kAlign; the front guard starts here
    int64_t total;      // front + size + tail
    int64_t size;       // payload bytes
    int64_t seq;        // allocation sequence number
    int device;
};

struct Desc {           // what the check kernel needs of one block
    const uint32_t* base;
    int64_t total;
    int64_t size;
};

}  // namespace

struct GuardViolation {           // one guard of one block that changed; guard_report copies these out
    int64_t seq;        // sequence number of the allocation (1 = first malloc of the process)
    int64_t size;       // its payload size in bytes
    int64_t first;      // first corrupted byte, as an offset from the payload's start (-1 = last front byte, size = first tail byte)
    int64_t last;       // last corrupted byte, same origin
    int32_t side;       // 0 front guard, 1 tail guard
    int32_t nfound;     // valid bytes in found[]
    uint8_t found[16];  // the bytes found from `first` on
};

namespace {

std::mutex g_mu;
std::unordered_map<char*, Block> g_live;                    // payload pointer -> block
std::vector<Block> g_quarantine;
std::unordered_map<int64_t, std::vector<Block>> g_pool;     // total -> checked blocks ready for reuse
std::vector<GuardViolation> g_violations;
std::string g_error;
int64_t g_seq = 0, g_quarantine_bytes = 0, g_pool_bytes = 0;
Desc* g_desc_dev = nullptr;
unsigned long long* g_hits_dev = nullptr;                   // [n][4]: front first/last, tail first/last
int64_t g_desc_cap = 0;

void cuda_ok(cudaError_t e, const char* what) {
    if (e != cudaSuccess) throw std::runtime_error(std::string("guard_alloc: ") + what + ": " + cudaGetErrorString(e));
}

__global__ void fill_kernel(uint4* p, int64_t n16) {
    const uint4 v = make_uint4(kPattern, kPattern, kPattern, kPattern);
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n16; i += int64_t(gridDim.x) * blockDim.x) p[i] = v;
}

// One CTA per block.  Byte b of the block (from base) is a guard byte when b < kFront or b >= kFront + size; each 32-bit
// word is compared with the pattern under a mask of its guard bytes, and the first and last differing guard byte of each
// side are kept with atomicMin / atomicMax.
__global__ void check_kernel(const Desc* desc, unsigned long long* hits) {
    const Desc d = desc[blockIdx.x];
    const int64_t t0 = kFront + d.size;
    const int64_t words_front = kFront / 4, w_tail0 = t0 / 4, words = d.total / 4;
    unsigned long long* h = hits + 4 * int64_t(blockIdx.x);
    const int64_t n = words_front + (words - w_tail0);
    for (int64_t k = threadIdx.x; k < n; k += blockDim.x) {
        const int64_t w = k < words_front ? k : w_tail0 + (k - words_front);
        uint32_t diff = d.base[w] ^ kPattern;
        if (!diff) continue;
        const bool tail = k >= words_front;
        for (int j = 0; j < 4; ++j) {
            const int64_t b = 4 * w + j;
            if (!((diff >> (8 * j)) & 0xFFu) || (tail ? b < t0 : b >= kFront)) continue;
            atomicMin(h + (tail ? 2 : 0), (unsigned long long)b);
            atomicMax(h + (tail ? 3 : 1), (unsigned long long)b);
        }
    }
}

void fill(const Block& b, cudaStream_t s) {
    const int64_t n16 = b.total / 16;
    const int grid = int(n16 / 256 + 1 < 1024 ? n16 / 256 + 1 : 1024);
    fill_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<uint4*>(b.base), n16);
    cuda_ok(cudaGetLastError(), "fill launch");
}

void release_pool() {
    for (auto& kv : g_pool)
        for (auto& b : kv.second) cudaFree(b.raw);
    g_pool.clear();
    g_pool_bytes = 0;
}

// Checks every live and quarantined block; returns the number of new violations.  Caller holds g_mu.
int check_locked() {
    cuda_ok(cudaDeviceSynchronize(), "synchronise before the check");
    std::vector<const Block*> blocks;
    blocks.reserve(g_live.size() + g_quarantine.size());
    for (auto& kv : g_live) blocks.push_back(&kv.second);
    for (auto& b : g_quarantine) blocks.push_back(&b);
    const int64_t n = int64_t(blocks.size());
    int found = 0;
    if (n) {
        if (n > g_desc_cap) {
            cudaFree(g_desc_dev);
            cudaFree(g_hits_dev);
            g_desc_cap = 2 * n;
            cuda_ok(cudaMalloc(&g_desc_dev, g_desc_cap * sizeof(Desc)), "check table");
            cuda_ok(cudaMalloc(&g_hits_dev, g_desc_cap * 4 * sizeof(unsigned long long)), "check table");
        }
        std::vector<Desc> desc(n);
        for (int64_t i = 0; i < n; ++i)
            desc[i] = {reinterpret_cast<const uint32_t*>(blocks[i]->base), blocks[i]->total, blocks[i]->size};
        std::vector<unsigned long long> hits(4 * n);
        for (int64_t i = 0; i < n; ++i) {
            hits[4 * i] = hits[4 * i + 2] = ~0ull;
            hits[4 * i + 1] = hits[4 * i + 3] = 0;
        }
        cuda_ok(cudaMemcpy(g_desc_dev, desc.data(), n * sizeof(Desc), cudaMemcpyHostToDevice), "check table upload");
        cuda_ok(cudaMemcpy(g_hits_dev, hits.data(), 4 * n * sizeof(unsigned long long), cudaMemcpyHostToDevice),
                "check table upload");
        for (int64_t i0 = 0; i0 < n; i0 += 65535) {
            const int64_t m = n - i0 < 65535 ? n - i0 : 65535;
            check_kernel<<<unsigned(m), 256>>>(g_desc_dev + i0, g_hits_dev + 4 * i0);
            cuda_ok(cudaGetLastError(), "check launch");
        }
        cuda_ok(cudaMemcpy(hits.data(), g_hits_dev, 4 * n * sizeof(unsigned long long), cudaMemcpyDeviceToHost),
                "check result download");
        for (int64_t i = 0; i < n; ++i)
            for (int side = 0; side < 2; ++side) {
                const unsigned long long first = hits[4 * i + 2 * side];
                if (first == ~0ull) continue;
                const Block& b = *blocks[i];
                GuardViolation v{};
                v.seq = b.seq;
                v.size = b.size;
                v.side = side;
                v.first = int64_t(first) - kFront;
                v.last = int64_t(hits[4 * i + 2 * side + 1]) - kFront;
                const int64_t end = side ? b.total : kFront;
                v.nfound = int32_t(end - int64_t(first) < 16 ? end - int64_t(first) : 16);
                cuda_ok(cudaMemcpy(v.found, b.base + first, v.nfound, cudaMemcpyDeviceToHost), "violation bytes");
                g_violations.push_back(v);
                ++found;
                // restore the guard, so that the next check reports only new damage
                const int64_t lo = side ? kFront + b.size : 0;
                std::vector<uint8_t> pattern(size_t(end - lo));
                for (int64_t k = lo; k < end; ++k) pattern[size_t(k - lo)] = (k & 1) ? 0xFF : 0xA5;
                cuda_ok(cudaMemcpy(b.base + lo, pattern.data(), pattern.size(), cudaMemcpyHostToDevice), "guard restore");
            }
    }
    for (auto& b : g_quarantine) {
        if (g_pool_bytes + b.total + kAlign > kPoolCap) {
            cudaFree(b.raw);
        } else {
            g_pool[b.total].push_back(b);
            g_pool_bytes += b.total + kAlign;
        }
    }
    g_quarantine.clear();
    g_quarantine_bytes = 0;
    return found;
}

}  // namespace

extern "C" {

void* guard_malloc(size_t size, int device, cudaStream_t stream) {
    if (size == 0) return nullptr;                  // as the caching allocator: no storage, no device work
    std::lock_guard<std::mutex> lock(g_mu);
    cuda_ok(cudaSetDevice(device), "set device");
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cuda_ok(cudaStreamIsCapturing(stream, &cap), "capture query");
    if (cap != cudaStreamCaptureStatusNone)
        throw std::runtime_error("guard_alloc: allocation on a capturing stream; the guard allocator cannot host "
                                 "CUDA graph capture");
    if (g_quarantine_bytes > kQuarantineCap) check_locked();
    Block b{};
    b.total = (kFront + int64_t(size) + kTailMin + kRound - 1) / kRound * kRound;
    auto it = g_pool.find(b.total);
    if (it != g_pool.end() && !it->second.empty() && it->second.back().device == device) {
        b = it->second.back();
        it->second.pop_back();
        g_pool_bytes -= b.total + kAlign;
    } else {
        void* raw = nullptr;
        if (cudaMalloc(&raw, b.total + kAlign) != cudaSuccess) {
            cudaGetLastError();
            check_locked();
            release_pool();
            cuda_ok(cudaMalloc(&raw, b.total + kAlign), "cudaMalloc");
        }
        b.raw = static_cast<char*>(raw);
        b.base = b.raw + (kAlign - reinterpret_cast<uintptr_t>(b.raw) % kAlign) % kAlign;
        b.device = device;
    }
    b.size = int64_t(size);
    b.seq = ++g_seq;
    fill(b, stream);
    char* payload = b.base + kFront;
    g_live[payload] = b;
    return payload;
}

void guard_free(void* ptr, size_t, int, cudaStream_t) {
    if (!ptr) return;
    std::lock_guard<std::mutex> lock(g_mu);
    auto it = g_live.find(static_cast<char*>(ptr));
    if (it == g_live.end()) throw std::runtime_error("guard_alloc: free of a pointer it did not allocate");
    g_quarantine_bytes += it->second.total;
    g_quarantine.push_back(it->second);
    g_live.erase(it);
}

// Synchronises the device and checks the guards of every live and quarantined block, then releases the quarantine.
// Returns the number of new violations, or -1 on a CUDA error, whose text guard_last_error() returns.
int guard_check() {
    std::lock_guard<std::mutex> lock(g_mu);
    try {
        return check_locked();
    } catch (const std::exception& e) {
        g_error = e.what();
        return -1;
    }
}

const char* guard_last_error() {
    return g_error.c_str();
}

// Copies up to `cap` violation records, oldest first, into `out`; returns how many have been recorded in all.
int64_t guard_report(GuardViolation* out, int64_t cap) {
    std::lock_guard<std::mutex> lock(g_mu);
    const int64_t n = int64_t(g_violations.size());
    if (out && cap > 0) std::memcpy(out, g_violations.data(), size_t(n < cap ? n : cap) * sizeof(GuardViolation));
    return n;
}

// out[0..5]: live blocks, live payload bytes, quarantined blocks, quarantined block bytes, allocations made, pooled bytes.
void guard_stats(int64_t* out) {
    std::lock_guard<std::mutex> lock(g_mu);
    int64_t live_bytes = 0;
    for (auto& kv : g_live) live_bytes += kv.second.size;
    out[0] = int64_t(g_live.size());
    out[1] = live_bytes;
    out[2] = int64_t(g_quarantine.size());
    out[3] = g_quarantine_bytes;
    out[4] = g_seq;
    out[5] = g_pool_bytes;
}

// Test support for the harness itself: sets one byte of the guard of the live block whose payload starts at `ptr`, at
// `offset` bytes from the payload's start (-kFront..-1 is the front guard, size.. the tail).  It writes memory the
// allocator owns, never a payload byte.  Returns 0, or -1 if ptr is not a live payload or offset is not a guard byte.
int guard_scribble_for_test(void* ptr, int64_t offset, int value) {
    std::lock_guard<std::mutex> lock(g_mu);
    auto it = g_live.find(static_cast<char*>(ptr));
    if (it == g_live.end()) return -1;
    const Block& b = it->second;
    if (offset < -kFront || (offset >= 0 && offset < b.size) || offset >= b.total - kFront) return -1;
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    if (cudaMemset(static_cast<char*>(ptr) + offset, value, 1) != cudaSuccess) return -1;
    return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}

// Bytes of the tail guard of the live block at `ptr` (-1 if it is not one): the last tail byte is at offset
// size + guard_tail_bytes(ptr) - 1.
int64_t guard_tail_bytes(void* ptr) {
    std::lock_guard<std::mutex> lock(g_mu);
    auto it = g_live.find(static_cast<char*>(ptr));
    return it == g_live.end() ? -1 : it->second.total - kFront - it->second.size;
}

}  // extern "C"

// Host build of pocketsphinx_b200/csrc/psb_mem.cuh against stub CUDA runtime functions: an allocator that fails on
// demand, so that the owners' behaviour after a failed allocation can be checked without a GPU.  Prints "ok" or the
// first failed check.
#include "psb_mem.cuh"

#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include <map>
#include <set>
#include <string>
#include <utility>

std::atomic<long long> g_psb_bytes_live{0};

static std::string g_msg;
void psb_set_error(const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_msg = buf;
}

static int g_fail_next = 0;                 // the next n allocations fail
static int g_allocs = 0;
static cudaError_t g_last = cudaSuccess;
static std::map<void *, bool> g_blocks;     // live block -> pinned
static std::set<void *> g_streams, g_events;

static cudaError_t stub_alloc(void **p, size_t bytes, bool pinned)
{
    ++g_allocs;
    if (g_fail_next > 0) {
        --g_fail_next;
        g_last = cudaErrorMemoryAllocation;
        return cudaErrorMemoryAllocation;
    }
    *p = malloc(bytes ? bytes : 1);
    g_blocks[*p] = pinned;
    return cudaSuccess;
}

static cudaError_t stub_free(void *p, bool pinned)
{
    if (!p) return cudaSuccess;
    auto it = g_blocks.find(p);
    if (it == g_blocks.end() || it->second != pinned) {
        printf("bad free of %p\n", p);
        exit(1);
    }
    g_blocks.erase(it);
    free(p);
    return cudaSuccess;
}

extern "C" {
cudaError_t cudaMalloc(void **p, size_t bytes) { return stub_alloc(p, bytes, false); }
cudaError_t cudaMallocHost(void **p, size_t bytes) { return stub_alloc(p, bytes, true); }
cudaError_t cudaFree(void *p) { return stub_free(p, false); }
cudaError_t cudaFreeHost(void *p) { return stub_free(p, true); }
cudaError_t cudaGetLastError(void)
{
    const cudaError_t e = g_last;
    g_last = cudaSuccess;
    return e;
}
const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "out of memory"; }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned int)
{
    *s = reinterpret_cast<cudaStream_t>(malloc(1));
    g_streams.insert(*s);
    return cudaSuccess;
}
cudaError_t cudaStreamDestroy(cudaStream_t s)
{
    if (!g_streams.erase(s)) { printf("bad stream destroy\n"); exit(1); }
    free(s);
    return cudaSuccess;
}
cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned int)
{
    *e = reinterpret_cast<cudaEvent_t>(malloc(1));
    g_events.insert(*e);
    return cudaSuccess;
}
cudaError_t cudaEventDestroy(cudaEvent_t e)
{
    if (!g_events.erase(e)) { printf("bad event destroy\n"); exit(1); }
    free(e);
    return cudaSuccess;
}
}

#define CHECK(c)                                                   \
    do {                                                           \
        if (!(c)) {                                                \
            printf("check failed at line %d: %s\n", __LINE__, #c); \
            return 1;                                              \
        }                                                          \
    } while (0)

int main()
{
    const long long live0 = g_psb_bytes_live.load();
    {
        DevBuf<int> d;
        HostBuf<double> h;
        CHECK(d.get() == nullptr && d.cap() == 0);

        // reserve allocates need + headroom and counts the bytes
        CHECK(d.reserve(100, 28) == PSB_OK);
        CHECK(d.get() != nullptr && d.cap() == 128);
        CHECK(g_psb_bytes_live.load() == live0 + 128 * 4);

        // within capacity: no new allocation
        int *p = d.get();
        const int n = g_allocs;
        CHECK(d.reserve(128) == PSB_OK && d.reserve(1, 1000) == PSB_OK);
        CHECK(d.get() == p && d.cap() == 128 && g_allocs == n);

        // a failed growth leaves the buffer empty with capacity 0, frees the old block, clears the last error
        g_fail_next = 1;
        CHECK(d.reserve(200, 8) == PSB_ERR_NOMEM);
        CHECK(d.get() == nullptr && d.cap() == 0);
        CHECK(cudaGetLastError() == cudaSuccess);
        CHECK(g_msg.find("832 bytes") != std::string::npos);
        CHECK(g_psb_bytes_live.load() == live0);
        CHECK(g_blocks.empty());

        // ... and the next reserve retries, even for a size the old block had room for
        CHECK(d.reserve(10) == PSB_OK && d.get() != nullptr && d.cap() == 10);

        // pinned memory the same way
        g_fail_next = 1;
        CHECK(h.reserve(4) == PSB_ERR_NOMEM && h.get() == nullptr && h.cap() == 0);
        CHECK(cudaGetLastError() == cudaSuccess);
        CHECK(h.reserve(4) == PSB_OK && h.cap() == 4 && g_blocks[h.get()]);
        CHECK(g_psb_bytes_live.load() == live0 + 10 * 4 + 4 * 8);

        // moves transfer ownership
        DevBuf<int> d2(std::move(d));
        CHECK(d.get() == nullptr && d.cap() == 0 && d2.cap() == 10);
        DevBuf<int> d3;
        CHECK(d3.reserve(5) == PSB_OK);
        d3 = std::move(d2);                         // frees d3's old block
        CHECK(d2.get() == nullptr && d3.cap() == 10 && g_blocks.size() == 2);
        CHECK(g_psb_bytes_live.load() == live0 + 10 * 4 + 4 * 8);

        // streams and events
        Stream s;
        Event e[2];
        CHECK(s.create() == cudaSuccess && e[0].create() == cudaSuccess && e[1].create(cudaEventDisableTiming) == cudaSuccess);
        CHECK((cudaStream_t)s != nullptr && g_streams.size() == 1 && g_events.size() == 2);
        Stream s2(std::move(s));
        CHECK((cudaStream_t)s == nullptr && (cudaStream_t)s2 != nullptr);
        Event e2;
        e2 = std::move(e[0]);
        CHECK((cudaEvent_t)e[0] == nullptr && g_events.size() == 2);
    }
    // destructors free everything
    CHECK(g_blocks.empty() && g_streams.empty() && g_events.empty());
    CHECK(g_psb_bytes_live.load() == live0);
    printf("ok\n");
    return 0;
}

// Host-only check of cphb_scratch and cphb_arena (cupoch_b200/csrc/cphb_internal.cuh) against recording stubs of the
// allocator: every buffer they hand out is freed exactly once, on its stream, whichever way the scope is left, and an
// arena lays its slices out at 256-byte-aligned running offsets.  Launches nothing and needs no device.  Exit code 0 =
// all checks passed.
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <vector>

#include "cphb_internal.cuh"

unsigned long long g_cphb_launches = 0;
static char g_err[256];
void cphb_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

struct Call {
    bool alloc;
    void *p;
    size_t bytes;
    cudaStream_t s;
};
static std::vector<Call> g_calls;
static int g_allocs = 0;    // cphb_alloc_async calls so far
static int g_fail_at = -1;  // this call (0-based) fails

int cphb_alloc_async(void **p, size_t bytes, cudaStream_t s) {
    if (g_allocs++ == g_fail_at) return CPHB_ERR_CUDA;
    *p = (void *)(uintptr_t)(0x10000 + 0x100 * g_allocs);
    g_calls.push_back({true, *p, bytes, s});
    return CPHB_OK;
}
void cphb_free_async(void *p, cudaStream_t s) { g_calls.push_back({false, p, 0, s}); }

static int g_failed = 0;
#define EXPECT(c)                                                   \
    do {                                                            \
        if (!(c)) {                                                 \
            fprintf(stderr, "%s:%d: EXPECT(%s)\n", __FILE__, __LINE__, #c); \
            ++g_failed;                                             \
        }                                                           \
    } while (0)

static const cudaStream_t S = (cudaStream_t)(uintptr_t)0x51;

static void reset(int fail_at = -1) {
    g_calls.clear();
    g_allocs = 0;
    g_fail_at = fail_at;
    g_err[0] = 0;
}
static int count(bool alloc) {
    int c = 0;
    for (const Call &k : g_calls) c += k.alloc == alloc;
    return c;
}
// every recorded allocation is freed exactly once, on S, after it was made; nothing else is freed (the stub hands out
// a new address per allocation)
static bool balanced() {
    for (size_t i = 0; i < g_calls.size(); ++i) {
        const Call &k = g_calls[i];
        int allocs = 0, frees = 0, later_frees = 0;
        for (size_t j = 0; j < g_calls.size(); ++j) {
            if (g_calls[j].p != k.p) continue;
            if (g_calls[j].alloc) {
                ++allocs;
            } else {
                ++frees;
                later_frees += j > i;
            }
        }
        if (k.s != S || allocs != 1 || frees != 1 || (k.alloc && later_frees != 1)) return false;
    }
    return true;
}

int main() {
    // scope exit frees every buffer once, sizes are count * sizeof(T)
    reset();
    {
        cphb_scratch sc(S);
        float *a = nullptr;
        int32_t *b = nullptr;
        double *c = nullptr;
        EXPECT(sc.alloc(&a, 10) == CPHB_OK && a);
        EXPECT(sc.alloc(&b, 3) == CPHB_OK && b);
        EXPECT(sc.alloc(&c, 1) == CPHB_OK && c);
        EXPECT(g_calls.size() == 3 && g_calls[0].bytes == 40 && g_calls[1].bytes == 12 && g_calls[2].bytes == 8);
        EXPECT(count(false) == 0);
    }
    EXPECT(count(true) == 3 && count(false) == 3 && balanced());

    // the k-th allocation fails: the k - 1 earlier buffers are freed, nothing else
    for (int k = 1; k <= 5; ++k) {
        reset(k - 1);
        int rc = CPHB_OK;
        {
            cphb_scratch sc(S);
            uint8_t *p[5] = {};
            for (int i = 0; i < 5; ++i)
                if (!rc) rc = sc.alloc(&p[i], 16);
            EXPECT(p[k - 1] == nullptr);
        }
        EXPECT(rc == CPHB_ERR_CUDA);
        EXPECT(count(true) == k - 1 && count(false) == k - 1 && balanced());
    }

    // release() frees now; the scope exit after it frees nothing twice, but still frees what came after
    reset();
    {
        cphb_scratch sc(S);
        float *a = nullptr, *b = nullptr, *c = nullptr;
        EXPECT(sc.alloc(&a, 4) == CPHB_OK);
        EXPECT(sc.alloc(&b, 4) == CPHB_OK);
        sc.release();
        EXPECT(count(false) == 2);
        EXPECT(sc.alloc(&c, 4) == CPHB_OK);
        EXPECT(count(false) == 2);
    }
    EXPECT(count(true) == 3 && count(false) == 3 && balanced());

    // past the slot capacity: an error, no allocation, and every earlier buffer is still freed once
    reset();
    {
        cphb_scratch sc(S);
        int rc = CPHB_OK;
        for (int i = 0; i < CPHB_SCRATCH_SLOTS && !rc; ++i) {
            float *p = nullptr;
            rc = sc.alloc(&p, 1);
        }
        EXPECT(rc == CPHB_OK);
        float *extra = nullptr;
        EXPECT(sc.alloc(&extra, 1) == CPHB_ERR_INVALID);
        EXPECT(extra == nullptr && g_allocs == CPHB_SCRATCH_SLOTS && g_err[0] != 0);
    }
    EXPECT(count(true) == CPHB_SCRATCH_SLOTS && count(false) == CPHB_SCRATCH_SLOTS && balanced());

    // cphb_arena: each slice starts at the running offset, which then moves to the next multiple of 256; an absent
    // slice is null and takes no bytes; one allocation of the total on the given stream, freed once on it at the end
    reset();
    {
        cphb_arena ar;
        float *a = nullptr;
        double *b = (double *)&ar;
        int32_t *c = nullptr;
        char *d = nullptr;
        uint8_t *e = nullptr;
        ar.slice(&a, 10);           // [0, 40)
        ar.slice(&b, 1000, false);  // absent
        ar.slice(&c, 64);           // [256, 512)
        ar.slice(&d, 0);            // empty, at 512
        ar.slice(&e, 257);          // [512, 769)
        EXPECT(ar.bytes() == 1024 && g_calls.empty() && !a && !b && !c);
        EXPECT(ar.alloc(S) == CPHB_OK);
        EXPECT(g_calls.size() == 1 && g_calls[0].alloc && g_calls[0].bytes == 1024 && g_calls[0].s == S);
        char *base = (char *)g_calls[0].p;
        EXPECT((char *)a == base && !b && (char *)c == base + 256 && d == base + 512 && (char *)e == base + 512);
    }
    EXPECT(count(true) == 1 && count(false) == 1 && balanced());

    // a failed allocation leaves every pointer null and frees nothing
    reset(0);
    {
        cphb_arena ar;
        float *a = nullptr, *b = nullptr;
        ar.slice(&a, 4);
        ar.slice(&b, 4);
        EXPECT(ar.alloc(S) == CPHB_ERR_CUDA && !a && !b);
    }
    EXPECT(g_calls.empty());

    // a move hands the block over: the moved-from arena frees nothing, the new owner frees it once
    reset();
    {
        cphb_arena *owner = nullptr;
        {
            cphb_arena ar;
            float *a = nullptr;
            ar.slice(&a, 4);
            EXPECT(ar.alloc(S) == CPHB_OK && a);
            owner = new cphb_arena(std::move(ar));
        }
        EXPECT(count(false) == 0);
        delete owner;
    }
    EXPECT(count(true) == 1 && count(false) == 1 && balanced());

    if (g_failed) {
        fprintf(stderr, "scratch_check: %d failed\n", g_failed);
        return 1;
    }
    printf("scratch_check: ok\n");
    return 0;
}

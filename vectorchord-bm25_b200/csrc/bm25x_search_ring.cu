// bm25x_search_ring.cu — instantiations of k_search_ring (bm25x_search_ring.cuh) for one pool size.
// Compiled once per pool capacity (-DBM25X_RING_KP=64|256|2048) so that the term-count classes build in parallel.
#include "bm25x_common.h"

#include "bm25x_search_ring.cuh"

#ifndef BM25X_RING_KP
#error "compile with -DBM25X_RING_KP=<pool capacity>"
#endif

namespace {

template <class C>
int launch_ring(int device, int sm_count, const SearchParams &sp_in, cudaStream_t stream) {
    static bool configured[64] = {false};
    auto kern = k_search_ring<C>;
    if (!configured[device & 63]) {
        BM25X_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::total));
        configured[device & 63] = true;
    }
    uint32_t grid = (uint32_t)sm_count;  // persistent: one CTA per SM, every warp pulls queries from the work counter
    const uint32_t need = (sp_in.nq + C::WARPS - 1) / C::WARPS;
    if (grid > need) grid = need;
    SearchParams sp = sp_in;
    sp.pool_scratch = nullptr;
    if (C::POOL_GLOBAL) {  // stream-ordered scratch for the per-warp pools, released right behind the kernel
        const size_t bytes = (size_t)grid * C::WARPS * (size_t)C::KP * 16;
        BM25X_CUDA_TRY(cudaMallocAsync((void **)&sp.pool_scratch, bytes, stream));
    }
    kern<<<grid, C::THREADS, C::total, stream>>>(sp);
    cudaError_t e = cudaGetLastError();
    if (sp.pool_scratch) cudaFreeAsync(sp.pool_scratch, stream);
    BM25X_CUDA_TRY(e);
    return BM25X_OK;
}

// a flavour / term-count class pair that is not built
int no_launch(int M) {
    bm25x_set_error("k_search_ring: no two-phase launch for %d terms / pool %d", M, (int)BM25X_RING_KP);
    return BM25X_ERR_INVALID;
}

// The term-count classes flavour F is built for: every class for the plain kernel (M = 64: two passes of the 32-term
// kernel); 2..4 terms for the two-phase flavours; 2..4 and 8 terms for the seeded launch and its hand-back.  The flavours
// other than plain only exist with the pool in shared memory (KP <= 256).
template <int F>
int launch_flavour(int device, int sm_count, const SearchParams &sp, int M, cudaStream_t stream) {
    constexpr int KP = BM25X_RING_KP;
    if constexpr (F == RING_PLAIN) {
        switch (M) {
            case 1: return launch_ring<RCfg<1, KP, F>>(device, sm_count, sp, stream);
            case 2: return launch_ring<RCfg<2, KP, F>>(device, sm_count, sp, stream);
            case 3: return launch_ring<RCfg<3, KP, F>>(device, sm_count, sp, stream);
            case 4: return launch_ring<RCfg<4, KP, F>>(device, sm_count, sp, stream);
            case 8: return launch_ring<RCfg<8, KP, F>>(device, sm_count, sp, stream);
            case 16: return launch_ring<RCfg<16, KP, F>>(device, sm_count, sp, stream);
            default: return launch_ring<RCfg<32, KP, F>>(device, sm_count, sp, stream);
        }
    } else if constexpr (KP <= 256) {
        switch (M) {
            case 2: return launch_ring<RCfg<2, KP, F>>(device, sm_count, sp, stream);
            case 3: return launch_ring<RCfg<3, KP, F>>(device, sm_count, sp, stream);
            case 4: return launch_ring<RCfg<4, KP, F>>(device, sm_count, sp, stream);
            case 8:
                if constexpr (F == RING_SEEDED || F == RING_HANDBACK) return launch_ring<RCfg<8, KP, F>>(device, sm_count, sp, stream);
                break;
            default: break;
        }
    }
    return no_launch(M);
}

}  // namespace

#if defined(BM25X_PHASE_PROF) && BM25X_RING_KP == 64
// diagnostic builds only (tools/phase_profile.py): copies the phase profile of the seeded k <= 32 classes to `out`
// (PP_SLOTS values: cycles per phase, then chunks, listed candidates, hits, hit-list flushes and rows) and zeroes it when `reset` is set
extern "C" int bm25x_phase_prof(unsigned long long *out, int reset) {
    if (out) BM25X_CUDA_TRY(cudaMemcpyFromSymbol(out, g_phase_prof, sizeof(g_phase_prof)));
    if (reset) {
        static const unsigned long long zero[PP_SLOTS] = {};
        BM25X_CUDA_TRY(cudaMemcpyToSymbol(g_phase_prof, zero, sizeof(zero)));
    }
    return PP_SLOTS;
}
#endif

#define BM25X_RING_ENTRY2(kp) bm25x_launch_ring_kp##kp
#define BM25X_RING_ENTRY(kp) BM25X_RING_ENTRY2(kp)

// M = term-count class of the launch (1, 2, 3, 4, 8, 16, 32)
int BM25X_RING_ENTRY(BM25X_RING_KP)(int device, int sm_count, const SearchParams &sp, int M, RingFlavour flavour,
                                    cudaStream_t stream) {
    switch (flavour) {
        case RING_PLAIN: return launch_flavour<RING_PLAIN>(device, sm_count, sp, M, stream);
        case RING_SUSPEND: return launch_flavour<RING_SUSPEND>(device, sm_count, sp, M, stream);
        case RING_RESUME: return launch_flavour<RING_RESUME>(device, sm_count, sp, M, stream);
        case RING_SEEDED: return launch_flavour<RING_SEEDED>(device, sm_count, sp, M, stream);
        case RING_HANDBACK: return launch_flavour<RING_HANDBACK>(device, sm_count, sp, M, stream);
    }
    return no_launch(M);
}

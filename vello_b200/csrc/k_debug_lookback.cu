// k_debug_lookback.cu -- test-only: vb_lookback (vb_device.cuh) run alone, under a schedule the caller forces.
//
// A look-back that finds an inclusive prefix at its nearest predecessor never combines more than one window, and never
// reduces a window of aggregates. Which case a frame kernel meets depends on timing. Here partition p, by ticket, first
// waits delay_ns[p]: a delayed partition keeps the ones after it from finishing, so they publish aggregates only and a later
// partition has to combine whole windows of them, in order. No frame kernel uses this file (vb_debug_lookback, vb_api.cu).
#include "../../include/vello_b200.h"
#include "vb_device.cuh"
#include "vb_stages.h"

// x -> a * x + b (mod 2^32), stored as (a - 1, b) so that all zeros is the identity. a (+) b applies a first: far from
// commutative, and every word depends on the order of the whole fold.
struct VbAffineOp {
    static constexpr bool commutative = false;
    template <int K> __device__ __forceinline__ static void combine(const uint32_t (&a)[K], const uint32_t (&b)[K], uint32_t (&r)[K]) {
        static_assert(K == 2, "VbAffineOp has two words");
        const uint32_t ma = a[0] + 1u, mb = b[0] + 1u, ab = a[1], bb = b[1];
        r[0] = mb * ma - 1u;
        r[1] = mb * ab + bb;
    }
};

__device__ __forceinline__ uint64_t lb_globaltimer() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// One warp per partition. The wait is bounded by the delay itself (the host caps it); the spins after it are vb_lookback's
// own, on predecessors that took their tickets first and so are already running.
template <int K, class Op>
__global__ void __launch_bounds__(32) k_debug_lookback(uint32_t *lb_mem, uint32_t n_parts, const uint32_t *agg, const uint32_t *delay_ns,
                                                       uint32_t *excl) {
    __shared__ uint32_t sh_ticket;
    const VbLookback lb = vb_lookback_view(lb_mem, n_parts, K);
    const uint32_t part = vb_take_ticket(lb, &sh_ticket);
    if (threadIdx.x == 0u) {
        const uint64_t d = delay_ns[part], t0 = lb_globaltimer();
        for (uint64_t t = t0; t - t0 < d; t = lb_globaltimer()) {
            const uint64_t left = d - (t - t0);
            __nanosleep(left < 1000u ? (uint32_t)left : 1000u);
        }
    }
    __syncwarp();
    uint32_t a[K], e[K];
#pragma unroll
    for (int k = 0; k < K; k++) a[k] = agg[(size_t)part * K + k];
    vb_lookback<K, Op>(lb, part, a, e);
    if (threadIdx.x == 0u) {
#pragma unroll
        for (int k = 0; k < K; k++) excl[(size_t)part * K + k] = e[k];
    }
}

extern "C" uint32_t vb_debug_lookback_words(int op) {
    switch (op) {
    case VB_LOOKBACK_SUM1: return 1;
    case VB_LOOKBACK_SUM5: return 5;
    case VB_LOOKBACK_BACKDROP: return 3;
    case VB_LOOKBACK_AFFINE: return 2;
    default: return 0;
    }
}

extern "C" uint32_t vb_launch_debug_lookback(int op, uint32_t n_parts, uint32_t *lb_mem, const uint32_t *agg, const uint32_t *delay_ns,
                                             uint32_t *excl, cudaStream_t st) {
    switch (op) {
    case VB_LOOKBACK_SUM1: k_debug_lookback<1, VbSumOp><<<n_parts, 32, 0, st>>>(lb_mem, n_parts, agg, delay_ns, excl); return 1;
    case VB_LOOKBACK_SUM5: k_debug_lookback<5, VbSumOp><<<n_parts, 32, 0, st>>>(lb_mem, n_parts, agg, delay_ns, excl); return 1;
    case VB_LOOKBACK_BACKDROP: k_debug_lookback<3, BdSegOp><<<n_parts, 32, 0, st>>>(lb_mem, n_parts, agg, delay_ns, excl); return 1;
    case VB_LOOKBACK_AFFINE: k_debug_lookback<2, VbAffineOp><<<n_parts, 32, 0, st>>>(lb_mem, n_parts, agg, delay_ns, excl); return 1;
    default: return 0;
    }
}

// k_recompose.cu -- the damage of the first frame after vb_recompose: which tiles differ between the composition the base
// frame rendered and the new one.
//
// The host (vb_compose.cu) matches the old instances to the new ones in order, by fragment id and transform, and unmatches an
// instance whose images moved in the atlas. A tile's pixels are a function of the ordered draw objects whose clipped box covers
// it, so it is damaged only by
//   - the draw objects of unmatched instances: their boxes in the base frame (old) and in this frame (new);
//   - a matched draw object whose box is not bit for bit its counterpart's (an enclosing clip that came or went): both boxes;
//   - the END_CLIPs after the last instance, paired from the end: an unpaired one, or both boxes of a pair that differs.
// Boxes are binning's clipped boxes, rounded out to tiles as tile_alloc rounds them (dm_or_box). The old boxes were copied
// from the base frame when the recompose was enqueued; the new ones are this frame's. Neither changes when the frame is run
// again after an arena overflow, so a re-run computes the same damage.
#include "vb_device.cuh"
#include "vb_stages.h"

#define RC_THREADS 256u

__device__ __forceinline__ bool rc_same_box(const VbBbox4 a, const VbBbox4 b) {
    return __float_as_uint(a.x0) == __float_as_uint(b.x0) && __float_as_uint(a.y0) == __float_as_uint(b.y0) &&
           __float_as_uint(a.x1) == __float_as_uint(b.x1) && __float_as_uint(a.y1) == __float_as_uint(b.y1);
}

// One warp per draw object: the new composition's first, then the old one's. Tables as vb_rcmp_tables lays them out.
__global__ void __launch_bounds__(RC_THREADS)
k_recompose_damage(const VbBbox4 *__restrict__ now_boxes, const VbBbox4 *__restrict__ old_boxes, const uint32_t *__restrict__ tables,
                   uint32_t n_old, uint32_t n_new, uint32_t old_draws, uint32_t new_draws, uint8_t *mask, uint32_t wt, uint32_t ht) {
    const uint32_t w = blockIdx.x * (RC_THREADS / 32u) + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
    const VbRcmpTables<const uint32_t> T = vb_rcmp_tables(tables, n_old, n_new);
    const uint32_t old_end = __ldg(T.old_pre + n_old), new_end = __ldg(T.new_pre + n_new); // the trailing END_CLIPs start here
    if (w < new_draws) {
        const uint32_t d = w;
        const VbBbox4 now = now_boxes[d];
        uint32_t od;
        if (d < new_end) {
            const uint32_t k = cp_find(T.new_pre, 0u, n_new - 1u, d), m = __ldg(T.map + k);
            if (m == VB_RCMP_NONE) {
                dm_or_box(mask, now, wt, ht, lane);
                return;
            }
            od = __ldg(T.old_pre + m) + (d - __ldg(T.new_pre + k));
        } else {
            const uint32_t t = new_draws - d; // 1 for the last END_CLIP
            if (t > old_draws - old_end) {
                dm_or_box(mask, now, wt, ht, lane);
                return;
            }
            od = old_draws - t;
        }
        const VbBbox4 was = old_boxes[od];
        if (rc_same_box(was, now)) return;
        dm_or_box(mask, was, wt, ht, lane);
        dm_or_box(mask, now, wt, ht, lane);
        return;
    }
    const uint32_t d = w - new_draws;
    if (d >= old_draws) return;
    // a matched old draw object is handled with its counterpart above
    const bool gone = d < old_end ? __ldg(T.unmatched + cp_find(T.old_pre, 0u, n_old - 1u, d)) != 0u : old_draws - d > new_draws - new_end;
    if (gone) dm_or_box(mask, old_boxes[d], wt, ht, lane);
}

extern "C" uint32_t vb_launch_recompose_damage(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    const VbDamage &D = b.dmg;
    if (!D.tables) return 0u;
    const uint32_t warps = D.new_draws + D.old_draws, per = RC_THREADS / 32u;
    if (warps == 0u) return 0u;
    k_recompose_damage<<<(warps + per - 1u) / per, RC_THREADS, 0, st>>>(b.draw_bboxes, D.old_boxes, D.tables, D.n_old, D.n_new, D.old_draws,
                                                                        D.new_draws, D.mask, cfg.width_in_tiles, cfg.height_in_tiles);
    return 1u;
}

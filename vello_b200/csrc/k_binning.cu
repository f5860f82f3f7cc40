// k_binning.cu -- draw-object bounding boxes -> 256x256 px bins.
//
// Reference: vello_shaders/shader/binning.wgsl:55-203, CPU twin cpu/binning.rs.
// Output layout is the reference's: draw_bboxes[draw], bin_headers[partition][bin]{count,offset},
// bin_data (appended after `info` in info_bin_data). Within one (partition, bin) chunk the draw
// indices are ascending; chunk offsets come from an atomic bump allocator (as in the WGSL, but one
// allocation per partition and bin block, with its chunks in bin order), so chunk ORDER in bin_data is
// not deterministic -- consumers only go through the headers.
// Extension: the bin-row window [win_by0, win_by1) restricts binning to this GPU's stripe.
#include "vb_device.cuh"
#include "vb_stages.h"

#define BN_THREADS 256
#define BN_N_SLICE 8
#define BN_N_SUBSLICE 4

__global__ void __launch_bounds__(BN_THREADS)
k_binning(VbConfig cfg, const VbDrawMonoid *__restrict__ draw_monoids, const VbPathBbox *__restrict__ path_bbox_buf,
          const VbBbox4 *__restrict__ clip_bbox_buf, VbBbox4 *intersected_bbox, VbBump *bump, uint32_t *info_bin_data,
          VbBinHeader *bin_header) {
    __shared__ uint32_t sh_bitmaps[BN_N_SLICE][VB_N_TILE];
    __shared__ uint32_t sh_count[BN_N_SUBSLICE][VB_N_TILE];
    __shared__ uint32_t sh_chunk_offset[VB_N_TILE];
    __shared__ uint32_t sh_scan[BN_THREADS / 32 + 1];
    const uint32_t lid = threadIdx.x;
    for (int i = 0; i < BN_N_SLICE; i++) sh_bitmaps[i][lid] = 0u;
    if (bump->failed & VB_STAGE_FLATTEN) return; // uniform
    __syncthreads();

    const uint32_t element_ix = blockIdx.x * BN_THREADS + lid;
    int32_t x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    const float SX = 1.0f / 256.0f, SY = 1.0f / 256.0f;
    if (element_ix < cfg.layout.n_draw_objects) {
        VbDrawMonoid dm = draw_monoids[element_ix];
        VbBbox4 cb = {-1e9f, -1e9f, 1e9f, 1e9f};
        if (dm.clip_ix > 0u) cb = clip_bbox_buf[min(dm.clip_ix - 1u, cfg.layout.n_clips - 1u)];
        VbPathBbox pb = path_bbox_buf[dm.path_ix];
        VbBbox4 b = {fmaxf(cb.x0, (float)pb.x0), fmaxf(cb.y0, (float)pb.y0), fminf(cb.x1, (float)pb.x1), fminf(cb.y1, (float)pb.y1)};
        intersected_bbox[element_ix] = b;
        if (b.x0 < b.x1 && b.y0 < b.y1) {
            x0 = vb_f2i_sat(floorf(b.x0 * SX));
            y0 = vb_f2i_sat(floorf(b.y0 * SY));
            x1 = vb_f2i_sat(ceilf(b.x1 * SX));
            y1 = vb_f2i_sat(ceilf(b.y1 * SY));
        }
    }
    const int32_t width_in_bins = (int32_t)((cfg.width_in_tiles + VB_N_TILE_X - 1u) / VB_N_TILE_X);
    const int32_t height_in_bins = (int32_t)((cfg.height_in_tiles + VB_N_TILE_Y - 1u) / VB_N_TILE_Y);
    const uint32_t n_bins = (uint32_t)(width_in_bins * height_in_bins) * cfg.n_cells;
    const uint32_t aligned_n_bins = (n_bins + VB_N_TILE - 1u) & ~(VB_N_TILE - 1u);
    x0 = vb_clampi(x0, 0, width_in_bins);
    x1 = vb_clampi(x1, 0, width_in_bins);
    y0 = vb_clampi(y0, (int32_t)cfg.win_by0, (int32_t)cfg.win_by1);
    y1 = vb_clampi(y1, (int32_t)cfg.win_by0, (int32_t)cfg.win_by1);
    if (x0 == x1) y1 = y0;
    // Batch: the draw's rectangle, clamped to its own cell above, moves down to the cell's bin rows; this partition walks only
    // the 256-bin blocks that hold bins of the cells its draws belong to (coarse reads no header of any other block).
    uint32_t block_lo = 0u, block_hi = n_bins;
    if (cfg.n_cells > 1u) {
        const uint32_t last_ix = min(blockIdx.x * BN_THREADS + BN_THREADS, cfg.layout.n_draw_objects) - 1u;
        const uint32_t c_first = vb_cell_of(cfg, blockIdx.x * BN_THREADS), c_last = vb_cell_of(cfg, last_ix);
        const uint32_t cell_bins = (uint32_t)(width_in_bins * height_in_bins);
        block_lo = (c_first * cell_bins) & ~(VB_N_TILE - 1u);
        block_hi = (c_last + 1u) * cell_bins;
        const int32_t row0 = (int32_t)(vb_cell_of(cfg, min(element_ix, cfg.layout.n_draw_objects - 1u)) * (uint32_t)height_in_bins);
        y0 += row0;
        y1 += row0;
    }
    const int32_t y0_width = y0 * width_in_bins, y1_width = y1 * width_in_bins;
    const uint32_t my_slice = lid / 32u, my_mask = 1u << (lid & 31u);

    uint32_t next_block = block_lo + VB_N_TILE;
    for (uint32_t block_start = block_lo; block_start < block_hi;) {
        for (int32_t y_offset = y0_width; y_offset < y1_width; y_offset += width_in_bins) {
            uint32_t start_bin = max((uint32_t)(y_offset + x0), block_start);
            uint32_t end_bin = min((uint32_t)(y_offset + x1), next_block);
            for (uint32_t bin_ix = start_bin; bin_ix < end_bin; bin_ix++) atomicOr(&sh_bitmaps[my_slice][bin_ix - block_start], my_mask);
        }
        __syncthreads();
        const uint32_t cur_bin_ix = block_start + lid;
        uint32_t element_count = 0u;
        for (uint32_t i = 0u; i < BN_N_SUBSLICE; i++) {
            element_count += __popc(sh_bitmaps[i * 2u][lid]);
            uint32_t lo = element_count;
            element_count += __popc(sh_bitmaps[i * 2u + 1u][lid]);
            sh_count[i][lid] = lo | (element_count << 16);
        }
        // the block's chunks are one allocation, laid out in bin order: one atomic per block instead of one per bin on the
        // same counter (a block of map-like draws reaches most of its 256 bins)
        uint32_t block_total;
        uint32_t chunk_offset = vb_block_excl_scan(element_count, sh_scan, &block_total);
        if (lid == 0u) sh_scan[0] = block_total != 0u ? atomicAdd(&bump->binning, block_total) : 0u;
        __syncthreads();
        chunk_offset = element_count != 0u ? sh_scan[0] + chunk_offset : 0u;
        if (element_count != 0u && chunk_offset + element_count > cfg.binning_size) {
            chunk_offset = 0u;
            atomicOr(&bump->failed, VB_STAGE_BINNING);
        }
        sh_chunk_offset[lid] = chunk_offset;
        const uint32_t header_ix = blockIdx.x * aligned_n_bins + cur_bin_ix;
        if (cur_bin_ix < aligned_n_bins) {
            VbBinHeader h = {element_count, chunk_offset};
            bin_header[header_ix] = h;
        }
        __syncthreads();
        const bool failed = (bump->failed & VB_STAGE_BINNING) != 0u;
        for (int32_t y_offset = y0_width; y_offset < y1_width; y_offset += width_in_bins) {
            uint32_t start_bin = max((uint32_t)(y_offset + x0), block_start);
            uint32_t end_bin = min((uint32_t)(y_offset + x1), next_block);
            for (uint32_t bin_ix = start_bin; bin_ix < end_bin; bin_ix++) {
                uint32_t sh_bin_ix = bin_ix - block_start;
                uint32_t out_mask = sh_bitmaps[my_slice][sh_bin_ix];
                uint32_t idx = __popc(out_mask & (my_mask - 1u));
                if (my_slice > 0u) {
                    uint32_t count_ix = my_slice - 1u;
                    uint32_t packed = sh_count[count_ix / 2u][sh_bin_ix];
                    idx += (packed >> (16u * (count_ix & 1u))) & 0xffffu;
                }
                uint32_t off = sh_chunk_offset[sh_bin_ix] + idx;
                if (!failed && off < cfg.binning_size) info_bin_data[cfg.layout.bin_data_start + off] = element_ix;
            }
        }
        block_start = next_block;
        if (next_block < block_hi) {
            __syncthreads();
            for (int i = 0; i < BN_N_SLICE; i++) sh_bitmaps[i][lid] = 0u;
            __syncthreads();
            next_block += VB_N_TILE;
        }
    }
}

extern "C" uint32_t vb_launch_binning(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    uint32_t n = cfg.layout.n_draw_objects;
    if (n == 0) return 0;
    k_binning<<<(n + BN_THREADS - 1) / BN_THREADS, BN_THREADS, 0, st>>>(cfg, b.draw_monoids, b.path_bboxes, b.clip_bboxes, b.draw_bboxes, b.bump(),
                                                                       b.info_bin_data, b.bin_headers);
    return 1;
}

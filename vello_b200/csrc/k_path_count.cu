// k_path_count.cu -- line -> tile DDA: backdrop deltas, per-tile segment counts, crossing worklist.
//
// Reference: vello_shaders/shader/path_count.wgsl:51-202 (+ path_count_setup.wgsl), CPU twin
// cpu/path_count.rs; the conservative line walk is Appendix C.1 of SURVEY.md. Comparisons follow
// the WGSL where the CPU twin differs (`s1.y <= bbox.y`, `max(s0.x,s1.x) <= bbox.x`); WGSL
// round() is ties-to-even -> rintf.
//
// Design: (i) no indirect dispatch -- the grid is sized from the arena capacity and reads bump.lines on the device.
// (ii) Lines are taken PC_LINES = PC_LPT x PC_THREADS at a time (a step): thread t sets up lines t, PC_THREADS + t, ... A
// frame too small to give every resident CTA (PC_MINB per SM) a step of PC_LINES is taken PC_THREADS at a time instead, so
// that its lines still spread over all the SMs (512 always cost the 1920 x 1080 tiger 2.5 us, 26 %). The per-line phase is
// the WGSL's, one thread per line: setup, box cull, imin / imax, and the backdrop of the rows left of the path's box (0.3 %
// of the headline frame's lines have such rows, 1 or 2 each). The seg_counts allocation is aggregated per CTA: one
// atomicAdd per step. Same-address atomics serialise, and they bound this kernel: one more per 256 lines made it 51 us
// slower on the headline frame; reserving per 512 lines instead of per 256 took the stage from 155 to 127 us, per 768 to 121
// us (per 1024 the line state needs more shared memory than 6 CTAs per SM allow: 138 us at 4; per-warp aggregation left
// ~133 k atomics a frame and was slower still). The line state is 45 B per line, with the signs and the top-edge test of
// step 0 in one flags byte, so that 768 lines fit 6 CTAs per SM.
// (iii) The crossing phase spreads the step's crossings over all its threads instead of walking each line in a serial
// loop: the state the walk needs goes to shared memory, and item k of the step's exclusive scan (in line order) is
// crossing i = imin + k - excl of the line found by a binary search over the scan. z and the previous z are recomputed from
// i exactly as the serial loop produced them, so every (line, i) record is bit-identical and lands at cta_base + k, where
// the serial loop put it. A line of 28 crossings no longer holds its CTA for 28 dependent atomic round trips.
// (iv) Slots are reserved once per (warp, tile): __match_any_sync groups the lanes of a tile, the first takes
// popc(peers) slots and the others theirs in lane order, so a tile's slots stay a permutation of 0..count-1. Backdrop
// updates are fire-and-forget RED operations (aggregating the top-edge ones per warp as well measured no faster).
// Per-tile slot order (seg_within_slice) is atomic-order dependent exactly as in the reference.
// Measured no faster on the headline frame: staging the next lines in shared memory with a bulk copy (10-15 us slower), a
// persistent grid, spreading the left-of-box rows over the CTA like the crossings, and taking the reservation's round
// trip off the barrier.
#include "vb_device.cuh"
#include "vb_stages.h"

#ifndef PC_THREADS
#define PC_THREADS 256
#endif
#ifndef PC_MINB
#define PC_MINB 6
#endif
#ifndef PC_LPT
#define PC_LPT 3 // lines per thread in a step
#endif
#define PC_LINES (PC_LPT * PC_THREADS) // lines per step of a CTA, whose crossings take one seg_counts reservation
#define PC_SEARCH (PC_LPT > 2 ? 512 : PC_LINES / 2) // the largest power of two below PC_LINES: the search's first step
static_assert(PC_SEARCH < PC_LINES && 2 * PC_SEARCH >= PC_LINES, "PC_SEARCH");
// PcLines::flags
#define PC_NEG_DELTA 1u // the line goes up: its backdrop delta is -1 (else +1)
#define PC_NEG_X 2u     // x_sign is -1 (else +1)
#define PC_TOP_AT_0 4u  // step 0 of the walk is a top edge (y0 == s0y)
#ifndef PC_CTAS_PER_SM
#define PC_CTAS_PER_SM 16
#endif
#define ONE_MINUS_ULP 0.99999994f
#define ROBUST_EPSILON 2e-7f
#define TILE_SCALE 0.0625f

// Phase timing (tools/path_count_phases.py), off by default: built with -DVB_PATH_COUNT_PHASES, thread 0 of every CTA reads
// %globaltimer after a CTA-wide barrier at the end of each phase (of each line of a thread, then of each step) and adds the
// time to the phase's total. Per CTA (row blockIdx.x): start, end, then the ns spent in line loads and set-up, in the
// left-of-box backdrop, in the scan and seg_counts reservation and in the crossing phase, the SM, the steps it took.
// pc_ph_rows counts lines by their left-of-box rows (the last bin: PC_PH_ROWS - 1 or more); its updates are kept out of
// every phase. vb_debug_path_count_phases copies both tables out and clears them.
#ifdef VB_PATH_COUNT_PHASES
#define PC_PH_CTAS 65536u
#define PC_PH_ROWS 64u
__device__ unsigned long long pc_ph_cta[PC_PH_CTAS][8];
__device__ unsigned long long pc_ph_rows[PC_PH_ROWS];
__device__ __forceinline__ unsigned long long pc_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define PC_STAMP(k)                                    \
    do {                                               \
        __syncthreads();                               \
        if (threadIdx.x == 0u) {                       \
            const unsigned long long n_ = pc_now();    \
            ph_##k += n_ - ph_t;                       \
            ph_t = n_;                                 \
        }                                              \
    } while (0)
// the rows histogram: counted in shared memory, outside the timed phases (the clock restarts after it)
#define PC_COUNT_ROWS(rows, valid)                                                \
    do {                                                                          \
        __syncthreads();                                                          \
        if (valid) atomicAdd(&sh_ph_rows[min((uint32_t)(rows), PC_PH_ROWS - 1u)], 1u); \
        __syncthreads();                                                          \
        if (threadIdx.x == 0u) ph_t = pc_now();                                   \
    } while (0)
extern "C" int vb_debug_path_count_phases(void *cta, size_t cta_bytes, void *rows, size_t rows_bytes) {
    if (cudaMemcpyFromSymbol(cta, pc_ph_cta, min(cta_bytes, sizeof pc_ph_cta)) != cudaSuccess) return 1;
    if (cudaMemcpyFromSymbol(rows, pc_ph_rows, min(rows_bytes, sizeof pc_ph_rows)) != cudaSuccess) return 1;
    void *p_cta, *p_rows;
    if (cudaGetSymbolAddress(&p_cta, pc_ph_cta) != cudaSuccess || cudaGetSymbolAddress(&p_rows, pc_ph_rows) != cudaSuccess) return 1;
    if (cudaMemset(p_cta, 0, sizeof pc_ph_cta) != cudaSuccess) return 1;
    return cudaMemset(p_rows, 0, sizeof pc_ph_rows) != cudaSuccess;
}
#else
#define PC_STAMP(k) do {} while (0)
#define PC_COUNT_ROWS(rows, valid) do {} while (0)
#endif

// What the crossing phase needs of each line of the current PC_LINES-line step, as structure-of-arrays (34 KB).
// Entries of lines without crossings are stale; the search over excl never lands on them.
struct PcLines {
    float a[PC_LINES], b[PC_LINES], x0[PC_LINES], y0[PC_LINES];
    int32_t bx0[PC_LINES], by0[PC_LINES], bx1[PC_LINES], by1[PC_LINES];
    uint32_t path_tiles[PC_LINES], imin[PC_LINES], excl[PC_LINES];
    uint8_t flags[PC_LINES];
};

__global__ void __launch_bounds__(PC_THREADS, PC_MINB)
k_path_count(VbConfig cfg, VbBump *bump, const VbLineSoup *__restrict__ lines, const VbPath *__restrict__ paths, VbTile *tile,
             VbSegmentCount *seg_counts, uint32_t pair_min) {
    __shared__ uint32_t sh_scan[PC_LPT][PC_THREADS / 32 + 1];
    __shared__ uint32_t sh_base;
    __shared__ PcLines sh;
    if (bump->failed != 0u) return;
    const uint32_t lane = vb_lane(), warp = threadIdx.x >> 5;
    const uint32_t n_lines = min(bump->lines, cfg.lines_size);
#ifdef VB_PATH_COUNT_PHASES
    __shared__ uint32_t sh_ph_rows[PC_PH_ROWS];
    if (threadIdx.x < PC_PH_ROWS) sh_ph_rows[threadIdx.x] = 0u;
    const unsigned long long ph_start = pc_now();
    unsigned long long ph_t = ph_start, ph_load = 0u, ph_backdrop = 0u, ph_scan = 0u, ph_cross = 0u, ph_steps = 0u;
#endif
    // a frame of fewer than pair_min lines, too few steps of PC_LINES to fill the GPU, takes PC_THREADS at a time
    const uint32_t lps = n_lines >= pair_min ? PC_LINES : PC_THREADS;
    for (uint32_t line_base = blockIdx.x * lps; line_base < n_lines; line_base += gridDim.x * lps) {
        // per-line phase: thread t takes lines t, PC_THREADS + t, ... of the step; each line's crossing count waits in
        // sh.excl until the scan
#pragma unroll 1
        for (uint32_t t = threadIdx.x; t < lps; t += PC_THREADS) {
            const uint32_t line_ix = line_base + t;
            bool active = line_ix < n_lines;
            uint32_t imin = 0u, imax = 0u;
            float a = 0.f, b = 0.f, x0 = 0.f, y0 = 0.f, x_sign = 1.f, s0y = 0.f;
            int32_t bx0 = 0, by0 = 0, bx1 = 0, by1 = 0, stride = 0, delta = 0, ymin = 0, ymax = 0;
            uint32_t path_tiles = 0;
            if (active) {
                const uint2 *lp = reinterpret_cast<const uint2 *>(lines + line_ix);
                uint2 w0 = __ldg(lp), w1 = __ldg(lp + 1), w2 = __ldg(lp + 2);
                const uint32_t path_ix = w0.x;
                const float p0x = __uint_as_float(w1.x), p0y = __uint_as_float(w1.y);
                const float p1x = __uint_as_float(w2.x), p1y = __uint_as_float(w2.y);
                const bool is_down = p1y >= p0y;
                const float xy0x = is_down ? p0x : p1x, xy0y = is_down ? p0y : p1y;
                const float xy1x = is_down ? p1x : p0x, xy1y = is_down ? p1y : p0y;
                const float s0x = xy0x * TILE_SCALE, s1x = xy1x * TILE_SCALE, s1y = xy1y * TILE_SCALE;
                s0y = xy0y * TILE_SCALE;
                const uint32_t count_x = vb_span(s0x, s1x) - 1u;
                const uint32_t count = count_x + vb_span(s0y, s1y);
                const float dx = fabsf(s1x - s0x);
                const float dy = s1y - s0y;
                if (dx + dy == 0.0f) active = false;
                if (dy == 0.0f && floorf(s0y) == s0y) active = false;
                if (active && path_ix >= cfg.layout.n_draw_objects) active = false;
                if (active) {
                    const float idxdy = 1.0f / (dx + dy);
                    a = dx * idxdy;
                    const bool is_positive_slope = s1x >= s0x;
                    x_sign = is_positive_slope ? 1.0f : -1.0f;
                    const float xt0 = floorf(s0x * x_sign);
                    const float c = s0x * x_sign - xt0;
                    y0 = floorf(s0y);
                    const float ytop = (s0y == s1y) ? ceilf(s0y) : y0 + 1.0f;
                    b = fminf((dy * c + dx * (ytop - s0y)) * idxdy, ONE_MINUS_ULP);
                    const float robust_err = floorf(a * ((float)count - 1.0f) + b) - (float)count_x;
                    if (robust_err != 0.0f) a -= ROBUST_EPSILON * vb_signf(robust_err);
                    x0 = xt0 * x_sign + (is_positive_slope ? 0.0f : -1.0f);
                    const VbPath path = paths[path_ix];
                    bx0 = (int32_t)path.bbox[0]; by0 = (int32_t)path.bbox[1]; bx1 = (int32_t)path.bbox[2];
                    by1 = (int32_t)path.bbox[3];
                    path_tiles = path.tiles;
                    const float xmin = fminf(s0x, s1x);
                    stride = bx1 - bx0;
                    if (s0y >= (float)by1 || s1y <= (float)by0 || xmin >= (float)bx1 || stride == 0) {
                        active = false;
                    } else {
                        if (s0y < (float)by0) {
                            float iminf = rintf(((float)by0 - y0 + b - a) / (1.0f - a)) - 1.0f;
                            if (y0 + iminf - floorf(a * iminf + b) < (float)by0) iminf += 1.0f;
                            imin = vb_f2u_sat(iminf);
                        }
                        imax = count;
                        if (s1y > (float)by1) {
                            float imaxf = rintf(((float)by1 - y0 + b - a) / (1.0f - a)) - 1.0f;
                            if (y0 + imaxf - floorf(a * imaxf + b) < (float)by1) imaxf += 1.0f;
                            imax = vb_f2u_sat(imaxf);
                        }
                        delta = is_down ? -1 : 1;
                        if (fmaxf(s0x, s1x) <= (float)bx0) {
                            ymin = vb_f2i_sat(ceilf(s0y));
                            ymax = vb_f2i_sat(ceilf(s1y));
                            imax = imin;
                        } else {
                            const float fudge = is_positive_slope ? 0.0f : 1.0f;
                            if (xmin < (float)bx0) {
                                float f = rintf((x_sign * ((float)bx0 - x0) - b + fudge) / a);
                                if ((x0 + x_sign * floorf(a * f + b) < (float)bx0) == is_positive_slope) f += 1.0f;
                                const int32_t ynext = vb_f2i_sat(y0 + f - floorf(a * f + b) + 1.0f);
                                if (is_positive_slope) {
                                    if (vb_f2u_sat(f) > imin) {
                                        ymin = vb_f2i_sat(y0 + ((y0 == s0y) ? 0.0f : 1.0f));
                                        ymax = ynext;
                                        imin = vb_f2u_sat(f);
                                    }
                                } else {
                                    if (vb_f2u_sat(f) < imax) {
                                        ymin = ynext;
                                        ymax = vb_f2i_sat(ceilf(s1y));
                                        imax = vb_f2u_sat(f);
                                    }
                                }
                            }
                            if (fmaxf(s0x, s1x) > (float)bx1) {
                                float f = rintf((x_sign * ((float)bx1 - x0) - b + fudge) / a);
                                if ((x0 + x_sign * floorf(a * f + b) < (float)bx1) == is_positive_slope) f += 1.0f;
                                if (is_positive_slope) imax = min(imax, vb_f2u_sat(f));
                                else imin = max(imin, vb_f2u_sat(f));
                            }
                        }
                        imax = max(imin, imax);
                        ymin = max(ymin, by0);
                        ymax = min(ymax, by1);
                    }
                }
            }
            PC_STAMP(load);
            for (int32_t y = ymin; y < ymax; y++) {
                const int32_t base = (int32_t)path_tiles + (y - by0) * stride;
                atomicAdd(&tile[base].backdrop, delta);
            }
            PC_STAMP(backdrop);
            PC_COUNT_ROWS(max(ymax - ymin, 0), line_ix < n_lines);
            const uint32_t n = active ? imax - imin : 0u;
            sh.excl[t] = n;
            if (n != 0u) {
                sh.a[t] = a; sh.b[t] = b; sh.x0[t] = x0; sh.y0[t] = y0;
                sh.bx0[t] = bx0; sh.by0[t] = by0; sh.bx1[t] = bx1; sh.by1[t] = by1;
                sh.flags[t] = (uint8_t)((delta < 0 ? PC_NEG_DELTA : 0u) | (x_sign < 0.0f ? PC_NEG_X : 0u) | (y0 == s0y ? PC_TOP_AT_0 : 0u));
                sh.path_tiles[t] = path_tiles; sh.imin[t] = imin;
            }
        }
        // exclusive scan of the step's crossing counts, in line order (segment u holds lines u x PC_THREADS .. + PC_THREADS - 1),
        // and the CTA-aggregated worklist allocation: one same-address atomic per step, taken by the lane that has the
        // step's total. These atomics serialise: one more per 256 lines measured +51 us on the headline frame.
        uint32_t n[PC_LPT], incl[PC_LPT];
#pragma unroll
        for (uint32_t u = 0; u < PC_LPT; u++) {
            n[u] = u * PC_THREADS < lps ? sh.excl[u * PC_THREADS + threadIdx.x] : 0u;
            incl[u] = vb_warp_incl_scan(n[u]);
            if (lane == 31u) sh_scan[u][warp] = incl[u];
        }
        __syncthreads();
        if (warp == 0u) {
            uint32_t run = 0u; // the segments before u
#pragma unroll
            for (uint32_t u = 0; u < PC_LPT; u++) {
                const uint32_t v = lane < PC_THREADS / 32 ? sh_scan[u][lane] : 0u;
                const uint32_t c = vb_warp_incl_scan(v);
                if (lane < PC_THREADS / 32) sh_scan[u][lane] = run + c - v;
                run += __shfl_sync(VB_FULL, c, 31);
            }
            if (lane == 31u) {
                sh_scan[0][PC_THREADS / 32] = run;
                if (run != 0u) sh_base = atomicAdd(&bump->seg_counts, run);
            }
        }
        __syncthreads();
        const uint32_t cta_total = sh_scan[0][PC_THREADS / 32];
#pragma unroll
        for (uint32_t u = 0; u < PC_LPT; u++) sh.excl[u * PC_THREADS + threadIdx.x] = sh_scan[u][warp] + incl[u] - n[u];
        __syncthreads(); // sh.excl and sh_base are complete; sh_scan is free for the next step
        PC_STAMP(scan);
        const uint32_t cta_base = sh_base;
        // crossing phase: item k of the CTA is crossing i = imin + k - excl of the last line whose excl <= k. Whole warps
        // step together (k0 is warp-uniform), so the warp-wide slot reservation below sees every lane.
        for (uint32_t k0 = threadIdx.x & ~31u; k0 < cta_total; k0 += PC_THREADS) {
            const uint32_t k = k0 + lane;
            bool inside = false, top_edge = false;
            int32_t tix = 0, x = 0, bx1j = 0, dj = 0;
            uint32_t j = 0, i = 0;
            if (k < cta_total) {
#pragma unroll
                for (uint32_t step = PC_SEARCH; step != 0u; step >>= 1)
                    if (j + step < PC_LINES && sh.excl[j + step] <= k) j += step;
                const float aj = sh.a[j], bj = sh.b[j], y0j = sh.y0[j];
                const uint32_t iminj = sh.imin[j];
                i = iminj + (k - sh.excl[j]);
                // the serial walk's carried last_z: at imin it started from imin - 1 in f32, later it is the previous z
                const float z = floorf(aj * (float)i + bj);
                const float last_z = (i == iminj) ? floorf(aj * ((float)iminj - 1.0f) + bj) : floorf(aj * (float)(i - 1u) + bj);
                const int32_t y = vb_f2i_sat(y0j + (float)i - z);
                const uint32_t fl = sh.flags[j];
                x = vb_f2i_sat(sh.x0[j] + ((fl & PC_NEG_X) ? -1.0f : 1.0f) * z);
                const int32_t bx0j = sh.bx0[j], by0j = sh.by0[j], by1j = sh.by1[j];
                bx1j = sh.bx1[j];
                dj = (fl & PC_NEG_DELTA) ? -1 : 1;
                tix = (int32_t)sh.path_tiles[j] + (y - by0j) * (bx1j - bx0j) - bx0j;
                top_edge = (i == 0u) ? (fl & PC_TOP_AT_0) != 0u : (last_z == z);
                // far from the frame the f32 walk can step off the path's tile box: such a crossing touches no tile
                inside = x >= bx0j && x < bx1j && y >= by0j && y < by1j;
            }
            if (inside && top_edge && x + 1 < bx1j) atomicAdd(&tile[tix + x + 1].backdrop, dj);
            // one slot fetch per (warp, tile): the leader takes popc(peers) slots and hands them out in lane order, so a
            // tile's slots stay a permutation of 0..count-1
            const uint32_t inmask = __ballot_sync(VB_FULL, inside);
            uint32_t peers = 0u, old = 0u;
            int leader = (int)lane;
            if (inside) {
                peers = __match_any_sync(inmask, tix + x);
                leader = __ffs((int)peers) - 1;
                if ((int)lane == leader) old = atomicAdd(&tile[tix + x].segment_count_or_ix, (uint32_t)__popc(peers));
            }
            old = __shfl_sync(VB_FULL, old, leader);
            if (k < cta_total) {
                const uint32_t seg_within_slice = inside ? old + (uint32_t)__popc(peers & ((1u << lane) - 1u)) : VB_SEG_OUTSIDE;
                const uint32_t seg_ix = cta_base + k;
                if (seg_ix < cfg.seg_counts_size) {
                    VbSegmentCount sc = {line_base + j, i, seg_within_slice};
                    seg_counts[seg_ix] = sc;
                }
            }
        }
        PC_STAMP(cross);
#ifdef VB_PATH_COUNT_PHASES
        ph_steps++;
#endif
        __syncthreads(); // the next step overwrites sh
    }
#ifdef VB_PATH_COUNT_PHASES
    __syncthreads();
    if (threadIdx.x < PC_PH_ROWS && sh_ph_rows[threadIdx.x] != 0u) atomicAdd(&pc_ph_rows[threadIdx.x], (unsigned long long)sh_ph_rows[threadIdx.x]);
    if (threadIdx.x == 0u && blockIdx.x < PC_PH_CTAS) {
        uint32_t smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        unsigned long long *row = pc_ph_cta[blockIdx.x];
        row[0] = ph_start; row[1] = pc_now(); row[2] = ph_load; row[3] = ph_backdrop; row[4] = ph_scan; row[5] = ph_cross;
        row[6] = smid; row[7] = ph_steps;
    }
#endif
}

// The seg_counts overflow check (the WGSL does it at the top of coarse) lives at the top of k_backdrop, the next kernel.

// The grid comes from the lines capacity (at most 16 CTAs per SM); the kernel strides over the count read on the device.
extern "C" uint32_t vb_launch_path_count(const VbConfig &cfg, const VbFrameBufs &b, cudaStream_t st) {
    const uint64_t blocks = ((uint64_t)cfg.lines_size + PC_THREADS - 1) / PC_THREADS, most = (uint64_t)b.sm_count * PC_CTAS_PER_SM;
    const uint32_t grid = (uint32_t)(blocks < most ? blocks : most);
    if (grid == 0) return 0;
    // steps of PC_LINES once they fill every SM's PC_MINB resident CTAs at least once
    const uint32_t pair_min = (uint32_t)b.sm_count * PC_MINB * PC_LINES;
    k_path_count<<<grid, PC_THREADS, 0, st>>>(cfg, b.bump(), b.lines, b.paths, b.tiles, b.seg_counts, pair_min);
    return 1;
}

// deodr_b200: the adjoint pass (replaces renderScene_B, DR.h:2903-3135) - kernels + their launch sequence.
//   k_raster_bwd + k_finalize_edges       (aux)  edge tiles: replay, reverse sweep, per-edge plane adjoints
//   k_interior_bwd                        (aux)  pixels of large triangles elsewhere
//   k_small_tri_bwd                              triangle-parallel adjoint of the small triangles
//   k_background_bwd                      (aux)  background gradient outside the edge tiles (only when asked for)
// Everything strides over device-side counts left by the forward pass of the same view slot (kernels.cu); a forward
// that overflowed its plan makes these kernels return at once (nothing is accumulated).
#include <cstdlib>
#include <cstring>

// -DDEODR_SMALLBWD_PHASE_CLOCKS (measurement builds only, scripts/small_bwd_phases.py): every thread of k_small_tri_bwd
// adds the clock64() cycles it spent in each phase of small_triangle_adjoint (phases.h: SB_*) to g_smallbwd_clocks,
// summed per warp first; the slots after the phases count the threads and the threads that own no pixel (hidden
// triangles), and g_smallbwd_hist counts the threads by pixels owned (0..64, before the edge-tile masking).  Read back
// (and cleared) with deodr_b200_small_bwd_phase_clocks.
#ifdef DEODR_SMALLBWD_PHASE_CLOCKS
constexpr int SB_SLOTS = 5 + 2;  // SB_PHASES, threads, hidden
constexpr int SB_HIST = 65;
__device__ unsigned long long g_smallbwd_clocks[SB_SLOTS];
__device__ unsigned int g_smallbwd_hist[SB_HIST];
struct SmallBwdClocks {
    unsigned int acc[5];
    int owned;
    long long prev;
    __host__ __device__ SmallBwdClocks() : acc{}, owned(0), prev(0) {
#if defined(__CUDA_ARCH__)
        prev = clock64();
#endif
    }
    __host__ __device__ void lap(int phase) {
#if defined(__CUDA_ARCH__)
        const long long now = clock64();
        acc[phase] += (unsigned int)(now - prev);
        prev = now;
#endif
    }
    __host__ __device__ void set_owned(unsigned long long mine) {
#if defined(__CUDA_ARCH__)
        owned = __popcll(mine);
#endif
    }
    __host__ __device__ void done() const {
#if defined(__CUDA_ARCH__)
        const unsigned int m = __activemask(), leader = __ffs(m) - 1, lane = threadIdx.x & 31;
#pragma unroll
        for (int k = 0; k < 5; k++) {
            const unsigned int v = __reduce_add_sync(m, acc[k]);
            if (lane == leader) atomicAdd(&g_smallbwd_clocks[k], (unsigned long long)v);
        }
        const unsigned int hidden = __popc(__ballot_sync(m, owned == 0));
        if (lane == leader) {
            atomicAdd(&g_smallbwd_clocks[5], (unsigned long long)__popc(m));
            atomicAdd(&g_smallbwd_clocks[6], (unsigned long long)hidden);
        }
        const unsigned int same = __match_any_sync(m, owned);
        if (lane == (unsigned int)(__ffs(same) - 1)) atomicAdd(&g_smallbwd_hist[owned], (unsigned int)__popc(same));
#endif
    }
};
#define SMALLBWD_START SmallBwdClocks sb_clocks_
#define SMALLBWD_LAP(phase) sb_clocks_.lap(phase)
#define SMALLBWD_OWNED(mine) sb_clocks_.set_owned(mine)
#define SMALLBWD_DONE sb_clocks_.done()
#endif

#include "kernels_common.cuh"

// antialiase_error adjoint, pixels outside every edge band: image_b = -2 (obs - image) err_b (DR.h:3054-3060), consumed
// unchanged by the interior adjoint kernels.
__global__ void k_error_image_b(const float *image, const float *obs, const float *err_b, float *image_b, size_t pixels,
                                int C, const int *scal) {
    if (scal[SC_OVERFLOW]) return;
    const size_t n = pixels * C;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        image_b[i] = (float)(-2.0 * ((double)obs[i] - (double)image[i]) * (double)err_b[i / C]);
}

// Background gradient, one pixel per thread, called by every thread of the CTA (NTHREADS of them): the pixel's colour
// adjoint g goes into background_image_b with one RED per channel (views may share the buffer); for background_color_b
// it is summed over the CTA first (per-warp shuffles, fp64 partials per warp in `sh`), then added with one atomic per
// channel per CTA.  acc[] is the thread's own sum (k_background_bwd: over the pixels of its grid-stride loop).
template <int MAXC, int NTHREADS>
static __device__ __forceinline__ void background_color_sum(int C, const float *acc, float *color_b,
                                                            double (*sh)[MAXC]) {
    const int lane = (int)(threadIdx.x & 31), warp = (int)(threadIdx.x >> 5);
#pragma unroll
    for (int c = 0; c < MAXC; c++) {
        if (c < C) {
            double x = (double)acc[c];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
            if (lane == 0) sh[warp][c] = x;
        }
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += NTHREADS) {
        double total = 0.0;
#pragma unroll
        for (int w = 0; w < NTHREADS / 32; w++) total += sh[w][c];
        atomicAdd(color_b + c, (float)total);
    }
}

// Adjoint of the tiles that have silhouette edges: fp64 forward replay of the tile's ordered edges, reverse sweep with
// un-blend (DR.h:1738), per-edge plane adjoints as fp64 moments, then the interior adjoint of all the tile's pixels with
// what is left of their colour adjoint.  ERR: the antialiase_error variant (DR.h:2296-2336, 2542-2576); compat = the
// reference's dropped row term reproduced (phase_edge_adjoint_error).  BG: what is left of the colour adjoint of the
// pixels that show the background (image_b times the transparencies of the edges over them; ERR: the residual's
// adjoint there) also goes to the background gradient `bg` (unused by the other instances).
// (register budgets are pinned: the allocator's own choice moved 64 -> 80 on an unrelated signature change)
template <int MAXC, bool TEX, bool ERR, bool BG>
__global__ void __launch_bounds__(EDGE_NT, DEODR_EDGE_MIN_CTAS) k_raster_bwd(SceneView s, double sigma, TileDiv tiles_x, EdgeTiles et,
                                                   const uint32_t *span_cache, TieTable ties,
                                                   const double *z_buffer,
                                                   const int *owner, const float *image_b, const float *obs,
                                                   const float *err_b, int compat, DeodrGrads grads,
                                                   double *edge_acc, const __grid_constant__ FrameMaps maps,
                                                   DeodrBackgroundGrads bg) {
    if (et.scal[SC_OVERFLOW]) return;
    fix_channel_count<MAXC, TEX>(s);
    s.perspective_correct = 0;  // the adjoint is only defined without it (validate_view rejects it): folds the branches
    __shared__ TileShared sh;
    // the tile's image_b / owner / z-buffer blocks arrive as three TMA tile loads (UTMALDG) issued by one thread
    __shared__ alignas(128) float t_img[MAXC <= 4 ? NT * MAXC : 4];
    __shared__ alignas(128) int t_own[NT];
    __shared__ alignas(128) double t_z[NT];
    __shared__ alignas(8) uint64_t tile_bar;
    const int tid = threadIdx.x;
    const bool tma_tiles = MAXC <= 4 && maps.ok;
    if (tma_tiles) {
        if (tid == 0) mbar_init(&tile_bar, 1);
        __syncthreads();
    }
    const int heavy = et.scal[SC_HEAVY_TILES], total = heavy + et.scal[SC_LIGHT_TILES];
    if ((int)blockIdx.x >= total) return;  // one CTA per entry of the list (launched for the plan's capacity)
    {
        const int tile_id = two_ended_at(et.list, et.num_tiles, heavy, blockIdx.x);
        const Tile tile = tile_of(tile_id, tiles_x);
        const int c = tid % TS, r = tid / TS;
        const int x = tile.x0 + c, y = tile.y0 + r;
        const bool inside = x < s.width && y < s.height;
        const size_t idx = inside ? (size_t)y * s.width + x : 0;
        const int n_edge = segment_size(et.seg, tile_id);

        PixelState<MAXC> p;
        AdjointState<MAXC> a;
        ErrorAdjointState<MAXC> ea;
        a.has_colour = false;
        ea.has = false;
        ea.g = 0.0;
        p.z = __longlong_as_double(0x7ff0000000000000LL);
        p.own = p.bown = -1;
        if (tma_tiles) {
            if (tid == 0) {
                mbar_expect_tx(&tile_bar, (uint32_t)(NT * (s.nb_colors * sizeof(float) + sizeof(int) + sizeof(double))));
                tma_load_tile(t_img, &maps.image, tile.x0 * s.nb_colors, tile.y0, &tile_bar);
                tma_load_tile(t_own, &maps.owner, tile.x0, tile.y0, &tile_bar);
                tma_load_tile(t_z, &maps.z, tile.x0, tile.y0, &tile_bar);
            }
            mbar_wait(&tile_bar, 0);
            if (inside) {
                p.z = t_z[tid];
                decode_owner(t_own[tid], ties, &p.own, &p.bown);
                for (int k = 0; k < channels<MAXC>(s); k++) a.g[k] = t_img[tid * channels<MAXC>(s) + k];
            }
        } else if (inside) {
            p.z = z_buffer[idx];
            decode_owner(owner[idx], ties, &p.own, &p.bown);
            for (int k = 0; k < channels<MAXC>(s); k++) a.g[k] = image_b[idx * channels<MAXC>(s) + k];
        }
        if (ERR && inside) ea.g = (double)err_b[idx];
        const float *obs_px = ERR ? obs + idx * channels<MAXC>(s) : nullptr;

        {
            const int edge_base = et.seg.offset[tile_id];
            const bool single = n_edge <= EDGE_CHUNK;
            auto load_spans = [&](int base, int m) {  // (all loads of a pass before its stores, see phase_edge_setup)
                const uint32_t *src = span_cache + (size_t)(edge_base + base) * TS;
                for (int first = tid; first < m * TS; first += 4 * EDGE_NT) {
                    uint32_t v[4];
#pragma unroll
                    for (int j = 0; j < 4; j++)
                        if (first + j * EDGE_NT < m * TS) v[j] = __ldg(src + first + j * EDGE_NT);
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const int item = first + j * EDGE_NT;
                        if (item < m * TS) sh.edge.span[item / TS][item % TS] = v[j];
                    }
                }
            };
            auto adjoint = [&](int m) {
                if (!inside) return;
                if (ERR) {
                    if (ea.has)
                        phase_edge_adjoint_error<MAXC, DevEnv>(s, x, y, r, m, &sh, p, obs_px, &ea, edge_acc,
                                                               grads.texture_b, compat != 0);
                } else if (a.has_colour) {
                    phase_edge_adjoint<MAXC, DevEnv>(s, x, y, r, m, &sh, p, &a, edge_acc, grads.texture_b);
                }
            };
            // pass A: forward replay (far to near) to obtain the final colour / residual in fp64
            for (int base = 0; base < n_edge; base += EDGE_CHUNK) {
                const int m = min(EDGE_CHUNK, n_edge - base);
                phase_edge_setup(tid, EDGE_NT, m, et.refs + edge_base + base, et.recs, &sh);
                load_spans(base, m);  // computed by the forward pass (k_edge_fwd)
                __syncthreads();
                if (inside) {
                    if (ERR) phase_edge_replay_error<MAXC>(s, x, y, r, m, &sh, p, obs_px, &ea);
                    else phase_edge_replay<MAXC>(s, x, y, r, m, &sh, p, &a);
                }
                if (single) adjoint(m);
                __syncthreads();
            }
            // pass B: reverse sweep (near to far), chunks in reverse order
            if (!single) {
                const int last = ((n_edge - 1) / EDGE_CHUNK) * EDGE_CHUNK;
                for (int base = last; base >= 0; base -= EDGE_CHUNK) {
                    const int m = min(EDGE_CHUNK, n_edge - base);
                    phase_edge_setup(tid, EDGE_NT, m, et.refs + edge_base + base, et.recs, &sh);
                    load_spans(base, m);
                    __syncthreads();
                    adjoint(m);
                    __syncthreads();
                }
            }
        }
        // a pixel overdrawn by edges in error mode: its colour adjoint comes from what is left of the residual's
        if (ERR && inside && ea.has) residual_adjoint<MAXC>(s, ea.col, obs_px, ea.g, a.g);
        interior_adjoint_warp<MAXC>(s, x, y, inside && p.bown >= 0, p, a.g, grads);
        if constexpr (BG) {
            const bool shows = inside && p.bown == -1;
            if (bg.background_image_b && shows)
                for (int k = 0; k < channels<MAXC>(s); k++) atomicAdd(bg.background_image_b + idx * channels<MAXC>(s) + k, a.g[k]);
            if (bg.background_color_b) {
                __shared__ double bg_partial[EDGE_NT / 32][MAXC];
                float g[MAXC];
#pragma unroll
                for (int k = 0; k < MAXC; k++) g[k] = shows ? a.g[k] : 0.0f;
                background_color_sum<MAXC, EDGE_NT>(channels<MAXC>(s), g, bg.background_color_b, bg_partial);
            }
        }
    }
}

// Background gradient of the tiles without silhouette edges (k_raster_bwd's BG instances take the others): the pixels
// whose owner code is -1 show the background as it is, so their colour adjoint (image_b; antialiase_error mode: the
// residual's, error_image_b) is the background's.  Pixels in row-major order, grid-stride (coalesced owner reads; image_b
// is read at background pixels only).
constexpr int BG_NT = 256;
template <int MAXC>
__global__ void __launch_bounds__(BG_NT) k_background_bwd(int width, int height, int C, int tiles_x, const int *scal,
                                                          const int *edge_cursor, const int *owner,
                                                          const float *image_b, DeodrBackgroundGrads bg) {
    if (scal[SC_OVERFLOW]) return;
    if (MAXC == 1 || MAXC == 3) C = MAXC;
    __shared__ double partial[BG_NT / 32][MAXC];
    float acc[MAXC];
#pragma unroll
    for (int k = 0; k < MAXC; k++) acc[k] = 0.0f;
    const int pixels = width * height;  // (sides <= 32767)
    for (int i = blockIdx.x * BG_NT + threadIdx.x; i < pixels; i += gridDim.x * BG_NT) {
        if (owner[i] != -1) continue;
        const int y = i / width, x = i - y * width;
        if (edge_cursor && edge_cursor[(y / TS) * tiles_x + x / TS] > 0) continue;  // handled by k_raster_bwd
        const float *g = image_b + (size_t)i * C;
        float *dst = bg.background_image_b ? bg.background_image_b + (size_t)i * C : nullptr;
#pragma unroll
        for (int k = 0; k < MAXC; k++) {
            if (k < C) {
                const float v = g[k];
                acc[k] += v;
                if (dst) atomicAdd(dst + k, v);
            }
        }
    }
    if (bg.background_color_b) background_color_sum<MAXC, BG_NT>(C, acc, bg.background_color_b, partial);
}

// Interior adjoint of the pixels owned by LARGE triangles in the tiles without silhouette edges: no shared memory, no
// z-buffer read; the gradients are summed per owner inside each warp before the scatter (interior_adjoint_warp).
template <int MAXC, bool TEX>
#ifndef DEODR_INTERIOR_MIN_CTAS
#define DEODR_INTERIOR_MIN_CTAS 3  // 85 registers
#endif
__global__ void __launch_bounds__(NT, DEODR_INTERIOR_MIN_CTAS) k_interior_bwd(SceneView s, TileDiv tiles_x, const int *large_tiles,
                                                     const int *scal, const int *edge_cursor, TieTable ties,
                                                     const int *owner, const float *image_b, DeodrGrads grads) {
    if (scal[SC_OVERFLOW]) return;
    fix_channel_count<MAXC, TEX>(s);
    s.perspective_correct = 0;  // the adjoint is only defined without it (validate_view rejects it): folds the branches
    const int tid = threadIdx.x, total = scal[SC_LARGE_TILES];
    for (int b = blockIdx.x; b < total; b += gridDim.x) {  // one CTA per tile with large triangles binned
        const int tile_id = large_tiles[b];
        if (edge_cursor && edge_cursor[tile_id] > 0) continue;  // handled by k_raster_bwd
        const Tile tile = tile_of(tile_id, tiles_x);
        const int x = tile.x0 + tid % TS, y = tile.y0 + tid / TS;
        const bool inside = x < s.width && y < s.height;
        PixelState<MAXC> p;
        p.z = 0.0;  // only read by the perspective-correct forward path
        p.own = p.bown = -1;
        float g[MAXC];
        if (inside) {
            const size_t idx = (size_t)y * s.width + x;
            decode_owner(owner[idx], ties, &p.own, &p.bown);
            if (p.bown >= 0 && (p.bown & SMALL_FLAG)) p.bown = -1;  // taken by k_small_tri_bwd (triangle-parallel)
            if (p.bown >= 0)
                for (int k = 0; k < channels<MAXC>(s); k++) g[k] = image_b[idx * channels<MAXC>(s) + k];
        }
        interior_adjoint_warp<MAXC>(s, x, y, inside && p.bown >= 0, p, g, grads);
    }
}

// Triangle-parallel interior adjoint of the small triangles (one thread per entry of the compacted small list).
template <int MAXC, bool TEX>
#ifndef DEODR_SMALL_MIN_CTAS
#define DEODR_SMALL_MIN_CTAS 8
#endif
__global__ void __launch_bounds__(128, DEODR_SMALL_MIN_CTAS) k_small_tri_bwd(SceneView s, int tiles_x, const int *small_ids, const int *scal,
                                                       const int *edge_cursor, TieTable ties, const int *owner,
                                                       const float *image_b, DeodrGrads grads) {
    if (scal[SC_OVERFLOW]) return;
    fix_channel_count<MAXC, TEX>(s);
    s.perspective_correct = 0;  // the adjoint is only defined without it (validate_view rejects it): folds the branches
    // one thread per entry (no stride loop: its registers cost this kernel its occupancy); the launch covers the exact
    // count when the forward's verdict has been read, every triangle otherwise
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= scal[SC_SMALL]) return;
    small_triangle_adjoint<MAXC, DevEnv>(s, small_ids[i], tiles_x, edge_cursor, owner, ties.pairs, image_b, grads.ij_b,
                                         grads.colors_b, grads.uv_b, grads.shade_b, grads.texture_b);
}

// Record-parallel interior adjoint of the small triangles (small_record_adjoint, phases.h; opt-in, see launch_bwd for the
// measurements that keep the triangle-parallel form the default): one CTA per tile without
// silhouette edges, one thread per pre-masked record of the tile's list (written by the binning pass for the z pass:
// consecutive threads read consecutive 64-byte records).  The tile's owner codes and colour adjoints arrive in shared
// memory as two TMA tile loads (UTMALDG.2D; cooperative loads when the buffers do not qualify): a record tests its 3-4
// covered pixels there instead of reading the 33 pixels of its triangle's bounding box from the owner map.
struct SharedTileFetch {
    const int *own;
    const float *img;
    int C;
    __device__ __forceinline__ int owner(int px) const { return own[px]; }
    __device__ __forceinline__ float g(int px, int q) const { return img[px * C + q]; }
};

template <int MAXC, bool TEX>
__global__ void __launch_bounds__(128, DEODR_SMALL_MIN_CTAS) k_small_rec_bwd(SceneView s, TileDiv tiles_x, TileSegments seg, const PreRec *recs,
                                                       const int *scal, const int *edge_cursor, TieTable ties,
                                                       const int *owner, const float *image_b, DeodrGrads grads,
                                                       const __grid_constant__ FrameMaps maps) {
    if (scal[SC_OVERFLOW]) return;
    fix_channel_count<MAXC, TEX>(s);
    s.perspective_correct = 0;  // the adjoint is only defined without it (validate_view rejects it): folds the branches
    const int tile_id = blockIdx.x, tid = threadIdx.x;
    const int n = segment_size(seg, tile_id);
    if (n == 0) return;
    if (edge_cursor && edge_cursor[tile_id] > 0) return;  // every pixel of that tile belongs to k_raster_bwd
    const Tile tile = tile_of(tile_id, tiles_x);
    const PreRec *list = recs + seg.offset[tile_id];
    if constexpr (MAXC <= 4) {
        __shared__ alignas(128) float t_img[NT * MAXC];
        __shared__ alignas(128) int t_own[NT];
        __shared__ alignas(8) uint64_t bar;
        if (maps.ok) {
            if (tid == 0) mbar_init(&bar, 1);
            __syncthreads();
            if (tid == 0) {
                mbar_expect_tx(&bar, (uint32_t)(NT * (s.nb_colors * sizeof(float) + sizeof(int))));
                tma_load_tile(t_img, &maps.image, tile.x0 * s.nb_colors, tile.y0, &bar);
                tma_load_tile(t_own, &maps.owner, tile.x0, tile.y0, &bar);  // (outside the image: zeros, no record's code)
            }
            mbar_wait(&bar, 0);
        } else {
            for (int px = tid; px < NT; px += blockDim.x) {
                const int x = tile.x0 + (px & (TS - 1)), y = tile.y0 + (px >> 4);
                const bool inside = x < s.width && y < s.height;
                const size_t idx = inside ? (size_t)y * s.width + x : 0;
                t_own[px] = inside ? owner[idx] : -1;
                for (int q = 0; q < s.nb_colors; q++) t_img[px * s.nb_colors + q] = inside ? image_b[idx * s.nb_colors + q] : 0.0f;
            }
            __syncthreads();
        }
        const SharedTileFetch fetch{t_own, t_img, s.nb_colors};
        for (int i = tid; i < n; i += blockDim.x)
            small_record_adjoint<MAXC, DevEnv>(s, list[i], tile, fetch, ties.pairs, grads.ij_b, grads.colors_b, grads.uv_b,
                                               grads.shade_b, grads.texture_b);
    } else {
        const GlobalTileFetch fetch{owner, image_b, tile, s.width, s.height, s.nb_colors};
        for (int i = tid; i < n; i += blockDim.x)
            small_record_adjoint<MAXC, DevEnv>(s, list[i], tile, fetch, ties.pairs, grads.ij_b, grads.colors_b, grads.uv_b,
                                               grads.shade_b, grads.texture_b);
    }
}

__global__ void k_finalize_edges(SceneView s, EdgeList edges, const int *scal, double sigma, const double *edge_acc,
                                 DeodrGrads grads) {
    if (scal[SC_OVERFLOW]) return;
    const int n = min(*edges.count, edges.capacity);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        finalize_edge<DevEnv>(s, edges.ids[i], sigma, edge_acc + (size_t)i * edge_acc_stride(s.nb_colors), grads.ij_b,
                              grads.colors_b, grads.uv_b, grads.shade_b);
}

template <int MAXC>
static void launch_bwd(DeodrWorkspace *ws, ViewSlot *v, Lane &lane, const SceneView &s, const DeodrViewIO &io,
                       double sigma, int flags, const DeodrGrads &g, const DeodrBackgroundGrads &bg) {
    // Three independent chains (disjoint pixel sets, all accumulate with atomics): edge tiles (longest tail: launched
    // first, on the lane's high-priority stream, so that its CTAs are dispatched first), small triangles (the longest
    // kernel: launched next), tiles with large triangles.  On an equal-priority stream the edge chain's CTAs were dispatched last in a graph replay: on the
    // 1M-triangle scene k_raster_bwd started 76 us after the adjoint began, and k_finalize_edges ran alone at the end.
    cudaStream_t st = lane.main;
    bool first = true;
    const FwdPlan &plan = v->plan;
    const bool tex = plan.tex != 0;
    const bool err_mode = (flags & DEODR_B200_ANTIALIASE_ERROR) != 0;
    const int compat = (flags & DEODR_B200_ERROR_ADJOINT_COMPLETE) ? 0 : 1;
    const int C = s.nb_colors;
    const bool edges = plan.cap_edges > 0;
    const TileDiv div = make_tile_div(v->tiles_x);
    const TieTable ties = tie_table(v);
    const int *edge_cursor = edges ? v->edge_cursor : nullptr;
    const float *image_b = io.image_b;
    const bool bg_on = bg.background_image_b || bg.background_color_b;  // (background gradients: a fourth chain)
    if (err_mode) {  // colour adjoint of the pixels outside the edge bands, before the three chains fork
        const size_t pixels = (size_t)s.height * s.width;
        k_error_image_b<<<grid_for(pixels * C, 256) < 4096 ? grid_for(pixels * C, 256) : 4096, 256, 0, st>>>(
            io.image, io.obs, io.err_buffer_b, v->error_image_b.as<float>(), pixels, C, v->scal);
        image_b = v->error_image_b.as<float>();
        ws->launches++;
    }
    // tensor maps of the tile-shaped reads of the adjoint (image_b / owner / z-buffer blocks): k_raster_bwd, k_small_rec_bwd
    FrameMaps maps;
    memset(&maps, 0, sizeof(maps));
    static const bool tma_allowed = !(getenv("DEODR_B200_TMA_TILES") && atoi(getenv("DEODR_B200_TMA_TILES")) == 0);
    maps.ok = tma_allowed && C <= 4 &&
              encode_tile_map(&maps.image, image_b, 4, true, s.height, s.width * C, TS, TS * C) &&
              encode_tile_map(&maps.owner, io.owner, 4, false, s.height, s.width, TS, TS) &&
              encode_tile_map(&maps.z, io.z_buffer, 8, false, s.height, s.width, TS, TS);
    if (edges) {
        cudaStream_t se = fork_stream(ws, lane, 0, &first);
        cudaMemsetAsync(v->edge_acc.ptr, 0, (size_t)plan.cap_edges * edge_acc_stride(C) * sizeof(double), se);
        const EdgeTiles et = edge_tiles_of(v);
        const int grid = at_least_one(v->hints_exact && !ws->capturing_internally ? plan.hint_edge_tiles : plan.cap_edge_tiles);
        {
            PhaseTimer timer(ws, DEODR_B200_PH_EDGE_BWD, se);
#define DEODR_RASTER_BWD(X, R, B) k_raster_bwd<MAXC, X, R, B><<<grid, EDGE_NT, 0, se>>>(s, sigma, div, et, v->edge_spans.as<uint32_t>(), ties, io.z_buffer, io.owner, image_b, io.obs, io.err_buffer_b, compat, g, v->edge_acc.as<double>(), maps, bg)
            if (!bg_on) {
                if (tex) { if (err_mode) DEODR_RASTER_BWD(true, true, false); else DEODR_RASTER_BWD(true, false, false); }
                else     { if (err_mode) DEODR_RASTER_BWD(false, true, false); else DEODR_RASTER_BWD(false, false, false); }
            } else {
                if (tex) { if (err_mode) DEODR_RASTER_BWD(true, true, true); else DEODR_RASTER_BWD(true, false, true); }
                else     { if (err_mode) DEODR_RASTER_BWD(false, true, true); else DEODR_RASTER_BWD(false, false, true); }
            }
#undef DEODR_RASTER_BWD
        }
        {
            PhaseTimer timer(ws, DEODR_B200_PH_EDGE_FINALIZE, se);
            const EdgeList el{v->scal + SC_EDGES, v->edge_ids.as<int>(), v->edge_keys.as<uint64_t>(), plan.cap_edges};
            k_finalize_edges<<<at_least_one(grid_for(plan.hint_edges, 128)), 128, 0, se>>>(s, el, v->scal, sigma,
                                                                                           v->edge_acc.as<double>(), g);
        }
        ws->launches += 2;
    }
    auto launch_small = [&]() {
        PhaseTimer timer(ws, DEODR_B200_PH_SMALL_BWD, st);
        // Triangle-parallel (default) or record-parallel (DEODR_B200_SMALL_ADJOINT=record) adjoint of the small triangles.
        // In the record-parallel form the vertex gathers and the fifteen atomics per thread are what it costs, not the
        // bounding-box reads, and more threads pay them; it also slows k_interior_bwd running beside it.
        if (!ws->small_by_record) {  // (read from the environment when the workspace is created)
            const int entries = v->hints_exact && !ws->capturing_internally ? plan.hint_small : s.nb_triangles;
            (tex ? k_small_tri_bwd<MAXC, true> : k_small_tri_bwd<MAXC, false>)<<<at_least_one(grid_for(entries, 128)), 128, 0, st>>>(
                s, v->tiles_x, v->small_ids.as<int>(), v->scal, edge_cursor, ties, io.owner, image_b, g);
        } else {
            const TileSegments seg{v->small_offset.as<int>(), v->small_cursor};
            (tex ? k_small_rec_bwd<MAXC, true> : k_small_rec_bwd<MAXC, false>)<<<v->num_tiles, 128, 0, st>>>(
                s, div, seg, v->small_recs.as<PreRec>(), v->scal, edge_cursor, ties, io.owner, image_b, g, maps);
        }
        ws->launches++;
    };
    bool small_done = false;  // launched before the interior chain when there is one, else after the others
    const bool large = plan.cap_large > 0 && plan.hint_large_tiles > 0;
    if (large) {  // pixels owned by large triangles, tiles without silhouette edges
        cudaStream_t sl = fork_stream(ws, lane, 2, &first);
        // k_small_tri_bwd is the adjoint's longest kernel.  Launched after k_interior_bwd, its CTAs were dispatched only
        // once the interior's had taken the SMs, and it ran alone at the end of the step (1M-triangle scene: it began
        // 54 us into the adjoint).  Launched first (the interior's stream has forked, so it does not wait for it), it
        // fills the SMs from the start and the interior's CTAs take the slots it leaves.
        launch_small();
        small_done = true;
        PhaseTimer timer(ws, DEODR_B200_PH_INTERIOR_BWD, sl);
        const int grid = at_least_one(plan.hint_large_tiles < v->num_tiles ? plan.hint_large_tiles : v->num_tiles);
        (tex ? k_interior_bwd<MAXC, true> : k_interior_bwd<MAXC, false>)<<<grid, NT, 0, sl>>>(
            s, div, v->large_tiles.as<int>(), v->scal, edge_cursor, ties, io.owner, image_b, g);
        ws->launches++;
    }
    if (bg_on) {  // background pixels of the tiles without silhouette edges (all of them when there are no edges)
        cudaStream_t sb = fork_stream(ws, lane, 1, &first);
        PhaseTimer timer(ws, DEODR_B200_PH_BACKGROUND_BWD, sb);
        const size_t pixels = (size_t)s.height * s.width;
        const int grid = at_least_one(std::min(grid_for(pixels, BG_NT), 2048));
        k_background_bwd<MAXC><<<grid, BG_NT, 0, sb>>>(s.width, s.height, C, v->tiles_x, v->scal, edge_cursor, io.owner,
                                                       image_b, bg);
        ws->launches++;
    }
    if (!small_done) launch_small();
    if (edges) join_stream(ws, lane, 0);
    if (large) join_stream(ws, lane, 2);
    if (bg_on) join_stream(ws, lane, 1);
}


// Adjoint of a scene with more than COLOR_SLAB channels (antialiase_error mode is refused there).  The adjoint is linear
// in image_b, and the blend weights, barycentrics and coverage do not depend on the channel: one adjoint pass of the
// 16-channel instances per slab of at most COLOR_SLAB channels, on compact copies of the slab's image_b, colours and
// texture.  The slab's colors_b / texture_b / background_image_b land in compact buffers that are then added into their
// channels of the caller's; ij_b, uv_b and shade_b accumulate over the slabs in place, background_color_b at offset c0.
// The edge accumulators are zeroed and finalised once per slab (launch_bwd), so they are sized for COLOR_SLAB channels.
static void launch_bwd_wide(DeodrWorkspace *ws, ViewSlot *v, Lane &lane, const SceneView &s, const DeodrViewIO &io,
                            double sigma, int flags, const DeodrGrads &g, const DeodrBackgroundGrads &bg) {
    cudaStream_t st = lane.main;
    const int C = s.nb_colors;
    const size_t pixels = (size_t)s.height * s.width, verts = (size_t)s.nb_vertices;
    const size_t texels = s.texture ? (size_t)s.texture_height * s.texture_width : 0;
    for (int c0 = 0; c0 < C; c0 += COLOR_SLAB) {
        const int n = std::min(COLOR_SLAB, C - c0);
        const SlabCopy image_b{io.image_b + c0, v->slab_image.as<float>(), pixels, C, n, n, 0};
        const SceneView slab = deodr_slab_inputs(ws, v, s, c0, &image_b, st);
        DeodrViewIO slab_io = io;
        slab_io.image_b = v->slab_image.as<float>();
        DeodrGrads slab_g = g;
        slab_g.colors_b = g.colors_b && verts ? v->slab_colors_b.as<float>() : nullptr;
        slab_g.texture_b = g.texture_b && texels ? v->slab_texture_b.as<float>() : nullptr;
        if (slab_g.colors_b) cudaMemsetAsync(slab_g.colors_b, 0, verts * n * sizeof(float), st);
        if (slab_g.texture_b) cudaMemsetAsync(slab_g.texture_b, 0, texels * n * sizeof(float), st);
        DeodrBackgroundGrads slab_bg;
        slab_bg.background_image_b = bg.background_image_b ? v->slab_background_b.as<float>() : nullptr;
        slab_bg.background_color_b = bg.background_color_b ? bg.background_color_b + c0 : nullptr;
        if (slab_bg.background_image_b) cudaMemsetAsync(slab_bg.background_image_b, 0, pixels * n * sizeof(float), st);
        launch_bwd<16>(ws, v, lane, slab, slab_io, sigma, flags, slab_g, slab_bg);
        SlabCopies out;
        memset(&out, 0, sizeof(out));
        if (slab_g.colors_b) out.job[out.n++] = SlabCopy{slab_g.colors_b, g.colors_b + c0, verts, n, C, n, 1};
        if (slab_g.texture_b) out.job[out.n++] = SlabCopy{slab_g.texture_b, g.texture_b + c0, texels, n, C, n, 1};
        if (slab_bg.background_image_b)
            out.job[out.n++] = SlabCopy{slab_bg.background_image_b, bg.background_image_b + c0, pixels, n, C, n, 1};
        deodr_slab_copy(ws, out, st);
    }
}

void deodr_launch_backward(DeodrWorkspace *ws, ViewSlot *v, Lane &lane, const SceneView &s, const DeodrViewIO &io,
                           double sigma, int flags, const DeodrGrads &g, const DeodrBackgroundGrads &bg) {
    const int C = s.nb_colors;
    if (C == 1) launch_bwd<1>(ws, v, lane, s, io, sigma, flags, g, bg);
    else if (C == 3) launch_bwd<3>(ws, v, lane, s, io, sigma, flags, g, bg);
    else if (C <= 4) launch_bwd<4>(ws, v, lane, s, io, sigma, flags, g, bg);
    else if (C <= COLOR_SLAB) launch_bwd<16>(ws, v, lane, s, io, sigma, flags, g, bg);
    else launch_bwd_wide(ws, v, lane, s, io, sigma, flags, g, bg);
}

#ifdef DEODR_SMALLBWD_PHASE_CLOCKS
// Measurement builds only: copies k_small_tri_bwd's per-phase cycle sums (SB_PHASES, then the threads and the hidden
// threads counted) and its owned-pixel histogram (SB_HIST) out of the device, then clears them.  Synchronises the device.
extern "C" int deodr_b200_small_bwd_phase_clocks(unsigned long long *clocks, unsigned int *hist) {
    if (cudaDeviceSynchronize() != cudaSuccess ||
        cudaMemcpyFromSymbol(clocks, g_smallbwd_clocks, sizeof(g_smallbwd_clocks)) != cudaSuccess ||
        cudaMemcpyFromSymbol(hist, g_smallbwd_hist, sizeof(g_smallbwd_hist)) != cudaSuccess)
        return DEODR_B200_ECUDA;
    static const unsigned long long zc[SB_SLOTS] = {};
    static const unsigned int zh[SB_HIST] = {};
    if (cudaMemcpyToSymbol(g_smallbwd_clocks, zc, sizeof(zc)) != cudaSuccess ||
        cudaMemcpyToSymbol(g_smallbwd_hist, zh, sizeof(zh)) != cudaSuccess)
        return DEODR_B200_ECUDA;
    return DEODR_B200_OK;
}
#endif

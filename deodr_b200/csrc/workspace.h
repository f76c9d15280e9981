// Host-side state shared by the translation units of libdeodr_b200.so (kernels.cu: device API, host_api.cu: the
// reference-shaped host entry points).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../include/deodr_b200.h"
#include "phases.h"

char *deodr_error_buffer();  // thread-local, 512 bytes (defined in kernels.cu)

static inline int set_error(int code, const char *fmt, const char *detail = "") {
    snprintf(deodr_error_buffer(), 512, fmt, detail);
    return code;
}

#define CUDA_TRY(expr)                                                                                \
    do {                                                                                              \
        cudaError_t err__ = (expr);                                                                   \
        if (err__ != cudaSuccess) {                                                                   \
            snprintf(deodr_error_buffer(), 512, "%s failed: %s", #expr, cudaGetErrorString(err__));   \
            return DEODR_B200_ECUDA;                                                                  \
        }                                                                                             \
    } while (0)

// growable device buffer
struct DevBuf {
    void *ptr = nullptr;
    size_t bytes = 0;
    int ensure(size_t need, int64_t *accounted) {
        if (need <= bytes) return DEODR_B200_OK;
        if (ptr) {
            CUDA_TRY(cudaFree(ptr));
            *accounted -= (int64_t)bytes;
            ptr = nullptr;
            bytes = 0;
        }
        size_t want = need + need / 4 + 256;
        CUDA_TRY(cudaMalloc(&ptr, want));
        bytes = want;
        *accounted += (int64_t)want;
        return DEODR_B200_OK;
    }
    void release() {
        if (ptr) cudaFree(ptr);
        ptr = nullptr;
        bytes = 0;
    }
    template <class T>
    T *as() const { return static_cast<T *>(ptr); }
};

// The plan of a view's forward pass: what the host knows WITHOUT asking the device.  Capacities of the per-tile
// segments (their offsets live on the device, in the slot) and of the edge list, the kernel instances to run, and
// launch-size hints (every kernel strides over the device-side counts, so a hint is never a correctness matter).
struct FwdPlan {
    bool valid = false;
    // what the plan was built for
    int T = -1, H = -1, W = -1;
    bool edges_possible = false;  // sigma > 0
    // reserved capacities
    int cap_small = 0, cap_large = 0, cap_edges = 0, cap_edge_refs = 0;
    int cap_edge_tiles = 0;  // tiles with silhouette edges the edge kernels are launched for (one CTA each)
    int tex = 1;  // kernel instances with the texture paths compiled in
    // hints
    int hint_small = 0, hint_edge_tiles = 0, hint_large_tiles = 0, hint_edges = 0;
};

// One view's forward state + plan (see include/deodr_b200.h: "view slots").
struct ViewSlot {
    FwdPlan plan;
    int64_t generation = 0;
    // geometry of the tiling
    int tiles_x = 0, tiles_y = 0, num_tiles = 0;
    // the last forward pass (what the adjoint checks / what a re-run after an overflow needs)
    int fwd_valid = 0;
    double sigma = -1;
    int fwd_C = 0, fwd_flags = 0;
    DeodrSceneView fwd_scene;
    DeodrViewIO fwd_io;
    bool fwd_check_indices = false;
    bool pending = false;     // a pass has been enqueued whose verdict has not been read yet
    bool head_enqueued = false;  // DEODR_B200_FORWARD_GEOMETRY has run; the RESUME call of the same pass must follow
    bool hints_exact = false; // the plan's hints are the counts of the slot's last pass (its verdict has been read)
    int totals_seq = 0;       // sequence number of the flag the publishing kernel raises in host_totals[SC_WORDS]
    int *host_totals = nullptr;  // pinned: SC_WORDS scalars + the sequence flag
    // device state
    DevBuf zeroed;            // [scalars(SC_WORDS) | small cursor | large cursor | edge cursor], one memset per forward
    int *scal = nullptr, *small_cursor = nullptr, *large_cursor = nullptr, *edge_cursor = nullptr;
    DevBuf small_offset, large_offset, edge_offset;  // [tiles + 1] segment offsets of the plan
    DevBuf small_recs, large_refs, small_ids;
    DevBuf edge_tiles_raw;    // tiles with silhouette edges in arrival order (k_bin_edges)
    DevBuf large_tiles, edge_tiles;  // compact lists of the tiles with large triangles / silhouette edges (two-ended)
    DevBuf edge_ids, edge_keys, edge_recs, edge_refs_tmp, edge_refs;
    DevBuf edge_spans;        // x spans of every (tile, edge, row), written by k_edge_fwd and reused by k_raster_bwd
    DevBuf edge_acc;          // per-edge fp64 plane adjoints of the backward pass
    DevBuf tie_pairs;
    int tie_capacity = 0;
    DevBuf error_image_b;     // antialiase_error adjoint: colour adjoint of the pixels outside every edge band
    // scenes with more than COLOR_SLAB channels: one slab's channels of the colours [V], texture [Ht*Wt], background
    // [H*W or 1] and image (forward) / image_b (adjoint) [H*W], and of the adjoint's colors_b [V] and texture_b [Ht*Wt],
    // COLOR_SLAB floats per row
    DevBuf slab_colors, slab_texture, slab_background, slab_image, slab_colors_b, slab_texture_b;
    DevBuf slab_background_b;  // one slab's background_image_b [H*W] (only when the adjoint is asked for it)
    DevBuf compare_scratch;    // k_compare: fp64 partial of every CTA + the count of finished CTAs (zeroed once)
};

// One lane = the stream a view's main chain runs on + auxiliary streams for its side chains: aux[0] (high priority)
// the silhouette-edge chains - the forward's short one, which the main chain waits for, and the adjoint's, whose
// crowded tiles set the pass's end; aux[1], aux[2] the adjoint's other concurrent kernels (background, large triangles).
constexpr int LANE_AUX = 3;
struct Lane {
    cudaStream_t main = nullptr;  // lane 0: the caller's stream (not owned)
    cudaStream_t aux[LANE_AUX] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev_fork = nullptr, ev_join[LANE_AUX] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev_begin = nullptr, ev_end = nullptr;  // lanes > 0: fork from / join to the caller's stream
};

constexpr int MAX_LANES = 8;

// A launch sequence captured once and replayed while nothing it depends on changes: a fitting loop calls the library
// with the same buffers, shapes and plans step after step, and a replayed graph has none of the per-launch gaps of a
// dozen dependent launches on four streams.  `key` is
// every byte the captured launches were built from; a different key re-captures.
struct GraphCache {
    cudaGraphExec_t exec = nullptr;
    std::vector<unsigned char> key;
    int launches = 0;  // kernels inside the graph (for deodr_b200_workspace_launches)
    int misses = 0;    // consecutive calls whose key differed: a caller that never repeats itself stops being captured
    void drop() {
        if (exec) cudaGraphExecDestroy(exec);
        exec = nullptr;
        key.clear();
    }
};

struct DeodrWorkspace {
    int device = 0;
    int64_t bytes = 0;
    int64_t launches = 0;
    int64_t generation_counter = 0;
    bool overlap = true;   // DEODR_B200_SERIAL=1 keeps every launch on the caller's stream (profiling, A/B)
    bool deferred = false; // the entry points never read the verdict (CUDA-graph capture); see deodr_b200_workspace_status
    int replans = 0;       // number of plans (re)built so far
    cudaEvent_t colors_ready = nullptr;  // one-shot: the next forward's colour readers wait for it (not owned)
    bool graphs = false;   // replay captured launch sequences (opt-in: DEODR_B200_GRAPHS=1)
    bool capturing_internally = false;  // the library itself is capturing: external event waits, capacity-sized grids
    GraphCache fwd_graph, bwd_graph;
    // the legacy default stream cannot be captured: a call made on it hops to this stream (event in, event out)
    cudaStream_t proxy = nullptr;
    cudaEvent_t proxy_in = nullptr, proxy_out = nullptr;
    // lanes a batch of views is spread over (DEODR_B200_LANES overrides); H100 (400 W), 16 renders of 200k triangles at
    // 512^2, graph replay: 0.94 ms per step with 6 lanes, 0.91 with 8
    int num_lanes = 8;
    bool small_by_record = false;  // DEODR_B200_SMALL_ADJOINT=record at creation: k_small_rec_bwd instead of k_small_tri_bwd
    Lane lanes[MAX_LANES];
    std::vector<ViewSlot *> slots;
    // optional per-phase event timing (bench / profiling)
    std::vector<cudaEvent_t> ev_start, ev_stop;
    std::vector<int> ev_phase;
    int ev_used = 0;
    DevBuf scalars;  // scratch of deodr_b200_check_scene
    int *host_scratch = nullptr;  // pinned, 32 ints
    // host-path staging (canonical device copies of a DeodrHostScene)
    DevBuf h_faces, h_faces_uv, h_ij, h_depths, h_uv, h_colors, h_shade, h_edgeflags, h_textured, h_shaded, h_texture,
        h_background, h_image, h_z, h_owner, h_image_b, h_grads, h_obs, h_err, h_err_b;
    struct HostPath *host = nullptr;  // pinned staging, copy threads, cache of the last host forward (host_api.cu)
    struct CollisionState *collision = nullptr;  // self-collision plan and buffers (collision.cu)
};

void deodr_host_path_destroy(DeodrWorkspace *ws);  // host_api.cu
void deodr_collision_destroy(DeodrWorkspace *ws);  // collision.cu

// forward pass of one view into slot 0 with optional on-device index validation (checkSceneValid, DR.h:2703-2714);
// always verified before it returns (the host path synchronises anyway)
int deodr_render_checked(DeodrWorkspace *ws, const DeodrSceneView *scene, const DeodrViewIO *io, double sigma, int flags,
                         void *stream);

// TEST INFRASTRUCTURE ONLY - CPU harness of the z pass's record phases (deodr_b200/csrc/phases.h).
//
// Runs one chunk of pre-masked records through the candidate scatter + pixel test the kernel uses for crowded chunks
// (phase_pre_scatter + phase_pix_test) and through the warp-local test of the other chunks (warp_candidates /
// phase_warp_test), each CTA phase as a `for (tid ...)` loop, and counts the pixels where they disagree.  Never part
// of the product.
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

#include "../../deodr_b200/csrc/phases.h"

using namespace deodr;

namespace {

struct HostEnv {
    static int shared_inc(int *p) { return (*p)++; }
};

// candidates of pixel tid by brute force: bit t <=> record t covers the pixel (n <= 128)
void brute_candidates(int tid, int n, const PreRec *pre, uint32_t out[4]) {
    out[0] = out[1] = out[2] = out[3] = 0u;
    for (int t = 0; t < n; t++)
        if ((pre[t].mask[tid / 32] >> (tid % 32)) & 1u) out[t / 32] |= 1u << (t % 32);
}

// candidates of pixel tid as left in the lists by a scatter; false if the count disagrees with `want` or a listed
// record is not a candidate / is listed twice
bool list_matches(int tid, const TileShared &sh, const uint32_t want[4]) {
    int expected = 0;
    for (int k = 0; k < 4; k++) expected += __builtin_popcount(want[k]);
    if (sh.tri.pix_cnt[tid] != expected) return false;
    if (expected > PIX_SLOTS) return true;  // the pixel scans the chunk's masks instead
    uint32_t seen[4] = {0u, 0u, 0u, 0u};
    for (int i = 0; i < expected; i++) {
        const int t = sh.tri.pix_list[i][tid];
        if (!((want[t / 32] >> (t % 32)) & 1u) || ((seen[t / 32] >> (t % 32)) & 1u)) return false;
        seen[t / 32] |= 1u << (t % 32);
    }
    return true;
}

bool same_state(const PixelState<1> &a, const PixelState<1> &b) {
    return std::memcmp(&a.z, &b.z, sizeof(double)) == 0 && a.own == b.own && a.bown == b.bown;
}

}  // namespace

extern "C" {

// One chunk of n (1..PRE_CHUNK) records on the tile at (x0, y0).  mismatch[0]: pixels whose scattered candidate list
// differs from the truth (brute force over the masks), [1]: pixels whose warp-local candidate set differs, [2]: pixels
// whose final (z, own, bown) from phase_warp_test differs from the scatter + pixel test's, [3]: candidate counters not
// left at zero.  z_out / own_out / bown_out[tid]: the final state of scatter + pixel test.
int wt_run_chunk(const PreRec *recs, int n, int x0, int y0, int persp, int *mismatch, double *z_out, int *own_out,
                 int *bown_out) {
    if (n < 1 || n > PRE_CHUNK) return -1;
    SceneView s;
    std::memset(&s, 0, sizeof(s));
    s.perspective_correct = persp;
    s.width = s.height = 1 << 14;
    const Tile tile{x0, y0};
    std::vector<PreRec> pre(recs, recs + n);
    TileShared *ref = new TileShared;
    std::memset(ref, 0, sizeof(TileShared));
    std::vector<PixelState<1>> p_ref(NT), p_warp(NT);
    for (int tid = 0; tid < NT; tid++) {
        for (auto *v : {&p_ref, &p_warp}) {
            (*v)[tid].z = std::numeric_limits<double>::infinity();
            (*v)[tid].own = (*v)[tid].bown = -1;
        }
    }
    for (int k = 0; k < 4; k++) mismatch[k] = 0;
    for (int tid = 0; tid < NT; tid++) phase_pre_scatter<HostEnv>(tid, n, pre.data(), ref);
    for (int tid = 0; tid < NT; tid++) {
        uint32_t want[4];
        brute_candidates(tid, n, pre.data(), want);
        if (!list_matches(tid, *ref, want)) mismatch[0]++;
        uint32_t got[4] = {0u, 0u, 0u, 0u};
        for (int g = 0; g < n; g += 32) got[g / 32] = warp_candidates(tid, n, g, pre.data());
        if (std::memcmp(got, want, sizeof(got)) != 0) mismatch[1]++;
    }
    for (int tid = 0; tid < NT; tid++) phase_pix_test<1>(s, tid, n, tile, pre.data(), ref, &p_ref[tid]);
    for (int tid = 0; tid < NT; tid++) phase_warp_test<1>(s, tid, n, tile, pre.data(), &p_warp[tid]);
    for (int tid = 0; tid < NT; tid++) {
        if (!same_state(p_warp[tid], p_ref[tid])) mismatch[2]++;
        z_out[tid] = p_ref[tid].z;
        own_out[tid] = p_ref[tid].own;
        bown_out[tid] = p_ref[tid].bown;
    }
    // phase_pix_test leaves the counters at zero for the next chunk
    for (int tid = 0; tid < NT; tid++)
        if (ref->tri.pix_cnt[tid] != 0) mismatch[3]++;
    delete ref;
    return 0;
}

}  // extern "C"

// Host binned-SAH BVH2 builder: the reference the device build (kjb_bvh_build.cuh) is checked against — same nodes and parent links byte
// for byte, same tri_info, same triangles per leaf.  The library ran this builder before the structure was built on the device; the CUDA
// library no longer compiles it.  Only the test emulator's build links it, which exports it as kjb_ref_* (bottom of this file).
#include "kjb_bvh.h"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace kjb {

struct HostBvh {
    std::vector<BvhNode> nodes;
    std::vector<BvhTri> tris;        // leaf order
    std::vector<TriInfo> info;       // by gid
    int32_t root_child = 0;          // encoded like a child reference (a 1-leaf scene has no inner node)
    std::vector<int32_t> parent;     // per inner node: (parent node << 1) | child slot, -1 for the root
};

namespace {

struct Box {
    float lo[3], hi[3];
    void reset() { for (int a = 0; a < 3; ++a) { lo[a] = 3.4e38f; hi[a] = -3.4e38f; } }
    void grow(const float* p) { for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], p[a]); hi[a] = std::max(hi[a], p[a]); } }
    void grow(const Box& b) { for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], b.lo[a]); hi[a] = std::max(hi[a], b.hi[a]); } }
    float area() const { float d0 = hi[0] - lo[0], d1 = hi[1] - lo[1], d2 = hi[2] - lo[2]; return (d0 < 0 || d1 < 0 || d2 < 0) ? 0.0f : 2.0f * (d0 * d1 + d1 * d2 + d2 * d0); }
};

struct Builder {
    const float* tris; uint32_t n;
    std::vector<Box> tbox; std::vector<float> cent;   // per triangle
    std::vector<uint32_t> order;
    HostBvh* out;
    static const int BINS = 16, LEAF = 4;

    Box padded(const Box& b) const {
        // the slab test only culls: pad so that rounding in (plane - origin) * inv_dir can never reject a true hit
        Box r = b;
        for (int a = 0; a < 3; ++a) { float pad = (b.hi[a] - b.lo[a]) * 1e-5f + 1e-6f + 1e-6f * std::max(std::fabs(b.lo[a]), std::fabs(b.hi[a])); r.lo[a] -= pad; r.hi[a] += pad; }
        return r;
    }
    // returns child reference
    int32_t build(uint32_t first, uint32_t count, const Box& bounds, const Box& cbounds, int depth = 0) {
        if (count <= (uint32_t)LEAF) return make_leaf(first, count);
        int best_axis = -1, best_split = -1; float best_cost = 3.4e38f;
        // past depth 40 fall back to median splits so the tree depth stays below the traversal stack (64 entries)
        for (int axis = 0; axis < 3 && depth < 40; ++axis) {
            const float lo = cbounds.lo[axis], ext = cbounds.hi[axis] - lo;
            if (!(ext > 1e-12f)) continue;
            Box bb[BINS]; uint32_t bc[BINS];
            for (int b = 0; b < BINS; ++b) { bb[b].reset(); bc[b] = 0; }
            const float scale = float(BINS) / ext;
            for (uint32_t i = first; i < first + count; ++i) {
                const uint32_t t = order[i];
                int b = int((cent[t * 3 + axis] - lo) * scale); b = b < 0 ? 0 : (b >= BINS ? BINS - 1 : b);
                bb[b].grow(tbox[t]); bc[b]++;
            }
            float right_area[BINS]; uint32_t right_cnt[BINS];
            Box acc; acc.reset(); uint32_t cnt = 0;
            for (int b = BINS - 1; b > 0; --b) { acc.grow(bb[b]); cnt += bc[b]; right_area[b] = acc.area(); right_cnt[b] = cnt; }
            acc.reset(); cnt = 0;
            for (int b = 0; b < BINS - 1; ++b) {
                acc.grow(bb[b]); cnt += bc[b];
                if (cnt == 0 || right_cnt[b + 1] == 0) continue;
                const float cost = acc.area() * float(cnt) + right_area[b + 1] * float(right_cnt[b + 1]);
                if (cost < best_cost) { best_cost = cost; best_axis = axis; best_split = b; }
            }
        }
        uint32_t mid;
        if (best_axis < 0) {
            mid = first + count / 2;   // all centroids coincide (or depth cap): split the list in half
            if (depth >= 40) {
                int axis = 0; float e = -1; for (int a = 0; a < 3; ++a) if (cbounds.hi[a] - cbounds.lo[a] > e) { e = cbounds.hi[a] - cbounds.lo[a]; axis = a; }
                std::nth_element(order.begin() + first, order.begin() + mid, order.begin() + first + count, [&](uint32_t a, uint32_t b) { return cent[a * 3 + axis] < cent[b * 3 + axis]; });
            }
        } else {
            const float lo = cbounds.lo[best_axis], scale = float(BINS) / (cbounds.hi[best_axis] - lo);
            auto it = std::partition(order.begin() + first, order.begin() + first + count, [&](uint32_t t) {
                int b = int((cent[t * 3 + best_axis] - lo) * scale); b = b < 0 ? 0 : (b >= BINS ? BINS - 1 : b);
                return b <= best_split; });
            mid = uint32_t(it - order.begin());
            if (mid == first || mid == first + count) mid = first + count / 2;
        }
        Box lb, lcb, rb, rcb; lb.reset(); lcb.reset(); rb.reset(); rcb.reset();
        for (uint32_t i = first; i < mid; ++i) { lb.grow(tbox[order[i]]); lcb.grow(&cent[order[i] * 3]); }
        for (uint32_t i = mid; i < first + count; ++i) { rb.grow(tbox[order[i]]); rcb.grow(&cent[order[i] * 3]); }
        const size_t idx = out->nodes.size();
        out->nodes.emplace_back();
        const int32_t c0 = build(first, mid - first, lb, lcb, depth + 1);
        const int32_t c1 = build(mid, first + count - mid, rb, rcb, depth + 1);
        const Box pl = padded(lb), pr = padded(rb);
        BvhNode& nd = out->nodes[idx];
        nd.n0[0] = pl.lo[0]; nd.n0[1] = pl.hi[0]; nd.n0[2] = pl.lo[1]; nd.n0[3] = pl.hi[1];
        nd.n1[0] = pr.lo[0]; nd.n1[1] = pr.hi[0]; nd.n1[2] = pr.lo[1]; nd.n1[3] = pr.hi[1];
        nd.n2[0] = pl.lo[2]; nd.n2[1] = pl.hi[2]; nd.n2[2] = pr.lo[2]; nd.n2[3] = pr.hi[2];
        nd.child[0] = c0; nd.child[1] = c1; nd.child[2] = nd.child[3] = 0;
        return int32_t(idx);
    }
    int32_t make_leaf(uint32_t first, uint32_t count) {
        const uint32_t base = uint32_t(out->tris.size());
        for (uint32_t i = first; i < first + count; ++i) {
            const uint32_t t = order[i]; const float* p = &tris[size_t(t) * 9];
            BvhTri bt{};
            for (int a = 0; a < 3; ++a) { bt.v0[a] = p[a]; bt.e1[a] = p[3 + a] - p[a]; bt.e2[a] = p[6 + a] - p[a]; }
            bt.gid = t;
            out->tris.push_back(bt);
        }
        return ~int32_t((base << 3) | (count - 1));
    }
};

}  // namespace

void build_bvh(const float* world_tris, const TriInfo* info, uint32_t tri_count, HostBvh& out) {
    out.nodes.clear(); out.tris.clear(); out.parent.clear(); out.info.assign(info, info + tri_count);
    out.root_child = 0;
    if (tri_count == 0) { out.root_child = ~int32_t(0); out.tris.emplace_back(); /* one degenerate (all-zero) triangle never hits */ return; }
    Builder b; b.tris = world_tris; b.n = tri_count; b.out = &out;
    b.tbox.resize(tri_count); b.cent.resize(size_t(tri_count) * 3); b.order.resize(tri_count);
    Box all, call; all.reset(); call.reset();
    for (uint32_t t = 0; t < tri_count; ++t) {
        Box bx; bx.reset();
        for (int v = 0; v < 3; ++v) bx.grow(&world_tris[size_t(t) * 9 + v * 3]);
        b.tbox[t] = bx;
        for (int a = 0; a < 3; ++a) b.cent[t * 3 + a] = 0.5f * (bx.lo[a] + bx.hi[a]);
        all.grow(bx); call.grow(&b.cent[t * 3]);
        b.order[t] = t;
    }
    out.nodes.reserve(tri_count);
    out.tris.reserve(tri_count);
    out.root_child = b.build(0, tri_count, all, call);
    out.parent.assign(out.nodes.size(), -1);
    for (size_t i = 0; i < out.nodes.size(); ++i) for (int k = 0; k < 2; ++k) if (out.nodes[i].child[k] >= 0) out.parent[size_t(out.nodes[i].child[k])] = int32_t(i << 1) | k;
}

}  // namespace kjb

// ---- C exports for the tests (emulator build only): build from gid-ordered world-space triangles (float[9] each), read the result back
extern "C" {
void* kjb_ref_bvh_build(const float* world_tris, uint32_t tri_count) {
    std::vector<kjb::TriInfo> info(tri_count);
    for (uint32_t t = 0; t < tri_count; ++t) { info[t].instance = 0; info[t].prim = t; }
    kjb::HostBvh* h = new kjb::HostBvh();
    kjb::build_bvh(world_tris, info.data(), tri_count, *h);
    return h;
}
void kjb_ref_bvh_counts(void* p, uint32_t out[2], int32_t* root) {
    const kjb::HostBvh* h = (const kjb::HostBvh*)p;
    out[0] = uint32_t(h->nodes.size()); out[1] = uint32_t(h->tris.size()); *root = h->root_child;
}
void kjb_ref_bvh_copy(void* p, void* nodes, void* tris, int32_t* parent) {
    const kjb::HostBvh* h = (const kjb::HostBvh*)p;
    memcpy(nodes, h->nodes.data(), h->nodes.size() * sizeof(kjb::BvhNode));
    memcpy(tris, h->tris.data(), h->tris.size() * sizeof(kjb::BvhTri));
    memcpy(parent, h->parent.data(), h->parent.size() * sizeof(int32_t));
}
void kjb_ref_bvh_free(void* p) { delete (kjb::HostBvh*)p; }
}

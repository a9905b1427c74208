// Device build of the acceleration structure: "rebuild tlas" when the instance list changes (kjb_api.cu, the one translation unit that
// includes this file).  It produces the tree the binned-SAH host builder this project used to run (kjb_bvh.cpp, now the test reference)
// produces, byte for byte:
//   - every split decision of that builder depends on sets only (box and centroid unions are min/max, bin counts are integers, the SAH
//     cost is evaluated per node in a fixed order: axis 0..2, bin 0..14, strict <), and the float expressions are the same on both sides
//     (no contraction, IEEE division), so the device picks the same split of the same set of triangles;
//   - leaves are slots [first, first + count) of the segment they came from, and inner nodes are numbered in DFS preorder, left child
//     first: the preorder index of an inner node is (leaves that start before its segment) + (left turns on its path from the root).
// Triangles keep ascending global id inside every segment (all partitions are stable).  Where the host builder's split depended on the
// order of its list (all centroids coincide, or depth >= 40, where it took the median of an arbitrary order) the device splits the
// gid-ordered segment at count / 2; only such subtrees can differ from the host's.  Hits do not depend on the order inside a leaf or on
// the topology (DESIGN.md "ray/triangle contract"), so frames are the same either way.
//
// Schedule, all on the context's stream, no host synchronisation:
//   flatten (one thread per triangle) -> root bounds -> per level of "large" segments (more than 32 triangles): binning into 3 x 16
//   bins (shared-memory privatised for the segment a block starts in), split choice (one thread per segment), a stable partition (a
//   scan of the go-left flags), child bounds -> every "small" segment (5..32 triangles) built depth-first by one thread -> leaf-start
//   scan -> nodes, parent links and leaf-order triangle records.
// The host does not know how many segments a level holds: every kernel reads the counts from device memory and returns early, and the
// number of levels is bounded from the triangle count (depth 40 is the last SAH level, then halving).
#pragma once
#include "kjb_context.h"
#include "kjb_ircache.cuh"

namespace kjb {
namespace bvhb {

enum { BINS = 16, LEAF = 4, SMALL = 32, SAH_DEPTH = 40, TILE = 8192, CHUNK = 2048 };
enum { BIN_WORDS = 7, SEG_BIN_WORDS = 3 * BINS * BIN_WORDS, ACC_WORDS = 12 };   // bin: 6 box keys + count; child bounds: box + centroid box keys
enum { CTR_REC = 0, CTR_ACT = 1, CTR_SMALL = 3, CTR_NODES = 4, CTR_ROOT = 5, CTR_WORDS = 32 };

struct Rec { uint32_t first, count, depth, lt; int32_t parent; uint32_t pfirst; float box[6]; };   // parent = (parent's left turns << 1) | slot, -1: root
struct Split { int32_t axis, bin; uint32_t lcount; int32_t cj[2]; uint32_t crec[2]; uint32_t pad; };

struct View {
    uint32_t n, act_cap;
    float* tbox; float* cent;
    uint32_t* ord[2]; int32_t* seg[2]; uint32_t* ord_final;
    uint32_t* scan; uint32_t* tiles;
    Rec* rec; Split* split; uint32_t* act[2]; float* cbox[2]; uint32_t* bins; uint32_t* acc; uint32_t* small; uint32_t* ctr;
};

// float <-> unsigned key whose integer order is the float order: min / max unions through integer atomics, in any order
KJB_DEV uint32_t fkey(float f) { const uint32_t u = kjb_f2u(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
KJB_DEV float fdec(uint32_t k) { return kjb_u2f((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }
KJB_DEV uint32_t empty_key(uint32_t w) { return (w % 6u) < 3u ? fkey(3.4e38f) : fkey(-3.4e38f); }   // lo words, then hi words
KJB_DEV void key_union(uint32_t* dst, const float* b6) {
    for (int a = 0; a < 3; ++a) { atom_min(dst + a, fkey(b6[a])); atom_max(dst + 3 + a, fkey(b6[3 + a])); }
}
KJB_DEV void key_union_point(uint32_t* dst, const float* p) {
    for (int a = 0; a < 3; ++a) { atom_min(dst + a, fkey(p[a])); atom_max(dst + 3 + a, fkey(p[a])); }
}
KJB_DEV void key_union_keys(uint32_t* dst, const uint32_t* src) {
    for (int a = 0; a < 3; ++a) { atom_min(dst + a, src[a]); atom_max(dst + 3 + a, src[3 + a]); }
}

// the host builder's Box, on float[6] = (lo, hi)
KJB_DEV void box_reset(float* b) { for (int a = 0; a < 3; ++a) { b[a] = 3.4e38f; b[3 + a] = -3.4e38f; } }
KJB_DEV void box_grow_point(float* b, const float* p) { for (int a = 0; a < 3; ++a) { b[a] = p[a] < b[a] ? p[a] : b[a]; b[3 + a] = b[3 + a] < p[a] ? p[a] : b[3 + a]; } }
KJB_DEV void box_grow(float* b, const float* o) { for (int a = 0; a < 3; ++a) { b[a] = o[a] < b[a] ? o[a] : b[a]; b[3 + a] = b[3 + a] < o[3 + a] ? o[3 + a] : b[3 + a]; } }
KJB_DEV float box_area(const float* b) {
    const float d0 = b[3] - b[0], d1 = b[4] - b[1], d2 = b[5] - b[2];
    return (d0 < 0 || d1 < 0 || d2 < 0) ? 0.0f : 2.0f * (d0 * d1 + d1 * d2 + d2 * d0);
}
KJB_DEV int bin_of(float c, float lo, float scale) { int b = int((c - lo) * scale); return b < 0 ? 0 : (b >= BINS ? BINS - 1 : b); }

// one axis of the SAH sweep over 16 bins, in the host builder's order; updates the best (cost, axis, split)
KJB_DEV void sah_axis(const float (*bb)[6], const uint32_t* bc, int axis, float& best_cost, int& best_axis, int& best_split) {
    float right_area[BINS]; uint32_t right_cnt[BINS];
    float acc[6]; box_reset(acc); uint32_t cnt = 0;
    for (int b = BINS - 1; b > 0; --b) { box_grow(acc, bb[b]); cnt += bc[b]; right_area[b] = box_area(acc); right_cnt[b] = cnt; }
    box_reset(acc); cnt = 0;
    for (int b = 0; b < BINS - 1; ++b) {
        box_grow(acc, bb[b]); cnt += bc[b];
        if (cnt == 0 || right_cnt[b + 1] == 0) continue;
        const float cost = box_area(acc) * float(cnt) + right_area[b + 1] * float(right_cnt[b + 1]);
        if (cost < best_cost) { best_cost = cost; best_axis = axis; best_split = b; }
    }
}

// ---- scan of u32 flags: tiles of 8192 scanned in place (inclusive), then the tile totals; scan_incl adds the tile's offset
KJB_DEV uint32_t scan_incl(const uint32_t* d, const uint32_t* tiles, uint32_t i) { const uint32_t t = i / TILE; return d[i] + (t ? tiles[t - 1] : 0u); }
KJB_DEV uint32_t scan_excl(const uint32_t* d, const uint32_t* tiles, uint32_t i) { return i ? scan_incl(d, tiles, i - 1) : 0u; }

// inclusive scan of one value per thread over a block of 1024 threads; every thread of the block must call it
__device__ __forceinline__ uint32_t block_scan(uint32_t v, uint32_t* sh, uint32_t& total) {
    const uint32_t t = threadIdx.x;
#if !defined(KJB_EMU)
    const uint32_t lane = t & 31u, warp = t >> 5, nw = blockDim.x >> 5;
    uint32_t a = v;
    for (uint32_t off = 1; off < 32u; off <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, a, off); if (lane >= off) a += u; }
    if (lane == 31u) sh[warp] = a;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < nw ? sh[lane] : 0u;
        for (uint32_t off = 1; off < 32u; off <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, w, off); if (lane >= off) w += u; }
        sh[lane] = w;
    }
    __syncthreads();
    const uint32_t r = a + (warp ? sh[warp - 1] : 0u);
    total = sh[nw - 1];
    __syncthreads();
    return r;
#else
    sh[t] = v;
    __syncthreads();
    if (t == 0) for (uint32_t i = 1; i < blockDim.x; ++i) sh[i] += sh[i - 1];
    __syncthreads();
    const uint32_t r = sh[t];
    total = sh[blockDim.x - 1];
    __syncthreads();
    return r;
#endif
}
// gate: a device counter; zero means there is nothing to scan this time
KJB_KERNEL(1024) k_bvhb_scan_tiles(uint32_t* d, uint32_t n, uint32_t* tiles, const uint32_t* gate, Rows kjb_rows) {
    __shared__ uint32_t sh[1024];
    if (gate && *gate == 0) return;
    const uint32_t base = blockIdx.x * TILE + threadIdx.x * 8u;
    uint32_t v[8], a = 0;
    for (uint32_t k = 0; k < 8u; ++k) { a += base + k < n ? d[base + k] : 0u; v[k] = a; }
    uint32_t total;
    const uint32_t before = block_scan(a, sh, total) - a;
    for (uint32_t k = 0; k < 8u; ++k) if (base + k < n) d[base + k] = v[k] + before;
    if (threadIdx.x == 0) tiles[blockIdx.x] = total;
}
KJB_KERNEL(1024) k_bvhb_scan_tile_totals(uint32_t* tiles, uint32_t n, const uint32_t* gate, Rows kjb_rows) {
    __shared__ uint32_t sh[1024];
    if (gate && *gate == 0) return;
    uint32_t carry = 0;
    for (uint32_t b = 0; b < n; b += blockDim.x) {
        const uint32_t i = b + threadIdx.x, v = i < n ? tiles[i] : 0u;
        uint32_t total;
        const uint32_t r = block_scan(v, sh, total);
        if (i < n) tiles[i] = r + carry;
        carry += total;
    }
}

// ---- flatten: one thread per triangle, gid in instance-major order
KJB_KERNEL(256) k_bvhb_init(View v, Rows kjb_rows) {
    for (uint32_t w = 0; w < CTR_WORDS; ++w) v.ctr[w] = 0;
    for (uint32_t w = 0; w < ACC_WORDS; ++w) v.ctr[CTR_ROOT + w] = empty_key(w);
}
KJB_KERNEL(256) k_bvhb_flatten(View v, SceneView sc, TriInfo* info, const uint32_t* prefix, uint32_t n_inst, Rows kjb_rows) {
    __shared__ uint32_t sh[ACC_WORDS];
    const uint32_t t = threadIdx.x, gid = blockIdx.x * blockDim.x + t;
    if (t < ACC_WORDS) sh[t] = empty_key(t);
    __syncthreads();
    if (gid < v.n) {
        uint32_t lo = 0, hi = n_inst;   // the last instance whose first triangle is <= gid (instances without triangles share a prefix value)
        while (lo < hi) { const uint32_t mid = (lo + hi + 1) >> 1; if (prefix[mid] <= gid) lo = mid; else hi = mid - 1; }
        const uint32_t prim = gid - prefix[lo];
        const kjb_instance& inst = sc.instances[lo];
        const kjb_gpu_mesh mesh = sc.meshes[inst.mesh_index];
        float b[6]; box_reset(b);
        for (int k = 0; k < 3; ++k) {
            const uint32_t idx = vb_u32(sc, mesh.index_offset + (prim * 3 + k) * 4);
            const float* p = reinterpret_cast<const float*>(sc.vertices + mesh.vertex_core_offset + size_t(idx) * 16);
            const float3 w = xform_point(inst.transform, f3(p[0], p[1], p[2]));
            const float wp[3] = {w.x, w.y, w.z};
            box_grow_point(b, wp);
        }
        float c[3];
        for (int a = 0; a < 3; ++a) c[a] = 0.5f * (b[a] + b[3 + a]);
        TriInfo ti; ti.instance = lo; ti.prim = prim; info[gid] = ti;
        for (int a = 0; a < 6; ++a) v.tbox[size_t(gid) * 6 + a] = b[a];
        for (int a = 0; a < 3; ++a) v.cent[size_t(gid) * 3 + a] = c[a];
        v.ord[0][gid] = gid; v.seg[0][gid] = 0; v.ord_final[gid] = gid;
        key_union(sh, b); key_union_point(sh + 6, c);
    }
    __syncthreads();
    if (t == 0) { key_union_keys(v.ctr + CTR_ROOT, sh); key_union_keys(v.ctr + CTR_ROOT + 6, sh + 6); }
}
KJB_DEV void init_bins(uint32_t* b) { for (uint32_t w = 0; w < SEG_BIN_WORDS; ++w) b[w] = (w % BIN_WORDS) == 6u ? 0u : empty_key(w % BIN_WORDS); }
// the root segment: a large one starts level 0, a small one goes to the depth-first builder, 4 or fewer triangles are the root leaf
KJB_KERNEL(256) k_bvhb_root(View v, Rows kjb_rows) {
    Rec r; r.first = 0; r.count = v.n; r.depth = 0; r.lt = 0; r.parent = -1; r.pfirst = 0;
    for (int a = 0; a < 6; ++a) r.box[a] = fdec(v.ctr[CTR_ROOT + a]);
    v.rec[0] = r; v.ctr[CTR_REC] = 1;
    if (v.n > SMALL) {
        v.act[0][0] = 0; v.ctr[CTR_ACT] = 1;
        for (int a = 0; a < 6; ++a) v.cbox[0][a] = fdec(v.ctr[CTR_ROOT + 6 + a]);
        init_bins(v.bins);
    } else if (v.n > LEAF) {
        v.small[0] = 0; v.ctr[CTR_SMALL] = 1;
    }
}

// ---- one level of large segments.  seg[cur][slot] = the slot's segment in this level's list, -1 once it left the level path.
KJB_KERNEL(256) k_bvhb_bin(View v, uint32_t cur, Rows kjb_rows) {
    __shared__ uint32_t sh[SEG_BIN_WORDS];
    const uint32_t t = threadIdx.x, base = blockIdx.x * CHUNK;
    if (blockIdx.x == 0 && t == 0) v.ctr[CTR_ACT + (cur ^ 1u)] = 0;   // the next level's list fills from k_bvhb_split on
    if (v.ctr[CTR_ACT + cur] == 0) return;
    const int32_t j0 = v.seg[cur][base];
    for (uint32_t w = t; w < SEG_BIN_WORDS; w += blockDim.x) sh[w] = (w % BIN_WORDS) == 6u ? 0u : empty_key(w % BIN_WORDS);
    __syncthreads();
    for (uint32_t s = base + t; s < base + CHUNK && s < v.n; s += blockDim.x) {
        const int32_t j = v.seg[cur][s];
        if (j < 0 || v.rec[v.act[cur][j]].depth >= SAH_DEPTH) continue;
        const float* cb = v.cbox[cur] + size_t(j) * 6;
        const uint32_t gid = v.ord[cur][s];
        for (int axis = 0; axis < 3; ++axis) {
            const float lo = cb[axis], ext = cb[3 + axis] - lo;
            if (!(ext > 1e-12f)) continue;
            const int b = bin_of(v.cent[size_t(gid) * 3 + axis], lo, float(BINS) / ext);
            uint32_t* dst = (j == j0 ? sh : v.bins + size_t(j) * SEG_BIN_WORDS) + (axis * BINS + b) * BIN_WORDS;
            key_union(dst, v.tbox + size_t(gid) * 6);
            atom_add(dst + 6, 1u);
        }
    }
    __syncthreads();
    if (j0 < 0) return;
    for (uint32_t i = t; i < 3u * BINS; i += blockDim.x) {
        const uint32_t* src = sh + i * BIN_WORDS;
        if (!src[6]) continue;
        uint32_t* dst = v.bins + size_t(j0) * SEG_BIN_WORDS + i * BIN_WORDS;
        key_union_keys(dst, src); atom_add(dst + 6, src[6]);
    }
}
// one thread per large segment: the host builder's split loop, then the two child records
KJB_KERNEL(256) k_bvhb_split(View v, uint32_t cur, Rows kjb_rows) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= v.ctr[CTR_ACT + cur]) return;
    const uint32_t nxt = cur ^ 1u;
    const Rec R = v.rec[v.act[cur][j]];
    const float* cb = v.cbox[cur] + size_t(j) * 6;
    const uint32_t* bins = v.bins + size_t(j) * SEG_BIN_WORDS;
    int best_axis = -1, best_split = -1; float best_cost = 3.4e38f;
    for (int axis = 0; axis < 3 && R.depth < SAH_DEPTH; ++axis) {
        if (!(cb[3 + axis] - cb[axis] > 1e-12f)) continue;
        float bb[BINS][6]; uint32_t bc[BINS];
        for (int b = 0; b < BINS; ++b) {
            const uint32_t* w = bins + (axis * BINS + b) * BIN_WORDS;
            for (int a = 0; a < 6; ++a) bb[b][a] = fdec(w[a]);
            bc[b] = w[6];
        }
        sah_axis(bb, bc, axis, best_cost, best_axis, best_split);
    }
    uint32_t lcount = 0;
    if (best_axis >= 0) {
        for (int b = 0; b <= best_split; ++b) lcount += bins[(best_axis * BINS + b) * BIN_WORDS + 6];
        if (lcount == 0 || lcount == R.count) best_axis = -1;
    }
    if (best_axis < 0) lcount = R.count / 2;   // all centroids coincide, or past the SAH depth: halve the gid-ordered segment
    Split sp; sp.axis = best_axis; sp.bin = best_split; sp.lcount = lcount; sp.pad = 0;
    const uint32_t c0 = atom_add(v.ctr + CTR_REC, 2u);
    for (uint32_t k = 0; k < 2; ++k) {
        Rec c; c.first = k ? R.first + lcount : R.first; c.count = k ? R.count - lcount : lcount; c.depth = R.depth + 1; c.lt = R.lt + (k ? 0u : 1u);
        c.parent = int32_t((R.lt << 1) | k); c.pfirst = R.first;
        for (int a = 0; a < 6; ++a) c.box[a] = 0.0f;
        v.rec[c0 + k] = c; sp.crec[k] = c0 + k; sp.cj[k] = -1;
        if (c.count > SMALL) {
            const uint32_t jn = atom_add(v.ctr + CTR_ACT + nxt, 1u);
            v.act[nxt][jn] = c0 + k; sp.cj[k] = int32_t(jn);
        } else if (c.count > LEAF) {
            v.small[atom_add(v.ctr + CTR_SMALL, 1u)] = c0 + k;
        }
        for (uint32_t w = 0; w < ACC_WORDS; ++w) v.acc[(size_t(j) * 2 + k) * ACC_WORDS + w] = empty_key(w);
    }
    v.split[j] = sp;
}
KJB_KERNEL(256) k_bvhb_flags(View v, uint32_t cur, Rows kjb_rows) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= v.n || v.ctr[CTR_ACT + cur] == 0) return;
    const int32_t j = v.seg[cur][s];
    uint32_t flag = 0;
    if (j >= 0) {
        const Split sp = v.split[j];
        if (sp.axis >= 0) {
            const float* cb = v.cbox[cur] + size_t(j) * 6;
            const float lo = cb[sp.axis], scale = float(BINS) / (cb[3 + sp.axis] - lo);
            flag = bin_of(v.cent[size_t(v.ord[cur][s]) * 3 + sp.axis], lo, scale) <= sp.bin ? 1u : 0u;
        } else {
            flag = s - v.rec[v.act[cur][j]].first < sp.lcount ? 1u : 0u;
        }
    }
    v.scan[s] = flag;
}
// stable partition: the k-th left slot of a segment goes to first + k, the k-th right slot to first + lcount + k; child bounds on the way
KJB_KERNEL(256) k_bvhb_scatter(View v, uint32_t cur, Rows kjb_rows) {
    __shared__ uint32_t sh[2 * ACC_WORDS];
    const uint32_t t = threadIdx.x, base = blockIdx.x * CHUNK, nxt = cur ^ 1u;
    if (v.ctr[CTR_ACT + cur] == 0) return;
    const int32_t j0 = v.seg[cur][base];
    if (t < 2 * ACC_WORDS) sh[t] = empty_key(t % ACC_WORDS);
    __syncthreads();
    for (uint32_t s = base + t; s < base + CHUNK && s < v.n; s += blockDim.x) {
        const int32_t j = v.seg[cur][s];
        if (j < 0) { v.seg[nxt][s] = -1; continue; }
        const Split sp = v.split[j];
        const uint32_t first = v.rec[v.act[cur][j]].first;
        const uint32_t es = scan_excl(v.scan, v.tiles, s), left = scan_incl(v.scan, v.tiles, s) - es, rank = es - scan_excl(v.scan, v.tiles, first);
        const uint32_t dst = left ? first + rank : first + sp.lcount + (s - first - rank), k = left ? 0u : 1u;
        const uint32_t gid = v.ord[cur][s];
        const int32_t cj = sp.cj[k];
        if (cj >= 0) { v.ord[nxt][dst] = gid; v.seg[nxt][dst] = cj; }
        else { v.ord_final[dst] = gid; v.seg[nxt][dst] = -1; }
        uint32_t* acc = j == j0 ? sh + k * ACC_WORDS : v.acc + (size_t(j) * 2 + k) * ACC_WORDS;
        key_union(acc, v.tbox + size_t(gid) * 6); key_union_point(acc + 6, v.cent + size_t(gid) * 3);
    }
    __syncthreads();
    if (j0 >= 0 && t < 4) key_union_keys(v.acc + size_t(j0) * 2 * ACC_WORDS + t * 6, sh + t * 6);
}
// one thread per large segment: the children's boxes, and the centroid bounds and fresh bins of the children that stay large
KJB_KERNEL(256) k_bvhb_finish(View v, uint32_t cur, Rows kjb_rows) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= v.ctr[CTR_ACT + cur]) return;
    const Split sp = v.split[j];
    for (uint32_t k = 0; k < 2; ++k) {
        const uint32_t* a = v.acc + (size_t(j) * 2 + k) * ACC_WORDS;
        for (int w = 0; w < 6; ++w) v.rec[sp.crec[k]].box[w] = fdec(a[w]);
        if (sp.cj[k] < 0) continue;
        for (int w = 0; w < 6; ++w) v.cbox[cur ^ 1u][size_t(sp.cj[k]) * 6 + w] = fdec(a[6 + w]);
    }
}
// the bins of the next level's segments: after k_bvhb_split has read this level's (one bins array serves both)
KJB_KERNEL(256) k_bvhb_clear_bins(View v, uint32_t nxt, Rows kjb_rows) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= v.ctr[CTR_ACT + nxt] * uint32_t(SEG_BIN_WORDS)) return;
    v.bins[i] = (i % BIN_WORDS) == 6u ? 0u : empty_key(i % BIN_WORDS);
}

// ---- small segments (5..32 triangles): one thread builds the whole subtree depth-first, exactly as the host builder, in ord_final
KJB_KERNEL(128) k_bvhb_small(View v, Rows kjb_rows) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= v.ctr[CTR_SMALL]) return;
    uint32_t stack[64]; int sp = 0;
    stack[sp++] = v.small[i];
    while (sp) {
        const Rec R = v.rec[stack[--sp]];
        uint32_t* o = v.ord_final + R.first;
        float cb[6]; box_reset(cb);
        for (uint32_t t = 0; t < R.count; ++t) box_grow_point(cb, v.cent + size_t(o[t]) * 3);
        int best_axis = -1, best_split = -1; float best_cost = 3.4e38f;
        for (int axis = 0; axis < 3 && R.depth < SAH_DEPTH; ++axis) {
            const float lo = cb[axis], ext = cb[3 + axis] - lo;
            if (!(ext > 1e-12f)) continue;
            const float scale = float(BINS) / ext;
            float bb[BINS][6]; uint32_t bc[BINS];
            for (int b = 0; b < BINS; ++b) { box_reset(bb[b]); bc[b] = 0; }
            for (uint32_t t = 0; t < R.count; ++t) {
                const uint32_t g = o[t]; const int b = bin_of(v.cent[size_t(g) * 3 + axis], lo, scale);
                box_grow(bb[b], v.tbox + size_t(g) * 6); bc[b]++;
            }
            sah_axis(bb, bc, axis, best_cost, best_axis, best_split);
        }
        uint32_t lcount = R.count / 2;
        if (best_axis >= 0) {
            const float lo = cb[best_axis], scale = float(BINS) / (cb[3 + best_axis] - lo);
            uint32_t tmp[SMALL], nl = 0, nr = 0; bool left[SMALL];
            for (uint32_t t = 0; t < R.count; ++t) { left[t] = bin_of(v.cent[size_t(o[t]) * 3 + best_axis], lo, scale) <= best_split; nl += left[t] ? 1u : 0u; }
            if (nl != 0 && nl != R.count) {
                for (uint32_t t = 0; t < R.count; ++t) { if (left[t]) tmp[nr++] = o[t]; }
                for (uint32_t t = 0; t < R.count; ++t) { if (!left[t]) tmp[nr++] = o[t]; }
                for (uint32_t t = 0; t < R.count; ++t) o[t] = tmp[t];
                lcount = nl;
            }
        }
        const uint32_t c0 = atom_add(v.ctr + CTR_REC, 2u);
        for (uint32_t k = 0; k < 2; ++k) {
            Rec c; c.first = k ? R.first + lcount : R.first; c.count = k ? R.count - lcount : lcount; c.depth = R.depth + 1; c.lt = R.lt + (k ? 0u : 1u);
            c.parent = int32_t((R.lt << 1) | k); c.pfirst = R.first;
            box_reset(c.box);
            for (uint32_t t = 0; t < c.count; ++t) box_grow(c.box, v.tbox + size_t(v.ord_final[c.first + t]) * 6);
            v.rec[c0 + k] = c;
            if (c.count > LEAF) stack[sp++] = c0 + k;
        }
    }
}

// ---- layout: leaf starts are scanned, then every record writes itself into its parent's slot
KJB_KERNEL(256) k_bvhb_leaf_flags(View v, Rows kjb_rows) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= v.ctr[CTR_REC]) return;
    if (v.rec[r].count <= LEAF) v.scan[v.rec[r].first] = 1u;
}
KJB_KERNEL(256) k_bvhb_emit(View v, BvhNode* nodes, int32_t* parent, Rows kjb_rows) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t nrec = v.ctr[CTR_REC];
    if (r == 0) v.ctr[CTR_NODES] = (nrec - 1) / 2;   // a binary tree of L leaves has L - 1 inner nodes
    if (r >= nrec) return;
    const Rec R = v.rec[r];
    const bool leaf = R.count <= LEAF;
    const int32_t self = leaf ? ~int32_t((R.first << 3) | (R.count - 1)) : int32_t(scan_excl(v.scan, v.tiles, R.first) + R.lt);
    if (R.parent < 0) { if (!leaf) parent[self] = -1; return; }
    const uint32_t pi = scan_excl(v.scan, v.tiles, R.pfirst) + uint32_t(R.parent >> 1), k = uint32_t(R.parent) & 1u;
    write_padded_slot(nodes[pi], int(k), R.box);
    nodes[pi].child[k] = self; nodes[pi].child[2 + k] = 0;
    if (!leaf) parent[self] = int32_t((pi << 1) | k);
}
// leaf-order triangle records: the global id here, the rest from k_refit_tris (kjb_api.cu), the same operations as every refit
KJB_KERNEL(256) k_bvhb_slots(View v, BvhTri* tris, Rows kjb_rows) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= v.n) return;
    BvhTri t; memset(&t, 0, sizeof(t)); t.gid = v.ord_final[s];
    tris[s] = t;
}

inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }
// the scratch of a build for up to `cap` triangles, carved from one allocation (null base: only the size)
inline size_t carve(uint32_t cap, uint8_t* base, View* v) {
    const size_t T = cap ? cap : 1, A = T / (SMALL + 1) + 1, tiles = T / TILE + 2;
    size_t off = 0;
    auto take = [&](size_t bytes) { uint8_t* p = base ? base + off : nullptr; off += align256(bytes); return (void*)p; };
    View w; memset(&w, 0, sizeof(w));
    w.tbox = (float*)take(T * 6 * 4); w.cent = (float*)take(T * 3 * 4);
    w.ord[0] = (uint32_t*)take(T * 4); w.ord[1] = (uint32_t*)take(T * 4); w.seg[0] = (int32_t*)take(T * 4); w.seg[1] = (int32_t*)take(T * 4);
    w.ord_final = (uint32_t*)take(T * 4); w.scan = (uint32_t*)take(T * 4); w.tiles = (uint32_t*)take(tiles * 4);
    w.rec = (Rec*)take(2 * T * sizeof(Rec)); w.split = (Split*)take(A * sizeof(Split));
    w.act[0] = (uint32_t*)take(A * 4); w.act[1] = (uint32_t*)take(A * 4); w.cbox[0] = (float*)take(A * 6 * 4); w.cbox[1] = (float*)take(A * 6 * 4);
    w.bins = (uint32_t*)take(A * SEG_BIN_WORDS * 4); w.acc = (uint32_t*)take(A * 2 * ACC_WORDS * 4);
    w.small = (uint32_t*)take((T / (LEAF + 1) + 1) * 4); w.ctr = (uint32_t*)take(CTR_WORDS * 4);
    w.act_cap = uint32_t(A);
    if (v) *v = w;
    return off;
}

}  // namespace bvhb

inline size_t bvh_build_scratch_bytes(uint32_t tri_cap) { return bvhb::carve(tri_cap, nullptr, nullptr); }
inline uint32_t* bvh_build_node_count(kjb_context* c) { bvhb::View v; bvhb::carve(c->bvh_tri_cap, (uint8_t*)c->d_bvh_scratch, &v); return v.ctr + bvhb::CTR_NODES; }

// Enqueues the build of `n` triangles from the instances and prefix already uploaded (c->g.scene.instances, c->d_inst_prefix) into the
// context's node, parent, tri_info and leaf-order gid arrays.  Capacities are the caller's (kjb_rebuild_tlas).
inline int bvh_build_on_device(kjb_context* c, uint32_t n_inst, uint32_t n) {
    using namespace bvhb;
    View v; carve(c->bvh_tri_cap, (uint8_t*)c->d_bvh_scratch, &v);
    v.n = n;
    const kjb::Rows kjb__rows = {0, 1};
    const dim3 b256(256), b1024(1024);
    const uint32_t chunks = (n + CHUNK - 1) / CHUNK, tiles = (n + TILE - 1) / TILE, recs = 2 * n, smalls = n / (LEAF + 1) + 1;
    KJB_LAUNCH(c, k_bvhb_init, KJB_DIMS(dim3(1), dim3(1)), v);
    KJB_LAUNCH_SYNC(c, k_bvhb_flatten, KJB_DIMS(dim3((n + 255) / 256), b256), v, c->g.scene, c->d_tri_info, (const uint32_t*)c->d_inst_prefix, n_inst);
    KJB_LAUNCH(c, k_bvhb_root, KJB_DIMS(dim3(1), dim3(1)), v);
    // levels of large segments: depth < 40 splits peel at least one triangle, later ones halve
    uint32_t levels = 0;
    if (n > SMALL) { uint32_t h = 0; while ((uint64_t(SMALL) << h) < n) ++h; levels = (n - SMALL < uint32_t(SAH_DEPTH) ? n - SMALL : uint32_t(SAH_DEPTH)) + h + 1; }
    for (uint32_t L = 0; L < levels; ++L) {
        const uint32_t cur = L & 1u;
        const uint32_t* gate = v.ctr + CTR_ACT + cur;
        KJB_LAUNCH_SYNC(c, k_bvhb_bin, KJB_DIMS(dim3(chunks), b256), v, cur);
        KJB_LAUNCH(c, k_bvhb_split, KJB_DIMS(dim3((v.act_cap + 255) / 256), b256), v, cur);
        KJB_LAUNCH(c, k_bvhb_clear_bins, KJB_DIMS(dim3(uint32_t((size_t(v.act_cap) * SEG_BIN_WORDS + 255) / 256)), b256), v, cur ^ 1u);
        KJB_LAUNCH(c, k_bvhb_flags, KJB_DIMS(dim3((n + 255) / 256), b256), v, cur);
        KJB_LAUNCH_SYNC(c, k_bvhb_scan_tiles, KJB_DIMS(dim3(tiles), b1024), v.scan, n, v.tiles, gate);
        KJB_LAUNCH_SYNC(c, k_bvhb_scan_tile_totals, KJB_DIMS(dim3(1), b1024), v.tiles, tiles, gate);
        KJB_LAUNCH_SYNC(c, k_bvhb_scatter, KJB_DIMS(dim3(chunks), b256), v, cur);
        KJB_LAUNCH(c, k_bvhb_finish, KJB_DIMS(dim3((v.act_cap + 255) / 256), b256), v, cur);
    }
    KJB_LAUNCH(c, k_bvhb_small, KJB_DIMS(dim3((smalls + 127) / 128), dim3(128)), v);
    if (dev_memset(c, v.scan, 0, size_t(n) * 4)) return c->fail("kjb_rebuild_tlas: memset failed");
    KJB_LAUNCH(c, k_bvhb_leaf_flags, KJB_DIMS(dim3((recs + 255) / 256), b256), v);
    KJB_LAUNCH_SYNC(c, k_bvhb_scan_tiles, KJB_DIMS(dim3(tiles), b1024), v.scan, n, v.tiles, (const uint32_t*)nullptr);
    KJB_LAUNCH_SYNC(c, k_bvhb_scan_tile_totals, KJB_DIMS(dim3(1), b1024), v.tiles, tiles, (const uint32_t*)nullptr);
    KJB_LAUNCH(c, k_bvhb_emit, KJB_DIMS(dim3((recs + 255) / 256), b256), v, c->d_nodes, c->d_node_parent);
    KJB_LAUNCH(c, k_bvhb_slots, KJB_DIMS(dim3((n + 255) / 256), b256), v, c->d_tris);
    return 0;
}

}  // namespace kjb

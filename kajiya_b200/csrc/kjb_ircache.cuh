// Irradiance cache: constants, grid addressing, sample parameters and the lookup-with-allocation used by every pass that
// binds the cache (ircache/{ircache_constants,ircache_grid,ircache_sampler_common.inc,lookup}.hlsl).
//
// The cache is a racy structure BY DESIGN upstream (docs/gi-overview.md "Irradiance cache"; ircache.rs:68-76 binds everything
// write_no_sync): cells are claimed with an atomic OR, entries popped with an atomic ADD, keep-alive is an atomic MIN and the
// reposition vote is last-writer-wins, so which thread wins is scheduling dependent.  Two schedules are built here:
//  * the reference's atomics as they land (KJB_OPTION_ORDERED_CACHE_SCHEDULE = 0, the CPU emulator's default, where launches run in
//    order; kjb_set_debug_serial runs them in launch order on the GPU too): the oracle's schedule, bit for bit;
//  * ordered (the default on the GPU): the same decisions made independently of the order the threads run in, so that the
//    same inputs give the same frames on every run.  A pass only reads the cache state it started with.  A claimed cell gets
//    its entry at the start of the next cache chain, where the claims of all passes take the lowest free entries in cell
//    order (k_ircache_det_*), and the winning vote of its claimers as its position at the chain's ageing; until then it
//    reads as just allocated, which is what every lookup of it returned anyway.  The
//    keep-alive of a lookup is applied there too.  Reposition votes keep the proposal whose hash is smallest (a 128-bit
//    compare-and-swap), i.e. a uniform choice among the voters like the reference's reservoir vote, but one that does not
//    depend on the order of the votes.  The precise lookups of the cache's own tracing passes read the per-entry reservoirs
//    as they were when the pass started (`aux_prev`), not as the pass is rewriting them.
#pragma once
#include "kjb_context.h"
#include "kjb_trace.cuh"

namespace kjb {

#define KJB_IRCACHE_GRID_CELL_DIAMETER (0.16f * 0.125f)
constexpr uint32_t IRCACHE_CASCADE_SIZE = 32, IRCACHE_CASCADE_COUNT = 12;
constexpr uint32_t IRCACHE_META_TRACING_ALLOC_COUNT = 0, IRCACHE_META_ENTRY_COUNT = 2, IRCACHE_META_ALLOC_COUNT = 3;   // u32 slots of meta_buf
constexpr uint32_t IRCACHE_ENTRY_META_OCCUPIED = 1u, IRCACHE_ENTRY_META_JUST_ALLOCATED = 2u;
constexpr uint32_t IRCACHE_ENTRY_LIFE_RECYCLE = 0x8000000u, IRCACHE_ENTRY_LIFE_RECYCLED = 0x8000001u;
constexpr uint32_t IRCACHE_ENTRY_LIFE_PER_RANK = 4, IRCACHE_ENTRY_RANK_COUNT = 3;
constexpr uint32_t IRCACHE_OCTA_DIMS = 4, IRCACHE_OCTA_DIMS2 = 16, IRCACHE_IRRADIANCE_STRIDE = 3, IRCACHE_AUX_STRIDE = 64;
constexpr uint32_t IRCACHE_SAMPLES_PER_FRAME = 4, IRCACHE_VALIDATION_SAMPLES_PER_FRAME = 4, IRCACHE_RESTIR_M_CLAMP = 30;
KJB_DEV bool is_ircache_entry_life_valid(uint32_t life) { return life < IRCACHE_ENTRY_LIFE_PER_RANK * IRCACHE_ENTRY_RANK_COUNT; }
KJB_DEV uint32_t ircache_entry_life_to_rank(uint32_t life) { return life / IRCACHE_ENTRY_LIFE_PER_RANK; }
KJB_DEV uint32_t ircache_entry_life_for_rank(uint32_t rank) { return rank * IRCACHE_ENTRY_LIFE_PER_RANK; }

// ---- device atomics (the CPU test emulator maps them to the compiler builtins)
#if defined(__CUDA_ARCH__)
KJB_DEV uint32_t atom_add(uint32_t* p, uint32_t v) { return atomicAdd(p, v); }
KJB_DEV uint32_t atom_or(uint32_t* p, uint32_t v) { return atomicOr(p, v); }
KJB_DEV uint32_t atom_and(uint32_t* p, uint32_t v) { return atomicAnd(p, v); }
KJB_DEV uint32_t atom_min(uint32_t* p, uint32_t v) { return atomicMin(p, v); }
KJB_DEV uint32_t atom_max(uint32_t* p, uint32_t v) { return atomicMax(p, v); }
#else
KJB_DEV uint32_t atom_add(uint32_t* p, uint32_t v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
KJB_DEV uint32_t atom_or(uint32_t* p, uint32_t v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
KJB_DEV uint32_t atom_and(uint32_t* p, uint32_t v) { return __atomic_fetch_and(p, v, __ATOMIC_RELAXED); }
KJB_DEV uint32_t atom_min(uint32_t* p, uint32_t v) { uint32_t c = *p; while (c > v && !__atomic_compare_exchange_n(p, &c, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {} return c; }
KJB_DEV uint32_t atom_max(uint32_t* p, uint32_t v) { uint32_t c = *p; while (c < v && !__atomic_compare_exchange_n(p, &c, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {} return c; }
#endif

KJB_DEV uint32_t kjb_popc(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __popc(x);
#else
    return uint32_t(__builtin_popcount(x));
#endif
}
// 128-bit compare-and-swap (sm_90); returns the value found
KJB_DEV uint4 atom_cas128(float4* p, uint4 expected, uint4 desired) {
#if defined(__CUDA_ARCH__)
    unsigned long long lo, hi;
    const unsigned long long elo = expected.x | (unsigned long long)expected.y << 32, ehi = expected.z | (unsigned long long)expected.w << 32;
    const unsigned long long dlo = desired.x | (unsigned long long)desired.y << 32, dhi = desired.z | (unsigned long long)desired.w << 32;
    asm volatile("{\n\t.reg .b128 e, d, r;\n\tmov.b128 e, {%2, %3};\n\tmov.b128 d, {%4, %5};\n\tatom.cas.b128 r, [%6], e, d;\n\tmov.b128 {%0, %1}, r;\n\t}"
                 : "=l"(lo), "=l"(hi) : "l"(elo), "l"(ehi), "l"(dlo), "l"(dhi), "l"(p) : "memory");
    return make_uint4(uint32_t(lo), uint32_t(lo >> 32), uint32_t(hi), uint32_t(hi >> 32));
#else
    unsigned __int128 e, d; memcpy(&e, &expected, 16); memcpy(&d, &desired, 16);
    const unsigned __int128 r = __sync_val_compare_and_swap(reinterpret_cast<unsigned __int128*>(p), e, d);
    uint4 out; memcpy(&out, &r, 16); return out;
#endif
}
KJB_DEV bool u4_eq(uint4 a, uint4 b) { return a.x == b.x && a.y == b.y && a.z == b.z && a.w == b.w; }
KJB_DEV bool vertex_vote_beats(uint4 a, uint4 b) {   // an empty (all-zero) slot loses to any vote; else the smaller hash, then the smaller bits
    if (b.x == 0u && b.y == 0u && b.z == 0u && b.w == 0u) return true;
    const uint32_t ka = hash1(a.x ^ hash1(a.y ^ hash1(a.z ^ hash1(a.w)))), kb = hash1(b.x ^ hash1(b.y ^ hash1(b.z ^ hash1(b.w))));
    if (ka != kb) return ka < kb;
    if (a.x != b.x) return a.x < b.x;
    if (a.y != b.y) return a.y < b.y;
    if (a.z != b.z) return a.z < b.z;
    return a.w < b.w;
}
// the slot ends up holding the winning vote of all the votes cast into it, whatever their order
KJB_DEV void vertex_vote(float4* slot, float4 v) {
    const uint4 nv = make_uint4(kjb_f2u(v.x), kjb_f2u(v.y), kjb_f2u(v.z), kjb_f2u(v.w));
    uint4 cur = atom_cas128(slot, make_uint4(0u, 0u, 0u, 0u), make_uint4(0u, 0u, 0u, 0u));   // an atomic read
    while (vertex_vote_beats(nv, cur)) {
        const uint4 prev = atom_cas128(slot, cur, nv);
        if (u4_eq(prev, cur)) return;
        cur = prev;
    }
}

// DEFINE_IRCACHE_BINDINGS (ircache/bindings.hlsl) + the aux buffer for IRCACHE_LOOKUP_PRECISE, + the scratch of the parallel schedule
struct IrcacheBufs {
    uint32_t *meta, *pool, *reposition_count, *grid_meta, *entry_cell, *life;
    float4 *reposition_proposal, *spatial, *irradiance, *aux;
    uint32_t* claim_rank = nullptr;      // per cell: RANK_COUNT - the lowest rank that claimed it since the last chain, 0 = unclaimed
    float4* claim_vertex = nullptr;      // per cell: the winning reposition vote of its claimers
    uint32_t* life_pending = nullptr;    // per entry: RECYCLE - the lowest life a lookup asked for, 0 = none
    const float4* aux_prev = nullptr;    // per entry: its 32 reservoir + contribution texels as the pass found them
    bool det = false;                    // the parallel schedule above
    KJB_DEV bool bound() const { return meta != nullptr; }
};
inline IrcacheBufs ircache_bufs(const kjb_ircache_bindings& b) {
    IrcacheBufs r; r.meta = (uint32_t*)b.meta_buf.data; r.pool = (uint32_t*)b.pool_buf.data; r.reposition_count = (uint32_t*)b.reposition_proposal_count_buf.data;
    r.grid_meta = (uint32_t*)b.grid_meta_buf.data; r.entry_cell = (uint32_t*)b.entry_cell_buf.data; r.life = (uint32_t*)b.life_buf.data;
    r.reposition_proposal = (float4*)b.reposition_proposal_buf.data; r.spatial = (float4*)b.spatial_buf.data; r.irradiance = (float4*)b.irradiance_buf.data; r.aux = nullptr;   /* not in the binding block: the rtdgi / rtr lookups are never IRCACHE_LOOKUP_PRECISE */
    return r;
}

// ---- ircache_grid.hlsl
struct IrcacheCoord { uint32_t cx, cy, cz, cascade; };
KJB_DEV uint32_t ircache_cell_idx(const IrcacheCoord& c) { return c.cx + c.cy * 32u + c.cz * 1024u + c.cascade * 32768u; }
KJB_DEV uint32_t ws_local_pos_to_cascade_idx(float3 local_pos, uint32_t reserved_cells) {   // :34-39
    const float3 fcoord = local_pos / KJB_IRCACHE_GRID_CELL_DIAMETER;
    const float max_coord = kjb_max(kjb_abs(fcoord.x), kjb_max(kjb_abs(fcoord.y), kjb_abs(fcoord.z)));
    const float cascade_float = kjb_log2(max_coord / float(IRCACHE_CASCADE_SIZE / 2 - reserved_cells));
    return kjb_cvt_u32(kjb_clamp(kjb_ceil(kjb_max(0.0f, cascade_float)), 0.0f, float(IRCACHE_CASCADE_COUNT - 1)));
}
KJB_DEV float ircache_grid_cell_diameter_in_cascade(uint32_t cascade) { return KJB_IRCACHE_GRID_CELL_DIAMETER * float(1u << cascade); }
KJB_DEV IrcacheCoord ws_pos_to_ircache_coord(const kjb_frame_constants& fc, float3 pos, float3 normal, float3 jitter) {   // :41-75
    const float3 center = f3(fc.ircache_grid_center[0], fc.ircache_grid_center[1], fc.ircache_grid_center[2]);
    const uint32_t reserved_cells = 1;
    {
        const uint32_t cascade = ws_local_pos_to_cascade_idx(pos - center, reserved_cells);
        pos = pos + ircache_grid_cell_diameter_in_cascade(cascade) * jitter;
    }
    const uint32_t cascade = ws_local_pos_to_cascade_idx(pos - center, reserved_cells);
    const float cell_diameter = ircache_grid_cell_diameter_in_cascade(cascade);
    const int32_t* co = fc.ircache_cascades[cascade].origin;
    const float3 cell_offset = normal * cell_diameter * 0.5f;
    const float3 q = (pos + cell_offset) / cell_diameter;
    const int ix = kjb_cvt_i32(kjb_floor(q.x)) - co[0], iy = kjb_cvt_i32(kjb_floor(q.y)) - co[1], iz = kjb_cvt_i32(kjb_floor(q.z)) - co[2];
    IrcacheCoord r; r.cascade = cascade;
    r.cx = uint32_t(ix < 0 ? 0 : (ix > 31 ? 31 : ix)); r.cy = uint32_t(iy < 0 ? 0 : (iy > 31 ? 31 : iy)); r.cz = uint32_t(iz < 0 ? 0 : (iz > 31 ? 31 : iz));
    return r;
}

// ---- pack_unpack.hlsl:79-88 / ircache_sampler_common.inc.hlsl
KJB_DEV float3 octa_decode(float2 f) {
    f = f * 2.0f - 1.0f;
    float3 n = f3(f.x, f.y, 1.0f - kjb_abs(f.x) - kjb_abs(f.y));
    const float t = kjb_clamp(-n.z, 0.0f, 1.0f);
    n.x -= (kjb_step(0.0f, n.x) * 2 - 1) * t;
    n.y -= (kjb_step(0.0f, n.y) * 2 - 1) * t;
    return normalize(n);
}
struct SampleParams {
    uint32_t value;
    KJB_DEV static SampleParams from_spf_entry_sample_frame(uint32_t spf, uint32_t entry_idx, uint32_t sample_idx, uint32_t frame_idx) {
        const uint32_t PERIOD = IRCACHE_OCTA_DIMS2 / spf;
        uint32_t xy = sample_idx * PERIOD + (frame_idx % PERIOD);
        xy ^= (xy & 4u) >> 2u;   // checkerboard
        SampleParams r; r.value = xy + ((frame_idx << 16u) ^ entry_idx) * IRCACHE_OCTA_DIMS2; return r;
    }
    KJB_DEV static SampleParams from_raw(uint32_t raw) { SampleParams r; r.value = raw; return r; }
    KJB_DEV uint32_t octa_idx() const { return value % IRCACHE_OCTA_DIMS2; }
    KJB_DEV uint32_t rng() const { return hash1(value >> 4u); }
    KJB_DEV float3 direction() const {
        const uint32_t oi = octa_idx();
        const float2 urand = r2_sequence(rng() % 1024u);
        return octa_decode((f2(float(oi % IRCACHE_OCTA_DIMS), float(oi / IRCACHE_OCTA_DIMS)) + urand) / 4.0f);
    }
};

// ---- inc/mesh.hlsl:25-46
struct IrcacheVertex { float3 position, normal; };
KJB_DEV IrcacheVertex unpack_vertex(float4 p) {
    const uint32_t pck = kjb_f2u(p.w);
    IrcacheVertex v; v.position = xyz(p);
    v.normal = f3(float(pck & 2047u) * (2.0f / 2047.0f) - 1.0f, float((pck >> 11u) & 1023u) * (2.0f / 1023.0f) - 1.0f, float(pck >> 21u) * (2.0f / 2047.0f) - 1.0f);
    return v;
}
KJB_DEV float4 pack_vertex(const IrcacheVertex& v) { return f4(v.position, kjb_u2f(pack_normal_11_10_11(v.normal))); }

KJB_DEV float eval_sh_geometrics(float4 sh, float3 normal) {   // lookup.hlsl:197-212
    const float R0 = sh.x;
    const float3 R1 = 0.5f * f3(sh.y, sh.z, sh.w);
    const float lenR1 = length(R1);
    const float q = 0.5f * (1.0f + dot(R1 / lenR1, normal));
    const float p = 1.0f + 2.0f * lenR1 / R0;
    const float a = (1.0f - lenR1 / R0) / (1.0f + lenR1 / R0);
    return R0 * (a + (1.0f - a) * (p + 1.0f) * kjb_pow(q, p));
}

template <bool PRECISE>
KJB_DEV float3 ircache_lookup_parallel(const Globals& g, const IrcacheBufs& b, float3 query_from_ws, float3 pt_ws, float3 normal_ws, uint32_t query_rank, uint32_t& rng, bool stochastic_interpolation);

// IrcacheLookupParams::lookup (lookup.hlsl:76-311) with the maybe-allocating lookup it wraps (:19-74,:120-190).
// PRECISE = IRCACHE_LOOKUP_PRECISE: sum the per-direction reservoirs instead of evaluating the SH (the cache's own tracing passes).
template <bool PRECISE>
KJB_DEV float3 ircache_lookup(const Globals& g, const IrcacheBufs& b, float3 query_from_ws, float3 pt_ws, float3 normal_ws, uint32_t query_rank, uint32_t& rng, bool stochastic_interpolation = false) {
    if (!b.bound()) return f3(0.0f);
    if (b.det) return ircache_lookup_parallel<PRECISE>(g, b, query_from_ws, pt_ws, normal_ws, query_rank, rng, stochastic_interpolation);
    const kjb_frame_constants& fc = g.fc;
    bool allocated_by_us = false, just_allocated = false;
    // lookup.hlsl:80-86: the three rng draws sit in the arguments of select(), i.e. they happen whether or not interpolation is on
    float3 jr; jr.x = rand01(rng); jr.y = rand01(rng); jr.z = rand01(rng);
    const IrcacheCoord rc = ws_pos_to_ircache_coord(fc, pt_ws, normal_ws, stochastic_interpolation ? jr - 0.5f : f3(0.0f));
    const uint32_t cell_idx = ircache_cell_idx(rc);
    {
        const int32_t* so = fc.ircache_cascades[rc.cascade].voxels_scrolled_this_frame;
        const int c3[3] = {int(rc.cx), int(rc.cy), int(rc.cz)};
        bool was_just_scrolled_in = false;
        for (int k = 0; k < 3; ++k) was_just_scrolled_in = was_just_scrolled_in || (so[k] > 0 ? (c3[k] + so[k] >= int(IRCACHE_CASCADE_SIZE)) : (c3[k] < -so[k]));
        const bool skip_allocation = query_rank >= IRCACHE_ENTRY_RANK_COUNT || (was_just_scrolled_in && query_rank > 0);
        const uint32_t entry_flags = b.grid_meta[cell_idx * 2 + 1];
        just_allocated = (entry_flags & IRCACHE_ENTRY_META_JUST_ALLOCATED) != 0;
        if (!skip_allocation && (entry_flags & IRCACHE_ENTRY_META_OCCUPIED) == 0) {
            const uint32_t prev = atom_or(&b.grid_meta[cell_idx * 2 + 1], IRCACHE_ENTRY_META_OCCUPIED | IRCACHE_ENTRY_META_JUST_ALLOCATED);
            if ((prev & IRCACHE_ENTRY_META_OCCUPIED) == 0) {   // we claimed the cell
                just_allocated = true; allocated_by_us = true;
                const uint32_t alloc_idx = atom_add(&b.meta[IRCACHE_META_ALLOC_COUNT], 1u);
                if (alloc_idx >= 1024u * 64u) {   // pool exhausted: undo
                    atom_add(&b.meta[IRCACHE_META_ALLOC_COUNT], uint32_t(-1));
                    atom_and(&b.grid_meta[cell_idx * 2 + 1], ~(IRCACHE_ENTRY_META_OCCUPIED | IRCACHE_ENTRY_META_JUST_ALLOCATED));
                } else {
                    const uint32_t entry_idx = b.pool[alloc_idx];
                    atom_max(&b.meta[IRCACHE_META_ENTRY_COUNT], entry_idx + 1);
                    b.life[entry_idx] = ircache_entry_life_for_rank(query_rank);   // clear dead state, mark used
                    b.entry_cell[entry_idx] = cell_idx;
                    b.grid_meta[cell_idx * 2 + 0] = entry_idx;
                }
            }
        }
    }
    uint32_t lookup_count = 0, lookup_entry = 0;
    if (b.grid_meta[cell_idx * 2 + 1] & IRCACHE_ENTRY_META_OCCUPIED) { lookup_entry = b.grid_meta[cell_idx * 2 + 0]; lookup_count = 1; }

    const float cell_diameter = ircache_grid_cell_diameter_in_cascade(rc.cascade);
    float3 offset_towards_query = query_from_ws - pt_ws;
    const float MAX_OFFSET = cell_diameter, MAX_OFFSET_AS_FRAC = 0.5f;
    offset_towards_query = offset_towards_query * (MAX_OFFSET / kjb_max(MAX_OFFSET / MAX_OFFSET_AS_FRAC, length(offset_towards_query)));
    IrcacheVertex new_entry; new_entry.position = pt_ws + offset_towards_query; new_entry.normal = normal_ws;
    if (allocated_by_us && lookup_count) b.reposition_proposal[lookup_entry] = pack_vertex(new_entry);
    if (just_allocated) return f3(0.0f);

    float3 irradiance_sum = f3(0.0f);
    if (lookup_count) {
        const uint32_t entry_idx = lookup_entry;
        float3 irradiance = f3(0.0f);
        if (PRECISE) {
            float weight_sum = 0;
            for (uint32_t octa_idx = 0; octa_idx < IRCACHE_OCTA_DIMS2; ++octa_idx) {
                const float4 ra = b.aux[entry_idx * IRCACHE_AUX_STRIDE + octa_idx];
                const Reservoir r = Reservoir::from_raw(u2(kjb_f2u(ra.x), kjb_f2u(ra.y)));
                const float3 dir = SampleParams::from_raw(r.payload).direction();
                const float wt = dot(dir, normal_ws);
                if (wt > 0.0f) {
                    const float4 contrib = b.aux[entry_idx * IRCACHE_AUX_STRIDE + IRCACHE_OCTA_DIMS2 + octa_idx];
                    irradiance += xyz(contrib) * wt * contrib.w;
                    weight_sum += wt;
                }
            }
            irradiance = irradiance / kjb_max(1.0f, weight_sum);
        } else {
            irradiance.x += eval_sh_geometrics(b.irradiance[entry_idx * 3 + 0], normal_ws);
            irradiance.y += eval_sh_geometrics(b.irradiance[entry_idx * 3 + 1], normal_ws);
            irradiance.z += eval_sh_geometrics(b.irradiance[entry_idx * 3 + 2], normal_ws);
        }
        irradiance = vmax(f3(0.0f), irradiance);
        irradiance_sum += irradiance * 1.0f;
        const uint32_t prev_life = b.life[entry_idx];
        if (prev_life < IRCACHE_ENTRY_LIFE_RECYCLE) {
            const uint32_t new_life = ircache_entry_life_for_rank(query_rank);
            if (new_life < prev_life) atom_min(&b.life[entry_idx], new_life);
            const uint32_t prev_rank = ircache_entry_life_to_rank(prev_life);
            if (query_rank <= prev_rank) {   // IRCACHE_USE_POSITION_VOTING + IRCACHE_USE_UNIFORM_VOTING
                const uint32_t prev_vote_count = atom_add(&b.reposition_count[entry_idx], 1u);
                const float dart = rand01(rng);
                const float prob = 1.0f / (float(prev_vote_count) + 1.0f);
                if (dart <= prob) b.reposition_proposal[entry_idx] = pack_vertex(new_entry);
            }
        }
    }
    return irradiance_sum;
}

// The same lookup on the parallel schedule (header comment): the same returned value and the same draws from `rng`; the cache
// updates go where their order cannot matter.
template <bool PRECISE>
KJB_DEV float3 ircache_lookup_parallel(const Globals& g, const IrcacheBufs& b, float3 query_from_ws, float3 pt_ws, float3 normal_ws, uint32_t query_rank, uint32_t& rng, bool stochastic_interpolation) {
    const kjb_frame_constants& fc = g.fc;
    float3 jr; jr.x = rand01(rng); jr.y = rand01(rng); jr.z = rand01(rng);
    const IrcacheCoord rc = ws_pos_to_ircache_coord(fc, pt_ws, normal_ws, stochastic_interpolation ? jr - 0.5f : f3(0.0f));
    const uint32_t cell_idx = ircache_cell_idx(rc);
    const float cell_diameter = ircache_grid_cell_diameter_in_cascade(rc.cascade);
    float3 offset_towards_query = query_from_ws - pt_ws;
    const float MAX_OFFSET = cell_diameter, MAX_OFFSET_AS_FRAC = 0.5f;
    offset_towards_query = offset_towards_query * (MAX_OFFSET / kjb_max(MAX_OFFSET / MAX_OFFSET_AS_FRAC, length(offset_towards_query)));
    IrcacheVertex new_entry; new_entry.position = pt_ws + offset_towards_query; new_entry.normal = normal_ws;

    const uint32_t entry_flags = b.grid_meta[cell_idx * 2 + 1];
    // no entry yet: unoccupied, or claimed (occupied + just allocated) and waiting for the next chain.  Every such lookup takes part in the
    // claim, whether or not another one got there first: the claim's rank and position do not depend on who read the flags when.
    if ((entry_flags & (IRCACHE_ENTRY_META_OCCUPIED | IRCACHE_ENTRY_META_JUST_ALLOCATED)) != IRCACHE_ENTRY_META_OCCUPIED) {
        const int32_t* so = fc.ircache_cascades[rc.cascade].voxels_scrolled_this_frame;
        const int c3[3] = {int(rc.cx), int(rc.cy), int(rc.cz)};
        bool was_just_scrolled_in = false;
        for (int k = 0; k < 3; ++k) was_just_scrolled_in = was_just_scrolled_in || (so[k] > 0 ? (c3[k] + so[k] >= int(IRCACHE_CASCADE_SIZE)) : (c3[k] < -so[k]));
        if (!(query_rank >= IRCACHE_ENTRY_RANK_COUNT || (was_just_scrolled_in && query_rank > 0))) {   // claim: the entry comes with the next chain
            atom_or(&b.grid_meta[cell_idx * 2 + 1], IRCACHE_ENTRY_META_OCCUPIED | IRCACHE_ENTRY_META_JUST_ALLOCATED);
            atom_max(&b.claim_rank[cell_idx], IRCACHE_ENTRY_RANK_COUNT - query_rank);
            vertex_vote(&b.claim_vertex[cell_idx], pack_vertex(new_entry));
        }
        return f3(0.0f);
    }

    const uint32_t entry_idx = b.grid_meta[cell_idx * 2 + 0];
    float3 irradiance = f3(0.0f);
    if (PRECISE) {
        float weight_sum = 0;
        for (uint32_t octa_idx = 0; octa_idx < IRCACHE_OCTA_DIMS2; ++octa_idx) {
            const float4 ra = b.aux_prev[entry_idx * 32u + octa_idx];
            const Reservoir r = Reservoir::from_raw(u2(kjb_f2u(ra.x), kjb_f2u(ra.y)));
            const float3 dir = SampleParams::from_raw(r.payload).direction();
            const float wt = dot(dir, normal_ws);
            if (wt > 0.0f) {
                const float4 contrib = b.aux_prev[entry_idx * 32u + IRCACHE_OCTA_DIMS2 + octa_idx];
                irradiance += xyz(contrib) * wt * contrib.w;
                weight_sum += wt;
            }
        }
        irradiance = irradiance / kjb_max(1.0f, weight_sum);
    } else {
        irradiance.x += eval_sh_geometrics(b.irradiance[entry_idx * 3 + 0], normal_ws);
        irradiance.y += eval_sh_geometrics(b.irradiance[entry_idx * 3 + 1], normal_ws);
        irradiance.z += eval_sh_geometrics(b.irradiance[entry_idx * 3 + 2], normal_ws);
    }
    irradiance = vmax(f3(0.0f), irradiance);
    const uint32_t prev_life = b.life[entry_idx];   // not written while a pass runs: the keep-alive waits in life_pending
    if (prev_life < IRCACHE_ENTRY_LIFE_RECYCLE) {
        const uint32_t new_life = ircache_entry_life_for_rank(query_rank);
        if (new_life < prev_life) atom_max(&b.life_pending[entry_idx], IRCACHE_ENTRY_LIFE_RECYCLE - new_life);
        if (query_rank <= ircache_entry_life_to_rank(prev_life)) {
            atom_add(&b.reposition_count[entry_idx], 1u);
            (void)rand01(rng);   // the serial schedule's dart: drawn all the same, so that the caller's stream does not depend on the schedule
            vertex_vote(&b.reposition_proposal[entry_idx], pack_vertex(new_entry));
        }
    }
    return irradiance;
}

// the ordered schedule's scratch of the cache whose life buffer is `life` (allocated zeroed on first use); false = the reference's atomics
inline bool ircache_parallel_scratch(kjb_context* c, const void* life, kjb_context::IrcacheScratch& out) {
    if (c->debug_serial || !c->ordered_cache || !life) return false;
    auto it = c->ircache_scratch.find(life);
    if (it == c->ircache_scratch.end()) {
        kjb_context::IrcacheScratch s;
        s.claim_rank = dev_alloc(4ull * KJB_IRCACHE_GRID_CELLS); s.claim_vertex = dev_alloc(16ull * KJB_IRCACHE_GRID_CELLS);
        s.life_pending = dev_alloc(4ull * KJB_IRCACHE_MAX_ENTRIES); s.scan = dev_alloc(4ull * (KJB_IRCACHE_MAX_ENTRIES + KJB_IRCACHE_GRID_CELLS / 32));
        s.claim_bits = dev_alloc(4ull * KJB_IRCACHE_GRID_CELLS / 32); s.aux_prev = dev_alloc(16ull * 32 * KJB_IRCACHE_MAX_ENTRIES); s.entry_vertex = dev_alloc(16ull * KJB_IRCACHE_MAX_ENTRIES);
        if (!s.claim_rank || !s.claim_vertex || !s.life_pending || !s.scan || !s.claim_bits || !s.aux_prev || !s.entry_vertex) {
            dev_free(s.claim_rank); dev_free(s.claim_vertex); dev_free(s.life_pending); dev_free(s.scan); dev_free(s.claim_bits); dev_free(s.aux_prev); dev_free(s.entry_vertex);
            return false;
        }
        it = c->ircache_scratch.emplace(life, s).first;
    }
    out = it->second;
    return true;
}
inline void ircache_attach_parallel(kjb_context* c, IrcacheBufs& b) {
    kjb_context::IrcacheScratch s;
    if (!b.bound() || !ircache_parallel_scratch(c, b.life, s)) return;
    b.claim_rank = (uint32_t*)s.claim_rank; b.claim_vertex = (float4*)s.claim_vertex; b.life_pending = (uint32_t*)s.life_pending; b.aux_prev = (const float4*)s.aux_prev;
    b.det = true;
}

}  // namespace kjb

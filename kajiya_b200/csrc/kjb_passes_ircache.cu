// Irradiance cache (ircache) as sm_90a kernels — one kernel per render-graph pass of
// crates/lib/kajiya/src/renderers/ircache.rs, shader sources under /root/reference/assets/shaders/ircache/.
// All passes are 1-D over cache entries / grid cells.  The reference's indirect dispatches become fixed-size launches that
// early-out on the counters in `meta_buf` (like the reference's own fixed-size validate/trace dispatches, ircache.rs:438-476),
// so no pass needs a host round trip.  Working set: 64 MB of per-entry reservoirs (aux) + 6 MB of grid metadata — L2-resident.
#include "kjb_context.h"
#include "kjb_ircache.cuh"

using namespace kjb;

#define MAX_ENTRIES KJB_IRCACHE_MAX_ENTRIES

KJB_DEV uint32_t tid1d() { return blockIdx.x * blockDim.x + threadIdx.x; }

// Slot 0 of the indirection table is never written (the compaction scan is inclusive, ircache_compact_entries.hlsl:17), so it keeps
// naming entry 0, which — when alive — is also slot 1.  On the reference's GPU both copies sit in adjacent lanes of one wave and run
// in lockstep: same reads, same writes, i.e. the entry is processed ONCE.  We get the same effect schedule-independently by
// skipping the stale slot when it duplicates slot 1.
KJB_DEV bool ircache_slot_is_stale_duplicate(const uint32_t* indirection, uint32_t alloc_count, uint32_t slot) {
    return slot == 0u && alloc_count > 1u && indirection[1] == indirection[0];
}

// ------------------------------------------------------------------ I1 clear_ircache_pool.hlsl
KJB_KERNEL(256) k_ircache_clear_pool(uint32_t* pool, uint32_t* life, Rows kjb_rows) {
    const uint32_t idx = tid1d(); if (idx >= MAX_ENTRIES) return;
    pool[idx] = idx; life[idx] = IRCACHE_ENTRY_LIFE_RECYCLED;
}

// ------------------------------------------------------------------ I2 scroll_cascades.hlsl:36-69
KJB_DEV void ircache_scroll_cell(const Globals& g, const uint32_t* gm, uint32_t* gm2, uint32_t* entry_cell, float4* irradiance, uint32_t* life, uint32_t* pool, uint32_t* meta, uint32_t dst_cell_idx,
                                 bool parallel = false) {
    const uint32_t x = dst_cell_idx & 31u, y = (dst_cell_idx >> 5) & 31u, z = (dst_cell_idx >> 10) & 31u, cascade = dst_cell_idx >> 15;
    const int32_t* sb = g.fc.ircache_cascades[cascade].voxels_scrolled_this_frame;
    const uint32_t ox = x - uint32_t(sb[0]), oy = y - uint32_t(sb[1]), oz = z - uint32_t(sb[2]);
    if (!(ox < 32u && oy < 32u && oz < 32u)) {   // about to be overwritten: deallocate_cell
        const uint32_t m0 = gm[dst_cell_idx * 2], m1 = gm[dst_cell_idx * 2 + 1];
        if (m1 & IRCACHE_ENTRY_META_OCCUPIED) {
            const uint32_t entry_idx = m0;
            life[entry_idx] = IRCACHE_ENTRY_LIFE_RECYCLED;
            for (uint32_t i = 0; i < IRCACHE_IRRADIANCE_STRIDE; ++i) irradiance[entry_idx * IRCACHE_IRRADIANCE_STRIDE + i] = f4(0.0f);
            const uint32_t entry_alloc_count = atom_add(&meta[IRCACHE_META_ALLOC_COUNT], uint32_t(-1));
            if (!parallel) pool[entry_alloc_count - 1] = entry_idx;   // the parallel schedule rebuilds the pool in entry order instead
        }
    }
    const uint32_t sx = x + uint32_t(sb[0]), sy = y + uint32_t(sb[1]), sz = z + uint32_t(sb[2]);
    if (sx < 32u && sy < 32u && sz < 32u) {
        const uint32_t src_cell_idx = sx + sy * 32u + sz * 1024u + cascade * 32768u;
        const uint32_t m0 = gm[src_cell_idx * 2], m1 = gm[src_cell_idx * 2 + 1];
        gm2[dst_cell_idx * 2] = m0; gm2[dst_cell_idx * 2 + 1] = m1;
        if (m1 & IRCACHE_ENTRY_META_OCCUPIED) entry_cell[m0] = dst_cell_idx;
    } else { gm2[dst_cell_idx * 2] = 0; gm2[dst_cell_idx * 2 + 1] = 0; }
}
// SERIAL (here and in the age, validate and trace passes): ONE thread walks the logical threads in launch order — the serial schedule
// (kjb_set_debug_serial, KJB_SERIAL_1D in kjb_context.h); the ordered schedule's scratch is never attached under it (`parallel` = 0)
template <bool SERIAL>
KJB_KERNEL(256) k_ircache_scroll_cascades(const __grid_constant__ Globals g, const uint32_t* gm, uint32_t* gm2, uint32_t* entry_cell, float4* irradiance, uint32_t* life, uint32_t* pool, uint32_t* meta,
                                          uint32_t parallel, Rows kjb_rows) {
    if constexpr (SERIAL) KJB_SERIAL_1D(KJB_IRCACHE_GRID_CELLS, ircache_scroll_cell(g, gm, gm2, entry_cell, irradiance, life, pool, meta, i, parallel != 0));
    else { const uint32_t i = tid1d(); if (i < KJB_IRCACHE_GRID_CELLS) ircache_scroll_cell(g, gm, gm2, entry_cell, irradiance, life, pool, meta, i, parallel != 0); }
}

// ------------------------------------------------------------------ I3 prepare_age_dispatch_args.hlsl / prepare_trace_dispatch_args.hlsl
KJB_KERNEL(32) k_ircache_prepare_age_args(const uint32_t* meta, uint32_t* args, Rows kjb_rows) {
    if (tid1d() != 0) return;
    args[0] = (meta[IRCACHE_META_ENTRY_COUNT] + 63u) / 64u; args[1] = 1; args[2] = 1; args[3] = 0;
}
KJB_KERNEL(32) k_ircache_prepare_trace_args(uint32_t* meta, uint32_t* args, Rows kjb_rows) {
    if (tid1d() != 0) return;
    const uint32_t alloc_count = meta[IRCACHE_META_ALLOC_COUNT];
    meta[IRCACHE_META_TRACING_ALLOC_COUNT] = alloc_count;
    args[8] = (alloc_count + 63u) / 64u; args[9] = 1; args[10] = 1; args[11] = 0;                      // reset, sum up irradiance
    const uint32_t a = alloc_count * IRCACHE_SAMPLES_PER_FRAME, b = alloc_count * IRCACHE_OCTA_DIMS2, v = alloc_count * IRCACHE_VALIDATION_SAMPLES_PER_FRAME;
    const uint32_t mx = a > b ? (a > v ? a : v) : (b > v ? b : v);
    args[0] = mx; args[1] = 1; args[2] = 1; args[3] = 0;  args[4] = mx; args[5] = 1; args[6] = 1; args[7] = 0;  args[12] = mx; args[13] = 1; args[14] = 1; args[15] = 0;
}

// ------------------------------------------------------------------ I4 age_ircache_entries.hlsl:55-94
KJB_DEV void ircache_age_entry(uint32_t* meta, uint32_t* gm, uint32_t* entry_cell, uint32_t* life, uint32_t* pool, float4* spatial, float4* proposal, uint32_t* proposal_count,
                               float4* irradiance, uint32_t* occupancy, uint32_t entry_idx, float4* entry_vertex = nullptr) {
    const uint32_t total_entry_count = meta[IRCACHE_META_ENTRY_COUNT];
    if (entry_idx >= (total_entry_count + 63u) / 64u * 64u) return;   // the reference dispatches ceil(entry_count / 64) groups
    if (entry_idx < total_entry_count) {
        const uint32_t prev_age = life[entry_idx];
        if (prev_age != IRCACHE_ENTRY_LIFE_RECYCLED) {
            const uint32_t new_age = prev_age + 1;
            if (is_ircache_entry_life_valid(new_age)) {
                life[entry_idx] = new_age;
                atom_and(&gm[entry_cell[entry_idx] * 2 + 1], ~IRCACHE_ENTRY_META_JUST_ALLOCATED);
            } else {
                life[entry_idx] = IRCACHE_ENTRY_LIFE_RECYCLED;
                for (uint32_t i = 0; i < IRCACHE_IRRADIANCE_STRIDE; ++i) irradiance[entry_idx * IRCACHE_IRRADIANCE_STRIDE + i] = f4(0.0f);
                const uint32_t entry_alloc_count = atom_add(&meta[IRCACHE_META_ALLOC_COUNT], uint32_t(-1));
                if (!entry_vertex) pool[entry_alloc_count - 1] = entry_idx;
                atom_and(&gm[entry_cell[entry_idx] * 2 + 1], ~(IRCACHE_ENTRY_META_OCCUPIED | IRCACHE_ENTRY_META_JUST_ALLOCATED));
            }
        }
        if (!entry_vertex) {
            spatial[entry_idx] = proposal[entry_idx];   // flush the reposition proposal (IRCACHE_USE_POSITION_VOTING)
        } else {                                        // parallel schedule: votes compete for an emptied slot, no vote = no move; a new entry starts at its claimers' vote
            float4 v = proposal[entry_idx];
            if (!(kjb_f2u(v.x) | kjb_f2u(v.y) | kjb_f2u(v.z) | kjb_f2u(v.w))) v = entry_vertex[entry_idx];
            if (kjb_f2u(v.x) | kjb_f2u(v.y) | kjb_f2u(v.z) | kjb_f2u(v.w)) spatial[entry_idx] = v;
            proposal[entry_idx] = f4(0.0f); entry_vertex[entry_idx] = f4(0.0f);
        }
        proposal_count[entry_idx] = 0;
    } else {
        spatial[entry_idx] = f4(0.0f);
    }
    const uint32_t l2 = life[entry_idx];
    occupancy[entry_idx] = (entry_idx < total_entry_count && is_ircache_entry_life_valid(l2)) ? 1u : 0u;
}
template <bool SERIAL>
KJB_KERNEL(256) k_ircache_age(uint32_t* meta, uint32_t* gm, uint32_t* entry_cell, uint32_t* life, uint32_t* pool, float4* spatial, float4* proposal, uint32_t* proposal_count,
                              float4* irradiance, uint32_t* occupancy, float4* entry_vertex, Rows kjb_rows) {
    if constexpr (SERIAL) KJB_SERIAL_1D(MAX_ENTRIES, ircache_age_entry(meta, gm, entry_cell, life, pool, spatial, proposal, proposal_count, irradiance, occupancy, i, entry_vertex));
    else { const uint32_t i = tid1d(); if (i < MAX_ENTRIES) ircache_age_entry(meta, gm, entry_cell, life, pool, spatial, proposal, proposal_count, irradiance, occupancy, i, entry_vertex); }
}

// ------------------------------------------------------------------ the parallel schedule's entry assignment (kjb_ircache.cuh), at the start of a chain
// per entry: apply the keep-alive the lookups asked for, mark the free entries (life RECYCLED, the ones the pool holds)
KJB_KERNEL(256) k_ircache_det_free(uint32_t* life, uint32_t* life_pending, uint32_t* free_scan, Rows kjb_rows) {
    const uint32_t e = tid1d(); if (e >= MAX_ENTRIES) return;
    uint32_t l = life[e];
    const uint32_t p = life_pending[e];
    if (p) {
        const uint32_t nl = IRCACHE_ENTRY_LIFE_RECYCLE - p;
        if (l < IRCACHE_ENTRY_LIFE_RECYCLE && nl < l) life[e] = l = nl;
        life_pending[e] = 0;
    }
    free_scan[e] = l == IRCACHE_ENTRY_LIFE_RECYCLED ? 1u : 0u;
}
// per entry (after the scan): the free entries in ascending order fill the pool above the allocated count, where the pops take them from
KJB_KERNEL(256) k_ircache_det_pool(const uint32_t* free_scan, uint32_t* pool, uint32_t* meta, Rows kjb_rows) {
    const uint32_t e = tid1d(); if (e >= MAX_ENTRIES) return;
    const uint32_t base = MAX_ENTRIES - free_scan[MAX_ENTRIES - 1];
    if (e == 0) meta[IRCACHE_META_ALLOC_COUNT] = base;
    if (free_scan[e] != (e ? free_scan[e - 1] : 0u)) pool[base + free_scan[e] - 1] = e;
}
// per 32 cells: which were claimed, and how many
KJB_KERNEL(256) k_ircache_det_claims(const uint32_t* claim_rank, uint32_t* claim_bits, uint32_t* claim_scan, Rows kjb_rows) {
    const uint32_t w = tid1d(); if (w >= KJB_IRCACHE_GRID_CELLS / 32) return;
    uint32_t m = 0;
    for (uint32_t k = 0; k < 32; ++k) m |= (claim_rank[w * 32 + k] ? 1u : 0u) << k;
    claim_bits[w] = m; claim_scan[w] = kjb_popc(m);
}
// per cell (after the scan of the claim counts): the n-th claimed cell in cell order takes the n-th free entry; beyond the pool the claim is dropped
KJB_KERNEL(256) k_ircache_det_assign(uint32_t* meta, uint32_t* gm, uint32_t* entry_cell, uint32_t* life, const uint32_t* pool, float4* entry_vertex, uint32_t* claim_rank, float4* claim_vertex,
                                     const uint32_t* free_scan, const uint32_t* claim_bits, const uint32_t* claim_scan, Rows kjb_rows) {
    const uint32_t cell = tid1d(); if (cell >= KJB_IRCACHE_GRID_CELLS) return;
    const uint32_t w = cell >> 5, k = cell & 31u, m = claim_bits[w];
    if (!((m >> k) & 1u)) return;
    const uint32_t n = (w ? claim_scan[w - 1] : 0u) + kjb_popc(m & ((1u << k) - 1u));
    const uint32_t free_count = free_scan[MAX_ENTRIES - 1];
    const uint32_t rank = IRCACHE_ENTRY_RANK_COUNT - claim_rank[cell];
    const float4 v = claim_vertex[cell];
    claim_rank[cell] = 0; claim_vertex[cell] = f4(0.0f);
    if (n >= free_count) { atom_and(&gm[cell * 2 + 1], ~(IRCACHE_ENTRY_META_OCCUPIED | IRCACHE_ENTRY_META_JUST_ALLOCATED)); return; }
    const uint32_t entry_idx = pool[MAX_ENTRIES - free_count + n];
    atom_max(&meta[IRCACHE_META_ENTRY_COUNT], entry_idx + 1);
    atom_add(&meta[IRCACHE_META_ALLOC_COUNT], 1u);
    life[entry_idx] = ircache_entry_life_for_rank(rank);
    entry_cell[entry_idx] = cell;
    gm[cell * 2 + 0] = entry_idx;
    entry_vertex[entry_idx] = v;
}
// per entry: its reservoirs and contributions as the coming pass finds them, for the precise lookups of that pass
KJB_KERNEL(256) k_ircache_det_snapshot_aux(const uint32_t* meta, const float4* aux, float4* aux_prev, Rows kjb_rows) {
    const uint32_t i = tid1d(), e = i / 32u; if (e >= MAX_ENTRIES || e >= meta[IRCACHE_META_ENTRY_COUNT]) return;
    aux_prev[i] = aux[e * IRCACHE_AUX_STRIDE + i % 32u];
}

// ------------------------------------------------------------------ I5 prefix_scan/*.hlsl: inclusive scan of <= 64 Ki u32 in one CTA
// Replaces the reference's 3-pass 1 Mi-element scan (prefix_scan.rs:10-39).  The array is cut into chunks of 8192; in chunk c thread t owns the 8
// consecutive values at c * 8192 + t * 8, read as two 16-byte loads (a warp reads 1 KiB contiguous) — all chunks' loads are issued before the
// first is consumed, so the kernel pays one memory round trip, not one per chunk.  Thread totals are scanned with warp shuffles (SHFL.UP inside
// each warp, then warp c scans the 32 warp totals of chunk c), chunk totals carry forward; two block barriers in all.
#define KJB_SCAN_CHUNKS 8
KJB_KERNEL(1024) k_inclusive_prefix_scan(uint32_t* d, uint32_t n, Rows kjb_rows) {
    __shared__ uint32_t warp_tot[KJB_SCAN_CHUNKS][32];
    const uint32_t t = threadIdx.x;
    const bool vec = (reinterpret_cast<uintptr_t>(d) & 15u) == 0;   // 16-byte loads need an aligned base (always true for kjb_buffer_alloc)
    uint32_t v[KJB_SCAN_CHUNKS][8], s[KJB_SCAN_CHUNKS];
#pragma unroll
    for (uint32_t c = 0; c < KJB_SCAN_CHUNKS; ++c) {
        const uint32_t b = c * 8192u + t * 8u;
        if (vec && b + 8u <= n) {
            const uint4 lo = *reinterpret_cast<const uint4*>(d + b), hi = *reinterpret_cast<const uint4*>(d + b + 4);
            v[c][0] = lo.x; v[c][1] = lo.y; v[c][2] = lo.z; v[c][3] = lo.w; v[c][4] = hi.x; v[c][5] = hi.y; v[c][6] = hi.z; v[c][7] = hi.w;
        } else {
#pragma unroll
            for (uint32_t k = 0; k < 8u; ++k) v[c][k] = b + k < n ? d[b + k] : 0u;
        }
    }
#pragma unroll
    for (uint32_t c = 0; c < KJB_SCAN_CHUNKS; ++c) {
        uint32_t a = 0;
#pragma unroll
        for (uint32_t k = 0; k < 8u; ++k) { a += v[c][k]; v[c][k] = a; }     // inclusive within the thread's 8 values
        s[c] = a;
    }
    uint32_t before[KJB_SCAN_CHUNKS];                                          // sum of everything in front of this thread's values of chunk c
#if !defined(KJB_EMU)
    const uint32_t lane = t & 31u, warp = t >> 5;
    uint32_t inc[KJB_SCAN_CHUNKS];
#pragma unroll
    for (uint32_t c = 0; c < KJB_SCAN_CHUNKS; ++c) {
        uint32_t a = s[c];
#pragma unroll
        for (uint32_t off = 1; off < 32u; off <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, a, off); if (lane >= off) a += u; }
        inc[c] = a;
        if (lane == 31u) warp_tot[c][warp] = a;
    }
    __syncthreads();
    if (warp < KJB_SCAN_CHUNKS) {
        uint32_t a = warp_tot[warp][lane];
#pragma unroll
        for (uint32_t off = 1; off < 32u; off <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, a, off); if (lane >= off) a += u; }
        warp_tot[warp][lane] = a;
    }
    __syncthreads();
    uint32_t carry = 0;
#pragma unroll
    for (uint32_t c = 0; c < KJB_SCAN_CHUNKS; ++c) {
        before[c] = carry + (warp ? warp_tot[c][warp - 1] : 0u) + (inc[c] - s[c]);
        carry += warp_tot[c][31];
    }
#else
    static thread_local uint32_t tot[KJB_SCAN_CHUNKS * 1024];
    (void)warp_tot;
    for (uint32_t c = 0; c < KJB_SCAN_CHUNKS; ++c) tot[c * 1024u + t] = s[c];
    __syncthreads();
    if (t == 0) { uint32_t a = 0; for (uint32_t i = 0; i < KJB_SCAN_CHUNKS * 1024u; ++i) { const uint32_t x = tot[i]; tot[i] = a; a += x; } }
    __syncthreads();
    for (uint32_t c = 0; c < KJB_SCAN_CHUNKS; ++c) before[c] = tot[c * 1024u + t];
    __syncthreads();
#endif
#pragma unroll
    for (uint32_t c = 0; c < KJB_SCAN_CHUNKS; ++c) {
        const uint32_t b = c * 8192u + t * 8u;
        if (vec && b + 8u <= n) {
            *reinterpret_cast<uint4*>(d + b) = make_uint4(v[c][0] + before[c], v[c][1] + before[c], v[c][2] + before[c], v[c][3] + before[c]);
            *reinterpret_cast<uint4*>(d + b + 4) = make_uint4(v[c][4] + before[c], v[c][5] + before[c], v[c][6] + before[c], v[c][7] + before[c]);
        } else {
#pragma unroll
            for (uint32_t k = 0; k < 8u; ++k) if (b + k < n) d[b + k] = v[c][k] + before[c];
        }
    }
}

// ------------------------------------------------------------------ I6 ircache_compact_entries.hlsl
KJB_KERNEL(256) k_ircache_compact(const uint32_t* meta, const uint32_t* life, const uint32_t* occupancy, uint32_t* indirection, Rows kjb_rows) {
    const uint32_t entry_idx = tid1d(); if (entry_idx >= MAX_ENTRIES) return;
    const uint32_t total_entry_count = meta[IRCACHE_META_ENTRY_COUNT];
    // the scan is INCLUSIVE, so slots are 1-based: slot 0 is never written and the last valid entry lands one past the traced range.
    // That is what the reference does (ircache_compact_entries.hlsl:17); kept for parity.
    if (entry_idx < total_entry_count && is_ircache_entry_life_valid(life[entry_idx])) indirection[occupancy[entry_idx]] = entry_idx;
}

// ------------------------------------------------------------------ I7 reset_entry.hlsl
KJB_KERNEL(256) k_ircache_reset(const uint32_t* meta, const float4* irradiance, float4* aux, const uint32_t* indirection, Rows kjb_rows) {
    // 64 threads per entry clear its 64 aux texels (coalesced 1 KB)
    const uint32_t gid = tid1d(), dispatch_idx = gid / IRCACHE_AUX_STRIDE, i = gid % IRCACHE_AUX_STRIDE;
    const uint32_t alloc_count = meta[IRCACHE_META_TRACING_ALLOC_COUNT];
    if (dispatch_idx >= alloc_count || ircache_slot_is_stale_duplicate(indirection, alloc_count, dispatch_idx)) return;
    const uint32_t entry_idx = indirection[dispatch_idx];
    const float4 v = irradiance[entry_idx * IRCACHE_IRRADIANCE_STRIDE];
    if (v.x == 0.0f && v.y == 0.0f && v.z == 0.0f && v.w == 0.0f) aux[entry_idx * IRCACHE_AUX_STRIDE + i] = f4(0.0f);
}

// ------------------------------------------------------------------ I8 trace_accessibility.rgen.hlsl:21-66
KJB_KERNEL(128) k_ircache_trace_access(const __grid_constant__ Globals g, const float4* spatial, const uint32_t* life, const uint32_t* meta, float4* aux, const uint32_t* indirection, Rows kjb_rows) {
    const uint32_t dispatch_idx = tid1d();
    const uint32_t alloc_count = meta[IRCACHE_META_TRACING_ALLOC_COUNT];
    if (dispatch_idx >= alloc_count * IRCACHE_OCTA_DIMS2 || dispatch_idx >= MAX_ENTRIES * IRCACHE_OCTA_DIMS2) return;
    if (ircache_slot_is_stale_duplicate(indirection, alloc_count, dispatch_idx / IRCACHE_OCTA_DIMS2)) return;
    const uint32_t entry_idx = indirection[dispatch_idx / IRCACHE_OCTA_DIMS2], octa_idx = dispatch_idx % IRCACHE_OCTA_DIMS2;
    if (!is_ircache_entry_life_valid(life[entry_idx])) return;
    const IrcacheVertex entry = unpack_vertex(spatial[entry_idx]);
    const uint32_t output_idx = entry_idx * IRCACHE_AUX_STRIDE + octa_idx;
    const float4 ra = aux[output_idx];
    Reservoir r = Reservoir::from_raw(u2(kjb_f2u(ra.x), kjb_f2u(ra.y)));
    const IrcacheVertex prev_entry = unpack_vertex(aux[output_idx + IRCACHE_OCTA_DIMS2 * 2]);
    // reduce the weight of samples whose trace origins are not accessible now
    if (rt_is_shadowed(g, entry.position, prev_entry.position - entry.position, 0.001f, 0.999f)) {
        r.M *= 0.8f;
        const uint2 raw = r.as_raw();
        aux[output_idx] = f4(kjb_u2f(raw.x), kjb_u2f(raw.y), ra.z, ra.w);
    }
}

// ------------------------------------------------------------------ ircache_trace_common.inc.hlsl:37-227
// MAX_PATH_LENGTH 1, USE_WORLD_RADIANCE_CACHE 0, IRCACHE_LOOKUP_PRECISE, SAMPLE_IRCACHE_AT_LAST_VERTEX
struct IrcacheTraceResult { float3 incident_radiance, direction, hit_pos; };
KJB_DEV IrcacheTraceResult ircache_trace(const Globals& g, const IrcacheBufs& b, const Img& sky_cube_tex, const IrcacheVertex& entry, SampleParams sample_params, uint32_t life) {
    uint32_t rng = sample_params.rng();
    Ray outgoing_ray; outgoing_ray.origin = entry.position; outgoing_ray.dir = sample_params.direction(); outgoing_ray.tmin = 0.0f; outgoing_ray.tmax = KJB_FLT_MAX;
    IrcacheTraceResult result; result.direction = outgoing_ray.dir; result.hit_pos = f3(0.0f);
    float3 irradiance_sum = f3(0.0f);
    RayCone cone; cone.width = 0; cone.spread_angle = 0.1f;
    const GbufferPathVertex primary_hit = gbuffer_raytrace(g, outgoing_ray, cone, 1, false);
    if (primary_hit.is_hit) {
        result.hit_pos = primary_hit.position;
        const float3 to_light_norm = sun_direction(g.fc);
        const bool is_shadowed = rt_is_shadowed(g, primary_hit.position, to_light_norm, 1e-4f, KJB_FLT_MAX);
        const GbufferData gbuffer = gbuffer_unpack(primary_hit.gbuffer_packed);
        const float3x3 tangent_to_world = build_orthonormal_basis(gbuffer.normal);
        const float3 wi = mul(to_light_norm, tangent_to_world);
        float3 wo = mul(-outgoing_ray.dir, tangent_to_world);
        if (wo.z < 0.0f) { wo.z *= -0.25f; wo = normalize(wo); }   // shading normal facing away: flip along it
        LayeredBrdf brdf = layered_brdf_from_gbuffer_ndotv(g, gbuffer, wo.z);
        brdf.specular_brdf.roughness = kjb_lerp(brdf.specular_brdf.roughness, 1.0f, 0.5f);   // FIREFLY_SUPPRESSION, roughness_bias 0.5
        const float3 brdf_value = layered_evaluate_directional_light(brdf, wo, wi);
        const float3 light_radiance = is_shadowed ? f3(0.0f) : f3(g.sun_color[0], g.sun_color[1], g.sun_color[2]);
        irradiance_sum += brdf_value * light_radiance * kjb_max(0.0f, wi.z);
        irradiance_sum += gbuffer.emissive;
        if (g.fc.triangle_light_count > 0) {
            const float light_selection_pmf = 1.0f / float(g.fc.triangle_light_count);
            const uint32_t light_idx = hash1_mut(rng) % g.fc.triangle_light_count;
            float2 urand; urand.x = rand01(rng); urand.y = rand01(rng);
            const kjb_triangle_light tl = g.lights[light_idx];
            const LightSample ls = sample_triangle_light(tl, urand);
            const float3 to_light_ws = ls.pos - primary_hit.position;
            const float dist_to_light2 = dot(to_light_ws, to_light_ws);
            const float3 to_light_norm_ws = to_light_ws * kjb_rsqrt(dist_to_light2);
            const float to_psa_metric = kjb_max(0.0f, dot(to_light_norm_ws, gbuffer.normal)) * kjb_max(0.0f, dot(to_light_norm_ws, -ls.normal)) / dist_to_light2;
            if (to_psa_metric > 0.0f) {
                const float3 wi2 = mul(to_light_norm_ws, tangent_to_world);
                const bool sh = rt_is_shadowed(g, primary_hit.position, to_light_norm_ws, 1e-3f, kjb_sqrt(dist_to_light2) - 2e-3f);
                irradiance_sum += sh ? f3(0.0f) : f3(tl.radiance[0], tl.radiance[1], tl.radiance[2]) * layered_evaluate(brdf, wo, wi2) / ls.pdf * to_psa_metric / light_selection_pmf;
            }
        }
        irradiance_sum += ircache_lookup<true>(g, b, entry.position, primary_hit.position, gbuffer.normal, 1 + ircache_entry_life_to_rank(life), rng) * gbuffer.albedo;
        // path ends here: the BRDF-sampled continuation of the reference's loop is never traced with MAX_PATH_LENGTH == 1
    } else {
        result.hit_pos = outgoing_ray.origin + outgoing_ray.dir * 1000.0f;
        irradiance_sum += xyz(sample_cube_rgba16f(sky_cube_tex, outgoing_ray.dir));
    }
    result.incident_radiance = irradiance_sum;
    return result;
}
KJB_DEV float self_lighting_limiter(float3 dir, float3 normal) { return kjb_lerp(0.5f, 1.0f, kjb_smoothstep(-0.1f, 0.0f, dot(dir, normal))); }   // USE_SELF_LIGHTING_LIMITER

// ------------------------------------------------------------------ I9 ircache_validate.rgen.hlsl:44-131
KJB_DEV void ircache_validate_sample(const Globals& g, const IrcacheBufs& b, const Img& sky_cube_tex, const uint32_t* indirection, uint32_t dispatch_idx) {
    const uint32_t alloc_count = b.meta[IRCACHE_META_TRACING_ALLOC_COUNT];
    if (dispatch_idx >= alloc_count * IRCACHE_VALIDATION_SAMPLES_PER_FRAME || dispatch_idx >= MAX_ENTRIES * IRCACHE_VALIDATION_SAMPLES_PER_FRAME) return;
    if (ircache_slot_is_stale_duplicate(indirection, alloc_count, dispatch_idx / IRCACHE_VALIDATION_SAMPLES_PER_FRAME)) return;
    const uint32_t entry_idx = indirection[dispatch_idx / IRCACHE_VALIDATION_SAMPLES_PER_FRAME], sample_idx = dispatch_idx % IRCACHE_VALIDATION_SAMPLES_PER_FRAME;
    const uint32_t life = b.life[entry_idx];
    const SampleParams sample_params = SampleParams::from_spf_entry_sample_frame(IRCACHE_VALIDATION_SAMPLES_PER_FRAME, entry_idx, sample_idx, g.fc.frame_index);
    const uint32_t output_idx = entry_idx * IRCACHE_AUX_STRIDE + sample_params.octa_idx();
    const float4 ra = b.aux[output_idx];
    Reservoir r = Reservoir::from_raw(u2(kjb_f2u(ra.x), kjb_f2u(ra.y)));
    if (r.M > 0) {
        const float ped = g.fc.pre_exposure_delta;
        float4 prev_value_and_count = b.aux[output_idx + IRCACHE_OCTA_DIMS2] * f4(ped, ped, ped, 1);
        const IrcacheVertex prev_entry = unpack_vertex(b.aux[output_idx + IRCACHE_OCTA_DIMS2 * 2]);
        const IrcacheTraceResult prev_traced = ircache_trace(g, b, sky_cube_tex, prev_entry, SampleParams::from_raw(r.payload), life);   // validate the previous sample
        const float3 av = prev_traced.incident_radiance * self_lighting_limiter(prev_traced.direction, prev_entry.normal), bv = xyz(prev_value_and_count);
        const float3 dist3 = vabs(av - bv) / (av + bv);
        const float dist = kjb_max(dist3.x, kjb_max(dist3.y, dist3.z));
        const float invalidity = kjb_smoothstep(0.1f, 0.5f, dist);
        r.M = kjb_max(0.0f, kjb_min(r.M, kjb_exp2(kjb_log2(float(IRCACHE_RESTIR_M_CLAMP)) * (1.0f - invalidity))));
        prev_value_and_count = f4(av, prev_value_and_count.w);   // update the stored value too
        const uint2 raw = r.as_raw();
        b.aux[output_idx] = f4(kjb_u2f(raw.x), kjb_u2f(raw.y), ra.z, ra.w);
        b.aux[output_idx + IRCACHE_OCTA_DIMS2] = prev_value_and_count;
    }
}
// the serial form (as k_ircache_trace's) walks the samples of the traced entries only: the parallel launch's threads beyond them return at once
template <bool SERIAL>
KJB_KERNEL(128) k_ircache_validate(const __grid_constant__ Globals g, IrcacheBufs b, Img sky_cube_tex, const uint32_t* indirection, Rows kjb_rows) {
    if constexpr (SERIAL) {
        const uint32_t n = b.meta[IRCACHE_META_TRACING_ALLOC_COUNT] * IRCACHE_VALIDATION_SAMPLES_PER_FRAME, n_max = MAX_ENTRIES * IRCACHE_VALIDATION_SAMPLES_PER_FRAME;
        KJB_SERIAL_1D(n < n_max ? n : n_max, ircache_validate_sample(g, b, sky_cube_tex, indirection, i));
    } else ircache_validate_sample(g, b, sky_cube_tex, indirection, tid1d());
}

// ------------------------------------------------------------------ I10 trace_irradiance.rgen.hlsl:44-145
KJB_DEV void ircache_trace_sample(const Globals& g, const IrcacheBufs& b, const Img& sky_cube_tex, const uint32_t* indirection, uint32_t dispatch_idx) {
    const uint32_t alloc_count = b.meta[IRCACHE_META_TRACING_ALLOC_COUNT];
    if (dispatch_idx >= alloc_count * IRCACHE_SAMPLES_PER_FRAME || dispatch_idx >= MAX_ENTRIES * IRCACHE_SAMPLES_PER_FRAME) return;
    if (ircache_slot_is_stale_duplicate(indirection, alloc_count, dispatch_idx / IRCACHE_SAMPLES_PER_FRAME)) return;
    const uint32_t entry_idx = indirection[dispatch_idx / IRCACHE_SAMPLES_PER_FRAME], sample_idx = dispatch_idx % IRCACHE_SAMPLES_PER_FRAME;
    const uint32_t life = b.life[entry_idx];
    const float4 packed_entry = b.spatial[entry_idx];
    const IrcacheVertex entry = unpack_vertex(packed_entry);
    uint32_t rng = hash1(hash1(entry_idx) + g.fc.frame_index);
    const SampleParams sample_params = SampleParams::from_spf_entry_sample_frame(IRCACHE_SAMPLES_PER_FRAME, entry_idx, sample_idx, g.fc.frame_index);
    const IrcacheTraceResult traced = ircache_trace(g, b, sky_cube_tex, entry, sample_params, life);
    const float3 new_value = traced.incident_radiance * self_lighting_limiter(traced.direction, entry.normal);
    const float new_lum = luminance(new_value);
    StreamState stream_state; Reservoir reservoir = Reservoir::create();
    reservoir.init_with_stream(new_lum, 1.0f, stream_state, sample_params.value);
    const uint32_t output_idx = entry_idx * IRCACHE_AUX_STRIDE + sample_params.octa_idx();
    const float ped = g.fc.pre_exposure_delta;
    const float4 prev_value_and_count = b.aux[output_idx + IRCACHE_OCTA_DIMS2] * f4(ped, ped, ped, 1);
    float3 val_sel = new_value; bool selected_new = true;
    const float4 ra = b.aux[output_idx];
    {
        Reservoir r = Reservoir::from_raw(u2(kjb_f2u(ra.x), kjb_f2u(ra.y)));
        if (r.M > 0) {
            r.M = kjb_min(r.M, 30.0f);
            if (reservoir.update_with_stream(r, luminance(xyz(prev_value_and_count)), 1.0f, stream_state, r.payload, rng)) { val_sel = xyz(prev_value_and_count); selected_new = false; }
        }
    }
    reservoir.finish_stream(stream_state);
    const uint2 raw = reservoir.as_raw();
    b.aux[output_idx] = f4(kjb_u2f(raw.x), kjb_u2f(raw.y), ra.z, ra.w);
    b.aux[output_idx + IRCACHE_OCTA_DIMS2] = f4(val_sel, reservoir.W);
    if (selected_new) b.aux[output_idx + IRCACHE_OCTA_DIMS2 * 2] = packed_entry;
}
template <bool SERIAL>
KJB_KERNEL(128) k_ircache_trace(const __grid_constant__ Globals g, IrcacheBufs b, Img sky_cube_tex, const uint32_t* indirection, Rows kjb_rows) {
    if constexpr (SERIAL) {
        const uint32_t n = b.meta[IRCACHE_META_TRACING_ALLOC_COUNT] * IRCACHE_SAMPLES_PER_FRAME, n_max = MAX_ENTRIES * IRCACHE_SAMPLES_PER_FRAME;
        KJB_SERIAL_1D(n < n_max ? n : n_max, ircache_trace_sample(g, b, sky_cube_tex, indirection, i));
    } else ircache_trace_sample(g, b, sky_cube_tex, indirection, tid1d());
}

// ------------------------------------------------------------------ I11 sum_up_irradiance.hlsl:34-89
KJB_KERNEL(256) k_ircache_sum(const __grid_constant__ Globals g, const uint32_t* meta, float4* irradiance, const float4* aux, const uint32_t* indirection, Rows kjb_rows) {
    const uint32_t dispatch_idx = tid1d();
    const uint32_t alloc_count = meta[IRCACHE_META_TRACING_ALLOC_COUNT];
    if (dispatch_idx >= alloc_count || dispatch_idx >= MAX_ENTRIES || ircache_slot_is_stale_duplicate(indirection, alloc_count, dispatch_idx)) return;
    const uint32_t entry_idx = indirection[dispatch_idx];
    float4 sh_rgb[3] = {f4(0.0f), f4(0.0f), f4(0.0f)};
    float valid_samples = 0;
    for (uint32_t octa_idx = 0; octa_idx < IRCACHE_OCTA_DIMS2; ++octa_idx) {
        const float4 ra = aux[entry_idx * IRCACHE_AUX_STRIDE + octa_idx];
        const Reservoir r = Reservoir::from_raw(u2(kjb_f2u(ra.x), kjb_f2u(ra.y)));
        const float3 dir = SampleParams::from_raw(r.payload).direction();
        const float4 contrib = aux[entry_idx * IRCACHE_AUX_STRIDE + IRCACHE_OCTA_DIMS2 + octa_idx];
        const float3 radiance = xyz(contrib) * contrib.w;
        const float4 sh = f4(0.282095f, dir.x * 0.488603f, dir.y * 0.488603f, dir.z * 0.488603f) * 4.0f;   // shEvaluateL1 x 4, pi cancelled in the BRDF
        sh_rgb[0] += sh * radiance.x; sh_rgb[1] += sh * radiance.y; sh_rgb[2] += sh * radiance.z;
        valid_samples += contrib.w > 0 ? 1.0f : 0.0f;
    }
    const float sc = 1.0f / kjb_max(1.0f, valid_samples);
    const float ped = g.fc.pre_exposure_delta;
    for (uint32_t basis_i = 0; basis_i < IRCACHE_IRRADIANCE_STRIDE; ++basis_i) {
        const float4 new_value = sh_rgb[basis_i] * sc;
        float4 prev_value = irradiance[entry_idx * IRCACHE_IRRADIANCE_STRIDE + basis_i] * ped;
        const bool should_reset = !(prev_value.x != 0.0f || prev_value.y != 0.0f || prev_value.z != 0.0f || prev_value.w != 0.0f);
        if (should_reset) prev_value = new_value;
        irradiance[entry_idx * IRCACHE_IRRADIANCE_STRIDE + basis_i] = vlerp(prev_value, new_value, 0.25f);
    }
}

// ================================================================== C-ABI entry points
// ------------------------------------------------------------------ tile-sharded frames: exchange of cache requests between the ranks' replicas (kjb.h)
KJB_KERNEL(256) k_ircache_export_requests(IrcacheBufs b, uint32_t* block, uint32_t max_records, Rows kjb_rows) {
    const uint32_t e = tid1d();
    if (e >= b.meta[IRCACHE_META_ENTRY_COUNT] || e >= MAX_ENTRIES) return;
    const uint32_t life = b.life[e];
    // Entries of rank <= 1 only: the ones a screen ray asked for (the diffuse and reflection rays look the cache up with query rank 1, rtdgi/trace_diffuse,
    // rtr/reflection).  Entries of higher rank exist because a cache ray of THIS replica landed there; every replica derives its own from the (now shared)
    // rank-1 set, as the single cache does — exporting them would make the union grow with the number of ranks.
    if (!is_ircache_entry_life_valid(life) || ircache_entry_life_to_rank(life) > 1u) return;
    const uint32_t slot = atom_add(&block[0], 1u);            // the header may end up above max_records: readers clamp
    if (slot >= max_records) return;
    uint32_t* rec = block + 4 + slot * 8u;
    float4 v = b.reposition_proposal[e];
    if (!(kjb_f2u(v.x) | kjb_f2u(v.y) | kjb_f2u(v.z) | kjb_f2u(v.w))) v = b.spatial[e];   // no vote yet (parallel schedule): where the entry is
    rec[0] = b.entry_cell[e]; rec[1] = life; rec[2] = b.reposition_count[e]; rec[3] = 0u;
    rec[4] = kjb_f2u(v.x); rec[5] = kjb_f2u(v.y); rec[6] = kjb_f2u(v.z); rec[7] = kjb_f2u(v.w);
}
// one launch per source rank: a cell appears at most once per block, so records of one launch never meet in the same entry
KJB_KERNEL(256) k_ircache_merge_requests(IrcacheBufs b, const uint32_t* block, uint32_t max_records, uint32_t seed, Rows kjb_rows) {
    const uint32_t i = tid1d();
    const uint32_t n = block[0] < max_records ? block[0] : max_records;
    if (i >= n) return;
    const uint32_t* rec = block + 4 + i * 8u;
    const uint32_t cell_idx = rec[0], life_r = rec[1], count_r = rec[2];
    if (cell_idx >= KJB_IRCACHE_GRID_CELLS || !is_ircache_entry_life_valid(life_r)) return;
    const float4 vote = f4(kjb_u2f(rec[4]), kjb_u2f(rec[5]), kjb_u2f(rec[6]), kjb_u2f(rec[7]));
    if (b.det && (b.grid_meta[cell_idx * 2 + 1] & (IRCACHE_ENTRY_META_OCCUPIED | IRCACHE_ENTRY_META_JUST_ALLOCATED)) != IRCACHE_ENTRY_META_OCCUPIED) {
        // parallel schedule: a cell without an entry yet is claimed like a lookup claims it, and gets its entry with the coming chain
        atom_or(&b.grid_meta[cell_idx * 2 + 1], IRCACHE_ENTRY_META_OCCUPIED | IRCACHE_ENTRY_META_JUST_ALLOCATED);
        atom_max(&b.claim_rank[cell_idx], IRCACHE_ENTRY_RANK_COUNT - ircache_entry_life_to_rank(life_r));
        vertex_vote(&b.claim_vertex[cell_idx], vote);
        return;
    }
    bool fresh = false;
    if ((b.grid_meta[cell_idx * 2 + 1] & IRCACHE_ENTRY_META_OCCUPIED) == 0) {      // no local ray asked for this cell: allocate it as the lookup would (lookup.hlsl:19-74)
        const uint32_t prev = atom_or(&b.grid_meta[cell_idx * 2 + 1], IRCACHE_ENTRY_META_OCCUPIED | IRCACHE_ENTRY_META_JUST_ALLOCATED);
        if ((prev & IRCACHE_ENTRY_META_OCCUPIED) == 0) {
            const uint32_t alloc_idx = atom_add(&b.meta[IRCACHE_META_ALLOC_COUNT], 1u);
            if (alloc_idx >= 1024u * 64u) {
                atom_add(&b.meta[IRCACHE_META_ALLOC_COUNT], uint32_t(-1));
                atom_and(&b.grid_meta[cell_idx * 2 + 1], ~(IRCACHE_ENTRY_META_OCCUPIED | IRCACHE_ENTRY_META_JUST_ALLOCATED));
                return;
            }
            const uint32_t entry_idx = b.pool[alloc_idx];
            atom_max(&b.meta[IRCACHE_META_ENTRY_COUNT], entry_idx + 1);
            b.life[entry_idx] = life_r; b.entry_cell[entry_idx] = cell_idx; b.grid_meta[cell_idx * 2 + 0] = entry_idx;
            b.reposition_proposal[entry_idx] = vote; b.reposition_count[entry_idx] = count_r;
            fresh = true;
        }
    }
    if (fresh || (b.grid_meta[cell_idx * 2 + 1] & IRCACHE_ENTRY_META_OCCUPIED) == 0) return;
    const uint32_t entry_idx = b.grid_meta[cell_idx * 2 + 0];
    const uint32_t prev_life = b.life[entry_idx];
    if (prev_life >= IRCACHE_ENTRY_LIFE_RECYCLE) return;
    if (life_r < prev_life) atom_min(&b.life[entry_idx], life_r);
    if (count_r > 0u) {
        const uint32_t prev_votes = atom_add(&b.reposition_count[entry_idx], count_r);
        uint32_t rng = hash1(cell_idx ^ hash1(seed));
        const float dart = rand01(rng);
        if (dart * (float(prev_votes) + float(count_r)) <= float(count_r)) b.reposition_proposal[entry_idx] = vote;
    }
}

#define BUF(b, T, min_elems, name) if (!(b).data || (b).size_bytes < uint64_t(min_elems) * sizeof(T)) return c->fail(std::string(P) + ": buffer '" name "' is null or too small")
#define U32P(b) ((uint32_t*)(b).data)
#define F4P(b) ((float4*)(b).data)
#define DIMS1D(n, bs) KJB_DIMS(dim3(unsigned(((n) + (bs) - 1) / (bs))), dim3(bs))
#define NO_SCISSOR const kjb::Rows kjb__rows = {0, 1}   /* cache passes are not pixel grids: the tile scissor does not apply */

extern "C" {

int kjb_pass_ircache_clear_pool(kjb_context* c, const kjb_ircache_clear_pool_args* a) {
    const char* P = "clear ircache pool"; BUF(a->pool_buf, uint32_t, MAX_ENTRIES, "pool_buf"); BUF(a->life_buf, uint32_t, MAX_ENTRIES, "life_buf");
    NO_SCISSOR;
    KJB_LAUNCH(c, k_ircache_clear_pool, DIMS1D(MAX_ENTRIES, 256), U32P(a->pool_buf), U32P(a->life_buf));
    kjb_context::IrcacheScratch s;   // an emptied cache has no pending claims or keep-alives
    if (ircache_parallel_scratch(c, a->life_buf.data, s) && (dev_memset(c, s.claim_rank, 0, 4ull * KJB_IRCACHE_GRID_CELLS) || dev_memset(c, s.claim_vertex, 0, 16ull * KJB_IRCACHE_GRID_CELLS)
                                                               || dev_memset(c, s.life_pending, 0, 4ull * MAX_ENTRIES) || dev_memset(c, s.entry_vertex, 0, 16ull * MAX_ENTRIES)))
        return c->fail(std::string(P) + ": memset failed");
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ircache_scroll_cascades(kjb_context* c, const kjb_ircache_scroll_cascades_args* a) {
    const char* P = "scroll cascades";
    BUF(a->grid_meta_buf, uint2, KJB_IRCACHE_GRID_CELLS, "grid_meta_buf"); BUF(a->grid_meta_buf2, uint2, KJB_IRCACHE_GRID_CELLS, "grid_meta_buf2");
    BUF(a->entry_cell_buf, uint32_t, MAX_ENTRIES, "entry_cell_buf"); BUF(a->irradiance_buf, float4, 3 * MAX_ENTRIES, "irradiance_buf"); BUF(a->life_buf, uint32_t, MAX_ENTRIES, "life_buf");
    BUF(a->pool_buf, uint32_t, MAX_ENTRIES, "pool_buf"); BUF(a->meta_buf, uint32_t, 8, "meta_buf");
    NO_SCISSOR;
    kjb_context::IrcacheScratch s;
    if (ircache_parallel_scratch(c, a->life_buf.data, s)) {   // the claims of the last frame's passes take their entries (kjb_ircache.cuh)
        uint32_t* free_scan = (uint32_t*)s.scan; uint32_t* claim_scan = free_scan + MAX_ENTRIES;
        KJB_LAUNCH(c, k_ircache_det_free, DIMS1D(MAX_ENTRIES, 256), U32P(a->life_buf), (uint32_t*)s.life_pending, free_scan);
        KJB_LAUNCH_SYNC(c, k_inclusive_prefix_scan, KJB_DIMS(dim3(1), dim3(1024)), free_scan, MAX_ENTRIES);
        KJB_LAUNCH(c, k_ircache_det_pool, DIMS1D(MAX_ENTRIES, 256), (const uint32_t*)free_scan, U32P(a->pool_buf), U32P(a->meta_buf));
        KJB_LAUNCH(c, k_ircache_det_claims, DIMS1D(KJB_IRCACHE_GRID_CELLS / 32, 256), (const uint32_t*)s.claim_rank, (uint32_t*)s.claim_bits, claim_scan);
        KJB_LAUNCH_SYNC(c, k_inclusive_prefix_scan, KJB_DIMS(dim3(1), dim3(1024)), claim_scan, KJB_IRCACHE_GRID_CELLS / 32);
        KJB_LAUNCH(c, k_ircache_det_assign, DIMS1D(KJB_IRCACHE_GRID_CELLS, 256), U32P(a->meta_buf), U32P(a->grid_meta_buf), U32P(a->entry_cell_buf), U32P(a->life_buf), (const uint32_t*)U32P(a->pool_buf),
                   (float4*)s.entry_vertex, (uint32_t*)s.claim_rank, (float4*)s.claim_vertex, (const uint32_t*)free_scan, (const uint32_t*)s.claim_bits, (const uint32_t*)claim_scan);
    }
    KJB_LAUNCH_CACHE(c, true, k_ircache_scroll_cascades, DIMS1D(KJB_IRCACHE_GRID_CELLS, 256), c->g, U32P(a->grid_meta_buf), U32P(a->grid_meta_buf2), U32P(a->entry_cell_buf), F4P(a->irradiance_buf),
                     U32P(a->life_buf), U32P(a->pool_buf), U32P(a->meta_buf), ircache_parallel_scratch(c, a->life_buf.data, s) ? 1u : 0u);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ircache_prepare_age_dispatch_args(kjb_context* c, const kjb_ircache_dispatch_args_args* a) {
    const char* P = "_ircache dispatch args"; BUF(a->meta_buf, uint32_t, 8, "meta_buf"); BUF(a->dispatch_args, uint32_t, 4, "dispatch_args");
    NO_SCISSOR;
    KJB_LAUNCH(c, k_ircache_prepare_age_args, DIMS1D(1, 32), U32P(a->meta_buf), U32P(a->dispatch_args));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ircache_prepare_trace_dispatch_args(kjb_context* c, const kjb_ircache_dispatch_args_args* a) {
    const char* P = "_ircache dispatch args"; BUF(a->meta_buf, uint32_t, 8, "meta_buf"); BUF(a->dispatch_args, uint32_t, 16, "dispatch_args");
    NO_SCISSOR;
    KJB_LAUNCH(c, k_ircache_prepare_trace_args, DIMS1D(1, 32), U32P(a->meta_buf), U32P(a->dispatch_args));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ircache_age_entries(kjb_context* c, const kjb_ircache_age_args* a) {
    const char* P = "age ircache entries";
    BUF(a->meta_buf, uint32_t, 8, "meta_buf"); BUF(a->grid_meta_buf, uint2, KJB_IRCACHE_GRID_CELLS, "grid_meta_buf"); BUF(a->entry_cell_buf, uint32_t, MAX_ENTRIES, "entry_cell_buf");
    BUF(a->life_buf, uint32_t, MAX_ENTRIES, "life_buf"); BUF(a->pool_buf, uint32_t, MAX_ENTRIES, "pool_buf"); BUF(a->spatial_buf, float4, MAX_ENTRIES, "spatial_buf");
    BUF(a->reposition_proposal_buf, float4, MAX_ENTRIES, "reposition_proposal_buf"); BUF(a->reposition_proposal_count_buf, uint32_t, MAX_ENTRIES, "reposition_proposal_count_buf");
    BUF(a->irradiance_buf, float4, 3 * MAX_ENTRIES, "irradiance_buf"); BUF(a->entry_occupancy_buf, uint32_t, MAX_ENTRIES, "entry_occupancy_buf");
    NO_SCISSOR;
    kjb_context::IrcacheScratch s;
    float4* entry_vertex = ircache_parallel_scratch(c, a->life_buf.data, s) ? (float4*)s.entry_vertex : nullptr;
    KJB_LAUNCH_CACHE(c, true, k_ircache_age, DIMS1D(MAX_ENTRIES, 256), U32P(a->meta_buf), U32P(a->grid_meta_buf), U32P(a->entry_cell_buf), U32P(a->life_buf), U32P(a->pool_buf), F4P(a->spatial_buf),
                     F4P(a->reposition_proposal_buf), U32P(a->reposition_proposal_count_buf), F4P(a->irradiance_buf), U32P(a->entry_occupancy_buf), entry_vertex);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_inclusive_prefix_scan_u32(kjb_context* c, const kjb_prefix_scan_args* a) {
    const char* P = "_prefix scan"; BUF(a->inout_buf, uint32_t, a->element_count, "inout_buf");
    if (a->element_count > 65536u) return c->fail("_prefix scan: at most 65536 elements (the irradiance cache's MAX_ENTRIES)");
    NO_SCISSOR;
    KJB_LAUNCH_SYNC(c, k_inclusive_prefix_scan, KJB_DIMS(dim3(1), dim3(1024)), U32P(a->inout_buf), a->element_count);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ircache_compact(kjb_context* c, const kjb_ircache_compact_args* a) {
    const char* P = "ircache compact";
    BUF(a->meta_buf, uint32_t, 8, "meta_buf"); BUF(a->life_buf, uint32_t, MAX_ENTRIES, "life_buf"); BUF(a->entry_occupancy_buf, uint32_t, MAX_ENTRIES, "entry_occupancy_buf");
    BUF(a->entry_indirection_buf, uint32_t, MAX_ENTRIES + 1, "entry_indirection_buf");
    NO_SCISSOR;
    KJB_LAUNCH(c, k_ircache_compact, DIMS1D(MAX_ENTRIES, 256), U32P(a->meta_buf), U32P(a->life_buf), U32P(a->entry_occupancy_buf), U32P(a->entry_indirection_buf));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ircache_reset(kjb_context* c, const kjb_ircache_reset_args* a) {
    const char* P = "ircache reset";
    BUF(a->meta_buf, uint32_t, 8, "meta_buf"); BUF(a->irradiance_buf, float4, 3 * MAX_ENTRIES, "irradiance_buf"); BUF(a->aux_buf, float4, 64 * MAX_ENTRIES, "aux_buf");
    BUF(a->entry_indirection_buf, uint32_t, MAX_ENTRIES + 1, "entry_indirection_buf");
    NO_SCISSOR;
    KJB_LAUNCH(c, k_ircache_reset, DIMS1D(MAX_ENTRIES * 64u, 256), U32P(a->meta_buf), F4P(a->irradiance_buf), F4P(a->aux_buf), U32P(a->entry_indirection_buf));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ircache_trace_access(kjb_context* c, const kjb_ircache_trace_access_args* a) {
    const char* P = "ircache trace access";
    BUF(a->spatial_buf, float4, MAX_ENTRIES, "spatial_buf"); BUF(a->life_buf, uint32_t, MAX_ENTRIES, "life_buf"); BUF(a->meta_buf, uint32_t, 8, "meta_buf");
    BUF(a->aux_buf, float4, 64 * MAX_ENTRIES, "aux_buf"); BUF(a->entry_indirection_buf, uint32_t, MAX_ENTRIES + 1, "entry_indirection_buf");
    if (!c->tlas_valid) return c->fail("ircache trace access: no acceleration structure (call kjb_rebuild_tlas)");
    NO_SCISSOR;
    KJB_LAUNCH(c, k_ircache_trace_access, DIMS1D(MAX_ENTRIES * 16u, 128), c->g, F4P(a->spatial_buf), U32P(a->life_buf), U32P(a->meta_buf), F4P(a->aux_buf), U32P(a->entry_indirection_buf));
    KJB_PASS_EPILOGUE(c, P);
}
static int check_trace_args(kjb_context* c, const char* P, const kjb_ircache_trace_args* a, IrcacheBufs& b) {
    BUF(a->spatial_buf, float4, MAX_ENTRIES, "spatial_buf"); BUF(a->grid_meta_buf, uint2, KJB_IRCACHE_GRID_CELLS, "grid_meta_buf"); BUF(a->life_buf, uint32_t, MAX_ENTRIES, "life_buf");
    BUF(a->reposition_proposal_buf, float4, MAX_ENTRIES, "reposition_proposal_buf"); BUF(a->reposition_proposal_count_buf, uint32_t, MAX_ENTRIES, "reposition_proposal_count_buf");
    BUF(a->meta_buf, uint32_t, 8, "meta_buf"); BUF(a->aux_buf, float4, 64 * MAX_ENTRIES, "aux_buf"); BUF(a->pool_buf, uint32_t, MAX_ENTRIES, "pool_buf");
    BUF(a->entry_indirection_buf, uint32_t, MAX_ENTRIES + 1, "entry_indirection_buf"); BUF(a->entry_cell_buf, uint32_t, MAX_ENTRIES, "entry_cell_buf");
    if (!check_img(c, a->sky_cube_tex, KJB_FMT_RGBA16_FLOAT, P, "sky_cube_tex")) return 1;
    if (!c->tlas_valid) return c->fail(std::string(P) + ": no acceleration structure (call kjb_rebuild_tlas)");
    b.meta = U32P(a->meta_buf); b.pool = U32P(a->pool_buf); b.reposition_count = U32P(a->reposition_proposal_count_buf); b.grid_meta = U32P(a->grid_meta_buf); b.entry_cell = U32P(a->entry_cell_buf);
    b.life = U32P(a->life_buf); b.reposition_proposal = F4P(a->reposition_proposal_buf); b.spatial = F4P(a->spatial_buf); b.irradiance = nullptr; b.aux = F4P(a->aux_buf);   // precise lookups read the per-entry reservoirs, not the SH
    ircache_attach_parallel(c, b);
    return 0;
}
static void snapshot_aux(kjb_context* c, const IrcacheBufs& b) {   // parallel schedule: what the pass's precise lookups read
    NO_SCISSOR;
    if (b.det) KJB_LAUNCH(c, k_ircache_det_snapshot_aux, DIMS1D(MAX_ENTRIES * 32u, 256), (const uint32_t*)b.meta, (const float4*)b.aux, (float4*)b.aux_prev);
}
int kjb_pass_ircache_validate(kjb_context* c, const kjb_ircache_trace_args* a) {
    const char* P = "ircache validate"; IrcacheBufs b; if (check_trace_args(c, P, a, b)) return 1;
    snapshot_aux(c, b);
    NO_SCISSOR;
    KJB_LAUNCH_CACHE(c, true, k_ircache_validate, DIMS1D(MAX_ENTRIES * 4u, 128), c->g, b, img_ro(a->sky_cube_tex), U32P(a->entry_indirection_buf));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ircache_trace(kjb_context* c, const kjb_ircache_trace_args* a) {
    const char* P = "ircache trace"; IrcacheBufs b; if (check_trace_args(c, P, a, b)) return 1;
    snapshot_aux(c, b);
    NO_SCISSOR;
    KJB_LAUNCH_CACHE(c, true, k_ircache_trace, DIMS1D(MAX_ENTRIES * 4u, 128), c->g, b, img_ro(a->sky_cube_tex), U32P(a->entry_indirection_buf));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ircache_sum(kjb_context* c, const kjb_ircache_sum_args* a) {
    const char* P = "ircache sum";
    BUF(a->meta_buf, uint32_t, 8, "meta_buf"); BUF(a->irradiance_buf, float4, 3 * MAX_ENTRIES, "irradiance_buf"); BUF(a->aux_buf, float4, 64 * MAX_ENTRIES, "aux_buf");
    BUF(a->entry_indirection_buf, uint32_t, MAX_ENTRIES + 1, "entry_indirection_buf");
    NO_SCISSOR;
    KJB_LAUNCH(c, k_ircache_sum, DIMS1D(MAX_ENTRIES, 256), c->g, U32P(a->meta_buf), F4P(a->irradiance_buf), F4P(a->aux_buf), U32P(a->entry_indirection_buf));
    KJB_PASS_EPILOGUE(c, P);
}

static bool share_bindings_ok(const kjb_ircache_bindings& b) {
    return b.meta_buf.data && b.pool_buf.data && b.reposition_proposal_buf.data && b.reposition_proposal_count_buf.data && b.grid_meta_buf.data && b.entry_cell_buf.data && b.life_buf.data;
}
int kjb_pass_ircache_export_requests(kjb_context* c, const kjb_ircache_share_args* a) {
    const char* P = "tile ircache export";
    if (!share_bindings_ok(a->ircache)) return c->fail(std::string(P) + ": the irradiance cache is not bound");
    BUF(a->block, uint8_t, KJB_IRCACHE_SHARE_BLOCK_BYTES(uint64_t(a->max_records)), "block");
    NO_SCISSOR;
    if (dev_memset(c, a->block.data, 0, 16)) return c->fail(std::string(P) + ": memset failed");
    KJB_LAUNCH_ORDERED(c, k_ircache_export_requests, DIMS1D(MAX_ENTRIES, 256), ircache_bufs(a->ircache), U32P(a->block), a->max_records);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ircache_merge_requests(kjb_context* c, const kjb_ircache_share_args* a) {
    const char* P = "tile ircache merge";
    if (!share_bindings_ok(a->ircache)) return c->fail(std::string(P) + ": the irradiance cache is not bound");
    BUF(a->block, uint8_t, KJB_IRCACHE_SHARE_BLOCK_BYTES(uint64_t(a->max_records)), "block");
    if (a->max_records == 0) return 0;
    NO_SCISSOR;
    IrcacheBufs b = ircache_bufs(a->ircache); ircache_attach_parallel(c, b);
    KJB_LAUNCH_ORDERED(c, k_ircache_merge_requests, DIMS1D(a->max_records, 256), b, (const uint32_t*)a->block.data, a->max_records, a->seed);
    KJB_PASS_EPILOGUE(c, P);
}

}  // extern "C"

/* Tile-sharded frames with the irradiance cache: the exact exchange of the replicas' pending requests, and the option query a frame driver
 * uses to choose it.  Entry points of the CUDA library and its emulator; kept out of kjb.h because the CPU oracle, which implements kjb.h,
 * has no ordered schedule and renders no tile-sharded frames. */
#ifndef KJB_IRCACHE_SHARE_H
#define KJB_IRCACHE_SHARE_H
#include "kjb.h"
#ifdef __cplusplus
extern "C" {
#endif
/* the option's value in effect; for KJB_OPTION_ORDERED_CACHE_SCHEDULE 1 only while kjb_set_debug_serial is off (the serial schedule overrides it) */
int  kjb_get_option(kjb_context *ctx, uint32_t option, uint32_t *value);

/* The exact exchange, on the ordered schedule only (KJB_OPTION_ORDERED_CACHE_SCHEDULE = 1; both passes fail on the reference's atomics, whose
 * outcome depends on thread timing).  On that schedule a frame's lookups never change what another lookup of the frame reads: every request
 * waits as pending state until the next cache chain, merged with operators that ignore order and repetition —
 *   claim a cell:        grid_meta flag bits |= OCCUPIED | JUST_ALLOCATED, claim_rank = max, claim_vertex = the vote with the smallest hash;
 *   keep an entry alive: life_pending = max;
 *   vote where it moves: reposition_proposal = the vote with the smallest hash; reposition_proposal_count_buf = max (see the option above).
 * So replicas that start a frame identical and merge the union of all ranks' pending state hold exactly what one GPU holds after all of the
 * frame's rays, frame after frame.  Call export after the frame's last cache user, all-gather the blocks, then merge them (before the next
 * cache chain).  A replica's own block may be among the merged ones: merging it changes nothing.
 * The block has a fixed size.  Entries are dense, by entry index (identical replicas share entry indices).  Claims are (cell, rank, vertex)
 * records in ascending cell order, at most KJB_IRCACHE_MAX_ENTRIES: the chain gives the n-th claimed cell in cell order the n-th free entry and
 * there are never more free entries than that, so a claim beyond a rank's first KJB_IRCACHE_MAX_ENTRIES can never get an entry.  (If a rank
 * holds more claims, the others' replicas lack those cells' pending flags until the next chain drops them on every replica alike.)
 * Layout: u32 header[64] = {claim records, claims held}, float4 proposal[E], float4 claim_vertex[E], u32 life_pending[E], vote_count[E],
 * claim_cell[E], claim_rank[E] with E = KJB_IRCACHE_MAX_ENTRIES; a multiple of 256 bytes, so blocks sit back to back in an all-gather. */
#define KJB_IRCACHE_PENDING_BLOCK_BYTES (256u + KJB_IRCACHE_MAX_ENTRIES * 48u)
typedef struct kjb_ircache_pending_args {
    kjb_ircache_bindings ircache;
    kjb_buffer blocks;           /* export: this replica's block (written).  merge: `block_count` blocks back to back (read) */
    uint32_t block_count;        /* merge: 1 to 4096 (all ranks' blocks in one launch); export: must be 1 */
} kjb_ircache_pending_args;
int kjb_pass_ircache_export_pending(kjb_context *ctx, const kjb_ircache_pending_args *a);
int kjb_pass_ircache_merge_pending(kjb_context *ctx, const kjb_ircache_pending_args *a);

#ifdef __cplusplus
}
#endif
#endif

/* Read-only introspection of the acceleration structure the CUDA library built (kjb_rebuild_tlas), for tests and tools.
 * The layout of the records is kajiya_b200/csrc/kjb_bvh.h: 64-byte nodes, 48-byte leaf-order triangle records, 8-byte tri_info by global
 * triangle id, one parent link per inner node.  Kept out of kjb.h: the CPU oracle implements kjb.h with a structure of its own. */
#ifndef KJB_TLAS_H
#define KJB_TLAS_H
#include "kjb.h"
#ifdef __cplusplus
extern "C" {
#endif
/* Synchronises the context, then writes out_counts = (inner nodes, triangle slots, triangles) and the root reference (a node index, or
 * ~((first << 3) | (count - 1)) for a single leaf, ~0 for an empty scene), and copies each array whose pointer is not null. */
int kjb_tlas_download(kjb_context *ctx, uint32_t out_counts[3], int32_t *out_root, void *nodes, void *tris, void *tri_info, int32_t *parent);

/* Traces n rays against the structure as built, synchronously (upload, one launch, download; not for the frame loop).  A ray is 8 floats
 * (o.xyz, tmin, d.xyz, tmax); a result is 4 words: t, u, v as float bits and the global triangle id, or 0, 0, 0, 0xffffffff for a miss.
 * With KJB_TLAS_TRACE_ANY_HIT only word 3 means something: 0 for a hit, 0xffffffff for none.  KJB_TLAS_TRACE_BRUTE_FORCE tests every
 * triangle record instead of walking the tree: the same triangle test and selection rule, with no culling at all. */
#define KJB_TLAS_TRACE_ANY_HIT 1u
#define KJB_TLAS_TRACE_CULL_BACK 2u
#define KJB_TLAS_TRACE_BRUTE_FORCE 4u
int kjb_tlas_trace(kjb_context *ctx, const float *rays, uint32_t n, uint32_t flags, float *out);
#ifdef __cplusplus
}
#endif
#endif

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
#ifdef __cplusplus
}
#endif
#endif

// Software acceleration structure for H100 (no RT cores, no Vulkan): a single flattened WORLD-SPACE BVH2.
//
// The reference keeps a two-level driver structure (BLAS per mesh + TLAS rebuilt per frame,
// crates/lib/kajiya-backend/src/vulkan/ray_tracing.rs:96-260,455-520) because RT hardware wants it.  Without
// RT hardware, one level wins: no per-instance ray transform, one traversal loop.  "rebuild tlas" re-flattens when transforms change.
//
// Layout (Aila-Laine style, 64-byte nodes holding BOTH children's boxes => one 64 B line per traversal step):
//   n0 = (c0.lo.x, c0.hi.x, c0.lo.y, c0.hi.y)   n1 = (c1.lo.x, c1.hi.x, c1.lo.y, c1.hi.y)
//   n2 = (c0.lo.z, c0.hi.z, c1.lo.z, c1.hi.z)   n3 = (child0, child1, -, -) as int bits; child < 0 => leaf ~((first << 3) | (count - 1))
// Triangles are stored in leaf order as 48-byte records (v0 | global id, e1, e2) in world space.
// Built on the device (kjb_bvh_build.cuh), refitted on the device when only transforms change (kjb_api.cu).
#pragma once
#include <stdint.h>

namespace kjb {

struct BvhNode { float n0[4], n1[4], n2[4]; int32_t child[4]; };          // 64 B
struct BvhTri { float v0[3]; uint32_t gid; float e1[3]; uint32_t pad0; float e2[3]; uint32_t pad1; };   // 48 B
struct TriInfo { uint32_t instance, prim; };                               // indexed by global triangle id

}  // namespace kjb

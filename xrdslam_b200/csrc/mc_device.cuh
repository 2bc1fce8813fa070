// Device helpers shared by the marching-cubes kernels of mesh.cu (dense lattices) and tsdf.cu
// (block-sparse TSDF volumes): the fp32 edge interpolation, the lattice-to-world affine and the
// lookup of an edge's vertex id from its owner's scan base and owned-edge flags.
#pragma once

namespace xrd {
namespace mc {

// t of the level crossing on the lattice edge v0 -> v1, round-to-nearest
__device__ __forceinline__ float edge_t(float level, float v0, float v1) {
  return __fdiv_rn(__fsub_rn(level, v0), __fsub_rn(v1, v0));
}

// world coordinate of one axis of a lattice position c: ((c * spacing + shift) * scale) + origin
__device__ __forceinline__ float world(float c, float spacing, float shift, float scale,
                                       float origin) {
  return __fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(c, spacing), shift), scale), origin);
}

// vertex id of the crossed edge along `axis` owned by a lattice point whose first vertex is
// `vbase` and whose owned crossed edges are the bits of `flags` (bit a = edge along axis a)
__device__ __forceinline__ int edge_vertex(int vbase, int flags, int axis) {
  return vbase + __popc(flags & ((1 << axis) - 1));
}

}  // namespace mc
}  // namespace xrd

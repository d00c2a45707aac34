// The kitchen build (two-level broad phase) with the support-map narrow phase for MESH geoms (-DB200_HULL: dmodel.h carries the
// reduced-hull vertex tables of the blob, sim_core.cuh's portal-refinement collider takes the hull's support function, plane-hull
// picks the deepest vertices).  A third translation unit -- kernels fetch_kernel_hull<W, 31>, unit kernel_unit_kitchen_hull --
// so that the two validated kitchen builds stay byte-identical; chosen by
// b200sim_create when the model blob has MESH geoms (models compiled with mjcf.py compile_mjcf(mesh_hull=True)).
#define B200_KITCHEN_GROUPS 1
#define B200_HULL 1
#include "b200sim_kitchen.cu"

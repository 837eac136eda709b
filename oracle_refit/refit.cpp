/* The parity oracle's mesh refit — TEST INFRASTRUCTURE, built by __graft_entry__.build_oracle() into oracle/_build/liboracle_refit.so
 * and loaded by oracle_refit/pyrefit.py. adaptive_refit.cpp adds the same entry point to the Adaptive-sampler oracle.
 *
 * This translation unit is the ray-query oracle (oracle_queries/queries.cpp, which includes oracle/oracle.cpp whole; both unchanged,
 * so every orc_* entry point of both is here too) plus
 *   orc_scene_refit_mesh  the mesh takes new positions, normals and / or texcoords (NULL keeps an array). With positions, the mesh's
 *                         BVH<Triangle> keeps its nodes, their order, second_child / axis / geom_offset / ngeom and ordered_geom, and
 *                         every FlatNode's bounds become the fold of bvh.rs:143 over that node's ordered_geom range at the new
 *                         positions: BBox::new() unioned with Triangle::bounds (mesh.rs:128-134) of each triangle, in range order.
 * An interior node's range runs from its first leaf's geom_offset to its last leaf's end; it is taken from the leaves' ranges, never
 * from the children's boxes, so the product's bottom-up union is checked rather than repeated. Instances see the new bounds through
 * Mesh::bounds (the root's); the TLAS is rebuilt by the next orc_scene_update_frame, as in the reference.
 */
#include "../oracle_queries/queries.cpp"
#include "refit.h"

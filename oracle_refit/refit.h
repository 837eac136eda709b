/* orc_scene_refit_mesh — TEST INFRASTRUCTURE: included after the oracle (oracle/oracle.cpp) by refit.cpp (with the ray queries) and
 * adaptive_refit.cpp (with the Adaptive sampler). See refit.cpp for the contract it restates. */
#pragma once

extern "C" {

int orc_scene_refit_mesh(orc_scene* s, uint32_t mesh, const float* positions, const float* normals, const float* texcoords) {
    if (!s) { g_err = "null scene"; return TRB_INVALID_ARG; }
    if (mesh >= s->meshes.size()) { g_err = "mesh index out of range"; return TRB_INVALID_ARG; }
    Mesh& m = *s->meshes[mesh];
    for (size_t v = 0; v < m.positions.size(); ++v) {
        if (positions) m.positions[v] = V3(positions[3 * v], positions[3 * v + 1], positions[3 * v + 2]);
        if (normals) m.normals[v] = V3(normals[3 * v], normals[3 * v + 1], normals[3 * v + 2]);
        if (texcoords) m.texcoords[v] = V3(texcoords[2 * v], texcoords[2 * v + 1], 0.0f);
    }
    if (!positions) return TRB_OK;
    BVH& b = m.bvh;
    const size_t n = b.tree.size();
    std::vector<uint32_t> lo(n), hi(n); /* the node's ordered_geom range; preorder puts both children after their parent */
    for (size_t i = n; i-- > 0;) {
        const FlatNode& f = b.tree[i];
        if (f.leaf) { lo[i] = f.a; hi[i] = f.a + f.b; }
        else { lo[i] = lo[i + 1]; hi[i] = hi[f.a]; }
    }
#pragma omp parallel for schedule(dynamic, 256)
    for (long i = 0; i < (long)n; ++i) {
        BBox box;
        for (uint32_t k = lo[i]; k < hi[i]; ++k) {
            const uint32_t t = b.ordered_geom[k];
            const V3 pa = m.positions[m.indices[3 * t]], pb = m.positions[m.indices[3 * t + 1]], pc = m.positions[m.indices[3 * t + 2]];
            box = box.box_union(BBox(pa, pa).point_union(pb).point_union(pc));
        }
        b.tree[i].bounds = box;
    }
    return TRB_OK;
}

} // extern "C"

/* tests/instance_tree_host.cpp — TEST INFRASTRUCTURE: raytracing_b200/csrc/rt_instances.h (the code rt_set_instances runs) behind a C
 * entry point for tests/test_instancing_cpu.py. */
#include <cstdint>
#include <cstring>
#include <vector>
#include "rt_instances.h"

/* n instances (matrices m: 12 floats each, mesh ids) over meshes given by their root boxes (6 floats each: lo xyz, hi xyz) and
 * triangle counts.  Outputs: the instance records (32 floats each), the world boxes (6 floats each), the top-level records
 * (16 floats each, room for max(n - 1, 1)), their count, the root box (6 floats), the root reference and the slack (a, b).
 * Returns 1, or 0 for a rejected list (err gets the message). */
extern "C" int inst_prepare(const float* m, const uint32_t* mesh, uint32_t n, const float* mesh_boxes, const uint32_t* mesh_tris,
                            uint32_t n_meshes, float* rec, float* boxes, float* records, uint32_t* n_records, float* root, int* root_ref,
                            float* slack, char* err, int err_len)
{
    std::vector<RtInstance> in(n);
    for (uint32_t i = 0; i < n; ++i) { memset(&in[i], 0, sizeof(RtInstance)); memcpy(in[i].object_to_world, m + 12 * i, 48); in[i].mesh = mesh[i]; }
    std::vector<rtinst::MeshInfo> meshes(n_meshes);
    uint32_t first = 0;
    for (uint32_t k = 0; k < n_meshes; ++k)
    {
        rtinst::MeshInfo& mi = meshes[k];
        mi.root_ref = 0; mi.rec_f4 = 0; mi.first_tri = first; mi.n_tris = mesh_tris[k]; mi.first_node = 0;
        memcpy(mi.lo, mesh_boxes + 6 * k, 12); memcpy(mi.hi, mesh_boxes + 6 * k + 3, 12);
        first += mesh_tris[k];
    }
    rtinst::Prepared pr;
    std::string e;
    if (!rtinst::prepare(in.data(), n, meshes, pr, e)) { strncpy(err, e.c_str(), err_len - 1); err[err_len - 1] = 0; return 0; }
    memcpy(rec, pr.rec.data(), pr.rec.size() * 4);
    for (uint32_t i = 0; i < n; ++i) { memcpy(boxes + 6 * i, pr.boxes[i].lo, 12); memcpy(boxes + 6 * i + 3, pr.boxes[i].hi, 12); }
    memcpy(records, pr.tree.records.data(), pr.tree.records.size() * 4);
    *n_records = (uint32_t)(pr.tree.records.size() / 16);
    memcpy(root, pr.tree.root.lo, 12); memcpy(root + 3, pr.tree.root.hi, 12);
    *root_ref = pr.tree.root_ref;
    slack[0] = pr.tree.slack[0]; slack[1] = pr.tree.slack[1];
    return 1;
}

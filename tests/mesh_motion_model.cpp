/*
 * mesh_motion_model.cpp — TEST INFRASTRUCTURE.  The velocity AOV of instanced scenes with deforming meshes (rt_update_mesh_triangles*
 * under RT_OPT_OBJECT_MOTION, include/rt_b200.h): the previous positions Q of every mesh triangle placed by the previous transform.
 * It compiles tests/instance_model.cpp into the same translation unit and evaluates, for the primary hits that model's frame
 * found, the rule of the header with the model's own building blocks (Interp, XPoint, ProjectScreen), all float without
 * contraction in the order written:  q = (q1 * w0 + q2 * u) + q3 * v;  velocity = project(M * p) - project(M_prev * q).
 * Built by tests/mesh_motion_model.py with -ffp-contract=off.
 */
#include "instance_model.cpp"

extern "C" {

/* velocity (float2 per pixel) of the primary hits (one RtHit per pixel, as im_render returns them) of the instanced scene of
 * im_render's arguments; prev (12 floats per instance) the previous transforms, NULL = the current ones; prev_positions (9 floats
 * per triangle of scene: q1, q2, q3) the previous mesh positions, NULL = the current ones; the camera is its own previous camera.
 * Returns 0, or -1 for a rejected list. */
int mm_velocity(const OrcScene* scene, const RtMeshDesc* meshes, uint32_t n_meshes, const RtInstance* instances, uint32_t n_inst,
                const float* prev, const float* prev_positions, const RtCamera* cam, uint32_t width, uint32_t height,
                const RtHit* primary_hits, float* velocity)
{
    Scene sc = to_scene(scene);
    Inst I;
    for (uint32_t k = 0; k < n_meshes; ++k)
    {
        const RtMeshDesc& m = meshes[k];
        const RtLinearBVHNode& r = sc.nodes[m.first_node];
        rtinst::MeshInfo mi = { 0, 0, (uint32_t)m.first_triangle, (uint32_t)m.n_triangles, (uint32_t)m.first_node,
                                { r.bounds_min.x, r.bounds_min.y, r.bounds_min.z }, { r.bounds_max.x, r.bounds_max.y, r.bounds_max.z } };
        I.meshes.push_back(mi);
    }
    std::string err;
    if (!rtinst::prepare(instances, n_inst, I.meshes, I.pr, err)) return -1;
    for (size_t pixel = 0; pixel < (size_t)width * height; ++pixel)
    {
        const RtHit& hit = primary_hits[pixel];
        velocity[2 * pixel] = 0.0f; velocity[2 * pixel + 1] = 0.0f;
        if (hit.primitive_id == RT_INVALID_ID) continue;
        const uint32_t inst = InstanceOf(I, hit.primitive_id);
        const float* rec = I.pr.rec.data() + 32 * (size_t)inst;
        uint32_t first_tri;
        memcpy(&first_tri, rec + 26, 4);
        const uint32_t tri_id = first_tri + (hit.primitive_id - I.pr.base[inst]);
        const RtTriangle& tri = sc.triangles[tri_id];
        const float u = hit.bc.x, v = hit.bc.y;
        const V3 obj = Interp(v3(tri.v1.position), v3(tri.v2.position), v3(tri.v3.position), u, v);
        const V3 position = XPoint(rec + 12, obj);
        const float* q = prev_positions ? prev_positions + 9 * (size_t)tri_id : nullptr;
        const V3 was_obj = q ? Interp(v3(q[0], q[1], q[2]), v3(q[3], q[4], q[5]), v3(q[6], q[7], q[8]), u, v) : obj;
        const V3 was = XPoint(prev ? prev + 12 * (size_t)inst : rec + 12, was_obj);
        const V2 a = ProjectScreen(position, *cam), b = ProjectScreen(was, *cam);
        velocity[2 * pixel] = a.x - b.x; velocity[2 * pixel + 1] = a.y - b.y;
    }
    return 0;
}

} // extern "C"

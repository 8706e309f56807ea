/*
 * bsdf_harness.cpp — TEST INFRASTRUCTURE.  Batch entry points for the BSDF sampler (the oracle's SampleBxdf, which the kernels'
 * sample_bxdf is held to bit for bit) and for the BSDF the sampled lights weigh against it (the model's BxdfEvalSampled, held to
 * rt_device.cuh's bxdf_eval_sampled the same way), so that tests/test_bsdf_sampling_cpu.py can check the sampler's directions
 * against the stated density p_b and its estimates against the stated integrand g.  Built by tests/bsdf_harness.py with
 * -ffp-contract=off.
 */
#include "emitter_model.cpp"

namespace
{

// mat: diffuse albedo rgb, roughness, specular albedo rgb, metalness, ior, transparency (the unpacked Material fields)
inline Material material_of(const float* mat)
{
    Material m;
    m.diffuse_albedo = v3(mat[0], mat[1], mat[2]); m.roughness = mat[3];
    m.specular_albedo = v3(mat[4], mat[5], mat[6]); m.metalness = mat[7];
    m.emission = splat(0.0f); m.ior = mat[8];
    m.transparency = mat[9];
    return m;
}

} // namespace

extern "C" {

/* n samples of SampleBxdf from draws s (s1, s.x, s.y per sample): out holds per sample outgoing xyz, pdf, bxdf rgb, offset */
void bh_sample(const float* mat, const float* normal, const float* incoming, const float* s, uint32_t n, float* out)
{
    const Material m = material_of(mat);
    const V3 nrm = v3(normal[0], normal[1], normal[2]), inc = v3(incoming[0], incoming[1], incoming[2]);
#pragma omp parallel for schedule(static)
    for (long long k = 0; k < (long long)n; ++k)
    {
        V3 o = v3(0, 0, 0);
        float pdf = 0.0f, offset = 0.0f;
        V3 f = SampleBxdf(s[3 * k], V2{ s[3 * k + 1], s[3 * k + 2] }, m, nrm, inc, false, &o, &pdf, &offset);
        float* r = out + 8 * k;
        r[0] = o.x; r[1] = o.y; r[2] = o.z; r[3] = pdf; r[4] = f.x; r[5] = f.y; r[6] = f.z; r[7] = offset;
    }
}

/* BxdfEvalSampled for n directions o (xyz): out holds per direction g rgb, p_b, spec_pdf, alpha */
void bh_eval(const float* mat, const float* normal, const float* incoming, const float* o, uint32_t n, float* out)
{
    const Material m = material_of(mat);
    const V3 nrm = v3(normal[0], normal[1], normal[2]), inc = v3(incoming[0], incoming[1], incoming[2]);
#pragma omp parallel for schedule(static)
    for (long long k = 0; k < (long long)n; ++k)
    {
        float p_b, spec_pdf, alpha;
        V3 g = BxdfEvalSampled(m, nrm, inc, v3(o[3 * k], o[3 * k + 1], o[3 * k + 2]), &p_b, &spec_pdf, &alpha);
        float* r = out + 6 * k;
        r[0] = g.x; r[1] = g.y; r[2] = g.z; r[3] = p_b; r[4] = spec_pdf; r[5] = alpha;
    }
}

/* EvaluateMaterial (the BRDF analytic-light samples weigh) for n directions o (xyz): out holds rgb per direction */
void bh_evaluate_material(const float* mat, const float* normal, const float* incoming, const float* o, uint32_t n, float* out)
{
    const Material m = material_of(mat);
    const V3 nrm = v3(normal[0], normal[1], normal[2]), inc = v3(incoming[0], incoming[1], incoming[2]);
    for (uint32_t k = 0; k < n; ++k)
    {
        V3 f = EvaluateMaterial(m, nrm, inc, v3(o[3 * k], o[3 * k + 1], o[3 * k + 2]));
        out[3 * k] = f.x; out[3 * k + 1] = f.y; out[3 * k + 2] = f.z;
    }
}

} // extern "C"

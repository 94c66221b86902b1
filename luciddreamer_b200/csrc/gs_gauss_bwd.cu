// Per-Gaussian backward (sm_90a): turns the 9-float accumulator rows of the tile pass into the FINAL dense gradient
// tensors.  Replaces, fused: computeCov2DCUDA (RAST/cuda_rasterizer/backward.cu:144-274), preprocessCUDA bwd (:346-396,
// with the SH backward :20-139 and the cov3D backward :278-341), the nine torch::zeros fills of the binding
// (RAST/rasterize_points.cu:154-162) and every read-modify-write the reference does on dense [P,*] intermediates
// (dL_dconic, dL_dcov3D, dL_dcolors never exist as dense tensors unless the caller asks for them).  Seven kernels:
//
//   k_grad_vis           over the compact visible list: one 44-float compact row per visible Gaussian in the scratch
//                        (the dL_dsh block kept factored as basis[16] x dRGB[3]), or, after k_fill_zero, the final rows
//                        scattered straight into the outputs
//   k_fill_zero          zeroes the six outputs by TMA on a side stream, beside the tile pass
//   k_grad_write         streaming over all P rows: expands the compact rows into the outputs, zeros for invisible rows
//   k_grad_write_tma     the same for the reference's own input mode, each block assembled in shared memory and stored
//                        by TMA
//   k_grad_dense         more than half of the Gaussians visible: the whole per-Gaussian backward in one TMA pipeline
//   k_grad_reduce_peers  data-parallel shared-model step: adds the visible rows into every rank's bucket
//   k_peer_barrier       that step's cross-rank barrier
//
// Routes, chosen once per call by grad_plan (gs_api.cu); "six outputs" = exactly the six gradients of the reference's
// input mode (16 stored SH coefficients), 16-byte aligned:
//   six outputs, scales + rotations, P % 4 = 0, a context   k_fill_zero + k_grad_vis scattering
//   six outputs otherwise                                    k_grad_vis + k_grad_write_tma
//   any other outputs                                        k_grad_vis + k_grad_write
//   peer reduce                                 [k_peer_barrier] k_grad_vis + k_grad_reduce_peers [k_peer_barrier]
// With six outputs, scales + rotations and no peer reduce, k_grad_dense is launched as well unless the scratch proves
// the sparse regime; the device decides from num_visible which of it and the sparse kernels does the work, and the
// others return at once.

#include "gs_common.cuh"

namespace {

constexpr int kT = 256;
// compact gradient row (floats), 11 float4: dmean3D[3], dmean2D[2], dopacity, dscale[3], drot[4], dRGB[3] (clamp
// masked), SH basis[16], dcolor[3] (raw), dcov3D[6], 3 floats of padding
constexpr int kRow = GS_GOUT_FLOATS;
struct Row {
    static constexpr int dmean3D = 0, dmean2D = 3, dopacity = 5, dscale = 6, drot = 9, dRGB = 13, basis = 16, dcolor = 32,
                         dcov3D = 35;
};

// The accumulator row of one Gaussian (a0, a1, a2, read from `src`: the row itself or a staged copy of it), re-armed in
// `aa` for the next backward: zeros, keeping the clamp bits (a2.y) and the compact slot (a2.w).
__device__ __forceinline__ void take_acc(float4* aa, const float4* src, float4& a0, float4& a1, float4& a2) {
    a0 = src[0]; a1 = src[1]; a2 = src[2];
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    aa[0] = z4; aa[1] = z4; aa[2] = make_float4(0.f, a2.y, 0.f, a2.w);
}

// Row i of the six dense outputs from a finished compact row o: dL_dmeans3D, dL_dmeans2D (its third component is zero,
// stored when kM2z), dL_dopacity, dL_dscales, dL_drotations and dL_dsh = basis x dRGB (16 coefficients).  The
// destinations are global memory or a shared-memory image of a block.  kVec: dL_drotations and dL_dsh leave as float4
// (16-byte aligned rows), else as scalars.  I is the caller's index type, which shapes the address arithmetic.
template <bool kVec, bool kM2z, typename I>
__device__ __forceinline__ void expand_row(const float4* o, float* m3, float* m2, float* op, float* sc, float* rot,
                                           float* sh, const I i) {
    m3[3 * i] = o[0].x; m3[3 * i + 1] = o[0].y; m3[3 * i + 2] = o[0].z;
    m2[3 * i] = o[0].w; m2[3 * i + 1] = o[1].x;
    if (kM2z) m2[3 * i + 2] = 0.f;
    op[i] = o[1].y;
    sc[3 * i] = o[1].z; sc[3 * i + 1] = o[1].w; sc[3 * i + 2] = o[2].x;
    const float bs[16] = {o[4].x, o[4].y, o[4].z, o[4].w, o[5].x, o[5].y, o[5].z, o[5].w,
                          o[6].x, o[6].y, o[6].z, o[6].w, o[7].x, o[7].y, o[7].z, o[7].w};
    const float dR[3] = {o[3].y, o[3].z, o[3].w};
    if (kVec) {
        reinterpret_cast<float4*>(rot)[i] = make_float4(o[2].y, o[2].z, o[2].w, o[3].x);
        float4* d4 = reinterpret_cast<float4*>(sh + (size_t)i * 48);
#pragma unroll
        for (int j = 0; j < 12; j++) {
            float w[4];
#pragma unroll
            for (int u = 0; u < 4; u++) { const int e = 4 * j + u; w[u] = bs[e / 3] * dR[e % 3]; }
            d4[j] = make_float4(w[0], w[1], w[2], w[3]);
        }
    } else {
        rot[4 * i] = o[2].y; rot[4 * i + 1] = o[2].z; rot[4 * i + 2] = o[2].w; rot[4 * i + 3] = o[3].x;
#pragma unroll
        for (int e = 0; e < 48; e++) sh[i * 48 + e] = bs[e / 3] * dR[e % 3];
    }
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tma_store(void* dst, uint32_t src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}

constexpr int kVisT = 64;              // small CTAs: P_vis is often only a few 10^4, spread it over all SMs

// One Gaussian's gradients from the 9 sums of the tile pass (a0, a1, a2 = its accumulator row): computeCov2DCUDA
// (backward.cu:144-274), preprocessCUDA bwd (:346-396), SH bwd (:20-139), cov3D bwd (:278-341).  `fill_cf(cf, n)` loads
// the first n SH coefficients of the Gaussian (global or shared memory).  Writes the 44-float row (11 float4) to o.
// `scales` true: sc / q hold the scale and the quaternion (cov3D is derived); false: c6 holds cov3D_precomp.
template <typename FillCf>
__device__ __forceinline__ void grad_row_core(const GsView& v, const GsCam& cam, const float4 a0, const float4 a1,
                                              const float4 a2, const uint32_t clamped, const float3 p, const bool has_sh,
                                              const bool scales, const float3 sc, const float4 q, float* c6,
                                              FillCf fill_cf, float4* o) {
    const float dm2x = a0.x, dm2y = a0.y, dop = a1.y;
    const float dcx = a0.z, dcy = a0.w, dcz = a1.x;     // dL_dconic (a, b, c)
    const float dcol0 = a1.z, dcol1 = a1.w, dcol2 = a2.x;
    if (scales) gs_cov3d(sc, v.scale_modifier, q, c6);
    // ---- computeCov2DCUDA (backward.cu:144-274)
    GsCov2D cc;
    gs_cov2d(p, v, cam.vm, c6, cc);
    const float a = cc.a, b = cc.b, cq = cc.c;
    const float denom = a * cq - b * b;
    float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
    const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
    const float (*Tm)[3] = cc.A;
    float dcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (denom2inv != 0.f) {
        dL_da = denom2inv * (-cq * cq * dcx + 2 * b * cq * dcy + (denom - a * cq) * dcz);
        dL_dc = denom2inv * (-a * a * dcz + 2 * a * b * dcy + (denom - a * cq) * dcx);
        dL_db = denom2inv * 2 * (b * cq * dcx - (denom + 2 * b * b) * dcy + a * b * dcz);
        dcov[0] = (Tm[0][0] * Tm[0][0] * dL_da + Tm[0][0] * Tm[1][0] * dL_db + Tm[1][0] * Tm[1][0] * dL_dc);
        dcov[3] = (Tm[0][1] * Tm[0][1] * dL_da + Tm[0][1] * Tm[1][1] * dL_db + Tm[1][1] * Tm[1][1] * dL_dc);
        dcov[5] = (Tm[0][2] * Tm[0][2] * dL_da + Tm[0][2] * Tm[1][2] * dL_db + Tm[1][2] * Tm[1][2] * dL_dc);
        dcov[1] = 2 * Tm[0][0] * Tm[0][1] * dL_da + (Tm[0][0] * Tm[1][1] + Tm[0][1] * Tm[1][0]) * dL_db + 2 * Tm[1][0] * Tm[1][1] * dL_dc;
        dcov[2] = 2 * Tm[0][0] * Tm[0][2] * dL_da + (Tm[0][0] * Tm[1][2] + Tm[0][2] * Tm[1][0]) * dL_db + 2 * Tm[1][0] * Tm[1][2] * dL_dc;
        dcov[4] = 2 * Tm[0][2] * Tm[0][1] * dL_da + (Tm[0][1] * Tm[1][2] + Tm[0][2] * Tm[1][1]) * dL_db + 2 * Tm[1][1] * Tm[1][2] * dL_dc;
    }
    const float S[3][3] = {{c6[0], c6[1], c6[2]}, {c6[1], c6[3], c6[4]}, {c6[2], c6[4], c6[5]}};
    float dT[2][3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float u0 = Tm[0][0] * S[k][0] + Tm[0][1] * S[k][1] + Tm[0][2] * S[k][2];
        const float u1 = Tm[1][0] * S[k][0] + Tm[1][1] * S[k][1] + Tm[1][2] * S[k][2];
        dT[0][k] = 2 * u0 * dL_da + u1 * dL_db;
        dT[1][k] = 2 * u1 * dL_dc + u0 * dL_db;
    }
    const float* vm = cam.vm;
    const float dJ00 = vm[0] * dT[0][0] + vm[4] * dT[0][1] + vm[8] * dT[0][2];
    const float dJ02 = vm[2] * dT[0][0] + vm[6] * dT[0][1] + vm[10] * dT[0][2];
    const float dJ11 = vm[1] * dT[1][0] + vm[5] * dT[1][1] + vm[9] * dT[1][2];
    const float dJ12 = vm[2] * dT[1][0] + vm[6] * dT[1][1] + vm[10] * dT[1][2];
    const float tz = 1.f / cc.tz, tz2 = tz * tz, tz3 = tz2 * tz;
    const float dtx = cc.xmul * -v.focal_x * tz2 * dJ02;
    const float dty = cc.ymul * -v.focal_y * tz2 * dJ12;
    const float dtz = -v.focal_x * tz2 * dJ00 - v.focal_y * tz2 * dJ11 + (2 * v.focal_x * cc.tx) * tz3 * dJ02 +
                      (2 * v.focal_y * cc.ty) * tz3 * dJ12;
    float dm3x = vm[0] * dtx + vm[1] * dty + vm[2] * dtz;     // assignment (backward.cu:273)
    float dm3y = vm[4] * dtx + vm[5] * dty + vm[6] * dtz;
    float dm3z = vm[8] * dtx + vm[9] * dty + vm[10] * dtz;

    // ---- preprocessCUDA backward (backward.cu:346-396): projection Jacobian
    const float* pj = cam.pm;
    const float4 m_hom = gs_xf4x4(p, pj);
    const float m_w = 1.0f / (m_hom.w + 0.0000001f);
    const float mul1 = (pj[0] * p.x + pj[4] * p.y + pj[8] * p.z + pj[12]) * m_w * m_w;
    const float mul2 = (pj[1] * p.x + pj[5] * p.y + pj[9] * p.z + pj[13]) * m_w * m_w;
    dm3x += (pj[0] * m_w - pj[3] * mul1) * dm2x + (pj[1] * m_w - pj[3] * mul2) * dm2y;
    dm3y += (pj[4] * m_w - pj[7] * mul1) * dm2x + (pj[5] * m_w - pj[7] * mul2) * dm2y;
    dm3z += (pj[8] * m_w - pj[11] * mul1) * dm2x + (pj[9] * m_w - pj[11] * mul2) * dm2y;

    // ---- SH backward (backward.cu:20-139)
    float bs[16];
#pragma unroll
    for (int k = 0; k < 16; k++) bs[k] = 0.f;
    float dRGB0 = 0.f, dRGB1 = 0.f, dRGB2 = 0.f;
    if (has_sh) {
        const float3 d0 = make_float3(p.x - cam.campos[0], p.y - cam.campos[1], p.z - cam.campos[2]);
        const float len = sqrtf(d0.x * d0.x + d0.y * d0.y + d0.z * d0.z);
        const float x = d0.x / len, y = d0.y / len, z = d0.z / len;
        dRGB0 = dcol0 * ((clamped & 1u) ? 0.f : 1.f);
        dRGB1 = dcol1 * ((clamped & 2u) ? 0.f : 1.f);
        dRGB2 = dcol2 * ((clamped & 4u) ? 0.f : 1.f);
        gs_sh_basis(v.D, x, y, z, bs);
        const int D = v.D;
        float ddx = 0.f, ddy = 0.f, ddz = 0.f;          // dL_ddir
        if (D > 0) {
            // all active coefficients in flight before use
            float cf[48];
            fill_cf(cf, (D + 1) * (D + 1) * 3);
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            const float dR[3] = {dRGB0, dRGB1, dRGB2};
            float ax[3], ay[3], az[3];
#pragma unroll
            for (int ch = 0; ch < 3; ch++) {
#define SHK(k) cf[3 * (k) + ch]
                float vx = -GS_C1 * SHK(3), vy = -GS_C1 * SHK(1), vz = GS_C1 * SHK(2);
                if (D > 1) {
                    vx += GS_C2_0 * y * SHK(4) + GS_C2_2 * 2.f * -x * SHK(6) + GS_C2_3 * z * SHK(7) + GS_C2_4 * 2.f * x * SHK(8);
                    vy += GS_C2_0 * x * SHK(4) + GS_C2_1 * z * SHK(5) + GS_C2_2 * 2.f * -y * SHK(6) + GS_C2_4 * 2.f * -y * SHK(8);
                    vz += GS_C2_1 * y * SHK(5) + GS_C2_2 * 2.f * 2.f * z * SHK(6) + GS_C2_3 * x * SHK(7);
                    if (D > 2) {
                        vx += (GS_C3_0 * SHK(9) * 3.f * 2.f * xy + GS_C3_1 * SHK(10) * yz + GS_C3_2 * SHK(11) * -2.f * xy +
                               GS_C3_3 * SHK(12) * -3.f * 2.f * xz + GS_C3_4 * SHK(13) * (-3.f * xx + 4.f * zz - yy) +
                               GS_C3_5 * SHK(14) * 2.f * xz + GS_C3_6 * SHK(15) * 3.f * (xx - yy));
                        vy += (GS_C3_0 * SHK(9) * 3.f * (xx - yy) + GS_C3_1 * SHK(10) * xz + GS_C3_2 * SHK(11) * (-3.f * yy + 4.f * zz - xx) +
                               GS_C3_3 * SHK(12) * -3.f * 2.f * yz + GS_C3_4 * SHK(13) * -2.f * xy +
                               GS_C3_5 * SHK(14) * -2.f * yz + GS_C3_6 * SHK(15) * -3.f * 2.f * xy);
                        vz += (GS_C3_1 * SHK(10) * xy + GS_C3_2 * SHK(11) * 4.f * 2.f * yz + GS_C3_3 * SHK(12) * 3.f * (2.f * zz - xx - yy) +
                               GS_C3_4 * SHK(13) * 4.f * 2.f * xz + GS_C3_5 * SHK(14) * (xx - yy));
                    }
                }
#undef SHK
                ax[ch] = vx; ay[ch] = vy; az[ch] = vz;
            }
            ddx = ax[0] * dR[0] + ax[1] * dR[1] + ax[2] * dR[2];
            ddy = ay[0] * dR[0] + ay[1] * dR[1] + ay[2] * dR[2];
            ddz = az[0] * dR[0] + az[1] * dR[1] + az[2] * dR[2];
        }
        // dnormvdv (auxiliary.h:107-117)
        const float sum2 = d0.x * d0.x + d0.y * d0.y + d0.z * d0.z;
        const float inv32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
        dm3x += ((+sum2 - d0.x * d0.x) * ddx - d0.y * d0.x * ddy - d0.z * d0.x * ddz) * inv32;
        dm3y += (-d0.x * d0.y * ddx + (sum2 - d0.y * d0.y) * ddy - d0.z * d0.y * ddz) * inv32;
        dm3z += (-d0.x * d0.z * ddx - d0.y * d0.z * ddy + (sum2 - d0.z * d0.z) * ddz) * inv32;
    }

    // ---- cov3D backward (backward.cu:278-341)
    float dsx = 0.f, dsy = 0.f, dsz = 0.f;
    float4 drot = make_float4(0.f, 0.f, 0.f, 0.f);
    if (scales) {
        float R[3][3], M[3][3];
        gs_quat_R(q, R);
        const float sv[3] = {v.scale_modifier * sc.x, v.scale_modifier * sc.y, v.scale_modifier * sc.z};
#pragma unroll
        for (int r_ = 0; r_ < 3; r_++)
#pragma unroll
            for (int c_ = 0; c_ < 3; c_++) M[r_][c_] = sv[r_] * R[c_][r_];
        const float dS[3][3] = {{dcov[0], 0.5f * dcov[1], 0.5f * dcov[2]},
                                {0.5f * dcov[1], dcov[3], 0.5f * dcov[4]},
                                {0.5f * dcov[2], 0.5f * dcov[4], dcov[5]}};
        float dM[3][3];
#pragma unroll
        for (int r_ = 0; r_ < 3; r_++)
#pragma unroll
            for (int c_ = 0; c_ < 3; c_++)
                dM[r_][c_] = 2.0f * (M[r_][0] * dS[0][c_] + M[r_][1] * dS[1][c_] + M[r_][2] * dS[2][c_]);
        dsx = R[0][0] * dM[0][0] + R[1][0] * dM[0][1] + R[2][0] * dM[0][2];
        dsy = R[0][1] * dM[1][0] + R[1][1] * dM[1][1] + R[2][1] * dM[1][2];
        dsz = R[0][2] * dM[2][0] + R[1][2] * dM[2][1] + R[2][2] * dM[2][2];
        float Q[3][3];
#pragma unroll
        for (int r_ = 0; r_ < 3; r_++)
#pragma unroll
            for (int c_ = 0; c_ < 3; c_++) Q[r_][c_] = dM[r_][c_] * sv[r_];
        const float r = q.x, x = q.y, y = q.z, z = q.w;
        drot.x = 2 * z * (Q[0][1] - Q[1][0]) + 2 * y * (Q[2][0] - Q[0][2]) + 2 * x * (Q[1][2] - Q[2][1]);
        drot.y = 2 * y * (Q[1][0] + Q[0][1]) + 2 * z * (Q[2][0] + Q[0][2]) + 2 * r * (Q[1][2] - Q[2][1]) - 4 * x * (Q[2][2] + Q[1][1]);
        drot.z = 2 * x * (Q[1][0] + Q[0][1]) + 2 * r * (Q[2][0] - Q[0][2]) + 2 * z * (Q[1][2] + Q[2][1]) - 4 * y * (Q[2][2] + Q[0][0]);
        drot.w = 2 * r * (Q[0][1] - Q[1][0]) + 2 * x * (Q[2][0] + Q[0][2]) + 2 * y * (Q[1][2] + Q[2][1]) - 4 * z * (Q[1][1] + Q[0][0]);
    }

    o[0] = make_float4(dm3x, dm3y, dm3z, dm2x);
    o[1] = make_float4(dm2y, dop, dsx, dsy);
    o[2] = make_float4(dsz, drot.x, drot.y, drot.z);
    o[3] = make_float4(drot.w, dRGB0, dRGB1, dRGB2);
    o[4] = make_float4(bs[0], bs[1], bs[2], bs[3]);
    o[5] = make_float4(bs[4], bs[5], bs[6], bs[7]);
    o[6] = make_float4(bs[8], bs[9], bs[10], bs[11]);
    o[7] = make_float4(bs[12], bs[13], bs[14], bs[15]);
    o[8] = make_float4(dcol0, dcol1, dcol2, dcov[0]);
    o[9] = make_float4(dcov[1], dcov[2], dcov[3], dcov[4]);
    o[10] = make_float4(dcov[5], 0.f, 0.f, 0.f);
}

// operands from global memory (compact-list kernel)
template <typename FillCf>
__device__ __forceinline__ void grad_row(const GsView& v, const GsCam& cam, const size_t i, const float4 a0, const float4 a1,
                                         const float4 a2, const uint32_t clamped, const float* __restrict__ means3D,
                                         const bool has_sh, const float* __restrict__ scales,
                                         const float* __restrict__ rotations, const float* __restrict__ cov3D_precomp,
                                         FillCf fill_cf, float4* o) {
    const float3 p = make_float3(means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2]);
    float c6[6];
    float3 sc = make_float3(0.f, 0.f, 0.f);
    float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
    if (cov3D_precomp) {
#pragma unroll
        for (int k = 0; k < 6; k++) c6[k] = cov3D_precomp[6 * i + k];
    } else {
        sc = make_float3(scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]);
        q = __ldg(reinterpret_cast<const float4*>(rotations) + i);
    }
    grad_row_core(v, cam, a0, a1, a2, clamped, p, has_sh, cov3D_precomp == nullptr, sc, q, c6, fill_cf, o);
}

// more than half of the Gaussians visible: the dense kernel (k_grad_dense) does the whole per-Gaussian backward
__device__ __forceinline__ bool gs_dense_regime(const GsDevStatus* status, int P) {
    return 2ull * status->num_visible > (unsigned long long)P;
}

__global__ void __launch_bounds__(kVisT)
k_grad_vis(const GsView v, const float* __restrict__ means3D, const float* __restrict__ shs,
           const float* __restrict__ scales, const float* __restrict__ rotations,
           const float* __restrict__ cov3D_precomp, const float4* __restrict__ rec, float4* __restrict__ acc,
           const uint32_t* __restrict__ vis_list, const GsDevStatus* __restrict__ status, float* __restrict__ gout,
           const bool dense_elsewhere, const bool scatter, const GsGradPtrs g) {
    if (dense_elsewhere && gs_dense_regime(status, v.P)) return;
    __shared__ GsCam cam;
    gs_load_cam(v, &cam);
    const uint32_t nvis = (uint32_t)status->num_visible;
    for (uint32_t c = blockIdx.x * kVisT + threadIdx.x; c < nvis; c += gridDim.x * kVisT) {
        const uint32_t i = vis_list[c];
        float4 a0, a1, a2;
        take_acc(acc + (size_t)3 * i, acc + (size_t)3 * i, a0, a1, a2);
        const uint32_t clamped = __float_as_uint(a2.y);
        const float* sh = shs ? shs + (size_t)i * v.M * 3 : nullptr;
        // 128-bit loads when the rows are 16-byte aligned (M * 3 a multiple of 4, base aligned like every input --
        // gsraster.h; k_shade_emit reads them the same way), scalar loads otherwise
        const bool sh_v4 = (v.M * 3) % 4 == 0;
        auto fill = [&](float* cf, int na3) {
            if (sh_v4) {
                const float4* s4 = reinterpret_cast<const float4*>(sh);
#pragma unroll
                for (int k = 0; k < 12; k++) {
                    const float4 t = 4 * k < na3 ? __ldg(s4 + k) : make_float4(0.f, 0.f, 0.f, 0.f);
                    cf[4 * k] = t.x; cf[4 * k + 1] = 4 * k + 1 < na3 ? t.y : 0.f;
                    cf[4 * k + 2] = 4 * k + 2 < na3 ? t.z : 0.f; cf[4 * k + 3] = 4 * k + 3 < na3 ? t.w : 0.f;
                }
            } else {
#pragma unroll
                for (int k = 0; k < 48; k++) cf[k] = k < na3 ? __ldg(sh + k) : 0.f;
            }
        };
        if (!scatter) {
            grad_row(v, cam, i, a0, a1, a2, clamped, means3D, shs != nullptr, scales, rotations, cov3D_precomp, fill,
                     reinterpret_cast<float4*>(gout + (size_t)c * kRow));
            continue;
        }
        // the dense outputs were zero-filled beside the tile pass (k_fill_zero): the final rows go straight into them
        float4 o[11];
        grad_row(v, cam, i, a0, a1, a2, clamped, means3D, true, scales, rotations, cov3D_precomp, fill, o);
        expand_row<true, false>(o, g.dmeans3D, g.dmeans2D, g.dopacity, g.dscales, g.drots, g.dsh, i);   // the fill left dmeans2D[.][2] zero
    }
}

// Zero-fill of the six dense gradient tensors by TMA, issued on a side stream BESIDE the tile pass of the backward
// (the first stage of gs_backward): a persistent grid of single-warp CTAs, each streaming 16 KB bulk stores out of one zeroed
// shared-memory page.  No loads, no index arithmetic; in the dense regime (k_grad_dense writes every row) it exits.
struct FillRuns { char* p[6]; long long bytes[6]; };

__global__ void __launch_bounds__(32)
k_fill_zero(const FillRuns runs, const GsDevStatus* __restrict__ status, const int P, const bool dense_elsewhere) {
    if (dense_elsewhere && gs_dense_regime(status, P)) return;
    __shared__ __align__(128) float4 zero[1024];           // 16 KB
    for (int f = threadIdx.x; f < 1024; f += 32) zero[f] = make_float4(0.f, 0.f, 0.f, 0.f);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();
    if (threadIdx.x != 0) return;
    const uint32_t z = smem_u32(zero);
    long long base = 0;
    for (int r = 0; r < 6; r++) {
        const long long nchunk = (runs.bytes[r] + 16383) / 16384;
        // chunks are numbered across the six runs; CTA b takes chunks b, b + grid, ...
        long long first = ((long long)blockIdx.x - base % gridDim.x + gridDim.x) % gridDim.x;
        for (long long c = first; c < nchunk; c += gridDim.x) {
            const long long off = c * 16384, left = runs.bytes[r] - off;
            tma_store(runs.p[r] + off, z, (uint32_t)(left < 16384 ? left : 16384));
        }
        base += nchunk;
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// Store phase shared by k_grad_write and k_grad_dense.  One CTA of NT threads = NT consecutive rows; s_slot[row] =
// CTA-local index of the row's staged gradient (RS floats apart in s_row), or -1 for an invisible row (zeros).
template <int NF, int NT, int RS>
__device__ __forceinline__ void cta_store_rows(float* __restrict__ dst, const float* s_row, const int* s_slot, int off,
                                               long long row0, long long P) {
    const long long base = row0 * NF, lim = P * NF;
#pragma unroll
    for (int k = 0; k < NF; k++) {
        const int e = threadIdx.x + NT * k;
        const int row = e / NF, comp = e - row * NF;
        const int cl = s_slot[row];
        if (base + e < lim) dst[base + e] = cl < 0 ? 0.f : s_row[cl * RS + off + comp];
    }
}

// zeroes rows [row0, row0 + NT) of a dense [P, nf] tensor (nf floats per row); NT * nf is a multiple of 4
template <int NT>
__device__ __forceinline__ void cta_zero_run(float* __restrict__ base, long long row0, int nf) {
    if (!base || nf <= 0) return;
    float* p = base + row0 * nf;
    const int total = NT * nf;
    if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) {
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int f = threadIdx.x; f < (total >> 2); f += NT) reinterpret_cast<float4*>(p)[f] = z4;
    } else {
        for (int f = threadIdx.x; f < total; f += NT) p[f] = 0.f;
    }
}

// One run of zeros by TMA: `bytes` (a multiple of 16) from the 16 KB zero buffer in shared memory, 16 KB at a time.
__device__ __forceinline__ bool tma_zero_run(float* base, long long row0, int nf, int rows, uint32_t zsrc) {
    if (!base || nf <= 0) return true;
    float* p = base + row0 * nf;
    if (reinterpret_cast<uintptr_t>(p) & 15) return false;
    long long bytes = (long long)rows * nf * 4;
    for (char* d = reinterpret_cast<char*>(p); bytes > 0; d += 16384, bytes -= 16384)
        tma_store(d, zsrc, (uint32_t)(bytes < 16384 ? bytes : 16384));
    return true;
}

// `cl` = s_slot[threadIdx.x]; `count` = number of visible rows of the CTA
template <int NT, int RS>
__device__ __forceinline__ void cta_write_block(const int P, const int M, const long long row0, const float* s_row,
                                                const int* s_slot, const int cl, const int count, const GsGradPtrs& g,
                                                float* zero_smem = nullptr) {
    const int tid = threadIdx.x;
    const long long i = row0 + tid;
    __shared__ int s_misaligned;
    if (count == 0 && row0 + NT <= P && zero_smem) {
        // no visible row in this CTA (the common case when only a few per cent of the Gaussians are on screen): the NT
        // rows of every output are one contiguous run -> the TMA streams zeros out of a 16 KB shared-memory buffer
        // (eight bulk stores per CTA instead of ~4000 store instructions)
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int f = tid; f < 1024; f += NT) reinterpret_cast<float4*>(zero_smem)[f] = z4;
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        if (tid == 0) {
            const uint32_t z = smem_u32(zero_smem);
            const int M3z = g.dsh ? M * 3 : 0;
            bool ok = ((NT * 4) & 15) == 0;
            ok = ok && tma_zero_run(g.dmeans3D, row0, 3, NT, z) && tma_zero_run(g.dmeans2D, row0, 3, NT, z) &&
                 tma_zero_run(g.dscales, row0, 3, NT, z) && tma_zero_run(g.dcolors, row0, 3, NT, z) &&
                 tma_zero_run(g.dcov3D, row0, 6, NT, z) && tma_zero_run(g.dopacity, row0, 1, NT, z) &&
                 tma_zero_run(g.drots, row0, 4, NT, z) && tma_zero_run(g.dsh, row0, M3z, NT, z);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // the source buffer is shared memory
            s_misaligned = ok ? 0 : 1;
        }
        __syncthreads();
        if (!s_misaligned) return;
    }
    if (count == 0 && row0 + NT <= P) {
        // no visible row in this CTA (the common case when only a few per cent of the Gaussians are on screen):
        // the NT rows of every output are one contiguous run -> straight 128-bit zero stores, no index maths
        const int M3z = g.dsh ? M * 3 : 0;
        cta_zero_run<NT>(g.dmeans3D, row0, 3); cta_zero_run<NT>(g.dmeans2D, row0, 3); cta_zero_run<NT>(g.dscales, row0, 3);
        cta_zero_run<NT>(g.dcolors, row0, 3);  cta_zero_run<NT>(g.dcov3D, row0, 6);   cta_zero_run<NT>(g.dopacity, row0, 1);
        cta_zero_run<NT>(g.drots, row0, 4);    cta_zero_run<NT>(g.dsh, row0, M3z);
        return;
    }
    if (g.dmeans3D) cta_store_rows<3, NT, RS>(g.dmeans3D, s_row, s_slot, Row::dmean3D, row0, P);
    if (g.dmeans2D) {
        const long long base = row0 * 3, lim = (long long)P * 3;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const int e = tid + NT * k;
            const int row = e / 3, comp = e - row * 3;
            const int c2 = s_slot[row];
            if (base + e < lim) g.dmeans2D[base + e] = (c2 < 0 || comp == 2) ? 0.f : s_row[c2 * RS + Row::dmean2D + comp];
        }
    }
    if (g.dscales) cta_store_rows<3, NT, RS>(g.dscales, s_row, s_slot, Row::dscale, row0, P);
    if (g.dcolors) cta_store_rows<3, NT, RS>(g.dcolors, s_row, s_slot, Row::dcolor, row0, P);
    if (g.dcov3D) cta_store_rows<6, NT, RS>(g.dcov3D, s_row, s_slot, Row::dcov3D, row0, P);
    if (i < P) {
        if (g.dopacity) g.dopacity[i] = cl < 0 ? 0.f : s_row[cl * RS + Row::dopacity];
        if (g.drots) {
            float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
            if (cl >= 0) { const float* q = s_row + cl * RS + Row::drot; r = make_float4(q[0], q[1], q[2], q[3]); }
            if ((reinterpret_cast<uintptr_t>(g.drots) & 15) == 0) reinterpret_cast<float4*>(g.drots)[i] = r;
            else { float* d = g.drots + 4 * i; d[0] = r.x; d[1] = r.y; d[2] = r.z; d[3] = r.w; }
        }
    }
    if (g.dsh && M > 0) {
        const int M3 = M * 3;
        const long long rows = min((long long)NT, (long long)P - row0);
        float* dst = g.dsh + row0 * M3;
        const int total = (int)rows * M3;
        if (M3 == 48 && (reinterpret_cast<uintptr_t>(g.dsh) & 15) == 0) {   // M = 16: 12 float4 per row
            const int total4 = total >> 2;
            for (int f = tid; f < total4; f += NT) {
                const int row = f / 12, j = f - row * 12;
                const int c2 = s_slot[row];
                float4 o4 = make_float4(0.f, 0.f, 0.f, 0.f);
                if (c2 >= 0) {
                    const float* sb = s_row + c2 * RS + Row::basis;
                    const float* sr = s_row + c2 * RS + Row::dRGB;
                    float o[4];
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        const int e = 4 * j + u;
                        const int k = e / 3, ch = e - 3 * k;
                        o[u] = sb[k] * sr[ch];
                    }
                    o4 = make_float4(o[0], o[1], o[2], o[3]);
                }
                reinterpret_cast<float4*>(dst)[f] = o4;
            }
        } else {
            for (int e = tid; e < total; e += NT) {
                const int row = e / M3, rem = e - row * M3;
                const int k = rem / 3, ch = rem - 3 * k;
                const int c2 = s_slot[row];
                dst[e] = (c2 < 0 || k >= 16) ? 0.f : s_row[c2 * RS + Row::basis + k] * s_row[c2 * RS + Row::dRGB + ch];
            }
        }
    }
}

// The kT rows [row0, row0 + kT) of one CTA: every visible row claims a CTA-local compact slot (s_slot[row], -1 for an
// invisible row; *s_count = visible rows; s_rowidx[slot] = row when kRowIdx) and stages its compact row (k_grad_vis) at
// s_row + slot * kRow.  Returns the calling thread's slot; the CTA is synchronised on return.
template <bool kRowIdx>
__device__ __forceinline__ int claim_and_stage(const int P, const int* __restrict__ radii, const float4* __restrict__ acc,
                                               const float* __restrict__ gout, const long long row0, float* s_row,
                                               int* s_slot, int* s_count, int* s_rowidx) {
    const int tid = threadIdx.x, lane = tid & 31;
    const long long i = row0 + tid;
    if (tid == 0) *s_count = 0;
    __syncthreads();
    const bool vis = i < P && radii[i] > 0;
    const unsigned m = __ballot_sync(0xffffffffu, vis);
    int cl = -1;
    if (m) {
        int base = 0;
        if (lane == __ffs(m) - 1) base = atomicAdd(s_count, __popc(m));
        base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
        if (vis) cl = base + __popc(m & ((1u << lane) - 1u));
    }
    s_slot[tid] = cl;
    if (vis) {
        if (kRowIdx) s_rowidx[cl] = tid;
        const uint32_t slot = __float_as_uint(__ldg(reinterpret_cast<const float*>(acc + (size_t)3 * i + 2) + 3));
        const float4* src = reinterpret_cast<const float4*>(gout + (size_t)slot * kRow);
        float4* dstr = reinterpret_cast<float4*>(s_row + cl * kRow);
#pragma unroll
        for (int k = 0; k < kRow / 4; k++) dstr[k] = __ldg(src + k);
    }
    __syncthreads();
    return cl;
}

__global__ void __launch_bounds__(kT)
k_grad_write(const int P, const int M, const int* __restrict__ radii, const float4* __restrict__ acc,
             const float* __restrict__ gout, const GsGradPtrs g, const GsDevStatus* __restrict__ status,
             const bool dense_elsewhere) {
    if (dense_elsewhere && gs_dense_regime(status, P)) return;
    extern __shared__ __align__(16) float s_row[];       // kT * kRow floats: staged compact rows of this CTA
    __shared__ int s_slot[kT];
    __shared__ int s_count;
    const long long row0 = (long long)blockIdx.x * kT;
    const int cl = claim_and_stage<false>(P, radii, acc, gout, row0, s_row, s_slot, &s_count, nullptr);
    cta_write_block<kT, kRow>(P, M, row0, s_row, s_slot, cl, s_count, g, s_row);   // s_row doubles as the zero buffer
}

// ---- the common input mode (SH with 16 stored coefficients, scales + rotations, 16-byte aligned outputs): the block's
// slice of all six dense gradient tensors is ASSEMBLED IN SHARED MEMORY -- zeros, plus the expanded rows of the few
// visible Gaussians -- and leaves the SM as six TMA bulk stores.  Replaces ~60 global store instructions per thread by
// ~16 shared-memory stores; the HBM write stream is issued by the copy engine of the SM at full width.
constexpr int kWT = 128;               // rows per block
struct WriteImg {                      // byte offsets of the block image in shared memory
    static constexpr int sh = 0, m3 = 24576, m2 = 26112, sc = 27648, op = 29184, rot = 29696, bytes = 31744;
};

__global__ void __launch_bounds__(kWT)
k_grad_write_tma(const int P, const int* __restrict__ radii, const float4* __restrict__ acc,
                 const float* __restrict__ gout, const GsGradPtrs g, const GsDevStatus* __restrict__ status,
                 const bool dense_elsewhere) {
    if (dense_elsewhere && gs_dense_regime(status, P)) return;
    __shared__ __align__(128) unsigned char img[WriteImg::bytes];
    const int tid = threadIdx.x;
    const int nblk = (P + kWT - 1) / kWT;
  for (int blk = blockIdx.x; blk < nblk; blk += gridDim.x) {        // persistent grid: an early exit costs one wave
    const long long row0 = (long long)blk * kWT, i = row0 + tid;
    const bool full = row0 + kWT <= P;
    const bool vis = i < P && radii[i] > 0;
    float4 o[11];
    if (vis) {                                             // the row's compact gradients (k_grad_vis), in flight early
        const uint32_t slot = __float_as_uint(__ldg(reinterpret_cast<const float*>(acc + (size_t)3 * i + 2) + 3));
        const float4* src = reinterpret_cast<const float4*>(gout + (size_t)slot * kRow);
#pragma unroll
        for (int k = 0; k < 11; k++) o[k] = __ldg(src + k);
    } else {
#pragma unroll
        for (int k = 0; k < 11; k++) o[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (full) {
        // every thread writes its own row of every tensor (zeros for an invisible row): conflict-free, no second pass
        const float bs[16] = {o[4].x, o[4].y, o[4].z, o[4].w, o[5].x, o[5].y, o[5].z, o[5].w,
                              o[6].x, o[6].y, o[6].z, o[6].w, o[7].x, o[7].y, o[7].z, o[7].w};
        const float dR[3] = {o[3].y, o[3].z, o[3].w};
        float4* d4 = reinterpret_cast<float4*>(img + WriteImg::sh) + tid * 12;
#pragma unroll
        for (int j = 0; j < 12; j++) {
            float w[4];
#pragma unroll
            for (int u = 0; u < 4; u++) { const int e = 4 * j + u; w[u] = bs[e / 3] * dR[e % 3]; }
            d4[j] = make_float4(w[0], w[1], w[2], w[3]);
        }
        float* m3 = reinterpret_cast<float*>(img + WriteImg::m3) + tid * 3;
        float* m2 = reinterpret_cast<float*>(img + WriteImg::m2) + tid * 3;
        float* sc = reinterpret_cast<float*>(img + WriteImg::sc) + tid * 3;
        m3[0] = o[0].x; m3[1] = o[0].y; m3[2] = o[0].z;
        m2[0] = o[0].w; m2[1] = o[1].x; m2[2] = 0.f;
        sc[0] = o[1].z; sc[1] = o[1].w; sc[2] = o[2].x;
        reinterpret_cast<float*>(img + WriteImg::op)[tid] = o[1].y;
        reinterpret_cast<float4*>(img + WriteImg::rot)[tid] = make_float4(o[2].y, o[2].z, o[2].w, o[3].x);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        if (tid == 0) {
            const uint32_t base = smem_u32(img);
            tma_store(g.dsh + row0 * 48, base + WriteImg::sh, 24576);
            tma_store(g.dmeans3D + row0 * 3, base + WriteImg::m3, 1536);
            tma_store(g.dmeans2D + row0 * 3, base + WriteImg::m2, 1536);
            tma_store(g.dscales + row0 * 3, base + WriteImg::sc, 1536);
            tma_store(g.dopacity + row0, base + WriteImg::op, 512);
            tma_store(g.drots + row0 * 4, base + WriteImg::rot, 2048);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // the image is read before it is rebuilt
        }
        __syncthreads();
        continue;
    }
    if (i < P)                                             // last, partial block: plain stores
        expand_row<false, true>(o, g.dmeans3D, g.dmeans2D, g.dopacity, g.dscales, g.drots, g.dsh, i);
  }
}

// ---- dense regime (more than half of the Gaussians visible -- LucidDreamer's own workload: every Gaussian comes from a
// pixel of a training view, luciddreamer.py:370-374): ONE persistent kernel over all P rows replaces k_grad_vis +
// k_grad_write, built as a TMA pipeline.  A CTA owns blocks of 128 CONSECUTIVE Gaussians; everything such a block reads
// (SH rows 24 KB, accumulator rows 6 KB, means, scales, rotations) and writes (the six dense gradient tensors) is one
// contiguous run per tensor, so
//   in :  5 cp.async.bulk loads per block into one of two shared-memory stages, completion on the stage's mbarrier;
//         the loads of block k+1 are in flight while block k is computed (double buffering);
//   out:  every thread leaves its row's gradients in shared memory (the dL_dsh row = basis x dRGB takes the place of
//         the consumed SH row) and 6 cp.async.bulk stores per block write them out -- no index arithmetic, no
//         uncoalesced access, and the compact 176-byte rows of the sparse path never exist.
constexpr int kDT = 128;               // rows per block = threads per CTA
struct DenseStage {                    // byte offsets inside one stage
    static constexpr int sh = 0, acc = 24576, means = 30720, scales = 32256, rot = 33792, dm2 = 35840, dop = 37376,
                         bytes = 37888;
};
constexpr int kDenseSmem = 2 * DenseStage::bytes;

__device__ __forceinline__ void tma_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__global__ void __launch_bounds__(kDT, 3)
k_grad_dense(const GsView v, const float* __restrict__ means3D, const float* __restrict__ shs,
             const float* __restrict__ scales, const float* __restrict__ rotations, const int* __restrict__ radii,
             float4* __restrict__ acc, const GsDevStatus* __restrict__ status, const GsGradPtrs g) {
    if (!gs_dense_regime(status, v.P)) return;
    extern __shared__ __align__(128) unsigned char s_dense[];
    __shared__ GsCam cam;
    __shared__ __align__(8) unsigned long long s_bar[2];
    const int tid = threadIdx.x;
    const int nfull = v.P / kDT;                           // full blocks take the TMA pipeline
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(&s_bar[0])), "r"(1));
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(&s_bar[1])), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    gs_load_cam(v, &cam);                                  // contains the __syncthreads that publishes the barriers

    auto issue_loads = [&](int blk, int st) {              // one thread
        const size_t row0 = (size_t)blk * kDT;
        const uint32_t base = smem_u32(s_dense + st * DenseStage::bytes), bar = smem_u32(&s_bar[st]);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(DenseStage::dm2) : "memory");
        tma_load(base + DenseStage::sh, shs + row0 * 48, 24576, bar);
        tma_load(base + DenseStage::acc, acc + row0 * 3, 6144, bar);
        tma_load(base + DenseStage::means, means3D + row0 * 3, 1536, bar);
        tma_load(base + DenseStage::scales, scales + row0 * 3, 1536, bar);
        tma_load(base + DenseStage::rot, rotations + row0 * 4, 2048, bar);
    };

    int it = 0;
    if (tid == 0 && (int)blockIdx.x < nfull) issue_loads(blockIdx.x, 0);
    for (int blk = blockIdx.x; blk < nfull; blk += gridDim.x, it++) {
        const int st = it & 1;
        unsigned char* S = s_dense + st * DenseStage::bytes;
        const size_t row0 = (size_t)blk * kDT, i = row0 + tid;
        if (tid == 0) {
            // the other stage is free once the bulk stores issued from it (previous iteration) have read it
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            if (blk + (int)gridDim.x < nfull) issue_loads(blk + gridDim.x, st ^ 1);
        }
        const bool vis = radii[i] > 0;
        {
            uint32_t done = 0;
            const uint32_t bar = smem_u32(&s_bar[st]), parity = (it >> 1) & 1;
            while (!done) {
                asm volatile("{.reg .pred p;\n\t"
                             "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                             "selp.u32 %0, 1, 0, p;}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
            }
        }
        float* s_sh = reinterpret_cast<float*>(S + DenseStage::sh) + tid * 48;
        float* s_m = reinterpret_cast<float*>(S + DenseStage::means) + tid * 3;
        float* s_s = reinterpret_cast<float*>(S + DenseStage::scales) + tid * 3;
        float4* s_r = reinterpret_cast<float4*>(S + DenseStage::rot) + tid;
        float* s_dm2 = reinterpret_cast<float*>(S + DenseStage::dm2) + tid * 3;
        float* s_dop = reinterpret_cast<float*>(S + DenseStage::dop) + tid;
        float4 o[11];
        if (vis) {
            float4 a0, a1, a2;
            take_acc(acc + i * 3, reinterpret_cast<const float4*>(S + DenseStage::acc) + tid * 3, a0, a1, a2);
            const float3 p = make_float3(s_m[0], s_m[1], s_m[2]);
            const float3 sc = make_float3(s_s[0], s_s[1], s_s[2]);
            const float4 q = *s_r;
            auto fill = [&](float* cf, int) {
                const float4* s4 = reinterpret_cast<const float4*>(s_sh);
#pragma unroll
                for (int k = 0; k < 12; k++) {
                    const float4 t = s4[k];
                    cf[4 * k] = t.x; cf[4 * k + 1] = t.y; cf[4 * k + 2] = t.z; cf[4 * k + 3] = t.w;
                }
            };
            float c6[6];
            grad_row_core(v, cam, a0, a1, a2, __float_as_uint(a2.y), p, true, true, sc, q, c6, fill, o);
        } else {
#pragma unroll
            for (int k = 0; k < 11; k++) o[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        // every thread writes only slots it alone read: its SH row, mean, scale, rotation (dm2 / dop have their own)
        expand_row<true, true>(o, s_m, s_dm2, s_dop, s_s, reinterpret_cast<float*>(s_r), s_sh, 0);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");             // generic writes -> visible to the TMA
        __syncthreads();
        if (tid == 0) {
            const uint32_t base = smem_u32(S);
            tma_store(g.dsh + row0 * 48, base + DenseStage::sh, 24576);
            tma_store(g.dmeans3D + row0 * 3, base + DenseStage::means, 1536);
            tma_store(g.dmeans2D + row0 * 3, base + DenseStage::dm2, 1536);
            tma_store(g.dopacity + row0, base + DenseStage::dop, 512);
            tma_store(g.dscales + row0 * 3, base + DenseStage::scales, 1536);
            tma_store(g.drots + row0 * 4, base + DenseStage::rot, 2048);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
    if (tid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");     // stores complete before the CTA exits

    // the last, partial block (P % 128 rows): plain loads and stores, one CTA
    if (blockIdx.x == 0 && nfull * kDT < v.P) {
        const size_t i = (size_t)nfull * kDT + tid;
        if (i < (size_t)v.P) {
            float4 o[11];
            if (radii[i] > 0) {
                float4 a0, a1, a2;
                take_acc(acc + i * 3, acc + i * 3, a0, a1, a2);
                const float* sh = shs + i * 48;
                auto fill = [&](float* cf, int) {
#pragma unroll
                    for (int k = 0; k < 48; k++) cf[k] = __ldg(sh + k);
                };
                grad_row(v, cam, i, a0, a1, a2, __float_as_uint(a2.y), means3D, true, scales, rotations, nullptr, fill, o);
            } else {
#pragma unroll
                for (int k = 0; k < 11; k++) o[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
            expand_row<false, true>(o, g.dmeans3D, g.dmeans2D, g.dopacity, g.dscales, g.drots, g.dsh, i);
        }
    }
}

// Fused "final gradient -> peer reduce" for the shared-model data-parallel step (SURVEY.md 8e): instead of writing
// a dense local gradient and all-reducing 59 floats x P over NCCL, every rank adds the rows of its VISIBLE
// Gaussians straight into every rank's (pre-zeroed, symmetric) gradient bucket with red.global.add.f32 over
// NVLink peer mappings -- or with ONE multimem.red per element through the NVSwitch multicast address when the
// buckets are bound to a multicast object.  Traffic is 59 floats x P_vis per rank and peer instead of a dense
// 2 x 59 x P all-reduce; rows of invisible Gaussians are never touched.  dL_dmeans2D stays local (it feeds the
// per-view densification statistic, scene/gaussian_model.py:405-407).
struct GsPeerArgs {
    // sig[r] = rank r's signal words (peer-mapped uint32 array): [0, 16) "bucket of rank j is cleared" epochs,
    // [16, 32) "rank j's adds have landed" epochs (k_peer_barrier)
    uint32_t* sig[GS_MAX_PEERS];
    int rank;
    float* peers[GS_MAX_PEERS];       // bucket base of every rank (peer-mapped), [0, world)
    float* mc;                        // multicast address of the bucket, or nullptr
    int world;
    long long off_m3, off_sh, off_op, off_sc, off_rot;   // segment offsets inside the bucket, in floats
};

__device__ __forceinline__ void peer_add(const GsPeerArgs& pa, long long off, float v) {
    if (v == 0.f) return;
    if (pa.mc) {
        asm volatile("multimem.red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(pa.mc + off), "f"(v) : "memory");
    } else {
        for (int r = 0; r < pa.world; r++) atomicAdd(pa.peers[r] + off, v);
    }
}
// 128-bit variant (off must be a multiple of 4 floats and the buckets 16-byte aligned)
__device__ __forceinline__ void peer_add4(const GsPeerArgs& pa, long long off, float4 v) {
    if (v.x == 0.f && v.y == 0.f && v.z == 0.f && v.w == 0.f) return;
    if (pa.mc) {
        asm volatile("multimem.red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(pa.mc + off), "f"(v.x),
                     "f"(v.y), "f"(v.z), "f"(v.w)
                     : "memory");
    } else {
        for (int r = 0; r < pa.world; r++) atomicAdd(reinterpret_cast<float4*>(pa.peers[r] + off), v);
    }
}

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ void peer_reduce_rows(const GsPeerArgs& pa, const float* s_row, const int* s_rowidx, int nv, int M,
                                                 long long row0);

__global__ void __launch_bounds__(kT)
k_grad_reduce_peers(const int P, const int M, const int* __restrict__ radii, const float4* __restrict__ acc,
                    const float* __restrict__ gout, float* __restrict__ dmeans2D, const GsPeerArgs pa) {
    extern __shared__ __align__(16) float s_row[];
    __shared__ int s_rowidx[kT];
    __shared__ int s_slot[kT];
    __shared__ int s_count;
    const int tid = threadIdx.x;
    const long long row0 = (long long)blockIdx.x * kT;
    claim_and_stage<true>(P, radii, acc, gout, row0, s_row, s_slot, &s_count, s_rowidx);
    if (dmeans2D) {                                      // local, dense (zeros for invisible rows)
        const long long base = row0 * 3, lim = (long long)P * 3;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const int e = tid + kT * k;
            const int row = e / 3, comp = e - row * 3;
            const int c2 = s_slot[row];
            if (base + e < lim) dmeans2D[base + e] = (c2 < 0 || comp == 2) ? 0.f : s_row[c2 * kRow + Row::dmean2D + comp];
        }
    }
    const int nv = s_count;
    if (nv > 0) peer_reduce_rows(pa, s_row, s_rowidx, nv, M, row0);
}

// Cross-rank barrier of the shared-model step, one warp: tell every rank `epoch` on channel `base` (0: "my bucket is
// cleared", 16: "my adds have landed" -- stream order puts the reduce kernel in front of it), then wait until every rank
// has said so.  Signal words are peer-mapped (GsGrads.peer_signals); release / acquire at system scope.
__global__ void k_peer_barrier(const GsPeerArgs pa, const int base, const uint32_t epoch) {
    const int tid = threadIdx.x;
    if (tid < pa.world) {
        st_release_sys(pa.sig[tid] + base + pa.rank, epoch);
        while ((int)(ld_acquire_sys(pa.sig[pa.rank] + base + tid) - epoch) < 0) {}
    }
}

__device__ __forceinline__ void peer_reduce_rows(const GsPeerArgs& pa, const float* s_row, const int* s_rowidx, int nv, int M,
                                                 long long row0) {
    const int tid = threadIdx.x;
    const int M3 = M * 3;
    if (M3 == 48 && ((pa.off_sh | pa.off_rot) & 3) == 0) {
        // M = 16: 20 reductions per visible Gaussian -- 3 (mean) + 12 x 128-bit (SH) + 1 (opacity) + 3 (scale)
        // + 1 x 128-bit (rotation)
        for (int e = tid; e < nv * 20; e += kT) {
            const int c2 = e / 20, k = e - c2 * 20;
            const long long gi = row0 + s_rowidx[c2];
            const float* r = s_row + c2 * kRow;
            if (k < 3) peer_add(pa, pa.off_m3 + gi * 3 + k, r[Row::dmean3D + k]);
            else if (k < 15) {
                const int j = k - 3;                     // float4 j of the row's 48 SH gradients
                float o[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int q = 4 * j + u;
                    const int kk = q / 3, ch = q - 3 * kk;
                    o[u] = r[Row::basis + kk] * r[Row::dRGB + ch];
                }
                peer_add4(pa, pa.off_sh + gi * 48 + 4 * j, make_float4(o[0], o[1], o[2], o[3]));
            } else if (k == 15) peer_add(pa, pa.off_op + gi, r[Row::dopacity]);
            else if (k < 19) peer_add(pa, pa.off_sc + gi * 3 + (k - 16), r[Row::dscale + (k - 16)]);
            else peer_add4(pa, pa.off_rot + gi * 4, make_float4(r[Row::drot], r[Row::drot + 1], r[Row::drot + 2], r[Row::drot + 3]));
        }
        return;
    }
    const int per = 3 + M3 + 1 + 3 + 4;                  // floats per Gaussian in the bucket
    for (int e = tid; e < nv * per; e += kT) {
        const int c2 = e / per;
        int k = e - c2 * per;
        const long long gi = row0 + s_rowidx[c2];
        const float* r = s_row + c2 * kRow;
        if (k < 3) { peer_add(pa, pa.off_m3 + gi * 3 + k, r[Row::dmean3D + k]); continue; }
        k -= 3;
        if (k < M3) {
            const int kk = k / 3, ch = k - 3 * kk;
            peer_add(pa, pa.off_sh + gi * M3 + k, kk < 16 ? r[Row::basis + kk] * r[Row::dRGB + ch] : 0.f);
            continue;
        }
        k -= M3;
        if (k < 1) { peer_add(pa, pa.off_op + gi, r[Row::dopacity]); continue; }
        k -= 1;
        if (k < 3) { peer_add(pa, pa.off_sc + gi * 3 + k, r[Row::dscale + k]); continue; }
        k -= 3;
        peer_add(pa, pa.off_rot + gi * 4 + k, r[Row::drot + k]);
    }
}

}  // namespace

static GsPeerArgs peer_args(float* const* peers, int world, float* mc, const long long* seg_off, uint32_t* const* signals,
                            int rank) {
    GsPeerArgs pa;
    for (int r = 0; r < GS_MAX_PEERS; r++) pa.peers[r] = (peers && r < world) ? peers[r] : nullptr;
    for (int r = 0; r < GS_MAX_PEERS; r++) pa.sig[r] = (signals && r < world) ? signals[r] : nullptr;
    pa.rank = rank;
    pa.mc = mc; pa.world = world;
    pa.off_m3 = pa.off_sh = pa.off_op = pa.off_sc = pa.off_rot = 0;
    if (seg_off) { pa.off_m3 = seg_off[0]; pa.off_sh = seg_off[1]; pa.off_op = seg_off[2]; pa.off_sc = seg_off[3]; pa.off_rot = seg_off[4]; }
    return pa;
}
void gs_launch_grad_reduce_peers(int P, int M, const int* radii, const float4* acc, const float* gout, float* dmeans2D,
                                 float* const* peers, int world, float* mc, const long long* seg_off,
                                 cudaStream_t s) {
    const GsPeerArgs pa = peer_args(peers, world, mc, seg_off, nullptr, 0);
    const int grid = (P + kT - 1) / kT;
    k_grad_reduce_peers<<<grid, kT, kT * kRow * sizeof(float), s>>>(P, M, radii, acc, gout, dmeans2D, pa);
}
void gs_launch_peer_barrier(uint32_t* const* signals, int world, int rank, int channel, uint32_t epoch, cudaStream_t s) {
    const GsPeerArgs pa = peer_args(nullptr, world, nullptr, nullptr, signals, rank);
    k_peer_barrier<<<1, 32, 0, s>>>(pa, channel ? 16 : 0, epoch);
}

void gs_launch_grad_vis(const GsView& v, int num_sms, const float* means3D, const float* shs, const float* scales,
                        const float* rotations, const float* cov3D_precomp, const float4* rec, float4* acc,
                        const uint32_t* vis_list, const GsDevStatus* status, float* gout, bool dense_elsewhere,
                        bool scatter, GsGradPtrs g, cudaStream_t s) {
    const int need = (v.P + kVisT - 1) / kVisT;
    const int grid = need < num_sms * 8 ? need : num_sms * 8;
    k_grad_vis<<<grid, kVisT, 0, s>>>(v, means3D, shs, scales, rotations, cov3D_precomp, rec, acc, vis_list, status, gout,
                                      dense_elsewhere, scatter, g);
}
void gs_launch_fill_zero(int P, int num_sms, const GsGradPtrs& g, const GsDevStatus* status, bool dense_elsewhere,
                         cudaStream_t s) {
    FillRuns r;
    r.p[0] = (char*)g.dsh;      r.bytes[0] = (long long)P * 192;
    r.p[1] = (char*)g.dmeans3D; r.bytes[1] = (long long)P * 12;
    r.p[2] = (char*)g.dmeans2D; r.bytes[2] = (long long)P * 12;
    r.p[3] = (char*)g.dscales;  r.bytes[3] = (long long)P * 12;
    r.p[4] = (char*)g.dopacity; r.bytes[4] = (long long)P * 4;
    r.p[5] = (char*)g.drots;    r.bytes[5] = (long long)P * 16;
    k_fill_zero<<<num_sms * 4, 32, 0, s>>>(r, status, P, dense_elsewhere);
}
// the dense-regime twin of (k_grad_vis, k_grad_write): returns at once on the device unless most Gaussians are visible
void gs_launch_grad_dense(const GsView& v, int num_sms, const float* means3D, const float* shs, const float* scales,
                          const float* rotations, const int* radii, float4* acc, const GsDevStatus* status, GsGradPtrs g,
                          cudaStream_t s) {
    const int need = (v.P + kDT - 1) / kDT;
    const int grid = need < num_sms * 3 ? need : num_sms * 3;      // persistent: 3 CTAs (2 x 37 KB stages each) per SM
    k_grad_dense<<<grid, kDT, kDenseSmem, s>>>(v, means3D, shs, scales, rotations, radii, acc, status, g);
}
void gs_grad_write_init() {
    cudaFuncSetAttribute(k_grad_write, cudaFuncAttributeMaxDynamicSharedMemorySize, kT * kRow * (int)sizeof(float));
    cudaFuncSetAttribute(k_grad_reduce_peers, cudaFuncAttributeMaxDynamicSharedMemorySize, kT * kRow * (int)sizeof(float));
    cudaFuncSetAttribute(k_grad_dense, cudaFuncAttributeMaxDynamicSharedMemorySize, kDenseSmem);
}
// tma: k_grad_write_tma (the six tensors of the reference's input mode, 16-byte aligned), else the generic k_grad_write
void gs_launch_grad_write(int P, int M, const int* radii, const float4* acc, const float* gout, GsGradPtrs g,
                          const GsDevStatus* status, bool dense_elsewhere, bool tma, cudaStream_t s) {
    if (tma) {
        const int need = (P + kWT - 1) / kWT;
        k_grad_write_tma<<<need < g_gs_num_sms * 7 * 2 ? need : g_gs_num_sms * 7 * 2, kWT, 0, s>>>(P, radii, acc, gout, g, status, dense_elsewhere);
        return;
    }
    const int grid = (P + kT - 1) / kT;
    k_grad_write<<<grid, kT, kT * kRow * sizeof(float), s>>>(P, M, radii, acc, gout, g, status, dense_elsewhere);
}

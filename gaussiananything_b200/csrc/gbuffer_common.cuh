// Device code shared by the G-buffer kernels (gbuffer_ops.cu, pcd_ops.cu).  Both files are compiled without FMA
// contraction, so every operation below is rounded to fp32 on its own and the two give the same bits.
#pragma once
#include <math.h>

namespace gbuf {

constexpr float XYZ_CLIP = 0.45f;

// RaySampler (include/ga_b200.h Part 7, encoder channels 12-14): the pixel at (u_cam, v_cam) = ((x + 0.5) / W,
// (y + 0.5) / H) is lifted with the skew term, transformed as a point by the whole c2w, the origin is subtracted and
// the direction normalised; p = o + depth * r is clipped to [-0.45, 0.45], then 0 where |p| == 0.45.
// cam: the view's 25 floats (c2w row-major 16 | K 9).
__device__ __forceinline__ void unproject(const float *cam, float u_cam, float v_cam, float depth, float xyz[3])
{
    const float ox = cam[3], oy = cam[7], oz = cam[11];
    const float fx = cam[16], sk = cam[17], cx = cam[18], fy = cam[20], cy = cam[21];
    const float lx = (u_cam - cx + cy * sk / fy - sk * v_cam / fy) / fx, ly = (v_cam - cy) / fy;
    float rx = cam[0] * lx + cam[1] * ly + cam[2] + cam[3] - ox;
    float ry = cam[4] * lx + cam[5] * ly + cam[6] + cam[7] - oy;
    float rz = cam[8] * lx + cam[9] * ly + cam[10] + cam[11] - oz;
    const float rn = fmaxf(sqrtf(rx * rx + ry * ry + rz * rz), 1e-12f);
    rx = rx / rn;
    ry = ry / rn;
    rz = rz / rn;
    const float p[3] = {ox + depth * rx, oy + depth * ry, oz + depth * rz};
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float q = fminf(fmaxf(p[c], -XYZ_CLIP), XYZ_CLIP);
        xyz[c] = fabsf(q) == XYZ_CLIP ? 0.0f : q;
    }
}

}  // namespace gbuf

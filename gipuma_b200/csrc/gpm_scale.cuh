// gpm_scale.cuh — what gpm_api.cu hands to the joint bilateral upsampling of gpm_scale.cu (DESIGN.md §19).
#pragma once
#include <cuda_runtime.h>

namespace gpm {

constexpr int kJbuMaxRadius = 4;
constexpr int kJbuSide = 2 * kJbuMaxRadius + 1;

// One upsampling of a coarse level's raw planes to the fine level of the context that holds the guide image.
struct JbuArgs {
    const float4* coarse;                  // Wc x Hc planes (n.xyz, d), packed
    int Wc, Hc;
    const float* guide;                    // fine reference image as uploaded, replicate-padded by `apron` texels
    int guide_pitch, apron, color;         // pitch in texels; color: texel = float4 (x, y, z compared), else float
    int W, H, radius;
    float kinv[9];                         // fine reference K^-1, row-major
    float depth_min, depth_max;
    float k_range;                         // fp32(1 / sigma_range^2)
    float ws[2 * 2 * kJbuSide * kJbuSide]; // spatial weights [y & 1][x & 1][j + 4][i + 4]
    float4* planes;                        // NULL or W x H
    float* depth;                          // NULL or W x H
};

// Launches the upsampling on `stream` (no synchronisation).
cudaError_t launch_jbu(const JbuArgs& a, cudaStream_t stream);

}  // namespace gpm

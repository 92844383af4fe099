// ex2probe.cu — does MUFU.EX2 return exactly 1.0 for the support weights of gamma = 1e30?  The bit-exact NCC tests
// (tests/test_gpu_ncc.py, DESIGN.md §15) assume w_s = 1 for every |r_s - centre| in 0..255 at that gamma; this checks it with
// setup_window's expression.  Prints one JSON line.
//   nvcc -gencode arch=compute_90a,code=sm_90a --use_fast_math -o ex2probe tools/ex2probe.cu && ./ex2probe
#include <cstdio>
#include <cuda_runtime.h>
#include "../gipuma_b200/csrc/gpm_device.cuh"

__global__ void k_probe(float gamma, int* not_one, float* worst)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;         // |left - centre| = i / 16, 0 .. 255.9375
    if (i >= 256 * 16) return;
    const float nrg = -gpm::frcp(gamma);
    const float w = gpm::fex2(gpm::fmul(gpm::fmul((float)i * 0.0625f, nrg), 1.4426950216293334961f));
    if (w != 1.0f) { atomicAdd(not_one, 1);  *worst = w; }
}

int main()
{
    int* d_n;  float* d_w;
    if (cudaMalloc(&d_n, sizeof(int)) != cudaSuccess || cudaMalloc(&d_w, sizeof(float)) != cudaSuccess) { printf("{\"error\": \"no device\"}\n");  return 1; }
    cudaMemset(d_n, 0, sizeof(int));  cudaMemset(d_w, 0, sizeof(float));
    k_probe<<<16, 256>>>(1e30f, d_n, d_w);
    int n = -1;  float w = 0.f;
    cudaMemcpy(&n, d_n, sizeof(int), cudaMemcpyDeviceToHost);
    cudaMemcpy(&w, d_w, sizeof(float), cudaMemcpyDeviceToHost);
    cudaDeviceProp p;  cudaGetDeviceProperties(&p, 0);
    printf("{\"device\": \"%s\", \"gamma\": 1e30, \"arguments\": 4096, \"not_one\": %d, \"a_value_not_one\": %.9g, \"error\": \"%s\"}\n",
           p.name, n, w, cudaGetErrorString(cudaGetLastError()));
    cudaFree(d_n);  cudaFree(d_w);
    return n == 0 ? 0 : 1;
}

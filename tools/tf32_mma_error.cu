// Error of the tensor-core actor's TF32 accumulation (mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 chains over K/8
// k-tiles, accumulator initialised with an fp32 bias) against the exact sum, on operands shaped like the tests' actors:
// |a| <= 1.5, b ~ N(0, 1.5^2 / K), bias ~ N(0, 0.3^2).  Prints max |error| / (2^-24 S), S = sum |a_k b_k| + |bias|, the
// unit of tests/mlp_helpers.tf32_accumulation_bound.  On one H100 80GB HBM3 (SXM, 400 W): 2.01, 2.93, 3.25 and 4.05
// for K = 8, 16, 32 and 64 (4096 x 128 sums each).
//   nvcc -O2 -gencode arch=compute_90a,code=sm_90a -o /tmp/tf32_mma_error tools/tf32_mma_error.cu && /tmp/tf32_mma_error
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cmath>
#include <cstring>
#include <vector>
#include <random>
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// A: [trials][16][K] row-major, B: [trials][8][K] (n, k), C: [trials][16][8], D out [trials][16][8]
__global__ void probe(const float *A, const float *B, const float *C, float *D, int K) {
    const int tr = blockIdx.x, lane = threadIdx.x, g = lane >> 2, q = lane & 3;
    const float *a = A + (size_t)tr * 16 * K, *b = B + (size_t)tr * 8 * K, *c = C + (size_t)tr * 128;
    float d[4] = {c[g * 8 + 2 * q], c[g * 8 + 2 * q + 1], c[(g + 8) * 8 + 2 * q], c[(g + 8) * 8 + 2 * q + 1]};
    for (int kt = 0; kt < K / 8; ++kt) {
        const int k0 = kt * 8 + q, k1 = k0 + 4;
        uint32_t af[4] = {__float_as_uint(a[g * K + k0]), __float_as_uint(a[(g + 8) * K + k0]),
                          __float_as_uint(a[g * K + k1]), __float_as_uint(a[(g + 8) * K + k1])};
        uint32_t bf[2] = {__float_as_uint(b[g * K + k0]), __float_as_uint(b[g * K + k1])};
        mma_tf32(d, af, bf);
    }
    float *o = D + (size_t)tr * 128;
    o[g * 8 + 2 * q] = d[0]; o[g * 8 + 2 * q + 1] = d[1]; o[(g + 8) * 8 + 2 * q] = d[2]; o[(g + 8) * 8 + 2 * q + 1] = d[3];
}
static float tf32(float x) { uint32_t u; memcpy(&u, &x, 4); u = (u + 0x1000u) & 0xFFFFE000u; float r; memcpy(&r, &u, 4); return r; }
int main() {
    const int trials = 4096;
    std::mt19937 rng(1);
    std::normal_distribution<float> N01(0, 1);
    std::uniform_real_distribution<float> U(-1.5f, 1.5f);
    for (int K : {8, 16, 32, 64}) {
        std::vector<float> A((size_t)trials * 16 * K), B((size_t)trials * 8 * K), C(trials * 128), D(trials * 128);
        for (auto &x : A) x = tf32(U(rng));
        for (auto &x : B) x = tf32(N01(rng) * 1.5f / sqrtf((float)K));
        for (auto &x : C) x = N01(rng) * 0.3f;
        float *dA, *dB, *dC, *dD;
        cudaMalloc(&dA, A.size() * 4); cudaMalloc(&dB, B.size() * 4); cudaMalloc(&dC, C.size() * 4); cudaMalloc(&dD, D.size() * 4);
        cudaMemcpy(dA, A.data(), A.size() * 4, cudaMemcpyHostToDevice); cudaMemcpy(dB, B.data(), B.size() * 4, cudaMemcpyHostToDevice);
        cudaMemcpy(dC, C.data(), C.size() * 4, cudaMemcpyHostToDevice);
        probe<<<trials, 32>>>(dA, dB, dC, dD, K);
        cudaError_t e = cudaMemcpy(D.data(), dD, D.size() * 4, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) { printf("cuda error %s\n", cudaGetErrorString(e)); return 1; }
        double worst = 0, worst_abs = 0, sum = 0; long cnt = 0;
        for (int t = 0; t < trials; ++t) for (int m = 0; m < 16; ++m) for (int n = 0; n < 8; ++n) {
            double ex = C[t * 128 + m * 8 + n], S = fabs(ex);
            for (int k = 0; k < K; ++k) { double p = (double)A[((size_t)t * 16 + m) * K + k] * B[((size_t)t * 8 + n) * K + k]; ex += p; S += fabs(p); }
            double err = fabs((double)D[t * 128 + m * 8 + n] - ex), r = err / (ldexp(1.0, -24) * S);
            worst = r > worst ? r : worst; worst_abs = err > worst_abs ? err : worst_abs; sum += r; ++cnt;
        }
        printf("K=%d: max err/(u S) = %.2f  mean %.3f  max abs err %.3g\n", K, worst, sum / cnt, worst_abs);
        cudaFree(dA); cudaFree(dB); cudaFree(dC); cudaFree(dD);
    }
    return 0;
}

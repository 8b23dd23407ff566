// mpe_gae.cu -- MAPPO's GAE advantages and returns over a finished buffer (GaeArgs in mpe_kernels.cu, mpe_gae in the C
// ABI), compiled as a translation unit of its own so that the build runs it alongside the rest of the library.
#define MPE_KERNEL_TEMPLATES_ONLY
#include "mpe_kernels.cu"

namespace mpe {

constexpr int kGaeChunk = 8;   // steps whose loads are issued before the dependent recurrence runs over them

// Sums (s, s2) over the scan block (kGaeThreads threads) in a fixed order (a shuffle tree per warp, then the warps in
// index order); thread 0 gets the result.
__device__ __forceinline__ double2 gae_block_sum(double s, double s2) {
    __shared__ double2 part[kGaeThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_down_sync(0xffffffffu, s, o);
        s2 += __shfl_down_sync(0xffffffffu, s2, o);
    }
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = make_double2(s, s2);
    __syncthreads();
    double2 r = make_double2(0.0, 0.0);
    if (threadIdx.x == 0)
        for (int w = 0; w < kGaeThreads / 32; ++w) { r.x += part[w].x; r.y += part[w].y; }
    __syncthreads();   // part may be reused by a second call
    return r;
}

// One thread per column c of [T][A][N] (agent c / N, world c % N): a warp reads 128 contiguous bytes per step.  The
// recurrence of mpe_b200.h, in its operation order; NORM also sums every gae (fp64) for the normalisation.
template <bool NORM>
__global__ void __launch_bounds__(kGaeThreads) mpe_gae_kernel(const __grid_constant__ GaeArgs a) {
    const int64_t c = static_cast<int64_t>(blockIdx.x) * kGaeThreads + threadIdx.x, cols = a.cols;
    double s = 0.0, s2 = 0.0;
    if (c < cols) {
        const bool vn = a.value_norm != nullptr;
        float mean = 0.0f, sd = 1.0f;
        if (vn) {
            const int64_t row = (a.flags & kGaePerAgentNorm) ? c / a.n : 0;
            mean = __ldg(a.value_norm + 2 * row);
            sd = __ldg(a.value_norm + 2 * row + 1);
        }
        auto denorm = [&](float v) { return vn ? __fadd_rn(__fmul_rn(v, sd), mean) : v; };
        const float g = a.gamma, gl = __fmul_rn(a.gamma, a.lambda);
        const bool boot = a.flags & kGaeBootstrap;
        float next = 0.0f, gae = 0.0f;
        // one step: dv, delta, gae, ret of mpe_b200.h; next and gae carry to step t - 1
        auto step = [&](float r, float v, float *pr, float *pa) {
            const float dv = denorm(v);
            const float delta = __fsub_rn(__fadd_rn(r, __fmul_rn(g, next)), dv);
            gae = __fadd_rn(delta, __fmul_rn(gl, gae));
            *pr = __fadd_rn(gae, dv);
            *pa = gae;
            next = dv;
            if (NORM) {
                const double d = static_cast<double>(gae);
                s += d;
                s2 += d * d;   // exact: a float's square fits a double's mantissa
            }
        };
        for (int e = a.T / a.L - 1; e >= 0; --e) {
            next = boot ? denorm(__ldg(a.final_val + static_cast<int64_t>(e) * cols + c)) : 0.0f;
            gae = 0.0f;
            int t = e * a.L + a.L - 1;
            const int t0 = e * a.L;
            int64_t off = static_cast<int64_t>(t) * cols + c;
            for (; t - (kGaeChunk - 1) >= t0; t -= kGaeChunk) {
                float r[kGaeChunk], v[kGaeChunk];
#pragma unroll
                for (int k = 0; k < kGaeChunk; ++k) {
                    r[k] = __ldg(a.rew + off - k * cols);
                    v[k] = __ldg(a.val + off - k * cols);
                }
#pragma unroll
                for (int k = 0; k < kGaeChunk; ++k) step(r[k], v[k], a.ret + off - k * cols, a.adv + off - k * cols);
                off -= kGaeChunk * cols;
            }
            for (; t >= t0; --t, off -= cols) step(__ldg(a.rew + off), __ldg(a.val + off), a.ret + off, a.adv + off);
        }
    }
    if (!NORM) return;
    __shared__ bool last;
    const double2 b = gae_block_sum(s, s2);
    if (threadIdx.x == 0) {
        a.partial[2 * blockIdx.x] = b.x;   // two 8-byte stores: see GaeArgs::partial
        a.partial[2 * blockIdx.x + 1] = b.y;
        __threadfence();
        last = atomicAdd(a.ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    // the last block to finish combines every block's partial: thread i sums blocks i, i + 128, ... in order, then
    // gae_block_sum combines the threads in its fixed order
    __threadfence();
    double cs = 0.0, cs2 = 0.0;
    for (unsigned i = threadIdx.x; i < gridDim.x; i += kGaeThreads) {
        cs += __ldcg(a.partial + 2 * i);
        cs2 += __ldcg(a.partial + 2 * i + 1);
    }
    const double2 tot = gae_block_sum(cs, cs2);
    if (threadIdx.x == 0) {
        const double m = static_cast<double>(cols) * a.T;
        const double mu = tot.x / m, var = tot.y / m - mu * mu;
        a.stats[0] = mu;
        a.stats[1] = sqrt(var > 0.0 ? var : 0.0);
    }
}

// advantages[i] = float((double(a) - mean) / (std + 1e-5)) in place, over all T * A * N entries (grid-stride)
__global__ void __launch_bounds__(kGaeNormThreads) mpe_gae_normalize_kernel(const __grid_constant__ GaeArgs a) {
    const double mu = __ldcg(a.stats), den = __dadd_rn(__ldcg(a.stats + 1), 1e-5);
    const int64_t total = a.cols * a.T, stride = static_cast<int64_t>(gridDim.x) * kGaeNormThreads;
    constexpr int U = 4;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * kGaeNormThreads + threadIdx.x; i < total; i += U * stride) {
        float x[U];
#pragma unroll
        for (int k = 0; k < U; ++k)
            if (i + k * stride < total) x[k] = a.adv[i + k * stride];
#pragma unroll
        for (int k = 0; k < U; ++k)
            if (i + k * stride < total)
                a.adv[i + k * stride] = __double2float_rn(__ddiv_rn(__dsub_rn(static_cast<double>(x[k]), mu), den));
    }
}

const void *gae_kernel(int which) {
    return which == 0 ? reinterpret_cast<const void *>(mpe_gae_kernel<false>)
         : which == 1 ? reinterpret_cast<const void *>(mpe_gae_kernel<true>)
                      : reinterpret_cast<const void *>(mpe_gae_normalize_kernel);
}

}  // namespace mpe

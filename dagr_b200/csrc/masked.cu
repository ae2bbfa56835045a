// masked.cu -- index-masked row kernels of the asynchronous engine (replaces asy_tools,
// src/dagr/asynchronous/asy_tools/main.cu:14-188), sm_90a.  One warp per selected row, lanes over
// channels, accumulation in registers (the reference accumulates through global memory, :151-157).  Every entry point
// checks its arguments before it launches anything (DAGR_E_ARG and a message naming the function).
#include "common.cuh"

__global__ void k_masked_lin(const int64_t *__restrict__ idx, int64_t K, const float *__restrict__ x_in,
                             float *__restrict__ x_out, const float *__restrict__ weight, const float *__restrict__ bias,
                             int Cin, int Cout, int add)
{
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= K) return;
    const int64_t r = idx[i];
    const float *xi = x_in + r * Cin;
    for (int co = lane; co < Cout; co += 32) {
        float acc = add ? x_out[r * Cout + co] : 0.f;
        const float *w = weight + (int64_t)co * Cin;
        for (int ci = 0; ci < Cin; ci++) acc = fmaf(xi[ci], w[ci], acc);   // same order as main.cu:154-156 (nvcc contracts it to FFMA there too)
        if (bias) acc = __fadd_rn(acc, bias[co]);
        x_out[r * Cout + co] = acc;
    }
}

extern "C" int dagr_masked_lin(const int64_t *idx, int64_t K, const float *x_in, float *x_out, const float *weight,
                               const float *bias, int Cin, int Cout, int add, void *stream)
{
    DAGR_CHECK_ARG(K >= 0, "K < 0");
    DAGR_CHECK_ARG(Cin >= 1 && Cout >= 1, "Cin and Cout must be >= 1");
    DAGR_CHECK_ARG(K == 0 || (idx && x_in && x_out && weight), "null pointer (only bias may be NULL)");
    if (K == 0) return DAGR_OK;
    k_masked_lin<<<dagr_div_up(K, 4), 128, 0, (cudaStream_t)stream>>>(idx, K, x_in, x_out, weight, bias, Cin, Cout, add);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

__global__ void k_masked_bn(const int64_t *__restrict__ idx, int64_t K, const float *__restrict__ x, float *__restrict__ x_out,
                            const float *__restrict__ mean, const float *__restrict__ var, const float *__restrict__ weight,
                            const float *__restrict__ bias, int C, float eps)
{
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= K * C) return;
    const int64_t i = t / C;
    const int c = (int)(t % C);
    const int64_t o = idx[i] * C + c;
    // (x - mean) / sqrt(var + eps) * weight + bias   (main.cu:66).  nvcc contracts the reference's `* weight + bias` to one
    // fma.rn, so the last step is an FMA too: a separate multiply and add would differ by an ulp, which the cancellation in
    // d * weight + bias near zero turns into a large relative error.
    const float d = __fdiv_rn(__fsub_rn(x[o], mean[c]), __fsqrt_rn(__fadd_rn(var[c], eps)));
    x_out[o] = __fmaf_rn(d, weight[c], bias[c]);
}

extern "C" int dagr_masked_inplace_bn(const int64_t *idx, int64_t K, const float *x, float *x_out, const float *mean,
                                      const float *var, const float *weight, const float *bias, int C, float eps,
                                      void *stream)
{
    DAGR_CHECK_ARG(K >= 0, "K < 0");
    DAGR_CHECK_ARG(C >= 1, "C must be >= 1");
    DAGR_CHECK_ARG(K == 0 || (idx && x && x_out && mean && var && weight && bias), "null pointer");
    if (K == 0) return DAGR_OK;
    k_masked_bn<<<dagr_div_up(K * C, 256), 256, 0, (cudaStream_t)stream>>>(idx, K, x, x_out, mean, var, weight, bias, C, eps);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

__global__ void k_masked_isdiff(int64_t *__restrict__ idx, int64_t K, const float *__restrict__ a, const float *__restrict__ b,
                                int C, float atol, float rtol)
{
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= K) return;
    const int64_t r = idx[i];
    bool diff = false;
    for (int c = lane; c < C; c += 32) {
        const float in = a[r * C + c], ot = b[r * C + c];
        // signed rtol * other (main.cu:36), where nvcc contracts `atol + rtol * other` to one fma.rn; written as the FMA
        // here so the decision does not depend on the build's contraction setting
        diff |= fabsf(__fsub_rn(in, ot)) > __fmaf_rn(rtol, ot, atol);
    }
    diff = __any_sync(0xffffffffu, diff);
    if (lane == 0 && !diff) idx[i] = -1;
}

extern "C" int dagr_masked_isdiff(int64_t *idx_inout, int64_t K, const float *a, const float *b, int C, float atol,
                                  float rtol, void *stream)
{
    DAGR_CHECK_ARG(K >= 0, "K < 0");
    DAGR_CHECK_ARG(C >= 1, "C must be >= 1");
    DAGR_CHECK_ARG(K == 0 || (idx_inout && a && b), "null pointer");
    if (K == 0) return DAGR_OK;
    k_masked_isdiff<<<dagr_div_up(K, 4), 128, 0, (cudaStream_t)stream>>>(idx_inout, K, a, b, C, atol, rtol);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// parallel-cnn_b200/csrc/norm_act.cuh -- the per-element device helpers batch normalization (batchnorm_nhwc.cu) and group
// normalization (groupnorm_nhwc.cu) share: the 16-byte bf16 vectors, xhat, the fused activations and their gradients.  Both
// normalizations state the same per-element rules in include/pcnn.h, so they run the same code.  Included inside each file's
// anonymous namespace.
#pragma once

// pixels a thread loads before it uses any: 2 x 16 bytes per operand on the 8-channel path, 4 elements on the scalar one
template <int VEC>
__host__ __device__ constexpr int bn_unroll() { return VEC == 8 ? 2 : 4; }

template <int VEC>
struct alignas(2 * VEC) BfVec {
    __nv_bfloat16 h[VEC];
};

template <int VEC>
__device__ __forceinline__ BfVec<VEC> ld(const __nv_bfloat16 *p) {
    return *reinterpret_cast<const BfVec<VEC> *>(p);
}
template <int VEC>
__device__ __forceinline__ void st(__nv_bfloat16 *p, const BfVec<VEC> &v) {
    *reinterpret_cast<BfVec<VEC> *>(p) = v;
}

// xhat = (float(x) - mean) * rstd, fp32, no contraction (the forward's and both backward passes')
__device__ __forceinline__ float bn_xhat(__nv_bfloat16 x, float mean, float rstd) {
    return __fmul_rn(__fsub_rn(__bfloat162float(x), mean), rstd);
}

// g~ = bf16_rn(act'(t)) with t = float(dy) (+ float(dy2)): without dy2 dy's bits pass; at act 3 y <= 0 gives +0 (a NaN y passes)
template <int ACT>
__device__ __forceinline__ __nv_bfloat16 bn_dgrad(__nv_bfloat16 dy, __nv_bfloat16 dy2, bool has_dy2, __nv_bfloat16 y) {
    __nv_bfloat16 g = has_dy2 ? __float2bfloat16_rn(__fadd_rn(__bfloat162float(dy), __bfloat162float(dy2))) : dy;
    if (ACT == PCNN_ACT_RELU && __bfloat162float(y) <= 0.0f) g = __ushort_as_bfloat16((unsigned short)0);
    return g;
}

// codes 4-6 take their backward from the recomputed fp32 pre-activation v rather than from y
template <int ACT>
__host__ __device__ constexpr bool bn_preact() { return ACT == PCNN_ACT_SILU || ACT == PCNN_ACT_HARDSWISH || ACT == PCNN_ACT_RELU6; }

// the pre-activation v = RN(RN(xhat * gamma) + beta) (+ float(r)), as the forward forms it
__device__ __forceinline__ float bn_pre(float xh, float ga, float be, const __nv_bfloat16 *r, __nv_bfloat16 rv) {
    const float v = __fadd_rn(__fmul_rn(xh, ga), be);
    return r ? __fadd_rn(v, __bfloat162float(rv)) : v;
}

// act(v) in fp32 before the one bf16 rounding (pcnn.h states each in its order).  Every "/" is __fdiv_rn, the IEEE quotient: ptxas
// shows a 0-byte stack and no spills in every instantiation with it, and a divisor of +Inf gives +-0 for a finite dividend.
template <int ACT>
__device__ __forceinline__ float bn_act_f32(float v) {
    if (ACT == PCNN_ACT_RELU) return pcnn_tc::relu_f32(v);
    if (ACT == PCNN_ACT_SILU) return __fdiv_rn(v, __fadd_rn(1.0f, exp_f32(-v)));
    if (ACT == PCNN_ACT_HARDSWISH) {
        float u = __fadd_rn(v, 3.0f);
        u = u < 0.0f ? 0.0f : u;
        u = u > 6.0f ? 6.0f : u;                                        // NaN passes both
        return __fdiv_rn(__fmul_rn(v, u), 6.0f);
    }
    if (ACT == PCNN_ACT_RELU6) {
        const float u = v < 0.0f ? 0.0f : v;                            // NaN and -0 pass
        return u > 6.0f ? 6.0f : u;
    }
    return v;
}

// g = bf16_rn(act'(t)) at the pre-activation v, t = float(dy) or RN(float(dy) + float(dy2)): a multiplied derivative gives
// bf16_rn(RN(t * d)); a passed t gives bf16_rn(t) (dy's bits without dy2); a cut one +0
template <int ACT>
__device__ __forceinline__ __nv_bfloat16 bn_dgrad_pre(__nv_bfloat16 dy, __nv_bfloat16 dy2, bool has_dy2, float v) {
    const float t = has_dy2 ? __fadd_rn(__bfloat162float(dy), __bfloat162float(dy2)) : __bfloat162float(dy);
    const __nv_bfloat16 pass = has_dy2 ? __float2bfloat16_rn(t) : dy, zero = __ushort_as_bfloat16((unsigned short)0);
    if (ACT == PCNN_ACT_RELU6) return v > 0.0f && v < 6.0f ? pass : zero;                       // NaN gives +0
    if (ACT == PCNN_ACT_HARDSWISH) {
        if (v <= -3.0f) return zero;
        if (v >= 3.0f) return pass;
        return __float2bfloat16_rn(__fmul_rn(t, __fadd_rn(__fdiv_rn(v, 3.0f), 0.5f)));  // NaN gives NaN
    }
    // SiLU: s = RN(1 / RN(1 + E(-v))), d = RN(s * RN(1 + RN(v * RN(1 - s))))
    const float s = __fdiv_rn(1.0f, __fadd_rn(1.0f, exp_f32(-v)));
    const float d = __fmul_rn(s, __fadd_rn(1.0f, __fmul_rn(v, __fsub_rn(1.0f, s))));
    return __float2bfloat16_rn(__fmul_rn(t, d));
}

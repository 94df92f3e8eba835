// The LSTM cell (gate order i, f, g, o like ATen): the activation policies of every LSTM kernel, and the cell of one
// hidden unit used by the per-step and persistent wgmma kernels.  Callers load, sum and store in their own layouts and
// pass the summed pre-activations (forward) or the saved activations (backward) in.
#pragma once
#include <cuda_bf16.h>
#include <math.h>

namespace {

// Activation policies.  Accurate: tanhf / expf, so that the fp32 parity path stays within 1e-4 of the reference.
// Fast: MUFU.TANH, one instruction, ~2^-11 relative error -- far below bf16 resolution of the stored activations.
struct CellAccurate {
    static __device__ __forceinline__ float th(float x) { return tanhf(x); }
    static __device__ __forceinline__ float sg(float x) { return 1.f / (1.f + expf(-x)); }
};
struct CellFast {
    static __device__ __forceinline__ float th(float x) { float y; asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
    static __device__ __forceinline__ float sg(float x) { return fmaf(0.5f, th(0.5f * x), 0.5f); }
};
// by storage type: fp32 is the parity path, bf16 the fast one
template <typename T> struct CellMath;
template <> struct CellMath<float> : CellAccurate {};
template <> struct CellMath<__nv_bfloat16> : CellFast {};

struct LstmUnit { float i, f, g, o, c, h; };   // activated gates, c_t, h_t
template <typename Act>
__device__ __forceinline__ LstmUnit lstm_unit_fwd(float pi, float pf, float pg, float po, float c_prev) {
    LstmUnit u;
    u.i = Act::sg(pi);
    u.f = Act::sg(pf);
    u.g = Act::th(pg);
    u.o = Act::sg(po);
    u.c = __fmaf_rn(u.i, u.g, u.f * c_prev);        // the rounding of c_t is fixed: i * g fused, f * c_prev rounded
    u.h = u.o * Act::th(u.c);
    return u;
}

struct LstmUnitGrad { float di, df, dg, do_, dc_prev; };   // pre-activation gate gradients, dc_{t-1}
// i, f, g, o: activated gates of step t; c: c_t; dh: dL/dh_t; dc: dL/dc_t from step t + 1
template <typename Act>
__device__ __forceinline__ LstmUnitGrad lstm_unit_bwd(float i, float f, float g, float o, float c, float c_prev, float dh,
                                                      float dc) {
    const float tc = Act::th(c);
    const float dct = dc + dh * o * (1.f - tc * tc);
    LstmUnitGrad r;
    r.di = dct * g * i * (1.f - i);
    r.df = dct * c_prev * f * (1.f - f);
    r.dg = dct * i * (1.f - g * g);
    r.do_ = dh * tc * o * (1.f - o);
    r.dc_prev = dct * f;
    return r;
}

}  // namespace

// common.cuh -- shared helpers for libstereo_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/stereo_b200.h"

extern unsigned long long g_sb_launches;  // defined in misc.cu

#define SB_LAUNCHED() (++g_sb_launches)

#define SB_CHECK_LAUNCH()                              \
    do {                                               \
        cudaError_t e__ = cudaGetLastError();          \
        if (e__ != cudaSuccess) return (int)e__;       \
    } while (0)

static inline cudaStream_t sb_cs(sb_stream_t s) { return (cudaStream_t)s; }

static inline int sb_div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// Per-device caches (function attributes and device properties belong to one device context; a process may drive
// several GPUs).  Races between host threads are benign: every writer stores the same value.
constexpr int kSbMaxDevices = 64;
static inline int sb_cur_device() {
    int d = 0;
    cudaGetDevice(&d);
    return (d < 0 || d >= kSbMaxDevices) ? 0 : d;
}
static inline int sb_num_sms() {
    static int sms[kSbMaxDevices] = {0};
    const int d = sb_cur_device();
    if (!sms[d]) {
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d);
        sms[d] = n > 0 ? n : 132;
    }
    return sms[d];
}

// Deterministic expf, bit-identical to oracle/csrc/oracle_ops.c:sb_expf (every step is a
// single IEEE operation: rintf, fmaf, integer scale).  Replaces torch.exp of
// lib/model/rpn/bbox_transform.py:93-94 so that decoded boxes -- and therefore NMS keep
// masks and proposal indices -- can be compared bit-exactly between CPU oracle and GPU.
__device__ __forceinline__ float sb_expf(float x) {
    if (x > 88.72283f) return __int_as_float(0x7f800000);
    if (x < -103.9f) return 0.0f;
    const float log2e = 1.44269504088896341f;
    const float ln2_hi = 0.693145751953125f;
    const float ln2_lo = 1.42860682030941723212e-6f;
    float n = rintf(__fmul_rn(x, log2e));
    float r = __fmaf_rn(n, -ln2_hi, x);
    r = __fmaf_rn(n, -ln2_lo, r);
    float p = 1.0f / 5040.0f;
    p = __fmaf_rn(p, r, 1.0f / 720.0f);
    p = __fmaf_rn(p, r, 1.0f / 120.0f);
    p = __fmaf_rn(p, r, 1.0f / 24.0f);
    p = __fmaf_rn(p, r, 1.0f / 6.0f);
    p = __fmaf_rn(p, r, 0.5f);
    p = __fmaf_rn(p, r, 1.0f);
    p = __fmaf_rn(p, r, 1.0f);
    int ni = (int)n;
    int n1 = ni / 2, n2 = ni - n1;
    float s1 = __int_as_float((n1 + 127) << 23);
    float s2 = __int_as_float((n2 + 127) << 23);
    return __fmul_rn(__fmul_rn(p, s1), s2);
}

// bbox_transform_inv + clip_boxes for one box (bbox_transform.py:79-104,177-185);
// explicit _rn intrinsics: no FMA contraction, one rounding per reference op.
__device__ __forceinline__ float4 sb_decode_clip(float4 b, float dx, float dy, float dw, float dh,
                                                 float xmax, float ymax) {
    float w = __fadd_rn(__fsub_rn(b.z, b.x), 1.0f);
    float h = __fadd_rn(__fsub_rn(b.w, b.y), 1.0f);
    float cx = __fadd_rn(b.x, __fmul_rn(0.5f, w));
    float cy = __fadd_rn(b.y, __fmul_rn(0.5f, h));
    float pcx = __fadd_rn(__fmul_rn(dx, w), cx);
    float pcy = __fadd_rn(__fmul_rn(dy, h), cy);
    float pw = __fmul_rn(sb_expf(dw), w);
    float ph = __fmul_rn(sb_expf(dh), h);
    float4 o;
    o.x = __fsub_rn(pcx, __fmul_rn(0.5f, pw));
    o.y = __fsub_rn(pcy, __fmul_rn(0.5f, ph));
    o.z = __fadd_rn(pcx, __fmul_rn(0.5f, pw));
    o.w = __fadd_rn(pcy, __fmul_rn(0.5f, ph));
    o.x = fminf(fmaxf(o.x, 0.f), xmax);
    o.y = fminf(fmaxf(o.y, 0.f), ymax);
    o.z = fminf(fmaxf(o.z, 0.f), xmax);
    o.w = fminf(fmaxf(o.w, 0.f), ymax);
    return o;
}

// devIoU (nms_cuda_kernel.cu:31-39), no contraction
__device__ __forceinline__ float sb_iou(const float4 a, const float4 b) {
    float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
    float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
    float width = fmaxf(__fadd_rn(__fsub_rn(right, left), 1.0f), 0.f);
    float height = fmaxf(__fadd_rn(__fsub_rn(bottom, top), 1.0f), 0.f);
    float interS = __fmul_rn(width, height);
    float Sa = __fmul_rn(__fadd_rn(__fsub_rn(a.z, a.x), 1.0f), __fadd_rn(__fsub_rn(a.w, a.y), 1.0f));
    float Sb = __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.0f), __fadd_rn(__fsub_rn(b.w, b.y), 1.0f));
    return __fdiv_rn(interS, __fsub_rn(__fadd_rn(Sa, Sb), interS));
}

// Sort key of a score: a larger key ranks first, in torch.sort(descending=True)'s order -- every NaN (either sign)
// maps to the one key just above +inf, and -0.0 to the key of +0.0.  Equal keys are ties, which callers break by
// ascending index.
__device__ __forceinline__ unsigned int sb_score_key(float s) {
    if (isnan(s)) return 0xff800001u;
    const unsigned int b = __float_as_uint(s) == 0x80000000u ? 0u : __float_as_uint(s);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// TF32 operand hygiene helpers (see sb_conv_desc.out_mode in the header)
__device__ __forceinline__ float sb_round_tf32(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
__device__ __forceinline__ float sb_bias_tf32(float x) { return __uint_as_float(__float_as_uint(x) + 0x1000u); }
__device__ __forceinline__ float sb_unbias_tf32(float x) { return __uint_as_float(__float_as_uint(x) - 0x1000u); }
__device__ __forceinline__ float sb_store_mode(float x, int mode) {
    return mode == 1 ? sb_round_tf32(x) : (mode == 2 ? sb_bias_tf32(x) : x);
}

// sb_iou(a,b) > thresh, bit-identical in outcome, without the IEEE division for the common cases:
// disjoint boxes have IoU == +0 (never > a non-negative thresh), and when inter and thresh*union differ by
// more than 1e-4 relative the rounded quotient cannot land on the other side of thresh.
__device__ __forceinline__ bool sb_iou_gt(const float4 a, const float4 b, float thresh) {
    float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
    float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
    float width = fmaxf(__fadd_rn(__fsub_rn(right, left), 1.0f), 0.f);
    float height = fmaxf(__fadd_rn(__fsub_rn(bottom, top), 1.0f), 0.f);
    float interS = __fmul_rn(width, height);
    if (interS == 0.f && thresh >= 0.f) return false;
    float Sa = __fmul_rn(__fadd_rn(__fsub_rn(a.z, a.x), 1.0f), __fadd_rn(__fsub_rn(a.w, a.y), 1.0f));
    float Sb = __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.0f), __fadd_rn(__fsub_rn(b.w, b.y), 1.0f));
    float uni = __fsub_rn(__fadd_rn(Sa, Sb), interS);
    float t = thresh * uni;
    if (uni > 0.f && thresh > 0.f && isfinite(t)) {
        if (interS > t * 1.0001f) return true;
        if (interS < t * 0.9999f) return false;
    }
    return __fdiv_rn(interS, uni) > thresh;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// dense_align.cu -- photometric 3D-box depth refinement in two launches (sm_90a).
//
// Replaces lib/model/dense_align/dense_align.py:13-69,175-300 + box_3d.py:12-106
// (align_parallel -> sample()/Box3d -> enumeration_depth x2).  The reference runs a Python
// loop over RoIs with ~150 tiny kernels and host scalar reads each, builds a 38 MB uv grid,
// then ~10 full passes over [50 x D x P x 3] intermediates per stage (3.7 GB each at D=2048).
//
// Here (round 2), for up to kStripMaxD = 48 RoIs (what a KITTI frame has): the 2x-upsampled pair is NOT materialised
// (round 1 wrote 2 x 76 MB of it per call); beyond that -- the D = 128 ... 2048 sweep -- it is, see further down.
//   K1/K2 dense_stage_kernel<0|1>: grid (RoI, row slice).  Thread 0 builds the 3D box (corners, the three visible
//      planes by the nearest-vertex rule).  The CTA then walks its lattice rows; per row
//        (a) one thread per lattice pixel runs the ray / plane / in-box test and samples the LEFT image -- each tap
//            of F.grid_sample is a pixel of the 2x image, recomputed from <= 4 source pixels with the exact
//            arithmetic of F.upsample(align_corners=True);
//        (b) the span of RIGHT-image columns that the row's hypotheses can reach is reduced over the row, and the
//            CTA builds that strip of the 2x image (one or two rows of it) ONCE in shared memory -- SURVEY 8(d)'s
//            compulsory traffic: R_rows * (W_span + D_span) pixels per RoI instead of 70 * P gathers;
//        (c) thread (pixel, hypothesis group) evaluates d = fb / (depth + dz), the bilinear taps out of the strip
//            (taps outside the strip are recomputed from the source) and keeps the SAD of its 13 / 25 hypotheses in
//            registers across rows.  Taps outside the strip are not rare: the coarse depths of a car nearer than
//            ~12.5 m are clamped to 1.5 m, so some hypotheses have zf + rdis <= 0, d flips sign through the pole and
//            h = 0 / NH-1 no longer bound the row's reach.  On the 24-RoI golden at 600x1987 (tests/golden/
//            dense_align.npz), 72 of 691 coarse lattice rows reach over more than kStripMax columns and 33 528 of
//            2.2 M coarse taps (1.5 %) take the fallback; the fine stage took none there;
//      then a warp-shuffle + shared-memory reduction to one partial row per CTA.  The fine stage re-derives the
//      coarse argmin from the partial rows (fixed slice order).
//   K3 dense_final_kernel: per-RoI argmins, outputs, and the reference's "no valid pixel anywhere ->
//      return dis_init" early-out.
// Strip path: only the source pair (28.6 MB, L2-resident), a few KB of partial sums and D x 2 outputs touch HBM.
//
// Arithmetic mirrors oracle/csrc/oracle_ops.c (which is pinned to the reference's Python):
// every fp32 step is an explicit _rn intrinsic in the reference's evaluation order.
#include "common.cuh"

namespace {

// One pixel (y, x) of F.upsample(im, scale 2, bilinear, align_corners=True) of a planar [3,H,W] image, with the
// arithmetic of the reference's materialised tensor (dense_align.py:255-257): same ratios, same operation order.
struct UpGeom { float rh, rw; int H, W; };
__device__ __forceinline__ float4 up_pixel(const float* __restrict__ src, const UpGeom& ug, int y, int x) {
    const float sy = __fmul_rn(ug.rh, (float)y);
    const int y1 = (int)sy;
    const int yp = (y1 < ug.H - 1) ? 1 : 0;
    const float ly1 = __fsub_rn(sy, (float)y1), ly0 = __fsub_rn(1.f, ly1);
    const float sx = __fmul_rn(ug.rw, (float)x);
    const int x1 = (int)sx;
    const int xp = (x1 < ug.W - 1) ? 1 : 0;
    const float lx1 = __fsub_rn(sx, (float)x1), lx0 = __fsub_rn(1.f, lx1);
    float o[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float* r0 = src + ((size_t)c * ug.H + y1) * ug.W;
        const float* r1 = r0 + (size_t)yp * ug.W;
        const float top = __fadd_rn(__fmul_rn(lx0, __ldg(r0 + x1)), __fmul_rn(lx1, __ldg(r0 + x1 + xp)));
        const float bot = __fadd_rn(__fmul_rn(lx0, __ldg(r1 + x1)), __fmul_rn(lx1, __ldg(r1 + x1 + xp)));
        o[c] = __fadd_rn(__fmul_rn(ly0, top), __fmul_rn(ly1, bot));
    }
    return make_float4(o[0], o[1], o[2], 0.f);
}

struct Consts {
    float s2f, f32, bl32, fb32, cx32, cy32, fw2, fh2;
    int FH, FW;
    UpGeom ug;
};

// dense_align_impl's calibration constants, formed on the device from 24 doubles in device memory (P2 then P3,
// row-major): calib4 = [p2[0], p2[2], p2[6], p2[3] - p3[3]] and then the host's fp64 operations in the host's order,
// each rounded explicitly so that nothing is contracted -- the same values the host puts in a launch's Consts.
__device__ __forceinline__ void calib_consts(Consts* k, const double* __restrict__ calib, double scale) {
    const double c0 = calib[0], c1 = calib[2], c2 = calib[6], c3 = __dsub_rn(calib[3], calib[15]);
    const double s2 = __dmul_rn(scale, 2.0);
    const double fd = __dmul_rn(c0, s2);
    const double bld = __ddiv_rn(__dmul_rn(c3, s2), fd);
    k->s2f = __double2float_rn(s2);
    k->f32 = __double2float_rn(fd);
    k->bl32 = __double2float_rn(bld);
    k->fb32 = __double2float_rn(__dmul_rn(fd, bld));
    k->cx32 = __double2float_rn(__dmul_rn(c1, s2));
    k->cy32 = __double2float_rn(__dmul_rn(c2, s2));
}

struct RoiCtx {
    float T[3];
    float c, s;
    float pmin[3], pmax[3];
    float planes[3][4];
    int u0, nu, su, v0, nv, sv;
    float z0, dis_init;
};

__device__ __forceinline__ void make_plane(const float* p1, const float* p2, const float* p3, float* pl) {
    float a1[3], a2[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { a1[k] = __fsub_rn(p2[k], p1[k]); a2[k] = __fsub_rn(p3[k], p1[k]); }
    float n0 = __fsub_rn(__fmul_rn(a1[1], a2[2]), __fmul_rn(a1[2], a2[1]));
    float n1 = __fsub_rn(__fmul_rn(a1[2], a2[0]), __fmul_rn(a1[0], a2[2]));
    float n2 = __fsub_rn(__fmul_rn(a1[0], a2[1]), __fmul_rn(a1[1], a2[0]));
    pl[0] = n0; pl[1] = n1; pl[2] = n2;
    pl[3] = __fsub_rn(__fsub_rn(__fmul_rn(-n0, p1[0]), __fmul_rn(n1, p1[1])), __fmul_rn(n2, p1[2]));
}

__device__ __forceinline__ int py_slice(int start, int stop, int step, int size, int* first) {
    if (start < 0) { start += size; if (start < 0) start = 0; }
    if (start > size) start = size;
    if (stop < 0) { stop += size; if (stop < 0) stop = 0; }
    if (stop > size) stop = size;
    *first = start;
    if (stop <= start) return 0;
    return (stop - start + step - 1) / step;
}

__device__ void setup_roi(const float* box_in, const float* kp, const float* pose, const Consts& k, RoiCtx* g) {
    const int PV[6][3] = {{0, 3, 4}, {2, 3, 6}, {1, 2, 5}, {0, 1, 4}, {0, 1, 2}, {4, 5, 6}};
    const int PG[8][3] = {{0, 3, 4}, {2, 3, 4}, {1, 2, 4}, {0, 1, 4}, {0, 3, 5}, {2, 3, 5}, {1, 2, 5}, {0, 1, 5}};
    float box[4], border[2];
#pragma unroll
    for (int i = 0; i < 4; ++i) box[i] = __fmul_rn(box_in[i], k.s2f);
    border[0] = __fmul_rn(kp[3], k.s2f);
    border[1] = __fmul_rn(kp[4], k.s2f);
    g->T[0] = pose[0]; g->T[1] = pose[1]; g->T[2] = pose[2];
    const float w = pose[3], h = pose[4], l = pose[5];
    g->c = (float)cos((double)pose[6]);
    g->s = (float)sin((double)pose[6]);
    const float hw = __fdiv_rn(w, 2.0f), hl = __fdiv_rn(l, 2.0f);
    float Po[8][3] = {{-hw, 0.f, -hl}, {-hw, 0.f, hl}, {hw, 0.f, hl}, {hw, 0.f, -hl},
                      {-hw, -h, -hl},  {-hw, -h, hl},  {hw, -h, hl},  {hw, -h, -hl}};
    float Pc[8][3];
    int nearest = 0;
    float best = 100000000.f;
    for (int i = 0; i < 8; ++i) {
        Pc[i][0] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(g->c, Po[i][0]), __fmul_rn(0.f, Po[i][1])), __fmul_rn(g->s, Po[i][2])), g->T[0]);
        Pc[i][1] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(0.f, Po[i][0]), __fmul_rn(1.f, Po[i][1])), __fmul_rn(0.f, Po[i][2])), g->T[1]);
        Pc[i][2] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(-g->s, Po[i][0]), __fmul_rn(0.f, Po[i][1])), __fmul_rn(g->c, Po[i][2])), g->T[2]);
        float nn = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(Pc[i][0], Pc[i][0]), __fmul_rn(Pc[i][1], Pc[i][1])), __fmul_rn(Pc[i][2], Pc[i][2])));
        if (nn < best) { best = nn; nearest = i; }
    }
    for (int q = 0; q < 3; ++q) {
        const int* v = PV[PG[nearest][q]];
        make_plane(Pc[v[0]], Pc[v[1]], Pc[v[2]], g->planes[q]);
    }
    g->pmin[0] = __fsub_rn(-hw, 0.01f); g->pmin[1] = __fsub_rn(-h, 0.01f); g->pmin[2] = __fsub_rn(-hl, 0.01f);
    g->pmax[0] = __fadd_rn(hw, 0.01f);  g->pmax[1] = __fadd_rn(0.f, 0.01f); g->pmax[2] = __fadd_rn(hl, 0.01f);
    int su = (int)__fdiv_rn(__fsub_rn(border[1], border[0]), 56.0f); if (su < 1) su = 1;
    int sv = (int)__fdiv_rn(__fsub_rn(box[3], box[1]), 56.0f);       if (sv < 1) sv = 1;
    int vs = (int)__fadd_rn(__fdiv_rn(__fadd_rn(box[1], box[3]), 2.0f), 0.5f);
    int ve = (int)__fadd_rn(__fsub_rn(box[3], __fmul_rn(__fsub_rn(box[3], box[1]), 0.1f)), 0.5f);
    int us = (int)__fadd_rn(border[0], 0.5f);
    int ue = (int)__fadd_rn(border[1], 0.5f);
    g->su = su; g->sv = sv;
    g->nv = py_slice(vs, ve, sv, k.FH, &g->v0);
    g->nu = py_slice(us, ue, su, k.FW, &g->u0);
    g->dis_init = __fdiv_rn(k.fb32, pose[2]);
    g->z0 = __fmul_rn(__fmul_rn(__fdiv_rn(1.0f, g->dis_init), k.f32), k.bl32);
}

__device__ __forceinline__ bool ray_test(const RoiCtx& g, float u, float v, const Consts& k, float* dz) {
    const float rx = __fdiv_rn(__fsub_rn(u, k.cx32), k.f32), ry = __fdiv_rn(__fsub_rn(v, k.cy32), k.f32);
    float oz = 0.f;
    bool m = false;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        if (m) break;
        const float* pl = g.planes[q];
        float t = __fadd_rn(__fadd_rn(__fmul_rn(rx, pl[0]), __fmul_rn(ry, pl[1])), __fmul_rn(1.0f, pl[2]));
        t = __fmul_rn(-__fdiv_rn(1.0f, t), pl[3]);
        const float ix = __fsub_rn(__fmul_rn(rx, t), g.T[0]);
        const float iy = __fsub_rn(__fmul_rn(ry, t), g.T[1]);
        const float iz = __fsub_rn(__fmul_rn(1.0f, t), g.T[2]);
        const float bx = __fadd_rn(__fadd_rn(__fmul_rn(g.c, ix), __fmul_rn(0.f, iy)), __fmul_rn(-g.s, iz));
        const float by = __fadd_rn(__fadd_rn(__fmul_rn(0.f, ix), __fmul_rn(1.f, iy)), __fmul_rn(0.f, iz));
        const float bz = __fadd_rn(__fadd_rn(__fmul_rn(g.s, ix), __fmul_rn(0.f, iy)), __fmul_rn(g.c, iz));
        m = (bx >= g.pmin[0]) && (by >= g.pmin[1]) && (bz >= g.pmin[2]) &&
            (bx <= g.pmax[0]) && (by <= g.pmax[1]) && (bz <= g.pmax[2]);
        oz = iz;
    }
    *dz = oz;
    return m;
}

// F.grid_sample(bilinear, border, align_corners=True): coordinates and weights of one sample
struct Samp {
    int xi0, yi0;
    bool okx, row1;          // tap columns / rows that exist and carry weight
    float nw, ne, sw, se;
};
__device__ __forceinline__ void samp_x(Samp& s, float gx, int W) {
    float ix = __fmul_rn(__fmul_rn(__fadd_rn(gx, 1.f), 0.5f), (float)(W - 1));
    ix = fminf(fmaxf(ix, 0.f), (float)(W - 1));
    const float x0 = floorf(ix);
    const float x1 = __fadd_rn(x0, 1.f);
    s.ne = __fsub_rn(ix, x0);     // wx1 (scaled by the row weights in samp_weights)
    s.nw = __fsub_rn(x1, ix);     // wx0
    s.xi0 = (int)x0;
    s.okx = s.xi0 + 1 <= W - 1;
}
__device__ __forceinline__ void samp_y(Samp& s, float gy, int H, float* wy0, float* wy1) {
    float iy = __fmul_rn(__fmul_rn(__fadd_rn(gy, 1.f), 0.5f), (float)(H - 1));
    iy = fminf(fmaxf(iy, 0.f), (float)(H - 1));
    const float y0 = floorf(iy);
    const float y1 = __fadd_rn(y0, 1.f);
    *wy1 = __fsub_rn(iy, y0);
    *wy0 = __fsub_rn(y1, iy);
    s.yi0 = (int)y0;
    s.row1 = (s.yi0 + 1 <= H - 1) && (*wy1 != 0.f);   // a zero-weight row adds +-0: skipping it does not change the sum
}
__device__ __forceinline__ void samp_weights(Samp& s, float wy0, float wy1) {
    const float wx0 = s.nw, wx1 = s.ne;
    s.nw = __fmul_rn(wx0, wy0); s.ne = __fmul_rn(wx1, wy0);
    s.sw = __fmul_rn(wx0, wy1); s.se = __fmul_rn(wx1, wy1);
}
// accumulate the (up to) four taps in the reference's order nw, ne, sw, se
__device__ __forceinline__ float3 samp_combine(const Samp& s, const float4 a, const float4 b, const float4 c, const float4 d) {
    float3 v = make_float3(__fmul_rn(a.x, s.nw), __fmul_rn(a.y, s.nw), __fmul_rn(a.z, s.nw));
    if (s.okx) { v.x = __fadd_rn(v.x, __fmul_rn(b.x, s.ne)); v.y = __fadd_rn(v.y, __fmul_rn(b.y, s.ne)); v.z = __fadd_rn(v.z, __fmul_rn(b.z, s.ne)); }
    if (s.row1) {
        v.x = __fadd_rn(v.x, __fmul_rn(c.x, s.sw)); v.y = __fadd_rn(v.y, __fmul_rn(c.y, s.sw)); v.z = __fadd_rn(v.z, __fmul_rn(c.z, s.sw));
        if (s.okx) { v.x = __fadd_rn(v.x, __fmul_rn(d.x, s.se)); v.y = __fadd_rn(v.y, __fmul_rn(d.y, s.se)); v.z = __fadd_rn(v.z, __fmul_rn(d.z, s.se)); }
    }
    return v;
}
// a sample straight from the source image (left-image samples; right-image taps that fall outside the strip)
__device__ __forceinline__ float3 sample_fly(const float* __restrict__ im, const Consts& k, const Samp& s) {
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 a = up_pixel(im, k.ug, s.yi0, s.xi0);
    const float4 b = s.okx ? up_pixel(im, k.ug, s.yi0, s.xi0 + 1) : z4;
    const float4 c = s.row1 ? up_pixel(im, k.ug, s.yi0 + 1, s.xi0) : z4;
    const float4 d = (s.row1 && s.okx) ? up_pixel(im, k.ug, s.yi0 + 1, s.xi0 + 1) : z4;
    return samp_combine(s, a, b, c, d);
}

constexpr int kStripMax = 2048;      // columns of the 2x image a CTA stages per lattice row (x 2 rows x 16 B = 64 KB)
constexpr int kMaxRowPix = 128;      // lattice pixels per row: ceil(span / max(int(span/56),1)) < 112 (dense_align.py:39-45)

// One stage of the depth search for one (RoI, row slice): rows a = slice, slice + nslices, ...  Thread t owns lattice
// column t % PB and the hypotheses h = t / PB + j * (256 / PB), j < NHG, and keeps their SADs in registers across rows;
// the CTA writes one partial row [NH costs, valid-pixel count] to `part`.
template <int NH, int PB>
__device__ __forceinline__ void stage_costs(const RoiCtx& g, const Consts& k, const float* __restrict__ imL,
                                            const float* __restrict__ imR, const float* __restrict__ rdis,
                                            float* __restrict__ red /*[8][NH+1]*/, float4* __restrict__ strip /*[2][kStripMax]*/,
                                            int slice, int nslices, float* __restrict__ part /*[NH+1] global*/) {
    constexpr int G = 256 / PB;                  // hypothesis groups
    constexpr int NHG = (NH + G - 1) / G;        // hypotheses per thread
    __shared__ float s_zf[kMaxRowPix];
    __shared__ float4 s_L[kMaxRowPix];           // left sample (x, y, z), w = 1 if the pixel is valid
    __shared__ int s_lo[2], s_hi[2];         // by row parity: a row's reset cannot race the previous row's readers
    float acc[NHG];
#pragma unroll
    for (int j = 0; j < NHG; ++j) acc[j] = 0.f;
    int cnt = 0;
    const int tid = threadIdx.x;
    const int pb = tid % PB, hg = tid / PB;
    int par = 0;
    for (int a = slice; a < g.nv; a += nslices, par ^= 1) {
        const float v = (float)(g.v0 + a * g.sv);
        const float gy = __fdiv_rn(__fsub_rn(v, k.fh2), k.fh2);
        Samp sy;
        float wy0, wy1;
        samp_y(sy, gy, k.FH, &wy0, &wy1);
        if (tid == 0) { s_lo[par] = 0x7fffffff; s_hi[par] = -1; }
        __syncthreads();
        // (a) ray test + left sample + reach of the right-image samples, one thread per lattice pixel
        if (tid < g.nu) {
            const float u = (float)(g.u0 + tid * g.su);
            float dz;
            float4 Lv = make_float4(0.f, 0.f, 0.f, 0.f);
            float zf = 0.f;
            if (ray_test(g, u, v, k, &dz)) {
                Samp s = sy;
                samp_x(s, __fdiv_rn(__fsub_rn(u, k.fw2), k.fw2), k.FW);
                samp_weights(s, wy0, wy1);
                const float3 L = sample_fly(imL, k, s);
                Lv = make_float4(L.x, L.y, L.z, 1.f);
                zf = __fdiv_rn(dz, k.fb32);
                // d = 1 / (zf + rdis[h]) falls with h: h = 0 reaches furthest left, h = NH-1 furthest right
                Samp e0 = sy, e1 = sy;
                samp_x(e0, __fdiv_rn(__fsub_rn(__fsub_rn(u, __fdiv_rn(1.0f, __fadd_rn(zf, rdis[0]))), k.fw2), k.fw2), k.FW);
                samp_x(e1, __fdiv_rn(__fsub_rn(__fsub_rn(u, __fdiv_rn(1.0f, __fadd_rn(zf, rdis[NH - 1]))), k.fw2), k.fw2), k.FW);
                atomicMin(&s_lo[par], min(e0.xi0, e1.xi0));
                atomicMax(&s_hi[par], max(e0.xi0, e1.xi0) + 1);
                ++cnt;
            }
            s_L[tid] = Lv;
            s_zf[tid] = zf;
        }
        __syncthreads();
        const int lo = s_lo[par];
        if (lo == 0x7fffffff) continue;              // no valid pixel in this row (uniform across the CTA)
        const int hi = min(min(s_hi[par], k.FW - 1), lo + kStripMax - 1);
        const int len = hi - lo + 1;
        // (b) the strip of the 2x right image this row can reach, built once
        for (int i = tid; i < len; i += 256) {
            strip[i] = up_pixel(imR, k.ug, sy.yi0, lo + i);
            if (sy.row1) strip[kStripMax + i] = up_pixel(imR, k.ug, sy.yi0 + 1, lo + i);
        }
        __syncthreads();
        // (c) SAD of this thread's hypotheses for its lattice pixel
        if (pb < g.nu) {
            const float4 Lv = s_L[pb];
            if (Lv.w != 0.f) {
                const float u = (float)(g.u0 + pb * g.su);
                const float zf = s_zf[pb];
#pragma unroll
                for (int j = 0; j < NHG; ++j) {
                    const int h = hg + j * G;
                    if (h < NH) {
                        const float d = __fdiv_rn(1.0f, __fadd_rn(zf, rdis[h]));
                        Samp s = sy;
                        samp_x(s, __fdiv_rn(__fsub_rn(__fsub_rn(u, d), k.fw2), k.fw2), k.FW);
                        samp_weights(s, wy0, wy1);
                        float3 R;
                        const int o = s.xi0 - lo;
                        if (o >= 0 && o + 1 < len + (s.okx ? 0 : 1)) {
                            const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
                            const float4 ta = strip[o], tb = s.okx ? strip[o + 1] : z4;
                            const float4 tc = s.row1 ? strip[kStripMax + o] : z4;
                            const float4 td = (s.row1 && s.okx) ? strip[kStripMax + o + 1] : z4;
                            R = samp_combine(s, ta, tb, tc, td);
                        } else {
                            R = sample_fly(imR, k, s);
                        }
                        acc[j] += fabsf(__fsub_rn(Lv.x, R.x)) + fabsf(__fsub_rn(Lv.y, R.y)) + fabsf(__fsub_rn(Lv.z, R.z));
                    }
                }
            }
        }
        // (the next row's first barrier orders these strip reads before the next fill)
    }
    __syncthreads();
    // reduce over the PB lattice columns: lanes first, then the warps of each hypothesis group
    const int lane = tid & 31, warp = tid >> 5;
    constexpr int WPG = PB / 32;                 // warps per hypothesis group
#pragma unroll
    for (int j = 0; j < NHG; ++j) {
        const float s = warp_sum(acc[j]);
        if (lane == 0) red[warp * NHG + j] = s;
    }
    {
        const float s = warp_sum((float)cnt);
        if (lane == 0) red[8 * NHG + warp] = s;
    }
    __syncthreads();
    if (tid < NH) {
        const int hgi = tid % G, j = tid / G;        // hypothesis tid = hgi + j * G
        float s = 0.f;
        for (int w = 0; w < WPG; ++w) s += red[(hgi * WPG + w) * NHG + j];
        part[tid] = s;
    }
    if (tid == NH) {
        float s = 0.f;
        for (int w = 0; w < 8; ++w) s += red[8 * NHG + w];
        part[NH] = s;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Many-RoI path (D > kStripMaxD): with hundreds of RoIs per image the 2x-upsampled pair is worth materialising
// once (59 us, 2 x 76 MB -- amortised over the RoIs: 3 % of the call at D = 2048) so that every tap is one 128-bit
// load and each thread keeps all hypotheses of its pixels in registers.  Measured (tests/tools/dense_align_sweep.py):
// 2.1 ms at D = 2048 against 5.3 ms for the strip kernel, which is built for the latency case (D <= 48: equal speed,
// no 152 MB of traffic per call).
__global__ void __launch_bounds__(256)
upsample2x_kernel(const float* __restrict__ im0, const float* __restrict__ im1, int H, int W,
                  float4* __restrict__ up0, float4* __restrict__ up1, const int* __restrict__ n_dev) {
    if (n_dev && *n_dev <= 0) return;        // no live RoI (device-resident count): the pair is never read
    const float* __restrict__ src = blockIdx.z ? im1 : im0;
    float4* __restrict__ dst = blockIdx.z ? up1 : up0;
    const int OH = 2 * H, OW = 2 * W;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= OW) return;
    const float rh = (OH > 1) ? __fdiv_rn((float)(H - 1), (float)(OH - 1)) : 0.f;
    const float rw = (OW > 1) ? __fdiv_rn((float)(W - 1), (float)(OW - 1)) : 0.f;
    const float sy = __fmul_rn(rh, (float)y);
    const int y1 = (int)sy;
    const int yp = (y1 < H - 1) ? 1 : 0;
    const float ly1 = __fsub_rn(sy, (float)y1), ly0 = __fsub_rn(1.f, ly1);
    const float sx = __fmul_rn(rw, (float)x);
    const int x1 = (int)sx;
    const int xp = (x1 < W - 1) ? 1 : 0;
    const float lx1 = __fsub_rn(sx, (float)x1), lx0 = __fsub_rn(1.f, lx1);
    float o[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float* r0 = src + ((size_t)c * H + y1) * W;
        const float* r1 = r0 + (size_t)yp * W;
        float top = __fadd_rn(__fmul_rn(lx0, __ldg(r0 + x1)), __fmul_rn(lx1, __ldg(r0 + x1 + xp)));
        float bot = __fadd_rn(__fmul_rn(lx0, __ldg(r1 + x1)), __fmul_rn(lx1, __ldg(r1 + x1 + xp)));
        o[c] = __fadd_rn(__fmul_rn(ly0, top), __fmul_rn(ly1, bot));
    }
    dst[(size_t)y * OW + x] = make_float4(o[0], o[1], o[2], 0.f);
}


// F.grid_sample(bilinear, border, align_corners=True) on the interleaved image
__device__ __forceinline__ float3 grid_sample(const float4* __restrict__ im, int H, int W, float gx, float gy) {
    float ix = __fmul_rn(__fmul_rn(__fadd_rn(gx, 1.f), 0.5f), (float)(W - 1));
    float iy = __fmul_rn(__fmul_rn(__fadd_rn(gy, 1.f), 0.5f), (float)(H - 1));
    ix = fminf(fmaxf(ix, 0.f), (float)(W - 1));
    iy = fminf(fmaxf(iy, 0.f), (float)(H - 1));
    const float x0 = floorf(ix), y0 = floorf(iy);
    const float x1 = __fadd_rn(x0, 1.f), y1 = __fadd_rn(y0, 1.f);
    const float wx1 = __fsub_rn(ix, x0), wx0 = __fsub_rn(x1, ix);
    const float wy1 = __fsub_rn(iy, y0), wy0 = __fsub_rn(y1, iy);
    const float nw = __fmul_rn(wx0, wy0), ne = __fmul_rn(wx1, wy0);
    const float sw = __fmul_rn(wx0, wy1), se = __fmul_rn(wx1, wy1);
    const int xi0 = (int)x0, yi0 = (int)y0;
    const bool okx = xi0 + 1 <= W - 1, oky = yi0 + 1 <= H - 1;
    const float4* p = im + (size_t)yi0 * W + xi0;
    const float4 a = __ldg(p);
    float3 v = make_float3(__fmul_rn(a.x, nw), __fmul_rn(a.y, nw), __fmul_rn(a.z, nw));
    if (okx) {
        const float4 b = __ldg(p + 1);
        v.x = __fadd_rn(v.x, __fmul_rn(b.x, ne)); v.y = __fadd_rn(v.y, __fmul_rn(b.y, ne)); v.z = __fadd_rn(v.z, __fmul_rn(b.z, ne));
    }
    if (oky && wy1 != 0.f) {   // a zero-weight row adds +-0 : skipped loads do not change the sum
        const float4 c = __ldg(p + W);
        v.x = __fadd_rn(v.x, __fmul_rn(c.x, sw)); v.y = __fadd_rn(v.y, __fmul_rn(c.y, sw)); v.z = __fadd_rn(v.z, __fmul_rn(c.z, sw));
        if (okx) {
            const float4 d = __ldg(p + W + 1);
            v.x = __fadd_rn(v.x, __fmul_rn(d.x, se)); v.y = __fadd_rn(v.y, __fmul_rn(d.y, se)); v.z = __fadd_rn(v.z, __fmul_rn(d.z, se));
        }
    }
    return v;
}

// One stage of the depth search for one (RoI, lattice slice).  Every thread owns lattice pixels
// q = slice*blockDim + tid (+ nslices*blockDim ...), keeps the SAD of all NH hypotheses in registers and the
// CTA writes one partial row [NH costs, valid-pixel count] to `part`.

template <int NH>
__device__ __forceinline__ void stage_costs_up(const RoiCtx& g, const Consts& k, const float4* __restrict__ upL,
                                            const float4* __restrict__ upR, const float* __restrict__ rdis,
                                            float* __restrict__ red /*[8][NH+1]*/, int slice, int nslices,
                                            float* __restrict__ part /*[NH+1] global*/) {
    float acc[NH];
#pragma unroll
    for (int h = 0; h < NH; ++h) acc[h] = 0.f;
    int cnt = 0;
    const int total = g.nu * g.nv;
    for (int q = slice * blockDim.x + threadIdx.x; q < total; q += nslices * blockDim.x) {
        const int a = q / g.nu, b = q - a * g.nu;
        const float u = (float)(g.u0 + b * g.su), v = (float)(g.v0 + a * g.sv);
        float dz;
        if (!ray_test(g, u, v, k, &dz)) continue;
        ++cnt;
        const float gy = __fdiv_rn(__fsub_rn(v, k.fh2), k.fh2);
        const float3 L = grid_sample(upL, k.FH, k.FW, __fdiv_rn(__fsub_rn(u, k.fw2), k.fw2), gy);
        const float zf = __fdiv_rn(dz, k.fb32);
#pragma unroll
        for (int h = 0; h < NH; ++h) {
            const float d = __fdiv_rn(1.0f, __fadd_rn(zf, rdis[h]));
            const float gx = __fdiv_rn(__fsub_rn(__fsub_rn(u, d), k.fw2), k.fw2);
            const float3 R = grid_sample(upR, k.FH, k.FW, gx, gy);
            acc[h] += fabsf(__fsub_rn(L.x, R.x)) + fabsf(__fsub_rn(L.y, R.y)) + fabsf(__fsub_rn(L.z, R.z));
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int h = 0; h < NH; ++h) {
        float s = warp_sum(acc[h]);
        if (lane == 0) red[warp * (NH + 1) + h] = s;
    }
    {
        float s = warp_sum((float)cnt);
        if (lane == 0) red[warp * (NH + 1) + NH] = s;
    }
    __syncthreads();
    const int nw = blockDim.x >> 5;
    if (threadIdx.x <= NH) {
        float s = 0.f;
        for (int w = 0; w < nw; ++w) s += red[w * (NH + 1) + threadIdx.x];
        part[threadIdx.x] = s;
    }
}


// coarse depths (dense_align.py:280-285) and the argmin over the slices' partial sums (fixed slice order)
__device__ __forceinline__ float coarse_depth(float z0, int h) {
    float d = __fadd_rn(__fsub_rn(z0, 12.5f), (float)(0.5 * h));
    return d < 1.5f ? 1.5f : d;
}
// one warp: lane h sums the slices' partials of hypotheses h and h+32 (fixed slice order), then a shuffle
// argmin with first-index tie break; every lane returns the result
__device__ __forceinline__ int argmin_partials(const float* __restrict__ part, int nslices, int nh, int row,
                                               float* npix) {
    const int lane = threadIdx.x & 31;
    float best = __int_as_float(0x7f800000);
    int bi = 0x7fffffff;
    for (int h = lane; h < nh; h += 32) {
        float c = 0.f;
        for (int s = 0; s < nslices; ++s) c += __ldcg(part + (size_t)s * row + h);
        if (c < best) { best = c; bi = h; }       // h ascending per lane: first minimum wins
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (npix) {
        float c = 0.f;
        for (int s = lane; s < nslices; s += 32) c += __ldcg(part + (size_t)s * row + nh);
        *npix = warp_sum(c);
    }
    return bi;
}

// grid (D, S): S row slices per RoI so that a few dozen RoIs still fill the machine; dynamic smem = the strip.
// DEV_CALIB: the calibration constants of `k0` are formed in the prologue from `calib` [24] (device memory) and
// `scale`; otherwise `k0` holds them and the last two arguments are unused.
template <int STAGE, bool DEV_CALIB>
__global__ void __launch_bounds__(256)
dense_stage_kernel(const float* __restrict__ imL, const float* __restrict__ imR, const float4* __restrict__ upL,
                   const float4* __restrict__ upR, Consts k0,
                   const float* __restrict__ box_left, const float* __restrict__ keypoints,
                   const float* __restrict__ poses, int box_ld, int pose_ld, float* __restrict__ part0 /*[D][S][51]*/,
                   float* __restrict__ part1 /*[D][S][21]*/, const int* __restrict__ n_dev,
                   const double* __restrict__ calib, double scale) {
    extern __shared__ float4 strip[];        // [2][kStripMax]
    if (n_dev && (int)blockIdx.x >= *n_dev) return;      // device-side RoI count (the solver's output): CTA-uniform
    __shared__ RoiCtx g;
    __shared__ float rdis[50];
    __shared__ float red[8 * 51];
    __shared__ float best_depth;
    __shared__ int best_idx;
    __shared__ Consts k_dev;
    const Consts& k = DEV_CALIB ? k_dev : k0;            // k_dev is written by thread 0 before the first barrier
    const int i = blockIdx.x, S = gridDim.y;
    if (threadIdx.x == 0) {
        if (DEV_CALIB) { k_dev = k0; calib_consts(&k_dev, calib, scale); }
        setup_roi(box_left + (size_t)box_ld * i, keypoints + 5 * i, poses + (size_t)pose_ld * i, k, &g);
    }
    if (STAGE == 1 && threadIdx.x >= 32 && threadIdx.x < 64) {      // warp 1, concurrently with the box setup
        const int bi = argmin_partials(part0 + (size_t)i * S * 51, S, 50, 51, nullptr);
        if (threadIdx.x == 32) best_idx = bi;
    }
    __syncthreads();
    if (STAGE == 1 && threadIdx.x == 0) best_depth = coarse_depth(g.z0, best_idx);
    if (STAGE == 1) __syncthreads();
    constexpr int NH = STAGE == 0 ? 50 : 20;
    if (threadIdx.x < NH) {
        // fine: depth_j = (best - 0.5) + 0.05 j (dense_align.py:290-294)
        const float d = STAGE == 0 ? coarse_depth(g.z0, threadIdx.x)
                                   : __fadd_rn(__fsub_rn(best_depth, 0.5f), (float)(0.05 * threadIdx.x));
        rdis[threadIdx.x] = __fdiv_rn(1.0f, __fmul_rn(__fdiv_rn(1.0f, d), k.fb32));
    }
    __syncthreads();
    float* part = STAGE == 0 ? part0 + ((size_t)i * S + blockIdx.y) * 51 : part1 + ((size_t)i * S + blockIdx.y) * 21;
    if (upL) stage_costs_up<NH>(g, k, upL, upR, rdis, red, blockIdx.y, S, part);          // materialised 2x pair
    else if (g.nu <= 64) stage_costs<NH, 64>(g, k, imL, imR, rdis, red, strip, blockIdx.y, S, part);
    else stage_costs<NH, 128>(g, k, imL, imR, rdis, red, strip, blockIdx.y, S, part);
}

// one CTA, one warp per RoI: argmins, outputs, and the reference's "no valid pixel anywhere -> dis_init" early-out
// (DEV_CALIB as in dense_stage_kernel)
template <bool DEV_CALIB>
__global__ void __launch_bounds__(256)
dense_final_kernel(Consts k0, const float* __restrict__ poses, int pose_ld, const float* __restrict__ part0,
                   const float* __restrict__ part1, int D, int S, float* __restrict__ status,
                   float* __restrict__ best_dis, const int* __restrict__ n_dev, const double* __restrict__ calib,
                   double scale) {
    __shared__ int any_valid;
    __shared__ Consts k_dev;
    const Consts& k = DEV_CALIB ? k_dev : k0;
    if (n_dev) D = min(D, *n_dev);
    if (threadIdx.x == 0) {
        any_valid = 0;
        if (DEV_CALIB) { k_dev = k0; calib_consts(&k_dev, calib, scale); }
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int i = warp; i < D; i += nw) {
        const float dis_init = __fdiv_rn(k.fb32, poses[(size_t)pose_ld * i + 2]);
        const float z0 = __fmul_rn(__fmul_rn(__fdiv_rn(1.0f, dis_init), k.f32), k.bl32);
        float npix;
        const float bd0 = coarse_depth(z0, argmin_partials(part0 + (size_t)i * S * 51, S, 50, 51, &npix));
        const int bj = argmin_partials(part1 + (size_t)i * S * 21, S, 20, 21, nullptr);
        if (lane == 0) {
            const float bd = __fadd_rn(__fsub_rn(bd0, 0.5f), (float)(0.05 * bj));
            status[i] = npix > 0.f ? 1.f : 0.f;
            best_dis[i] = __fadd_rn(__fdiv_rn(k.fb32, __fmul_rn(bd, k.s2f)), 0.5f);
            if (npix > 0.f) any_valid = 1;
        }
    }
    __syncthreads();
    if (!any_valid) {   // dense_align.py:272-273
        for (int i = threadIdx.x; i < D; i += blockDim.x) {
            status[i] = 0.f;
            best_dis[i] = __fdiv_rn(k.fb32, poses[(size_t)pose_ld * i + 2]);
        }
    }
}

constexpr int kMaxSlices = 16;

constexpr int kStripMaxD = 48;       // up to this many RoIs: strip kernel; beyond: materialise the 2x pair once

struct DaLayout { size_t upL, upR, part0, part1, total; };
DaLayout da_layout(int H, int W, int D) {
    DaLayout l;
    size_t off = 0;
    auto take = [&](size_t b) { size_t o = off; off += (b + 255) & ~(size_t)255; return o; };
    const size_t d = (size_t)(D > 0 ? D : 1);
    const size_t px = D > kStripMaxD ? (size_t)4 * H * W : 0;
    l.upL = take(px * sizeof(float4));
    l.upR = take(px * sizeof(float4));
    l.part0 = take(d * kMaxSlices * 51 * sizeof(float));
    l.part1 = take(d * kMaxSlices * 21 * sizeof(float));
    l.total = off;
    return l;
}

}  // namespace

extern "C" size_t sb_dense_align_workspace_bytes(int H, int W, int D) { return da_layout(H, W, D).total; }

// exactly one of calib4 (host, [4]) and dcalib (device, [24]) is non-null
static int dense_align_impl(const float* im_left, const float* im_right, int H, int W, const double* calib4,
                            const double* dcalib, double scale, const float* box_left, int box_ld,
                            const float* keypoints, const float* poses, int pose_ld, int D, const int* n_dev,
                            float* status, float* best_dis, void* workspace, size_t workspace_bytes,
                            sb_stream_t stream);

extern "C" int sb_dense_align(const float* im_left, const float* im_right, int H, int W, const double* calib4,
                              double scale, const float* box_left, const float* keypoints, const float* poses,
                              int D, float* status, float* best_dis, void* workspace, size_t workspace_bytes,
                              sb_stream_t stream) {
    if (D != 0 && !calib4) return SB_EINVAL;
    return dense_align_impl(im_left, im_right, H, W, calib4, nullptr, scale, box_left, 4, keypoints, poses, 7, D, nullptr,
                            status, best_dis, workspace, workspace_bytes, stream);
}

// D_cap rows are launched; rows >= *n_dev (a device-resident count, e.g. sb_box_solve's n_out) do no work and get no
// output, and with *n_dev == 0 the workspace is not written at all (not even the materialised 2x pair).
// box / pose rows may be wider than 4 / 7 floats (boxes_all [cap,5], poses_all [cap,8] of the solver).
extern "C" int sb_dense_align_n(const float* im_left, const float* im_right, int H, int W, const double* calib4,
                                double scale, const float* box_left, int box_ld, const float* keypoints,
                                const float* poses, int pose_ld, int D_cap, const int* n_dev, float* status,
                                float* best_dis, void* workspace, size_t workspace_bytes, sb_stream_t stream) {
    if (!n_dev || box_ld < 4 || pose_ld < 7) return SB_EINVAL;
    if (D_cap != 0 && !calib4) return SB_EINVAL;
    return dense_align_impl(im_left, im_right, H, W, calib4, nullptr, scale, box_left, box_ld, keypoints, poses, pose_ld,
                            D_cap, n_dev, status, best_dis, workspace, workspace_bytes, stream);
}

// sb_dense_align_n with the calibration read on the device: calib = P2 then P3, 24 row-major doubles in device
// memory.  The constants the host forms from calib4 are formed in each CTA's prologue, in the same fp64 operations.
extern "C" int sb_dense_align_n_devcalib(const float* im_left, const float* im_right, int H, int W,
                                         const double* calib, double scale, const float* box_left, int box_ld,
                                         const float* keypoints, const float* poses, int pose_ld, int D_cap,
                                         const int* n_dev, float* status, float* best_dis, void* workspace,
                                         size_t workspace_bytes, sb_stream_t stream) {
    if (!calib || !n_dev || box_ld < 4 || pose_ld < 7) return SB_EINVAL;
    return dense_align_impl(im_left, im_right, H, W, nullptr, calib, scale, box_left, box_ld, keypoints, poses, pose_ld,
                            D_cap, n_dev, status, best_dis, workspace, workspace_bytes, stream);
}

static int dense_align_impl(const float* im_left, const float* im_right, int H, int W, const double* calib4,
                            const double* dcalib, double scale, const float* box_left, int box_ld,
                            const float* keypoints, const float* poses, int pose_ld, int D, const int* n_dev,
                            float* status, float* best_dis, void* workspace, size_t workspace_bytes,
                            sb_stream_t stream) {
    if (D == 0) return SB_OK;
    if (D < 0 || H < 2 || W < 2 || !im_left || !im_right || !workspace) return SB_EINVAL;
    DaLayout l = da_layout(H, W, D);
    if (workspace_bytes < l.total) return SB_EINVAL;
    char* ws = (char*)workspace;
    cudaStream_t st = sb_cs(stream);
    float* part0 = (float*)(ws + l.part0);
    float* part1 = (float*)(ws + l.part1);
    const bool materialise = D > kStripMaxD;
    float4* upL = materialise ? (float4*)(ws + l.upL) : nullptr;
    float4* upR = materialise ? (float4*)(ws + l.upR) : nullptr;
    // dense_align.py:255-266 (python floats = doubles, cast to fp32 where they meet a tensor); with dcalib the
    // kernels form these six from device memory (calib_consts) and they stay zero here
    Consts k = {};
    if (calib4) {
        const double s2 = scale * 2.0;
        const double fd = calib4[0] * s2;
        const double bld = calib4[3] * s2 / fd;
        k.s2f = (float)s2;
        k.f32 = (float)fd;
        k.bl32 = (float)bld;
        k.fb32 = (float)(fd * bld);
        k.cx32 = (float)(calib4[1] * s2);
        k.cy32 = (float)(calib4[2] * s2);
    }
    k.FH = 2 * H;
    k.FW = 2 * W;
    k.fw2 = (float)(((double)k.FW - 1.0) / 2.0);
    k.fh2 = (float)(((double)k.FH - 1.0) / 2.0);
    k.ug.H = H;
    k.ug.W = W;
    k.ug.rh = (float)(H - 1) / (float)(k.FH - 1);       // F.upsample(align_corners=True) source ratios, fp32 division
    k.ug.rw = (float)(W - 1) / (float)(k.FW - 1);
    constexpr size_t kStripBytes = (size_t)2 * kStripMax * sizeof(float4);
    static bool attr_done[kSbMaxDevices] = {false};
    if (!attr_done[sb_cur_device()]) {
        const void* stage[4] = {(const void*)dense_stage_kernel<0, false>, (const void*)dense_stage_kernel<1, false>,
                                (const void*)dense_stage_kernel<0, true>, (const void*)dense_stage_kernel<1, true>};
        for (const void* f : stage) {
            const cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kStripBytes);
            if (e != cudaSuccess) return (int)e;
        }
        attr_done[sb_cur_device()] = true;
    }
    int S = (materialise ? 296 : 592) / D;     // strip kernel: ~4 CTAs per SM (its per-row phases are latency bound)
    if (materialise) {
        dim3 ugrid((k.FW + 255) / 256, k.FH, 2);
        upsample2x_kernel<<<ugrid, 256, 0, st>>>(im_left, im_right, H, W, upL, upR, n_dev);
        SB_LAUNCHED();
        SB_CHECK_LAUNCH();
    }
    S = S < 1 ? 1 : (S > kMaxSlices ? kMaxSlices : S);
    const size_t smem = materialise ? 0 : kStripBytes;
    if (dcalib) {
        dense_stage_kernel<0, true><<<dim3(D, S), 256, smem, st>>>(im_left, im_right, upL, upR, k, box_left, keypoints, poses, box_ld, pose_ld, part0, part1, n_dev, dcalib, scale);
        SB_LAUNCHED();
        dense_stage_kernel<1, true><<<dim3(D, S), 256, smem, st>>>(im_left, im_right, upL, upR, k, box_left, keypoints, poses, box_ld, pose_ld, part0, part1, n_dev, dcalib, scale);
        SB_LAUNCHED();
        dense_final_kernel<true><<<1, 256, 0, st>>>(k, poses, pose_ld, part0, part1, D, S, status, best_dis, n_dev, dcalib, scale);
        SB_LAUNCHED();
    } else {
        dense_stage_kernel<0, false><<<dim3(D, S), 256, smem, st>>>(im_left, im_right, upL, upR, k, box_left, keypoints, poses, box_ld, pose_ld, part0, part1, n_dev, nullptr, 0.0);
        SB_LAUNCHED();
        dense_stage_kernel<1, false><<<dim3(D, S), 256, smem, st>>>(im_left, im_right, upL, upR, k, box_left, keypoints, poses, box_ld, pose_ld, part0, part1, n_dev, nullptr, 0.0);
        SB_LAUNCHED();
        dense_final_kernel<false><<<1, 256, 0, st>>>(k, poses, pose_ld, part0, part1, D, S, status, best_dis, n_dev, nullptr, 0.0);
        SB_LAUNCHED();
    }
    SB_CHECK_LAUNCH();
    return SB_OK;
}

// fdgs_common.cuh -- shared device helpers of the H100-native 4D Gaussian rasterizer.
//
// Arithmetic contract.  "Tile assignment bit-exact" (BASELINE.json north_star) means the
// per-Gaussian quantities that decide tiles, depth order and the blend thresholds must be
// bit-identical to what the reference's kernels compute *as compiled by nvcc* (default
// -fmad=true).  nvcc's mul+add -> fma contraction depends on use counts and inlining, so
// this code does not rely on it: every operation on those paths is spelled with an explicit
// round-to-nearest intrinsic (__fmul_rn / __fadd_rn / __fmaf_rn ... are never re-contracted),
// in the association order read off the reference's PTX (tools/ptx2expr.py).  The CPU oracle
// (oracle/fdgs_oracle.c) spells the same operations with fmaf()/plain ops under
// -ffp-contract=off, so oracle and CUDA agree bit for bit except for MUFU.EX2.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fdgs {

constexpr int TILE_X = 16;   // reference: config.h:16  BLOCK_X
constexpr int TILE_Y = 16;   // reference: config.h:17  BLOCK_Y
constexpr int TILE_PIX = TILE_X * TILE_Y;

// ---- exact fp32 primitives -------------------------------------------------------------
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float fsqrt(float a) { return __fsqrt_rn(a); }
__device__ __forceinline__ float frcp(float a) { return __frcp_rn(a); }

// a0*b0 + a1*b1 + a2*b2 as nvcc contracts a left-associated sum of single-use products:
// the SECOND product stays a plain multiply, the first is fused onto it, the rest chain.
__device__ __forceinline__ float dot3c(float a0, float b0, float a1, float b1, float a2, float b2) {
    return ffma(a2, b2, ffma(a0, b0, fmul(a1, b1)));
}
__device__ __forceinline__ float dot4c(float a0, float b0, float a1, float b1, float a2, float b2,
                                       float a3, float b3) {
    return ffma(a3, b3, ffma(a2, b2, ffma(a0, b0, fmul(a1, b1))));
}

// reference: auxiliary.h:59-67 transformPoint4x3 / :69-78 transformPoint4x4, one row:
// m[r]*x + m[4+r]*y + m[8+r]*z + m[12+r]  ->  m12 + fma(z, m8, fma(x, m0, y*m4))
__device__ __forceinline__ float xform_row(float m0, float m4, float m8, float m12, float x, float y,
                                           float z) {
    return fadd(m12, ffma(z, m8, ffma(x, m0, fmul(y, m4))));
}

// Camera constants, loaded once per thread (broadcast through the constant/L1 path).
struct Camera {
    float view[16];
    float proj[16];
    float cam[3];
};

// ---- parameter activations (raw-parameter entry, SURVEY.md section 8(f) row 1) ---------------------------------
// The reference applies these in PyTorch before every render (scene/gaussian_model.py:179-219 getters:
// scaling_activation = torch.exp, opacity_activation = torch.sigmoid, rotation_activation = F.normalize); with
// fdgs_forward_args.raw_params the kernels apply them to the raw parameters instead.  Spelled like the ATen CUDA
// kernels so that the activated values -- and with them radii, tiles, depth order -- do not change:
//   exp      : expf (full-precision libdevice, what std::exp resolves to in ATen's exp kernel)
//   sigmoid  : 1 / (1 + expf(-x))                                  (ATen sigmoid kernel, opmath = float)
//   normalize: q / max(||q||_2, 1e-12); ATen's norm reduction of a 4-element row adds the rounded squares as
//              (x^2 + z^2) + (y^2 + w^2).  Other plain-fp32 orders differ from F.normalize in the last bit of some
//              rows; tests/test_gpu_raw_entry.py (test_activations_bit_identical_to_torch) checks all three
//              activations word for word against torch over 1M rows.
__device__ __forceinline__ float act_exp(float x) { return expf(x); }
__device__ __forceinline__ float act_sigmoid(float x) { return fdiv(1.0f, fadd(1.0f, expf(-x))); }
__device__ __forceinline__ float quat_norm(const float4 q) {
    return fsqrt(fadd(fadd(fmul(q.x, q.x), fmul(q.z, q.z)), fadd(fmul(q.y, q.y), fmul(q.w, q.w))));
}
__device__ __forceinline__ float4 act_normalize(const float4 q) {
    const float d = fmaxf(quat_norm(q), 1e-12f);
    return make_float4(fdiv(q.x, d), fdiv(q.y, d), fdiv(q.z, d), fdiv(q.w, d));
}
// gradient w.r.t. the raw quaternion given the gradient g w.r.t. the normalised one (autograd of q / clamp_min(||q||, eps))
__device__ __forceinline__ float4 act_normalize_bwd(const float4 q, const float4 g) {
    const float n = quat_norm(q);
    const float d = fmaxf(n, 1e-12f);
    const float inv = 1.0f / d;
    const float dot = g.x * q.x + g.y * q.y + g.z * q.z + g.w * q.w;
    const float coef = (n > 1e-12f) ? -dot * inv * inv / n : 0.f;
    return make_float4(g.x * inv + coef * q.x, g.y * inv + coef * q.y, g.z * inv + coef * q.z, g.w * inv + coef * q.w);
}

// ---- 4D covariance slice -----------------------------------------------------------------
// reference: forward.cu:279-352 computeCov3D_conditional.  Produces the 10 distinct entries of
// Sigma = (S R)^T (S R), R = M_r * M_l, in the reference's evaluation order.
struct Sigma4 {
    float s00, s01, s02, s03, s11, s12, s13, s22, s23, s33;
    float M[4][4];   // M[c][r] = s_r * R[c][r]   (needed again by the backward)
};

template <bool WANT_R = false>
__device__ __forceinline__ void build_M4(float sx, float sy, float sz, float st,  // already * mod
                                         const float4 rot, const float4 rot_r, float M[4][4],
                                         float (*Rout)[4] = nullptr) {
    const float a = rot.x, b = rot.y, c = rot.z, d = rot.w;
    const float p = rot_r.x, q = rot_r.y, r = rot_r.z, s = rot_r.w;
    // R = M_r * M_l with M_l = (a,b,-c,d | -b,a,d,c | c,-d,a,b | -d,-c,-b,a) and
    // M_r = (p,q,-r,-s | -q,p,s,-r | r,-s,p,-q | s,r,q,p) (glm column-major, forward.cu:315-329).
    // Each entry is a signed sum of four products; which products are fused into FFMAs is what
    // ptxas decided for the reference kernel (read from its SASS with tools/sass2expr.py) -- it
    // differs from entry to entry because the 16 products a*p .. d*s are shared between entries.
    float R[4][4];
    R[0][0] = ffma(d, s, fadd(ffma(a, p, -fmul(b, q)), -fmul(c, r)));
    R[0][1] = ffma(d, r, ffma(c, s, ffma(a, q, fmul(b, p))));
    R[0][2] = fadd(ffma(-c, p, ffma(b, s, -fmul(a, r))), fmul(d, q));
    R[0][3] = ffma(d, p, ffma(c, q, ffma(b, -r, -fmul(a, s))));
    R[1][0] = ffma(c, s, ffma(d, r, ffma(a, -q, -fmul(b, p))));
    R[1][1] = fadd(fmul(c, r), ffma(-d, s, ffma(a, p, -fmul(b, q))));
    R[1][2] = ffma(c, q, ffma(d, p, ffma(b, r, fmul(a, s))));
    R[1][3] = ffma(c, p, fadd(ffma(b, s, -fmul(a, r)), -fmul(d, q)));
    R[2][0] = ffma(b, s, fadd(fmul(a, r), ffma(c, p, fmul(d, q))));
    R[2][1] = ffma(b, r, fadd(-fmul(a, s), ffma(c, q, -fmul(d, p))));
    R[2][2] = fadd(fmul(b, q), ffma(a, p, ffma(-d, s, -fmul(c, r))));
    R[2][3] = fadd(fmul(b, p), ffma(-a, q, ffma(d, r, -fmul(c, s))));
    R[3][0] = fadd(fmul(a, s), ffma(-b, r, ffma(c, q, -fmul(d, p))));
    R[3][1] = fadd(fmul(a, r), ffma(b, s, ffma(-c, p, -fmul(d, q))));
    R[3][2] = ffma(a, q, fadd(-fmul(b, p), ffma(d, r, -fmul(c, s))));
    R[3][3] = ffma(a, p, fadd(fmul(b, q), ffma(d, s, fmul(c, r))));
    const float sc[4] = {sx, sy, sz, st};
#pragma unroll
    for (int col = 0; col < 4; ++col) {
#pragma unroll
        for (int row = 0; row < 4; ++row) {
            if (WANT_R) Rout[col][row] = R[col][row];
            M[col][row] = fmul(sc[row], R[col][row]);   // M = S * R, S diagonal
        }
    }
}

__device__ __forceinline__ float col_dot4(const float A[4], const float B[4]) {
    // Sigma = transpose(M) * M: entry = sum_k A[k]*B[k], contracted as dot4c
    return dot4c(A[0], B[0], A[1], B[1], A[2], B[2], A[3], B[3]);
}

__device__ __forceinline__ void sigma_from_M(Sigma4& S) {
    S.s00 = col_dot4(S.M[0], S.M[0]);
    S.s01 = col_dot4(S.M[1], S.M[0]);
    S.s02 = col_dot4(S.M[2], S.M[0]);
    S.s03 = col_dot4(S.M[3], S.M[0]);
    S.s11 = col_dot4(S.M[1], S.M[1]);
    S.s12 = col_dot4(S.M[2], S.M[1]);
    S.s13 = col_dot4(S.M[3], S.M[1]);
    S.s22 = col_dot4(S.M[2], S.M[2]);
    S.s23 = col_dot4(S.M[3], S.M[2]);
    S.s33 = col_dot4(S.M[3], S.M[3]);
}

// 4x4 helper, glm convention: A[c][r], (A*B)[c][r] = sum_k A[k][r] * B[c][k]
template <typename T>
__device__ __forceinline__ void mat4_mul(const T A[4][4], const T B[4][4], T C[4][4]) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int r = 0; r < 4; ++r)
            C[c][r] = A[0][r] * B[c][0] + A[1][r] * B[c][1] + A[2][r] * B[c][2] + A[3][r] * B[c][3];
}

// Backward of the 4D covariance Sigma = M^T M (build_M4 + sigma_from_M), reference: backward.cu:784-834.  Gradient in
// the rasterizer's convention -- every symmetric pair is one variable: d[6] = dL/d(Sigma_xyz upper triangle, as
// dL_dcov3D), dc12[3] = dL/d(Sigma[0..2][3]), dcovt = dL/d(Sigma[3][3]).  M, R = build_M4's matrices, sc = the scales
// it was given, rot / rot_r = the normalised quaternions.  Out: gs = dL/d(sc), g_rot / g_rotr = dL/d(rot / rot_r).
// Shared by geom_bwd_kernel (preprocess_bwd.cu, T = float, Q = float4) and the rigidity backward (regularize.cu, in
// double: T = double, Q = double4).
template <typename T, typename Q>
__device__ __forceinline__ void cov4_bwd(const T d[6], const T dc12[3], T dcovt, const T M[4][4], const T R4[4][4],
                                         const T sc[4], const Q rot, const Q rotr, T gs[4], T g_rot[4], T g_rotr[4]) {
    T dS[4][4];
    dS[0][0] = d[0]; dS[1][1] = d[3]; dS[2][2] = d[5]; dS[3][3] = dcovt;
    dS[0][1] = dS[1][0] = 0.5f * d[1];
    dS[0][2] = dS[2][0] = 0.5f * d[2];
    dS[1][2] = dS[2][1] = 0.5f * d[4];
    dS[0][3] = dS[3][0] = 0.5f * dc12[0];
    dS[1][3] = dS[3][1] = 0.5f * dc12[1];
    dS[2][3] = dS[3][2] = 0.5f * dc12[2];
    T M2[4][4], dM[4][4];
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int r = 0; r < 4; ++r) M2[c][r] = 2.0f * M[c][r];
    mat4_mul(M2, dS, dM);   // dL_dM = 2 * M * dL_dSigma
    // dL_dscale_i = sum_c R[c][i] * dL_dM[c][i]
    T N[4][4];   // N[i][j] = s_i * dL_dM[j][i]   (= scaled dL_dMt)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        T acc = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            acc += R4[c][i] * dM[c][i];
            N[i][c] = sc[i] * dM[c][i];
        }
        gs[i] = acc;
    }
    const T qa = rot.x, qb = rot.y, qc = rot.z, qd = rot.w;
    const T qp = rotr.x, qq = rotr.y, qr = rotr.z, qs = rotr.w;
    const T Ml[4][4] = {{qa, qb, -qc, qd}, {-qb, qa, qd, qc}, {qc, -qd, qa, qb}, {-qd, -qc, -qb, qa}};
    const T Mr[4][4] = {{qp, qq, -qr, -qs}, {-qq, qp, qs, -qr}, {qr, -qs, qp, -qq}, {qs, qr, qq, qp}};
    T X[4][4], Y[4][4];
    mat4_mul(N, Mr, X);    // dL_dml_t = dL_dMt * M_r
    mat4_mul(Ml, N, Y);    // dL_dmr_t = M_l * dL_dMt
    g_rot[0] = X[0][0] + X[1][1] + X[2][2] + X[3][3];
    g_rot[1] = -X[0][1] + X[1][0] - X[2][3] + X[3][2];
    g_rot[2] = X[0][2] - X[1][3] - X[2][0] + X[3][1];
    g_rot[3] = -X[0][3] - X[1][2] + X[2][1] + X[3][0];
    g_rotr[0] = Y[0][0] + Y[1][1] + Y[2][2] + Y[3][3];
    g_rotr[1] = -Y[0][1] + Y[1][0] + Y[2][3] - Y[3][2];
    g_rotr[2] = Y[0][2] + Y[1][3] - Y[2][0] - Y[3][1];
    g_rotr[3] = Y[0][3] - Y[1][2] + Y[2][1] - Y[3][0];
}

// marginal_t = __expf(-0.5*dt*dt / cov_t')   reference: forward.cu:333 (double-promoted argument)
__device__ __forceinline__ float marginal_from(float dt, float cov_t, float prefilter_var) {
    const float den = (prefilter_var > 0.0f) ? fadd(prefilter_var, cov_t) : cov_t;
    const double arg = ((double)dt * -0.5) * (double)dt / (double)den;
    return __expf((float)arg);
}

// ---- 3D covariance -------------------------------------------------------------------------
// reference: forward.cu:242-276 computeCov3D (quaternion NOT normalised, :251)
__device__ __forceinline__ void build_M3(float sx, float sy, float sz, const float4 q, float M[3][3]) {
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    // fusion pattern as in the reference kernel's SASS (tools/sass2expr.py)
    const float yy = fmul(y, y), zz = fmul(z, z);
    const float rz = fmul(r, z), xz = fmul(x, z), rx = fmul(r, x);
    const float A = fadd(yy, zz);
    const float B = ffma(x, x, zz);
    const float C = ffma(x, x, yy);
    float R[3][3];
    float t;
    R[0][0] = fsub(1.f, fadd(A, A));
    t = ffma(x, y, -rz); R[0][1] = fadd(t, t);
    t = ffma(r, y, xz);  R[0][2] = fadd(t, t);
    t = ffma(x, y, rz);  R[1][0] = fadd(t, t);
    R[1][1] = fsub(1.f, fadd(B, B));
    t = ffma(y, z, -rx); R[1][2] = fadd(t, t);
    t = ffma(-r, y, xz); R[2][0] = fadd(t, t);
    t = ffma(y, z, rx);  R[2][1] = fadd(t, t);
    R[2][2] = fsub(1.f, fadd(C, C));
    const float sc[3] = {sx, sy, sz};
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int rr = 0; rr < 3; ++rr) M[c][rr] = fmul(sc[rr], R[c][rr]);
}

__device__ __forceinline__ void cov3_from_M3(const float M[3][3], float cov[6]) {
    cov[0] = dot3c(M[0][0], M[0][0], M[0][1], M[0][1], M[0][2], M[0][2]);
    cov[1] = dot3c(M[1][0], M[0][0], M[1][1], M[0][1], M[1][2], M[0][2]);
    cov[2] = dot3c(M[2][0], M[0][0], M[2][1], M[0][1], M[2][2], M[0][2]);
    cov[3] = dot3c(M[1][0], M[1][0], M[1][1], M[1][1], M[1][2], M[1][2]);
    cov[4] = dot3c(M[2][0], M[1][0], M[2][1], M[1][1], M[2][2], M[1][2]);
    cov[5] = dot3c(M[2][0], M[2][0], M[2][1], M[2][1], M[2][2], M[2][2]);
}

// ---- EWA projection ------------------------------------------------------------------------
// reference: forward.cu:198-237 computeCov2D (forward) and backward.cu:507-537 (recompute).
// T = W * J (only the two non-zero columns), then cov = T^T Vrk^T T.
struct Proj2D {
    float T00, T01, T02, T10, T11, T12;   // T[c][r]
    float tx, ty, tz;                     // clamped view-space mean
    float txtz, tytz;
};

__device__ __forceinline__ void build_T(const float* __restrict__ view, float mx, float my, float mz,
                                        float focal_x, float focal_y, float tan_fovx, float tan_fovy,
                                        Proj2D& P) {
    const float tx0 = xform_row(view[0], view[4], view[8], view[12], mx, my, mz);
    const float ty0 = xform_row(view[1], view[5], view[9], view[13], mx, my, mz);
    const float tz = xform_row(view[2], view[6], view[10], view[14], mx, my, mz);
    const float limx = fmul(1.3f, tan_fovx);
    const float limy = fmul(1.3f, tan_fovy);
    P.txtz = fdiv(tx0, tz);
    P.tytz = fdiv(ty0, tz);
    // min(limx, max(-limx, txtz)) * t.z   (forward.cu:210-211)
    P.tx = fmul(fminf(limx, fmaxf(-limx, P.txtz)), tz);
    P.ty = fmul(fminf(limy, fmaxf(-limy, P.tytz)), tz);
    P.tz = tz;
    const float tz2 = fmul(tz, tz);
    const float j00 = fdiv(focal_x, tz);
    const float j11 = fdiv(focal_y, tz);
    const float j02 = fdiv(fmul(focal_x, -P.tx), tz2);   // -(focal_x * t.x) / (t.z * t.z)
    const float j12 = fdiv(fmul(focal_y, -P.ty), tz2);
    P.T00 = ffma(view[2], j02, fmul(view[0], j00));
    P.T01 = ffma(view[6], j02, fmul(view[4], j00));
    P.T02 = ffma(j02, view[10], fmul(view[8], j00));
    P.T10 = ffma(view[2], j12, fmul(j11, view[1]));
    P.T11 = ffma(view[6], j12, fmul(j11, view[5]));
    P.T12 = ffma(j12, view[10], fmul(j11, view[9]));
}

// cov2D (before the +0.3 low-pass): a = cov[0][0], b = cov[0][1], c = cov[1][1]
__device__ __forceinline__ void cov2d_from_T(const Proj2D& P, const float c3[6], float& a, float& b,
                                             float& c) {
    const float X00 = dot3c(P.T00, c3[0], P.T01, c3[1], P.T02, c3[2]);
    const float X01 = dot3c(P.T10, c3[0], P.T11, c3[1], P.T12, c3[2]);
    const float X10 = dot3c(P.T00, c3[1], P.T01, c3[3], P.T02, c3[4]);
    const float X11 = dot3c(P.T10, c3[1], P.T11, c3[3], P.T12, c3[4]);
    const float X20 = dot3c(P.T00, c3[2], P.T01, c3[4], P.T02, c3[5]);
    const float X21 = dot3c(P.T10, c3[2], P.T11, c3[4], P.T12, c3[5]);
    a = dot3c(P.T00, X00, P.T01, X10, P.T02, X20);
    b = dot3c(P.T00, X01, P.T01, X11, P.T02, X21);
    c = dot3c(P.T10, X01, P.T11, X11, P.T12, X21);
}

// reference: auxiliary.h:42-45 ndc2Pix -- evaluated in double, contracted to a double fma
__device__ __forceinline__ float ndc2pix(float v, int S) {
    return (float)(__fma_rn((double)v + 1.0, (double)S, -1.0) * 0.5);
}

// reference: auxiliary.h:47-57 getRect (max_radius is an int there)
__device__ __forceinline__ void get_rect(float px, float py, int radius, int gx, int gy, int& x0, int& y0,
                                         int& x1, int& y1) {
    const float r = (float)radius;
    x0 = min(gx, max(0, (int)fmul(fsub(px, r), 0.0625f)));
    y0 = min(gy, max(0, (int)fmul(fsub(py, r), 0.0625f)));
    x1 = min(gx, max(0, (int)fmul(fadd(fadd(fadd(px, r), 16.0f), -1.0f), 0.0625f)));
    y1 = min(gy, max(0, (int)fmul(fadd(fadd(fadd(py, r), 16.0f), -1.0f), 0.0625f)));
}

// SH constants, reference: auxiliary.h:23-40
__device__ constexpr float kSH_C0 = 0.28209479177387814f;
__device__ constexpr float kSH_C1 = 0.4886025119029199f;
__device__ constexpr float kSH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                        -1.0925484305920792f, 0.5462742152960396f};
__device__ constexpr float kSH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                        0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                                        -0.5900435899266435f};
#define FDGS_MY_PI 3.14159265   /* double literal, reference: auxiliary.h:20 */

// ---- per-instance record consumed by the blend kernels -------------------------------------
// One 64-byte record per (tile, Gaussian) instance, stored in tile-sorted order, so that a
// tile's work list is one contiguous byte range that cp.async.bulk can stream into shared
// memory.  Four float4 "planes":
//   q0 = { x, y, pmin, gaussian_id (bits) }   pixel-space mean; pmin = log(1/(255*opacity)) - slack
//   q1 = { A, B, C, opacity }                 conic (reference conic_opacity)
//   q2 = { r, g, b, depth }
//   q3 = { flow_x, flow_y, ex, ey }           ex/ey = half-extents of the alpha >= 1/255 box
struct __align__(16) InstRec {
    float4 q0, q1, q2, q3;
};
static_assert(sizeof(InstRec) == 64, "InstRec must be 64 bytes");

// The same record as it is stored in the tile-sorted instance stream (`recs`) and staged in shared memory by the
// blend kernels: padded to 80 bytes.  With a 64-byte stride the culling loads -- lane j reads plane q of record j,
// LDS.128 at address 64 j + 16 q -- hit only two 4-bank groups (4-way conflict, 16 wavefronts per load, measured
// 61 M of the ~110-190 M shared-memory wavefronts of each blend kernel); with an 80-byte stride 8 consecutive
// records cover all 32 banks (20 j mod 32 = 0, 20, 8, 28, 16, 4, 24, 12) and the loads are conflict-free.  The
// extra 16 bytes per instance are HBM traffic the blend kernels, at < 8 % of DRAM bandwidth, do not feel.
struct __align__(16) StageRec {
    float4 q0, q1, q2, q3, pad;
};
static_assert(sizeof(StageRec) == 80, "StageRec must be 80 bytes");
constexpr uint32_t kStageRecBytes = 80u;

// Can the instance (centre x0,y0; conic A,B,C; pmin; slopes sbc=-B/C, sba=-B/A) contribute to any
// pixel of the rectangle [bx0,bx1] x [by0,by1]?  It contributes at offset d only if
// q(d) = 0.5*(A dx^2 + C dy^2) + B dx dy <= -pmin.  q is convex, so its minimum over the rectangle is
// 0 if the centre is inside, else it lies on the edge(s) facing the centre, where it is a clamped
// 1-D quadratic minimum.  Exact up to round-off, which the 0.02 slack inside pmin and the 1e-3 here
// absorb; pmin = +inf means "never", pmin = -inf means "always" (irregular inputs).
__device__ __forceinline__ bool rect_may_contribute(float x0, float y0, float A, float B, float C, float pmin,
                                                    float sbc, float sba, float bx0, float bx1, float by0,
                                                    float by1) {
    const float ddx = fminf(fmaxf(x0, bx0), bx1) - x0;   // offset of the nearest rectangle point
    const float ddy = fminf(fmaxf(y0, by0), by1) - y0;
    // edge x = x0 + ddx, y free in the rectangle
    const float ty = fminf(fmaxf(sbc * ddx, by0 - y0), by1 - y0);
    const float q1 = 0.5f * (A * ddx * ddx + C * ty * ty) + B * ddx * ty;
    // edge y = y0 + ddy, x free in the rectangle
    const float tx = fminf(fmaxf(sba * ddy, bx0 - x0), bx1 - x0);
    const float q2 = 0.5f * (A * tx * tx + C * ddy * ddy) + B * tx * ddy;
    // if the centre is outside in one axis only, only that axis' edge applies; inside: q = 0
    float qmin = (ddx != 0.f) ? ((ddy != 0.f) ? fminf(q1, q2) : q1) : ((ddy != 0.f) ? q2 : 0.f);
    // thin, rotated Gaussians far from their centre: the three terms of q are large and cancel, so the fp32 rounding
    // error of q -- and of the blend loop's own power -- grows with their magnitude.  Both are bounded by ~6 roundings
    // of 2^-24 each relative to `mag`; the cull keeps 2e-6 * mag of extra slack, i.e. it only rejects when even the
    // worst-case rounding leaves q above the cut.  (A fixed "never cull above mag = 128" guard was measured to triple
    // the survivors of cfg3: an ordinary 1-pixel Gaussian 12 pixels away already has A ddx^2 = 144.)
    const float mag = fmaxf(fabsf(A * ddx * ddx) + fabsf(C * ty * ty) + 2.f * fabsf(B * ddx * ty),
                            fabsf(A * tx * tx) + fabsf(C * ddy * ddy) + 2.f * fabsf(B * tx * ddy));
    // also true for pmin = -inf (and for a non-finite mag), false for pmin = +inf
    return !(qmin > -pmin + 1e-3f + 2.0e-6f * mag);
}

// ---- mbarrier / bulk-copy (TMA 1-D) PTX wrappers ----------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// same, but a warp that has to wait gives its issue slots to the warps that are still working
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) __nanosleep(64);
}
// global -> shared bulk copy (SASS: UBLKCP), completion signalled on `bar` (complete_tx::bytes).
// dst, src and bytes must be multiples of 16.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// shared -> global bulk copy (bulk async-group completion)
__device__ __forceinline__ void bulk_s2g(void* dst_gmem, const void* src_smem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem),
                 "r"(smem_u32(src_smem)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() {
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// 4-byte asynchronous global -> shared copy (SASS: LDGSTS): no register staging, any 4-byte alignment -- used for the
// split SH rows (12-byte + 564-byte pieces) that the bulk-copy engine cannot address
__device__ __forceinline__ void cp_async4(void* dst_smem, const void* src_gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// One split SH row (3 floats at dc, row_floats - 3 at rest) -> dst[0 .. row_floats), by the 32 lanes of a warp
__device__ __forceinline__ void split_row_to_smem(float* dst, const float* __restrict__ dc, const float* __restrict__ rest,
                                                  int row_floats, int lane) {
    for (int f = lane; f < row_floats; f += 32) cp_async4(dst + f, (f < 3) ? dc + f : rest + (f - 3));
}
// make generic-proxy smem writes visible to the async proxy before a bulk store reads them
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

}  // namespace fdgs

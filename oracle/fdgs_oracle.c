/*
 * fdgs_oracle.c -- CPU restatement of the reference's differentiable 4D Gaussian rasterizer.
 *
 * TEST INFRASTRUCTURE.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * reference arm may load this; the product (4d-gaussian-splatting_b200/) never does.
 *
 * It follows the reference's CUDA code function by function (citations at each function) and is
 * written independently of the product's kernels: plain C, one Gaussian / one pixel at a time,
 * the reference's data layout (per-Gaussian arrays + sorted index list), no instance records, no
 * culling, no reductions.  fp32 arithmetic is spelled operation by operation (compile with
 * -ffp-contract=off): products that nvcc fuses into FMAs in the reference's kernels are fmaf()
 * here, in the association order read from the reference's PTX, so that integer outputs (radii,
 * tiles, sorted list, n_contrib) come out bit-identical to the reference kernels.  Known,
 * documented exceptions: MUFU.EX2-based __expf()/expf() and the double cos/sin are replaced by
 * libm (differences of a few ulp; they only matter on measure-zero threshold ties).
 *
 * Pinning: validated against golden vectors produced by the UNMODIFIED reference kernels
 * (oracle/_ref, built by oracle/build_ref.py) -- see tests/golden/ and tests/test_oracle_golden.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define BLOCK_X 16 /* reference: config.h:16 */
#define BLOCK_Y 16 /* reference: config.h:17 */
#define MY_PI 3.14159265 /* reference: auxiliary.h:20 (a double literal) */

/* reference: auxiliary.h:23-40 */
static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                               -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                               -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};

typedef struct {
    int P, D, D_t, M;
    int W, H;
    const float* background; /* [3] */
    const float* means3D;    /* [P,3] */
    const float* shs;        /* [P,M,3] or NULL */
    const float* colors_precomp;
    const float* flows;      /* [P,2] */
    const float* opacities;
    const float* ts;
    const float* scales;
    const float* scales_t;
    float scale_modifier;
    const float* rotations;
    const float* rotations_r;
    const float* cov3D_precomp;
    float prefilter_var;
    const float* viewmatrix; /* [16] column-major */
    const float* projmatrix;
    const float* cam_pos;
    float timestamp, time_duration;
    int rot_4d, gaussian_dim, force_sh_3d;
    float tan_fovx, tan_fovy;
} OracleScene;

/* per-Gaussian forward state == the reference's GeometryState (rasterizer_impl.h:29-44) */
typedef struct {
    float* out_means3D; /* [P,3] */
    int* radii;
    float* depths;
    float* means2D;       /* [P,2] */
    float* cov3D;         /* [P,6] */
    float* conic_opacity; /* [P,4] */
    float* rgb;           /* [P,3] */
    uint8_t* clamped;     /* [P,3] */
    uint32_t* tiles_touched;
} OracleGeom;

/* ---- exact float helpers -------------------------------------------------------------- */
static inline float fmul(float a, float b) { return a * b; }
static inline float fadd(float a, float b) { return a + b; }
static inline float fsub(float a, float b) { return a - b; }
static inline float ffma(float a, float b, float c) { return fmaf(a, b, c); }
static inline float fdivf_(float a, float b) { return a / b; }

/* float -> int, round toward zero, saturating, NaN -> 0 (PTX cvt.rzi.s32.f32) */
static inline int f2i_rz(float f) {
    if (f != f) return 0;
    if (f >= 2147483648.0f) return 2147483647;
    if (f <= -2147483648.0f) return (-2147483647 - 1);
    return (int)f;
}
static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

/* sum of products as the reference's kernels evaluate "a0*b0 + a1*b1 + a2*b2 (+ a3*b3)" after
 * nvcc's contraction: second product plain, first fused onto it, then the rest in order. */
static inline float dot3(float a0, float b0, float a1, float b1, float a2, float b2) {
    return ffma(a2, b2, ffma(a0, b0, fmul(a1, b1)));
}
static inline float dot4(float a0, float b0, float a1, float b1, float a2, float b2, float a3, float b3) {
    return ffma(a3, b3, ffma(a2, b2, ffma(a0, b0, fmul(a1, b1))));
}

/* reference: auxiliary.h:59-78 transformPoint4x3/4x4, one output row */
static inline float xform(const float* m, int r, float x, float y, float z) {
    return fadd(m[12 + r], ffma(z, m[8 + r], ffma(x, m[r], fmul(y, m[4 + r]))));
}

/* reference: auxiliary.h:42-45 (double; the multiply-add is contracted to a double fma) */
static inline float ndc2Pix(float v, int S) { return (float)(fma((double)v + 1.0, (double)S, -1.0) * 0.5); }

/* reference: auxiliary.h:47-57 */
static void getRect(float px, float py, int max_radius, int gx, int gy, int* x0, int* y0, int* x1, int* y1) {
    const float r = (float)max_radius;
    *x0 = imin(gx, imax(0, f2i_rz(fmul(fsub(px, r), 0.0625f))));
    *y0 = imin(gy, imax(0, f2i_rz(fmul(fsub(py, r), 0.0625f))));
    *x1 = imin(gx, imax(0, f2i_rz(fmul(fadd(fadd(fadd(px, r), 16.0f), -1.0f), 0.0625f))));
    *y1 = imin(gy, imax(0, f2i_rz(fmul(fadd(fadd(fadd(py, r), 16.0f), -1.0f), 0.0625f))));
}

/* __expf(x) = ex2.approx(x * log2(e)); libm stand-in for the hardware approximation */
static inline float fast_expf(float x) { return exp2f(fmul(x, 1.44269502f)); }

/* reference: forward.cu:333 / :434 -- the argument is evaluated in double */
static float marginal_of(float dt, float var, float prefilter_var) {
    const float den = (prefilter_var > 0.0f) ? fadd(prefilter_var, var) : var;
    const double arg = (((double)dt * -0.5) * (double)dt) / (double)den;
    return fast_expf((float)arg);
}

/* reference: forward.cu:279-331 -- M = S * (M_r * M_l), glm column-major: M[c][r] */
static void build_M4(const float sc[4], const float* rot, const float* rot_r, float M[4][4], float R[4][4]) {
    const float a = rot[0], b = rot[1], c = rot[2], d = rot[3];
    const float p = rot_r[0], q = rot_r[1], r = rot_r[2], s = rot_r[3];
    /* R = M_r * M_l, M_l = (a,b,-c,d | -b,a,d,c | c,-d,a,b | -d,-c,-b,a),
     * M_r = (p,q,-r,-s | -q,p,s,-r | r,-s,p,-q | s,r,q,p)  (glm columns, forward.cu:315-329).
     * Mathematically R[c][r] = sum_k M_r[k][r]*M_l[c][k]; the rounding sequence below (which of
     * the shared products a*p..d*s end up inside an FFMA) is the one in the reference kernel's
     * machine code, entry by entry. */
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
    for (int col = 0; col < 4; ++col)
        for (int row = 0; row < 4; ++row) M[col][row] = fmul(sc[row], R[col][row]);
}
static inline float coldot4(const float* A, const float* B) { return dot4(A[0], B[0], A[1], B[1], A[2], B[2], A[3], B[3]); }

/* reference: forward.cu:242-276 */
static void build_M3(const float sc[3], const float* q, float M[3][3], float R[3][3]) {
    const float r = q[0], x = q[1], y = q[2], z = q[3];
    const float yy = fmul(y, y), zz = fmul(z, z), rz = fmul(r, z), xz = fmul(x, z), rx = fmul(r, x);
    const float A = fadd(yy, zz), B = ffma(x, x, zz), C = ffma(x, x, yy);
    float t;
    /* 2*(x*y - r*z) etc.: the second product of each pair is fused in the reference's machine code */
    R[0][0] = fsub(1.f, fadd(A, A));
    t = ffma(x, y, -rz); R[0][1] = fadd(t, t);
    t = ffma(r, y, xz);  R[0][2] = fadd(t, t);
    t = ffma(x, y, rz);  R[1][0] = fadd(t, t);
    R[1][1] = fsub(1.f, fadd(B, B));
    t = ffma(y, z, -rx); R[1][2] = fadd(t, t);
    t = ffma(-r, y, xz); R[2][0] = fadd(t, t);
    t = ffma(y, z, rx);  R[2][1] = fadd(t, t);
    R[2][2] = fsub(1.f, fadd(C, C));
    for (int c = 0; c < 3; ++c)
        for (int rr = 0; rr < 3; ++rr) M[c][rr] = fmul(sc[rr], R[c][rr]);
}

typedef struct {
    float T[2][3]; /* T[c][r], third column is zero */
    float tx, ty, tz, txtz, tytz;
} ProjT;

/* reference: forward.cu:204-223 (forward) == backward.cu:509-535 (recompute) */
static void build_T(const float* V, float mx, float my, float mz, float fx, float fy, float tanx, float tany, ProjT* P) {
    const float tx0 = xform(V, 0, mx, my, mz), ty0 = xform(V, 1, mx, my, mz), tz = xform(V, 2, mx, my, mz);
    const float limx = fmul(1.3f, tanx), limy = fmul(1.3f, tany);
    P->txtz = tx0 / tz;
    P->tytz = ty0 / tz;
    P->tx = fmul(fminf(limx, fmaxf(-limx, P->txtz)), tz);
    P->ty = fmul(fminf(limy, fmaxf(-limy, P->tytz)), tz);
    P->tz = tz;
    const float tz2 = fmul(tz, tz);
    const float j00 = fx / tz, j11 = fy / tz;
    const float j02 = fmul(fx, -P->tx) / tz2, j12 = fmul(fy, -P->ty) / tz2;
    P->T[0][0] = ffma(V[2], j02, fmul(V[0], j00));
    P->T[0][1] = ffma(V[6], j02, fmul(V[4], j00));
    P->T[0][2] = ffma(j02, V[10], fmul(V[8], j00));
    P->T[1][0] = ffma(V[2], j12, fmul(j11, V[1]));
    P->T[1][1] = ffma(V[6], j12, fmul(j11, V[5]));
    P->T[1][2] = ffma(j12, V[10], fmul(j11, V[9]));
}

/* reference: forward.cu:225-236: cov = T^T * Vrk^T * T (before the 0.3 low-pass) */
static void cov2d(const ProjT* P, const float* c, float* a, float* b, float* cc) {
    const float (*T)[3] = P->T;
    const float X00 = dot3(T[0][0], c[0], T[0][1], c[1], T[0][2], c[2]);
    const float X01 = dot3(T[1][0], c[0], T[1][1], c[1], T[1][2], c[2]);
    const float X10 = dot3(T[0][0], c[1], T[0][1], c[3], T[0][2], c[4]);
    const float X11 = dot3(T[1][0], c[1], T[1][1], c[3], T[1][2], c[4]);
    const float X20 = dot3(T[0][0], c[2], T[0][1], c[4], T[0][2], c[5]);
    const float X21 = dot3(T[1][0], c[2], T[1][1], c[4], T[1][2], c[5]);
    *a = dot3(T[0][0], X00, T[0][1], X10, T[0][2], X20);
    *b = dot3(T[0][0], X01, T[0][1], X11, T[0][2], X21);
    *cc = dot3(T[1][0], X01, T[1][1], X11, T[1][2], X21);
}

/* ---- SH colour ---------------------------------------------------------------------------- */
/* degree-3 basis l[9..15] (forward.cu:53-59 / :125-131).  "3*xx - yy" and friends are single
 * FFMAs in the reference's machine code. */
static void sh_l3(float x, float y, float z, float xx, float yy, float zz, float xy, float l[16]) {
    const float w = fadd(-yy, ffma(zz, 4.f, -xx)); /* 4zz - xx - yy */
    l[9] = fmul(fmul(y, SH_C3[0]), ffma(xx, 3.f, -yy));
    l[10] = fmul(fmul(xy, SH_C3[1]), z);
    l[11] = fmul(fmul(y, SH_C3[2]), w);
    l[12] = fmul(fmul(z, SH_C3[3]), ffma(yy, -3.f, ffma(xx, -3.f, fadd(zz, zz))));
    l[13] = fmul(w, fmul(x, SH_C3[4]));
    l[14] = fmul(fsub(xx, yy), fmul(z, SH_C3[5]));
    l[15] = fmul(fmul(x, SH_C3[6]), ffma(yy, -3.f, xx));
}

/* reference: forward.cu:20-71 computeColorFromSH; returns the value before "+0.5, clamp".
 * The whole expression is one FFMA chain in the reference's machine code. */
static void sh_color_3d(const float* sh, int deg, float x, float y, float z, float out[3]) {
    const float xx = fmul(x, x), yy = fmul(y, y), zz = fmul(z, z), xy = fmul(x, y), yz = fmul(y, z), xz = fmul(x, z);
    float l[16];
    if (deg > 2) sh_l3(x, y, z, xx, yy, zz, xy, l);
    for (int ch = 0; ch < 3; ++ch) {
#define S(k) sh[3 * (k) + ch]
        float r = fmul(S(0), SH_C0);
        if (deg > 0) {
            r = ffma(-fmul(y, SH_C1), S(1), r);
            r = ffma(fmul(z, SH_C1), S(2), r);
            r = ffma(-fmul(x, SH_C1), S(3), r);
            if (deg > 1) {
                r = ffma(fmul(xy, SH_C2[0]), S(4), r);
                r = ffma(fmul(yz, SH_C2[1]), S(5), r);
                r = ffma(fmul(fsub(fsub(fadd(zz, zz), xx), yy), SH_C2[2]), S(6), r);
                r = ffma(fmul(xz, SH_C2[3]), S(7), r);
                r = ffma(fmul(fsub(xx, yy), SH_C2[4]), S(8), r);
                if (deg > 2)
                    for (int k = 9; k < 16; ++k) r = ffma(l[k], S(k), r);
            }
        }
#undef S
        out[ch] = r;
    }
}

/* reference: forward.cu:73-195 computeColorFromSH_4D; the basis l[16] */
static void sh_basis_4d(float x, float y, float z, int deg, float l[16]) {
    for (int i = 0; i < 16; ++i) l[i] = 0.f;
    l[0] = SH_C0;
    if (deg > 0) {
        l[1] = fmul(y, -SH_C1);
        l[2] = fmul(z, SH_C1);
        l[3] = fmul(x, -SH_C1);
        if (deg > 1) {
            const float xx = fmul(x, x), yy = fmul(y, y), zz = fmul(z, z), xy = fmul(x, y), yz = fmul(y, z),
                        xz = fmul(x, z);
            l[4] = fmul(xy, SH_C2[0]);
            l[5] = fmul(yz, SH_C2[1]);
            l[6] = (float)(((((double)zz + (double)zz) - (double)xx) - (double)yy) * (double)SH_C2[2]); /* :112 */
            l[7] = fmul(xz, SH_C2[3]);
            l[8] = fmul(fsub(xx, yy), SH_C2[4]);
            if (deg > 2) sh_l3(x, y, z, xx, yy, zz, xy, l);
        }
    }
}

static void sh_color_4d(const float* sh, int deg, int deg_t, float x, float y, float z, float dir_t, float duration,
                        float out[3]) {
    float l[16];
    sh_basis_4d(x, y, z, deg, l);
    for (int ch = 0; ch < 3; ++ch) {
#define S(k) sh[3 * (k) + ch]
        float r = fmul(S(0), SH_C0);
        if (deg > 0) {
            r = fadd(r, ffma(l[3], S(3), ffma(l[1], S(1), fmul(l[2], S(2)))));
            if (deg > 1) {
                float b = ffma(l[4], S(4), fmul(l[5], S(5)));
                b = ffma(S(6), l[6], b);
                b = ffma(l[8], S(8), ffma(l[7], S(7), b));
                r = fadd(r, b);
                if (deg > 2) {
                    float c = ffma(l[11], S(11), ffma(l[9], S(9), fmul(l[10], S(10))));
                    c = ffma(l[13], S(13), ffma(l[12], S(12), c));
                    c = ffma(l[15], S(15), ffma(l[14], S(14), c));
                    r = fadd(r, c);
                    /* temporal terms live under deg > 2 only (forward.cu:142 nested in :123) */
                    for (int n = 1; n <= deg_t && n <= 2; ++n) {
                        double ang = (double)dir_t * (2 * MY_PI);
                        if (n == 2) ang = ang * 2.0;
                        const float tn = (float)cos(ang / (double)duration);
                        float s = ffma(S(16 * n), l[0], fmul(l[1], S(16 * n + 1)));
                        for (int k = 2; k < 16; ++k) s = ffma(l[k], S(16 * n + k), s);
                        r = ffma(s, tn, r);
                    }
                }
            }
        }
#undef S
        out[ch] = r;
    }
}

/* ---- forward: per-Gaussian preprocessing ------------------------------------------------- */
/* reference: forward.cu:355-496 preprocessCUDA.  Returns num visible. */
int oracle_preprocess(const OracleScene* s, OracleGeom* g) {
    const int gx = (s->W + BLOCK_X - 1) / BLOCK_X, gy = (s->H + BLOCK_Y - 1) / BLOCK_Y;
    /* reference: rasterizer_impl.cu:235-236 */
    const float focal_y = s->H / (2.0f * s->tan_fovy);
    const float focal_x = s->W / (2.0f * s->tan_fovx);
    int nvis = 0;
#ifdef _OPENMP
#pragma omp parallel for schedule(static) reduction(+ : nvis)
#endif
    for (int idx = 0; idx < s->P; ++idx) {
        g->radii[idx] = 0;
        g->tiles_touched[idx] = 0;
        float px = s->means3D[3 * idx], py = s->means3D[3 * idx + 1], pz = s->means3D[3 * idx + 2];
        /* rasterize_points.cu:85: out_means3D starts as a clone */
        g->out_means3D[3 * idx] = px; g->out_means3D[3 * idx + 1] = py; g->out_means3D[3 * idx + 2] = pz;
        float opacity = s->opacities[idx];
        const float* cov3D;
        if (s->cov3D_precomp) {
            cov3D = s->cov3D_precomp + 6 * idx;
        } else if (s->rot_4d) {
            /* forward.cu:279-352 computeCov3D_conditional */
            const float dt = fsub(s->timestamp, s->ts[idx]);
            const float sc[4] = {fmul(s->scale_modifier, s->scales[3 * idx]), fmul(s->scale_modifier, s->scales[3 * idx + 1]),
                                 fmul(s->scale_modifier, s->scales[3 * idx + 2]), fmul(s->scale_modifier, s->scales_t[idx])};
            float M[4][4], R[4][4];
            build_M4(sc, s->rotations + 4 * idx, s->rotations_r + 4 * idx, M, R);
            const float s00 = coldot4(M[0], M[0]), s01 = coldot4(M[1], M[0]), s02 = coldot4(M[2], M[0]),
                        s03 = coldot4(M[3], M[0]), s11 = coldot4(M[1], M[1]), s12 = coldot4(M[2], M[1]),
                        s13 = coldot4(M[3], M[1]), s22 = coldot4(M[2], M[2]), s23 = coldot4(M[3], M[2]),
                        cov_t = coldot4(M[3], M[3]);
            const float marginal = marginal_of(dt, cov_t, s->prefilter_var);
            if (!((double)marginal > 0.05)) continue;
            opacity = fmul(opacity, marginal);
            float* c = g->cov3D + 6 * idx;
            c[0] = fsub(s00, fmul(s03, s03) / cov_t);
            c[1] = fsub(s01, fmul(s13, s03) / cov_t);
            c[2] = fsub(s02, fmul(s23, s03) / cov_t);
            c[3] = fsub(s11, fmul(s13, s13) / cov_t);
            c[4] = fsub(s12, fmul(s23, s13) / cov_t);
            c[5] = fsub(s22, fmul(s23, s23) / cov_t);
            px = ffma(dt, s03 / cov_t, px);
            py = ffma(dt, s13 / cov_t, py);
            pz = ffma(dt, s23 / cov_t, pz);
            g->out_means3D[3 * idx] = px; g->out_means3D[3 * idx + 1] = py; g->out_means3D[3 * idx + 2] = pz;
            cov3D = c;
        } else {
            const float sc[3] = {fmul(s->scale_modifier, s->scales[3 * idx]), fmul(s->scale_modifier, s->scales[3 * idx + 1]),
                                 fmul(s->scale_modifier, s->scales[3 * idx + 2])};
            float M[3][3], R[3][3];
            build_M3(sc, s->rotations + 4 * idx, M, R);
            float* c = g->cov3D + 6 * idx;
            c[0] = dot3(M[0][0], M[0][0], M[0][1], M[0][1], M[0][2], M[0][2]);
            c[1] = dot3(M[1][0], M[0][0], M[1][1], M[0][1], M[1][2], M[0][2]);
            c[2] = dot3(M[2][0], M[0][0], M[2][1], M[0][1], M[2][2], M[0][2]);
            c[3] = dot3(M[1][0], M[1][0], M[1][1], M[1][1], M[1][2], M[1][2]);
            c[4] = dot3(M[2][0], M[1][0], M[2][1], M[1][1], M[2][2], M[1][2]);
            c[5] = dot3(M[2][0], M[2][0], M[2][1], M[2][1], M[2][2], M[2][2]);
            cov3D = c;
            if (s->gaussian_dim == 4) { /* forward.cu:431-437: sigma used as a variance */
                const float dt = fsub(s->ts[idx], s->timestamp);
                const float sigma = fmul(s->scale_modifier, s->scales_t[idx]);
                const float marginal = marginal_of(dt, sigma, s->prefilter_var);
                if ((double)marginal <= 0.05) continue;
                opacity = fmul(opacity, marginal);
            }
        }
        /* in_frustum, auxiliary.h:140-163 */
        const float* V = s->viewmatrix;
        const float* Pm = s->projmatrix;
        const float vz = xform(V, 2, px, py, pz);
        if (vz <= 0.2f) continue;
        const float hx = xform(Pm, 0, px, py, pz), hy = xform(Pm, 1, px, py, pz), hw = xform(Pm, 3, px, py, pz);
        const float p_w = 1.0f / fadd(hw, 0.0000001f);
        const float projx = fmul(hx, p_w), projy = fmul(hy, p_w);
        ProjT Pj;
        build_T(V, px, py, pz, focal_x, focal_y, s->tan_fovx, s->tan_fovy, &Pj);
        float ca, cb, cc;
        cov2d(&Pj, cov3D, &ca, &cb, &cc);
        ca = fadd(ca, 0.3f);
        cc = fadd(cc, 0.3f);
        const float det = ffma(ca, cc, -fmul(cb, cb)); /* forward.cu:454, first product fused */
        if (det == 0.0f) continue;
        const float det_inv = 1.f / det;
        const float conx = fmul(cc, det_inv), cony = fmul(det_inv, -cb), conz = fmul(ca, det_inv);
        const float mid = fmul(fadd(ca, cc), 0.5f);
        const float sq = sqrtf(fmaxf(ffma(mid, mid, -det), 0.1f)); /* :465 */
        const float lam = fmaxf(fadd(mid, sq), fsub(mid, sq));
        const float my_radius = ceilf(fmul(sqrtf(lam), 3.f));
        const float ix = ndc2Pix(projx, s->W), iy = ndc2Pix(projy, s->H);
        const int radius = f2i_rz(my_radius);
        int x0, y0, x1, y1;
        getRect(ix, iy, radius, gx, gy, &x0, &y0, &x1, &y1);
        if ((x1 - x0) * (y1 - y0) == 0 || radius < 1) continue;
        if (!s->colors_precomp) {
            /* direction from the UNSHIFTED mean (forward.cu:480,482 pass orig_points) */
            const float dx = fsub(s->means3D[3 * idx], s->cam_pos[0]), dy = fsub(s->means3D[3 * idx + 1], s->cam_pos[1]),
                        dz = fsub(s->means3D[3 * idx + 2], s->cam_pos[2]);
            const float len = sqrtf(ffma(dz, dz, ffma(dx, dx, fmul(dy, dy))));
            const float x = dx / len, y = dy / len, z = dz / len;
            float res[3];
            const float* sh = s->shs + (size_t)idx * s->M * 3;
            if (s->gaussian_dim == 3 || s->force_sh_3d) sh_color_3d(sh, s->D, x, y, z, res);
            else sh_color_4d(sh, s->D, s->D_t, x, y, z, fsub(s->ts[idx], s->timestamp), s->time_duration, res);
            for (int ch = 0; ch < 3; ++ch) {
                const float r = fadd(res[ch], 0.5f);
                g->clamped[3 * idx + ch] = (r < 0.f);
                g->rgb[3 * idx + ch] = (r < 0.f) ? 0.f : r;
            }
        }
        g->depths[idx] = vz;
        g->radii[idx] = radius;
        g->means2D[2 * idx] = ix;
        g->means2D[2 * idx + 1] = iy;
        g->conic_opacity[4 * idx] = conx; g->conic_opacity[4 * idx + 1] = cony;
        g->conic_opacity[4 * idx + 2] = conz; g->conic_opacity[4 * idx + 3] = opacity;
        g->tiles_touched[idx] = (uint32_t)((x1 - x0) * (y1 - y0));
        ++nvis;
    }
    return nvis;
}

/* ---- binning ----------------------------------------------------------------------------- */
/* reference: rasterizer_impl.cu:298 (inclusive scan), :71-112 duplicateWithKeys, :325-330 SortPairs
 * (stable LSD radix sort of 64-bit keys), :117-139 identifyTileRanges.
 * point_list must hold sum(tiles_touched) entries; ranges holds 2*gx*gy entries. Returns R. */
int64_t oracle_count_instances(const OracleGeom* g, int P) {
    int64_t R = 0;
    for (int i = 0; i < P; ++i) R += g->tiles_touched[i];
    return R;
}

int oracle_bin(int P, int W, int H, const OracleGeom* g, int64_t R, uint32_t* point_list, uint32_t* ranges) {
    const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
    memset(ranges, 0, sizeof(uint32_t) * 2 * (size_t)gx * gy);
    if (R == 0) return 0;
    uint64_t* keys = (uint64_t*)malloc(sizeof(uint64_t) * R);
    uint64_t* keys2 = (uint64_t*)malloc(sizeof(uint64_t) * R);
    uint32_t* vals = (uint32_t*)malloc(sizeof(uint32_t) * R);
    uint32_t* vals2 = (uint32_t*)malloc(sizeof(uint32_t) * R);
    if (!keys || !keys2 || !vals || !vals2) return -1;
    int64_t off = 0;
    for (int idx = 0; idx < P; ++idx) {
        if (g->radii[idx] <= 0) continue;
        int x0, y0, x1, y1;
        getRect(g->means2D[2 * idx], g->means2D[2 * idx + 1], g->radii[idx], gx, gy, &x0, &y0, &x1, &y1);
        uint32_t dbits;
        memcpy(&dbits, &g->depths[idx], 4);
        for (int y = y0; y < y1; ++y)
            for (int x = x0; x < x1; ++x) {
                keys[off] = ((uint64_t)(uint32_t)(y * gx + x) << 32) | dbits;
                vals[off] = (uint32_t)idx;
                ++off;
            }
    }
    if (off != R) return -2;
    /* stable LSD radix sort, 8 passes of 8 bits over all 64 key bits */
    for (int pass = 0; pass < 8; ++pass) {
        size_t cnt[257];
        memset(cnt, 0, sizeof(cnt));
        const int sh = 8 * pass;
        for (int64_t i = 0; i < R; ++i) cnt[((keys[i] >> sh) & 255) + 1]++;
        for (int i = 0; i < 256; ++i) cnt[i + 1] += cnt[i];
        for (int64_t i = 0; i < R; ++i) {
            const size_t d = cnt[(keys[i] >> sh) & 255]++;
            keys2[d] = keys[i];
            vals2[d] = vals[i];
        }
        uint64_t* tk = keys; keys = keys2; keys2 = tk;
        uint32_t* tv = vals; vals = vals2; vals2 = tv;
    }
    for (int64_t i = 0; i < R; ++i) {
        point_list[i] = vals[i];
        const uint32_t tile = (uint32_t)(keys[i] >> 32);
        if (i == 0) ranges[2 * tile] = 0;
        else {
            const uint32_t prev = (uint32_t)(keys[i - 1] >> 32);
            if (prev != tile) {
                ranges[2 * prev + 1] = (uint32_t)i;
                ranges[2 * tile] = (uint32_t)i;
            }
        }
        if (i == R - 1) ranges[2 * tile + 1] = (uint32_t)R;
    }
    free(keys); free(keys2); free(vals); free(vals2);
    return 0;
}

/* ---- forward blend ---------------------------------------------------------------------------- */
/* reference: forward.cu:501-626 renderCUDA.  One pixel at a time; `done` semantics identical
 * (the block-wide early exit of the reference does not change any result). */
void oracle_render_forward(int W, int H, const uint32_t* ranges, const uint32_t* point_list, const float* means2D,
                           const float* features, const float* flows, const float* depths, const float* conic_opacity,
                           const float* bg, float* final_T, uint32_t* n_contrib, float* out_color, float* out_flow,
                           float* out_depth) {
    const int gx = (W + BLOCK_X - 1) / BLOCK_X;
    const size_t HW = (size_t)H * W;
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 4)
#endif
    for (int py = 0; py < H; ++py) {
        for (int px = 0; px < W; ++px) {
            const int tile = (py / BLOCK_Y) * gx + (px / BLOCK_X);
            const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
            const float pixfx = (float)px, pixfy = (float)py;
            float T = 1.0f, C[3] = {0, 0, 0}, Fl[2] = {0, 0}, D = 0;
            uint32_t contributor = 0, last_contributor = 0;
            for (uint32_t i = r0; i < r1; ++i) {
                contributor++;
                const uint32_t id = point_list[i];
                const float dx = fsub(means2D[2 * id], pixfx), dy = fsub(means2D[2 * id + 1], pixfy);
                const float* co = conic_opacity + 4 * id;
                /* forward.cu:581 as compiled: fma(fma(dx, dx*A, dy*(dy*C)), -0.5, -(dy*(dx*B))) */
                const float power = ffma(ffma(dx, fmul(dx, co[0]), fmul(dy, fmul(dy, co[2]))), -0.5f,
                                         -fmul(dy, fmul(dx, co[1])));
                if (power > 0.0f) continue;
                const float alpha = fminf(fmul(co[3], expf(power)), 0.99f);
                if (alpha < 1.0f / 255.0f) continue;
                const float test_T = fmul(T, fsub(1.0f, alpha));
                if (test_T < 0.0001f) break; /* done = true */
                for (int ch = 0; ch < 3; ++ch) C[ch] = ffma(T, fmul(alpha, features[3 * id + ch]), C[ch]);
                for (int ch = 0; ch < 2; ++ch) Fl[ch] = ffma(T, fmul(alpha, flows[2 * id + ch]), Fl[ch]);
                D = ffma(T, fmul(alpha, depths[id]), D);
                T = test_T;
                last_contributor = contributor;
            }
            const size_t pid = (size_t)py * W + px;
            final_T[pid] = T;
            n_contrib[pid] = last_contributor;
            for (int ch = 0; ch < 3; ++ch) out_color[ch * HW + pid] = ffma(T, bg[ch], C[ch]);
            out_flow[pid] = Fl[0];
            out_flow[HW + pid] = Fl[1];
            out_depth[pid] = D;
        }
    }
}

/* ---- backward blend --------------------------------------------------------------------------- */
/* reference: backward.cu:926-1137 renderCUDA.  Accumulates into zero-initialised per-Gaussian
 * arrays: dL_dmean2D [P,3], dL_dconic [P,4] (x,y,-,w), dL_dopacity [P], dL_dcolors [P,3], dL_dflows [P,2]. */
void oracle_render_backward(int W, int H, const uint32_t* ranges, const uint32_t* point_list, const float* bg,
                            const float* means2D, const float* conic_opacity, const float* colors, const float* depths,
                            const float* flows, const float* final_Ts, const uint32_t* n_contrib, const float* dL_dpixels,
                            const float* dL_depths, const float* dL_masks, const float* dL_dpix_flow, float* dL_dmean2D,
                            float* dL_dconic, float* dL_dopacity, float* dL_dcolors, float* dL_dflows) {
    const int gx = (W + BLOCK_X - 1) / BLOCK_X;
    const size_t HW = (size_t)H * W;
    const float ddelx_dx = (float)(0.5 * W), ddely_dy = (float)(0.5 * H);
    /* double accumulators are not used: the reference sums in fp32 (atomicAdd); order differs anyway */
    for (int py = 0; py < H; ++py) {
        for (int px = 0; px < W; ++px) {
            const int tile = (py / BLOCK_Y) * gx + (px / BLOCK_X);
            const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
            const size_t pid = (size_t)py * W + px;
            const float pixfx = (float)px, pixfy = (float)py;
            const float T_final = final_Ts[pid];
            float T = T_final;
            const uint32_t last_contributor = n_contrib[pid];
            float accum_rec[3] = {0, 0, 0}, accum_flow[2] = {0, 0}, accum_depth = 0, accum_mask = 0;
            float dL_dpixel[3], dL_dflow[2];
            for (int i = 0; i < 3; ++i) dL_dpixel[i] = dL_dpixels[i * HW + pid];
            for (int i = 0; i < 2; ++i) dL_dflow[i] = dL_dpix_flow[i * HW + pid];
            const float dL_depth = dL_depths[pid], dL_mask = dL_masks[pid];
            float last_alpha = 0, last_color[3] = {0, 0, 0}, last_flow[2] = {0, 0}, last_depth = 0;
            uint32_t contributor = r1 - r0;
            for (uint32_t i = r1; i-- > r0;) {
                contributor--;
                if (contributor >= last_contributor) continue;
                const uint32_t id = point_list[i];
                const float dx = fsub(means2D[2 * id], pixfx), dy = fsub(means2D[2 * id + 1], pixfy);
                const float* co = conic_opacity + 4 * id;
                const float power = ffma(ffma(dx, fmul(dx, co[0]), fmul(dy, fmul(dy, co[2]))), -0.5f,
                                         -fmul(dy, fmul(dx, co[1])));
                if (power > 0.0f) continue;
                const float G = expf(power);
                const float alpha = fminf(fmul(co[3], G), 0.99f);
                if (alpha < 1.0f / 255.0f) continue;
                T = T / (1.f - alpha);
                const float dchannel_dcolor = alpha * T;
                float dL_dalpha = 0.0f;
                for (int ch = 0; ch < 3; ++ch) {
                    const float c = colors[3 * id + ch];
                    accum_rec[ch] = last_alpha * last_color[ch] + (1.f - last_alpha) * accum_rec[ch];
                    last_color[ch] = c;
                    dL_dalpha += (c - accum_rec[ch]) * dL_dpixel[ch];
                    dL_dcolors[3 * id + ch] += dchannel_dcolor * dL_dpixel[ch];
                }
                for (int ch = 0; ch < 2; ++ch) {
                    const float f = flows[2 * id + ch];
                    accum_flow[ch] = last_alpha * last_flow[ch] + (1.f - last_alpha) * accum_flow[ch];
                    last_flow[ch] = f;
                    dL_dalpha += (f - accum_flow[ch]) * dL_dflow[ch];
                    dL_dflows[2 * id + ch] += dchannel_dcolor * dL_dflow[ch];
                }
                const float c_d = depths[id];
                accum_depth = last_alpha * last_depth + (1.f - last_alpha) * accum_depth;
                last_depth = c_d;
                dL_dalpha += ((c_d - accum_depth) * dL_depth);
                accum_mask = last_alpha + (1.f - last_alpha) * accum_mask;
                dL_dalpha = (float)((double)dL_dalpha + ((1.0 - (double)accum_mask) * (double)dL_mask)); /* :1102 */
                dL_dalpha *= T;
                last_alpha = alpha;
                float bg_dot_dpixel = 0;
                for (int k = 0; k < 3; ++k) bg_dot_dpixel += bg[k] * dL_dpixel[k];
                dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot_dpixel;
                const float dL_dG = co[3] * dL_dalpha;
                const float gdx = G * dx, gdy = G * dy;
                const float dG_ddelx = -gdx * co[0] - gdy * co[1];
                const float dG_ddely = -gdy * co[2] - gdx * co[1];
                dL_dmean2D[3 * id + 0] += dL_dG * dG_ddelx * ddelx_dx;
                dL_dmean2D[3 * id + 1] += dL_dG * dG_ddely * ddely_dy;
                dL_dmean2D[3 * id + 2] += dL_depth * dchannel_dcolor;
                dL_dconic[4 * id + 0] += -0.5f * gdx * dx * dL_dG;
                dL_dconic[4 * id + 1] += -0.5f * gdx * dy * dL_dG;
                dL_dconic[4 * id + 3] += -0.5f * gdy * dy * dL_dG;
                dL_dopacity[id] += G * dL_dalpha;
            }
        }
    }
}

/* ---- backward preprocess ------------------------------------------------------------------- */
static void dnormvdv(const float v[3], const float dv[3], float out[3]) { /* auxiliary.h:108-118 */
    const float sum2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    const float inv = 1.0f / sqrtf(sum2 * sum2 * sum2);
    out[0] = ((+sum2 - v[0] * v[0]) * dv[0] - v[1] * v[0] * dv[1] - v[2] * v[0] * dv[2]) * inv;
    out[1] = (-v[0] * v[1] * dv[0] + (sum2 - v[1] * v[1]) * dv[1] - v[2] * v[1] * dv[2]) * inv;
    out[2] = (-v[0] * v[2] * dv[0] - v[1] * v[2] * dv[1] + (sum2 - v[2] * v[2]) * dv[2]) * inv;
}

/* glm-style products on [c][r] arrays */
static void mul4(const float A[4][4], const float B[4][4], float C[4][4]) {
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 4; ++r) C[c][r] = A[0][r] * B[c][0] + A[1][r] * B[c][1] + A[2][r] * B[c][2] + A[3][r] * B[c][3];
}
static void mul3(const float A[3][3], const float B[3][3], float C[3][3]) {
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) C[c][r] = A[0][r] * B[c][0] + A[1][r] * B[c][1] + A[2][r] * B[c][2];
}

/* SH backward: reference backward.cu:20-139 (3D) and :144-481 (4D, with its observable bugs:
 * dL_dsh[1] = l0m0*dL_dRGB (:190), no minus sign in dt*_dt (:303,:384), dRGBdt overwritten (:403)). */
static void sh_backward(const OracleScene* s, int idx, int is4d, const float mean[3], const uint8_t* clamped,
                        const float* dL_dcolor, float* dL_dmeans, float* dL_dsh, float* dL_dts) {
    const int deg = s->D, deg_t = s->D_t, M = s->M;
    const float* sh = s->shs + (size_t)idx * M * 3;
    float* dsh = dL_dsh + (size_t)idx * M * 3;
    const float dir_orig[3] = {mean[0] - s->cam_pos[0], mean[1] - s->cam_pos[1], mean[2] - s->cam_pos[2]};
    const float len = sqrtf(dir_orig[0] * dir_orig[0] + dir_orig[1] * dir_orig[1] + dir_orig[2] * dir_orig[2]);
    const float x = dir_orig[0] / len, y = dir_orig[1] / len, z = dir_orig[2] / len;
    float dRGB[3];
    for (int ch = 0; ch < 3; ++ch) dRGB[ch] = clamped[3 * idx + ch] ? 0.f : dL_dcolor[3 * idx + ch];
    float l[16], dlx[16], dly[16], dlz[16];
    for (int i = 0; i < 16; ++i) l[i] = dlx[i] = dly[i] = dlz[i] = 0.f;
    int nb = 1;
    l[0] = SH_C0;
    if (deg > 0) {
        nb = 4;
        l[1] = -SH_C1 * y; dly[1] = -SH_C1;
        l[2] = SH_C1 * z; dlz[2] = SH_C1;
        l[3] = -SH_C1 * x; dlx[3] = -SH_C1;
        if (deg > 1) {
            nb = 9;
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            l[4] = SH_C2[0] * xy; dlx[4] = SH_C2[0] * y; dly[4] = SH_C2[0] * x;
            l[5] = SH_C2[1] * yz; dly[5] = SH_C2[1] * z; dlz[5] = SH_C2[1] * y;
            l[6] = SH_C2[2] * (2.f * zz - xx - yy); dlx[6] = -2 * SH_C2[2] * x; dly[6] = -2 * SH_C2[2] * y; dlz[6] = 4 * SH_C2[2] * z;
            l[7] = SH_C2[3] * xz; dlx[7] = SH_C2[3] * z; dlz[7] = SH_C2[3] * x;
            l[8] = SH_C2[4] * (xx - yy); dlx[8] = 2 * SH_C2[4] * x; dly[8] = -2 * SH_C2[4] * y;
            if (deg > 2) {
                nb = 16;
                l[9] = SH_C3[0] * y * (3 * xx - yy); dlx[9] = SH_C3[0] * y * 6 * x; dly[9] = SH_C3[0] * (3 * xx - 3 * yy);
                l[10] = SH_C3[1] * xy * z; dlx[10] = SH_C3[1] * yz; dly[10] = SH_C3[1] * xz; dlz[10] = SH_C3[1] * xy;
                l[11] = SH_C3[2] * y * (4 * zz - xx - yy); dlx[11] = -SH_C3[2] * y * 2 * x;
                dly[11] = SH_C3[2] * (4 * zz - xx - 3 * yy); dlz[11] = SH_C3[2] * y * 8 * z;
                l[12] = SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy); dlx[12] = -SH_C3[3] * z * 6 * x;
                dly[12] = -SH_C3[3] * z * 6 * y; dlz[12] = SH_C3[3] * (6 * zz - 3 * xx - 3 * yy);
                l[13] = SH_C3[4] * x * (4 * zz - xx - yy); dlx[13] = SH_C3[4] * (4 * zz - 3 * xx - yy);
                dly[13] = -SH_C3[4] * x * 2 * y; dlz[13] = SH_C3[4] * x * 8 * z;
                l[14] = SH_C3[5] * z * (xx - yy); dlx[14] = SH_C3[5] * z * 2 * x; dly[14] = -SH_C3[5] * z * 2 * y;
                dlz[14] = SH_C3[5] * (xx - yy);
                l[15] = SH_C3[6] * x * (xx - 3 * yy); dlx[15] = SH_C3[6] * (3 * xx - 3 * yy); dly[15] = -SH_C3[6] * x * 6 * y;
            }
        }
    }
    float dRGBdx[3] = {0, 0, 0}, dRGBdy[3] = {0, 0, 0}, dRGBdz[3] = {0, 0, 0}, dRGBdt[3] = {0, 0, 0};
    const int nblk = (is4d && deg > 2) ? 1 + (deg_t > 2 ? 2 : deg_t) : 1;
    for (int blk = 0; blk < nblk; ++blk) {
        float tw = 1.f, dtw = 0.f;
        if (blk > 0) {
            const float dir_t = s->ts[idx] - s->timestamp;
            const double w = 2 * MY_PI * (double)dir_t * (blk == 2 ? 2.0 : 1.0) / (double)s->time_duration;
            tw = (float)cos(w);
            dtw = (float)(sin(w) * 2 * MY_PI * (blk == 2 ? 2.0 : 1.0) / (double)s->time_duration);
        }
        for (int k = 0; k < nb; ++k) {
            const int c = 16 * blk + k;
            float wk = tw * l[k];
            if (blk == 0) wk = (is4d && k == 1) ? l[0] : l[k]; /* quirk :190 */
            for (int ch = 0; ch < 3; ++ch) {
                dsh[3 * c + ch] = wk * dRGB[ch];
                dRGBdx[ch] += tw * dlx[k] * sh[3 * c + ch];
                dRGBdy[ch] += tw * dly[k] * sh[3 * c + ch];
                dRGBdz[ch] += tw * dlz[k] * sh[3 * c + ch];
            }
        }
        if (blk > 0)
            for (int ch = 0; ch < 3; ++ch) {
                float acc = 0.f;
                for (int k = 0; k < 16; ++k) acc += l[k] * sh[3 * (16 * blk + k) + ch];
                dRGBdt[ch] = dtw * acc; /* assignment: the t2 term overwrites the t1 term (:403) */
            }
    }
    float dL_ddir[3] = {0, 0, 0};
    for (int ch = 0; ch < 3; ++ch) {
        dL_ddir[0] += dRGBdx[ch] * dRGB[ch];
        dL_ddir[1] += dRGBdy[ch] * dRGB[ch];
        dL_ddir[2] += dRGBdz[ch] * dRGB[ch];
    }
    float dm[3];
    dnormvdv(dir_orig, dL_ddir, dm);
    for (int k = 0; k < 3; ++k) dL_dmeans[3 * idx + k] += dm[k];
    if (is4d) dL_dts[idx] += dRGBdt[0] * dRGB[0] + dRGBdt[1] * dRGB[1] + dRGBdt[2] * dRGB[2];
}

/* reference: backward.cu:486-617 computeCov2DCUDA followed by backward.cu:839-923 preprocessCUDA.
 * All outputs except dL_dopacity (in/out) must be zero-initialised by the caller. */
void oracle_preprocess_backward(const OracleScene* s, const float* means /* shifted, [P,3] */, const int* radii,
                                const uint8_t* clamped, const uint32_t* tiles_touched, const float* cov3Ds,
                                const float* dL_dmean2D, const float* dL_dconics, float* dL_dopacity,
                                const float* dL_dcolor, float* dL_dmeans, float* dL_dcov, float* dL_dsh, float* dL_dts,
                                float* dL_dscale, float* dL_dscale_t, float* dL_drot, float* dL_drot_r) {
    const float h_y = s->H / (2.0f * s->tan_fovy);
    const float h_x = s->W / (2.0f * s->tan_fovx);
    const float* V = s->viewmatrix;
    const float* proj = s->projmatrix;
    for (int idx = 0; idx < s->P; ++idx) {
        if (!(radii[idx] > 0)) continue;
        const float* cov3D = cov3Ds + 6 * idx;
        const float mean[3] = {means[3 * idx], means[3 * idx + 1], means[3 * idx + 2]};
        { /* computeCov2DCUDA */
            const float dcx = dL_dconics[4 * idx], dcy = dL_dconics[4 * idx + 1], dcz = dL_dconics[4 * idx + 3];
            ProjT Pj;
            build_T(V, mean[0], mean[1], mean[2], h_x, h_y, s->tan_fovx, s->tan_fovy, &Pj);
            const float limx = 1.3f * s->tan_fovx, limy = 1.3f * s->tan_fovy;
            const float x_grad_mul = (Pj.txtz < -limx || Pj.txtz > limx) ? 0.f : 1.f;
            const float y_grad_mul = (Pj.tytz < -limy || Pj.tytz > limy) ? 0.f : 1.f;
            float a, b, c;
            cov2d(&Pj, cov3D, &a, &b, &c);
            a += 0.3f;
            c += 0.3f;
            const float (*T)[3] = Pj.T;
            const float denom = a * c - b * b;
            float dL_da = 0, dL_db = 0, dL_dc = 0;
            const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
            float* dc = dL_dcov + 6 * idx;
            if (denom2inv != 0) {
                dL_da = denom2inv * (-c * c * dcx + 2 * b * c * dcy + (denom - a * c) * dcz);
                dL_dc = denom2inv * (-a * a * dcz + 2 * a * b * dcy + (denom - a * c) * dcx);
                dL_db = denom2inv * 2 * (b * c * dcx - (denom + 2 * b * b) * dcy + a * b * dcz);
                dc[0] = (T[0][0] * T[0][0] * dL_da + T[0][0] * T[1][0] * dL_db + T[1][0] * T[1][0] * dL_dc);
                dc[3] = (T[0][1] * T[0][1] * dL_da + T[0][1] * T[1][1] * dL_db + T[1][1] * T[1][1] * dL_dc);
                dc[5] = (T[0][2] * T[0][2] * dL_da + T[0][2] * T[1][2] * dL_db + T[1][2] * T[1][2] * dL_dc);
                dc[1] = 2 * T[0][0] * T[0][1] * dL_da + (T[0][0] * T[1][1] + T[0][1] * T[1][0]) * dL_db + 2 * T[1][0] * T[1][1] * dL_dc;
                dc[2] = 2 * T[0][0] * T[0][2] * dL_da + (T[0][0] * T[1][2] + T[0][2] * T[1][0]) * dL_db + 2 * T[1][0] * T[1][2] * dL_dc;
                dc[4] = 2 * T[0][2] * T[0][1] * dL_da + (T[0][1] * T[1][2] + T[0][2] * T[1][1]) * dL_db + 2 * T[1][1] * T[1][2] * dL_dc;
            } else {
                for (int i = 0; i < 6; ++i) dc[i] = 0;
            }
            const float Vrk[3][3] = {{cov3D[0], cov3D[1], cov3D[2]}, {cov3D[1], cov3D[3], cov3D[4]}, {cov3D[2], cov3D[4], cov3D[5]}};
            float dL_dT[2][3];
            for (int j = 0; j < 3; ++j) {
                const float r0 = T[0][0] * Vrk[j][0] + T[0][1] * Vrk[j][1] + T[0][2] * Vrk[j][2];
                const float r1 = T[1][0] * Vrk[j][0] + T[1][1] * Vrk[j][1] + T[1][2] * Vrk[j][2];
                dL_dT[0][j] = 2 * r0 * dL_da + r1 * dL_db;
                dL_dT[1][j] = 2 * r1 * dL_dc + r0 * dL_db;
            }
            /* W[c][r] = V[4*r + c] */
            const float dL_dJ00 = V[0] * dL_dT[0][0] + V[4] * dL_dT[0][1] + V[8] * dL_dT[0][2];
            const float dL_dJ02 = V[2] * dL_dT[0][0] + V[6] * dL_dT[0][1] + V[10] * dL_dT[0][2];
            const float dL_dJ11 = V[1] * dL_dT[1][0] + V[5] * dL_dT[1][1] + V[9] * dL_dT[1][2];
            const float dL_dJ12 = V[2] * dL_dT[1][0] + V[6] * dL_dT[1][1] + V[10] * dL_dT[1][2];
            const float tz = 1.f / Pj.tz, tz2 = tz * tz, tz3 = tz2 * tz;
            const float dL_dtx = x_grad_mul * -h_x * tz2 * dL_dJ02;
            const float dL_dty = y_grad_mul * -h_y * tz2 * dL_dJ12;
            const float dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * Pj.tx) * tz3 * dL_dJ02 +
                                 (2 * h_y * Pj.ty) * tz3 * dL_dJ12;
            const float vx = dL_dtx, vy = dL_dty, vz = dL_dtz + dL_dmean2D[3 * idx + 2];
            dL_dmeans[3 * idx + 0] = V[0] * vx + V[1] * vy + V[2] * vz; /* assignment, :616 */
            dL_dmeans[3 * idx + 1] = V[4] * vx + V[5] * vy + V[6] * vz;
            dL_dmeans[3 * idx + 2] = V[8] * vx + V[9] * vy + V[10] * vz;
        }
        if (tiles_touched[idx] == 0) continue; /* backward.cu:875 */
        { /* mean2D -> mean3D, backward.cu:877-894 */
            const float m_w = 1.0f / ((proj[3] * mean[0] + proj[7] * mean[1] + proj[11] * mean[2] + proj[15]) + 0.0000001f);
            const float mul1 = (proj[0] * mean[0] + proj[4] * mean[1] + proj[8] * mean[2] + proj[12]) * m_w * m_w;
            const float mul2 = (proj[1] * mean[0] + proj[5] * mean[1] + proj[9] * mean[2] + proj[13]) * m_w * m_w;
            const float gx = dL_dmean2D[3 * idx], gy = dL_dmean2D[3 * idx + 1];
            dL_dmeans[3 * idx + 0] += (proj[0] * m_w - proj[3] * mul1) * gx + (proj[1] * m_w - proj[3] * mul2) * gy;
            dL_dmeans[3 * idx + 1] += (proj[4] * m_w - proj[7] * mul1) * gx + (proj[5] * m_w - proj[7] * mul2) * gy;
            dL_dmeans[3 * idx + 2] += (proj[8] * m_w - proj[11] * mul1) * gx + (proj[9] * m_w - proj[11] * mul2) * gy;
        }
        if (s->shs) {
            const int is4d = !(s->gaussian_dim == 3 || s->force_sh_3d);
            sh_backward(s, idx, is4d, mean, clamped, dL_dcolor, dL_dmeans, dL_dsh, dL_dts);
        }
        if (!s->scales) continue;
        const float mod = s->scale_modifier;
        const float* d = dL_dcov + 6 * idx;
        if (s->rot_4d) { /* backward.cu:689-834 */
            const float dt = s->timestamp - s->ts[idx];
            const float sc[4] = {mod * s->scales[3 * idx], mod * s->scales[3 * idx + 1], mod * s->scales[3 * idx + 2], mod * s->scales_t[idx]};
            float M[4][4], R[4][4];
            build_M4(sc, s->rotations + 4 * idx, s->rotations_r + 4 * idx, M, R);
            const float cov_t = coldot4(M[3], M[3]);
            const float ctp = (s->prefilter_var > 0.0f) ? (s->prefilter_var + cov_t) : cov_t;
            const float marginal = marginal_of(dt, cov_t, s->prefilter_var);
            if (!((double)marginal > 0.05)) continue;
            const float c12[3] = {coldot4(M[3], M[0]), coldot4(M[3], M[1]), coldot4(M[3], M[2])};
            float dc12[3];
            dc12[0] = -(d[0] * c12[0] + d[1] * c12[1] * 0.5f + d[2] * c12[2] * 0.5f) * 2.0f / cov_t;
            dc12[1] = -(d[1] * c12[0] * 0.5f + d[3] * c12[1] + d[4] * c12[2] * 0.5f) * 2.0f / cov_t;
            dc12[2] = -(d[2] * c12[0] * 0.5f + d[4] * c12[1] * 0.5f + d[5] * c12[2]) * 2.0f / cov_t;
            float dcovt = (c12[0] * c12[0] * d[0] + c12[0] * c12[1] * d[1] + c12[0] * c12[2] * d[2] + c12[1] * c12[1] * d[3] +
                           c12[1] * c12[2] * d[4] + c12[2] * c12[2] * d[5]) / (cov_t * cov_t);
            const float dmarg = dL_dopacity[idx] * s->opacities[idx];
            dL_dopacity[idx] *= marginal;
            dcovt += (marginal * dt * dt / 2 / (ctp * ctp)) * dmarg;
            float dL_dt = dmarg * (marginal * dt / ctp);
            const float* dm = dL_dmeans + 3 * idx;
            for (int k = 0; k < 3; ++k) dc12[k] += dm[k] / cov_t * dt;
            const float ddot = dm[0] * c12[0] + dm[1] * c12[1] + dm[2] * c12[2];
            dcovt += -ddot / (cov_t * cov_t) * dt;
            dL_dt += -ddot / cov_t;
            dL_dts[idx] += dL_dt;
            const float dS[4][4] = {{d[0], 0.5f * d[1], 0.5f * d[2], 0.5f * dc12[0]},
                                    {0.5f * d[1], d[3], 0.5f * d[4], 0.5f * dc12[1]},
                                    {0.5f * d[2], 0.5f * d[4], d[5], 0.5f * dc12[2]},
                                    {0.5f * dc12[0], 0.5f * dc12[1], 0.5f * dc12[2], dcovt}};
            float M2[4][4], dM[4][4], N[4][4];
            for (int c = 0; c < 4; ++c)
                for (int r = 0; r < 4; ++r) M2[c][r] = 2.0f * M[c][r];
            mul4(M2, dS, dM);
            float gs[4];
            for (int i = 0; i < 4; ++i) { /* dot(Rt[i], dL_dMt[i]); then dL_dMt[i] *= s_i */
                gs[i] = 0.f;
                for (int c = 0; c < 4; ++c) {
                    gs[i] += R[c][i] * dM[c][i];
                    N[i][c] = sc[i] * dM[c][i];
                }
            }
            dL_dscale[3 * idx] = gs[0]; dL_dscale[3 * idx + 1] = gs[1]; dL_dscale[3 * idx + 2] = gs[2];
            dL_dscale_t[idx] = gs[3];
            const float* rot = s->rotations + 4 * idx;
            const float* rr = s->rotations_r + 4 * idx;
            const float Ml[4][4] = {{rot[0], rot[1], -rot[2], rot[3]}, {-rot[1], rot[0], rot[3], rot[2]},
                                    {rot[2], -rot[3], rot[0], rot[1]}, {-rot[3], -rot[2], -rot[1], rot[0]}};
            const float Mr[4][4] = {{rr[0], rr[1], -rr[2], -rr[3]}, {-rr[1], rr[0], rr[3], -rr[2]},
                                    {rr[2], -rr[3], rr[0], -rr[1]}, {rr[3], rr[2], rr[1], rr[0]}};
            float X[4][4], Y[4][4];
            mul4(N, Mr, X);
            mul4(Ml, N, Y);
            float* q = dL_drot + 4 * idx;
            q[0] = X[0][0] + X[1][1] + X[2][2] + X[3][3];
            q[1] = -X[0][1] + X[1][0] - X[2][3] + X[3][2];
            q[2] = X[0][2] - X[1][3] - X[2][0] + X[3][1];
            q[3] = -X[0][3] - X[1][2] + X[2][1] + X[3][0];
            float* qr = dL_drot_r + 4 * idx;
            qr[0] = Y[0][0] + Y[1][1] + Y[2][2] + Y[3][3];
            qr[1] = -Y[0][1] + Y[1][0] + Y[2][3] - Y[3][2];
            qr[2] = Y[0][2] + Y[1][3] - Y[2][0] - Y[3][1];
            qr[3] = Y[0][3] - Y[1][2] + Y[2][1] - Y[3][0];
        } else { /* backward.cu:621-684 */
            const float sc[3] = {mod * s->scales[3 * idx], mod * s->scales[3 * idx + 1], mod * s->scales[3 * idx + 2]};
            const float* q = s->rotations + 4 * idx;
            const float r = q[0], x = q[1], y = q[2], z = q[3];
            const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                                   {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                                   {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
            float M2[3][3], dM[3][3], Nt[3][3];
            for (int c = 0; c < 3; ++c)
                for (int rr = 0; rr < 3; ++rr) M2[c][rr] = 2.0f * sc[rr] * R[c][rr];
            const float dS[3][3] = {{d[0], 0.5f * d[1], 0.5f * d[2]}, {0.5f * d[1], d[3], 0.5f * d[4]}, {0.5f * d[2], 0.5f * d[4], d[5]}};
            mul3(M2, dS, dM);
            for (int i = 0; i < 3; ++i) {
                float acc = 0.f;
                for (int c = 0; c < 3; ++c) {
                    acc += R[c][i] * dM[c][i];
                    Nt[i][c] = sc[i] * dM[c][i];
                }
                dL_dscale[3 * idx + i] = acc;
            }
            float* dq = dL_drot + 4 * idx;
            dq[0] = 2 * z * (Nt[0][1] - Nt[1][0]) + 2 * y * (Nt[2][0] - Nt[0][2]) + 2 * x * (Nt[1][2] - Nt[2][1]);
            dq[1] = 2 * y * (Nt[1][0] + Nt[0][1]) + 2 * z * (Nt[2][0] + Nt[0][2]) + 2 * r * (Nt[1][2] - Nt[2][1]) - 4 * x * (Nt[2][2] + Nt[1][1]);
            dq[2] = 2 * x * (Nt[1][0] + Nt[0][1]) + 2 * r * (Nt[2][0] - Nt[0][2]) + 2 * z * (Nt[1][2] + Nt[2][1]) - 4 * y * (Nt[2][2] + Nt[0][0]);
            dq[3] = 2 * r * (Nt[0][1] - Nt[1][0]) + 2 * x * (Nt[2][0] + Nt[0][2]) + 2 * y * (Nt[1][2] + Nt[2][1]) - 4 * z * (Nt[1][1] + Nt[0][0]);
        }
    }
}

/* The camera's per-row gradient terms: the reference backward's own per-Gaussian arithmetic (computeCov2DCUDA,
 * preprocessCUDA's projection, the SH view direction) applied to the view matrix V, the projection Pm and the camera
 * position instead of the mean.  terms [P,27], zero-initialised by the caller, row idx written when the row is rendered
 * (radius > 0 and at least one tile), in this order:
 *   3c + r (c, r < 3)  dL/dV[4c + r] = m_c g_r + sum_i J[i][r] dL/dT[i][c]   (t = W m + V[12..14], T = J W)
 *   9 + r              dL/dV[12 + r] = g_r                                   (g: the view-space point's gradient)
 *   12 + 3c + j        dL/dPm[4c + r_j] = m_c gp_j, m_3 = 1, r_j = 0, 1, 3    (gp = dL/d(clip x, y, w))
 *   24 + k             dL/dcampos[k] = -(the SH direction part of dL/dmean[k])
 * Inputs as oracle_preprocess_backward's. */
void oracle_camera_terms(const OracleScene* s, const float* means /* shifted, [P,3] */, const int* radii,
                         const uint8_t* clamped, const uint32_t* tiles_touched, const float* cov3Ds,
                         const float* dL_dmean2D, const float* dL_dconics, const float* dL_dcolor, float* terms) {
    const float h_y = s->H / (2.0f * s->tan_fovy);
    const float h_x = s->W / (2.0f * s->tan_fovx);
    const float* V = s->viewmatrix;
    const float* proj = s->projmatrix;
    float* sh_mean = NULL;
    float* sh_dsh = NULL;
    float* sh_dts = NULL;
    if (s->shs) {
        sh_mean = (float*)calloc((size_t)s->P * 3, sizeof(float));
        sh_dsh = (float*)calloc((size_t)s->P * (s->M > 0 ? s->M : 1) * 3, sizeof(float));
        sh_dts = (float*)calloc((size_t)s->P, sizeof(float));
        if (!sh_mean || !sh_dsh || !sh_dts) abort();
    }
    for (int idx = 0; idx < s->P; ++idx) {
        if (!(radii[idx] > 0) || tiles_touched[idx] == 0) continue;
        float* out = terms + 27 * (size_t)idx;
        const float* cov3D = cov3Ds + 6 * idx;
        const float mean[3] = {means[3 * idx], means[3 * idx + 1], means[3 * idx + 2]};
        { /* computeCov2DCUDA */
            const float dcx = dL_dconics[4 * idx], dcy = dL_dconics[4 * idx + 1], dcz = dL_dconics[4 * idx + 3];
            ProjT Pj;
            build_T(V, mean[0], mean[1], mean[2], h_x, h_y, s->tan_fovx, s->tan_fovy, &Pj);
            const float limx = 1.3f * s->tan_fovx, limy = 1.3f * s->tan_fovy;
            const float x_grad_mul = (Pj.txtz < -limx || Pj.txtz > limx) ? 0.f : 1.f;
            const float y_grad_mul = (Pj.tytz < -limy || Pj.tytz > limy) ? 0.f : 1.f;
            float a, b, c;
            cov2d(&Pj, cov3D, &a, &b, &c);
            a += 0.3f;
            c += 0.3f;
            const float (*T)[3] = Pj.T;
            const float denom = a * c - b * b;
            float dL_da = 0, dL_db = 0, dL_dc = 0;
            const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
            if (denom2inv != 0) {
                dL_da = denom2inv * (-c * c * dcx + 2 * b * c * dcy + (denom - a * c) * dcz);
                dL_dc = denom2inv * (-a * a * dcz + 2 * a * b * dcy + (denom - a * c) * dcx);
                dL_db = denom2inv * 2 * (b * c * dcx - (denom + 2 * b * b) * dcy + a * b * dcz);
            }
            const float Vrk[3][3] = {{cov3D[0], cov3D[1], cov3D[2]}, {cov3D[1], cov3D[3], cov3D[4]}, {cov3D[2], cov3D[4], cov3D[5]}};
            float dL_dT[2][3];
            for (int j = 0; j < 3; ++j) {
                const float r0 = T[0][0] * Vrk[j][0] + T[0][1] * Vrk[j][1] + T[0][2] * Vrk[j][2];
                const float r1 = T[1][0] * Vrk[j][0] + T[1][1] * Vrk[j][1] + T[1][2] * Vrk[j][2];
                dL_dT[0][j] = 2 * r0 * dL_da + r1 * dL_db;
                dL_dT[1][j] = 2 * r1 * dL_dc + r0 * dL_db;
            }
            const float dL_dJ00 = V[0] * dL_dT[0][0] + V[4] * dL_dT[0][1] + V[8] * dL_dT[0][2];
            const float dL_dJ02 = V[2] * dL_dT[0][0] + V[6] * dL_dT[0][1] + V[10] * dL_dT[0][2];
            const float dL_dJ11 = V[1] * dL_dT[1][0] + V[5] * dL_dT[1][1] + V[9] * dL_dT[1][2];
            const float dL_dJ12 = V[2] * dL_dT[1][0] + V[6] * dL_dT[1][1] + V[10] * dL_dT[1][2];
            const float tz = 1.f / Pj.tz, tz2 = tz * tz, tz3 = tz2 * tz;
            const float vx = x_grad_mul * -h_x * tz2 * dL_dJ02;
            const float vy = y_grad_mul * -h_y * tz2 * dL_dJ12;
            const float vz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * Pj.tx) * tz3 * dL_dJ02 +
                             (2 * h_y * Pj.ty) * tz3 * dL_dJ12 + dL_dmean2D[3 * idx + 2];
            /* the Jacobian J of forward.cu:204-223 with the clamped tx, ty */
            const float j00 = h_x / Pj.tz, j11 = h_y / Pj.tz;
            const float j02 = (h_x * -Pj.tx) / (Pj.tz * Pj.tz), j12 = (h_y * -Pj.ty) / (Pj.tz * Pj.tz);
            for (int cc = 0; cc < 3; ++cc) {
                out[3 * cc + 0] = mean[cc] * vx + j00 * dL_dT[0][cc];
                out[3 * cc + 1] = mean[cc] * vy + j11 * dL_dT[1][cc];
                out[3 * cc + 2] = mean[cc] * vz + (j02 * dL_dT[0][cc] + j12 * dL_dT[1][cc]);
            }
            out[9] = vx;
            out[10] = vy;
            out[11] = vz;
        }
        { /* backward.cu:877-894: the homogeneous projection p = Pm [m, 1] */
            const float m_w = 1.0f / ((proj[3] * mean[0] + proj[7] * mean[1] + proj[11] * mean[2] + proj[15]) + 0.0000001f);
            const float mul1 = (proj[0] * mean[0] + proj[4] * mean[1] + proj[8] * mean[2] + proj[12]) * m_w * m_w;
            const float mul2 = (proj[1] * mean[0] + proj[5] * mean[1] + proj[9] * mean[2] + proj[13]) * m_w * m_w;
            const float gx = dL_dmean2D[3 * idx], gy = dL_dmean2D[3 * idx + 1];
            const float gp[3] = {gx * m_w, gy * m_w, -(mul1 * gx + mul2 * gy)};
            const float m4[4] = {mean[0], mean[1], mean[2], 1.f};
            for (int cc = 0; cc < 4; ++cc)
                for (int j = 0; j < 3; ++j) out[12 + 3 * cc + j] = m4[cc] * gp[j];
        }
        if (s->shs) { /* the view direction is m - campos */
            const int is4d = !(s->gaussian_dim == 3 || s->force_sh_3d);
            sh_backward(s, idx, is4d, mean, clamped, dL_dcolor, sh_mean, sh_dsh, sh_dts);
            for (int k = 0; k < 3; ++k) out[24 + k] = -sh_mean[3 * idx + k];
        }
    }
    free(sh_mean);
    free(sh_dsh);
    free(sh_dts);
}

/* reference: rasterizer_impl.cu:54-67 checkFrustum */
void oracle_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present) {
    for (int i = 0; i < P; ++i)
        present[i] = xform(viewmatrix, 2, means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2]) > 0.2f;
}

int oracle_num_threads(void) {
#ifdef _OPENMP
    extern int omp_get_max_threads(void);
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* n <= 0 restores the default (all host cores); used by bench.py to time cfg1 with one thread and with all */
void oracle_set_num_threads(int n) {
#ifdef _OPENMP
    extern void omp_set_num_threads(int);
    extern int omp_get_num_procs(void);
    omp_set_num_threads(n > 0 ? n : omp_get_num_procs());
#else
    (void)n;
#endif
}

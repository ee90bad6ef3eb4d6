/*
 * splat_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * A plain-C, CPU restatement of the reference's differentiable Gaussian
 * rasterizer with opaque-surfel depth (RTG-SLAM,
 * submodules/diff-gaussian-rasterizer-depth, "RAST/" below). Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may load it; the product path (rtg_slam_b200/csrc) never does.
 *
 * Parity pinning: the reference ships no golden vectors for this path
 * (SURVEY.md section 4). This restatement is pinned against outputs of the
 * reference's own CUDA code (RAST built unmodified for sm_90 into
 * oracle/_ref/, run on an H100) stored under tests/golden/ -- see
 * tests/golden/README.md and tests/test_oracle_raster.py.
 *
 * Build twice from this one file: -DREAL=float (mirrors the reference's fp32
 * arithmetic incl. its accidental double-precision sub-expressions) and
 * -DREAL=double (arbiter / finite-difference target).
 *
 * Each function cites the reference lines it follows.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#ifndef REAL
#define REAL float
#endif
typedef REAL real;

#define TILE 16 /* RAST/cuda_rasterizer/config.h:16-17 BLOCK_X, BLOCK_Y */

static const real SH_C0 = (real)0.28209479177387814;
static const real SH_C1 = (real)0.4886025119029199;
static const real SH_C2[5] = {(real)1.0925484305920792, (real)-1.0925484305920792, (real)0.31539156525252005,
                              (real)-1.0925484305920792, (real)0.5462742152960396};
static const real SH_C3[7] = {(real)-0.5900435899266435, (real)2.890611442640554, (real)-0.4570457994644658,
                              (real)0.3731763325901154, (real)-0.4570457994644658, (real)1.445305721320277,
                              (real)-0.5900435899266435};

/* Per-view constants: GaussianRasterizationSettings, RAST/diff_gaussian_rasterization_depth/__init__.py:284-303 */
typedef struct {
    int32_t H, W;
    real tanfovx, tanfovy, cx, cy;
    real scale_modifier, color_sigma;
    real opaque_threshold, depth_threshold, normal_threshold, T_threshold;
    real view[16], proj[16], campos[3], bg[3];
    int32_t sh_degree;
    real tie_eps; /* relative margin under which a discrete decision is flagged in `tie` */
} OracleView;

typedef struct {
    int P, M, H, W, tiles_x, tiles_y;
    OracleView v;
    /* geometry state (GeometryState, rasterizer_impl.cu:159-174) */
    real *depth, *xy, *conic_o, *rgb, *cov3D;
    uint8_t *clamped;
    int32_t *radii, *tiles_touched;
    /* binning state (BinningState :188-201), sorted */
    int64_t R;
    uint64_t *keys;
    int32_t *point_list;
    int64_t *ranges; /* per tile [start,end) */
    /* image state (ImageState :176-186) */
    real *final_T, *hit_normal_c, *hit_point_c, *weight_sum;
    int32_t *n_contrib;
    /* copies of the inputs the backward re-reads; colors_precomp replaces shs and cov3D_precomp replaces
     * scales / rots when given (NULL otherwise) */
    const real *means, *shs, *opac, *scales, *rots, *colors_precomp, *cov3D_precomp;
} OracleState;

/* ------------------------------------------------------------------ helpers */
/* auxiliary.h:59-97 */
static void xform4x3(const real *p, const real *m, real *o) {
    o[0] = m[0] * p[0] + m[4] * p[1] + m[8] * p[2] + m[12];
    o[1] = m[1] * p[0] + m[5] * p[1] + m[9] * p[2] + m[13];
    o[2] = m[2] * p[0] + m[6] * p[1] + m[10] * p[2] + m[14];
}
static void xform4x4(const real *p, const real *m, real *o) {
    o[0] = m[0] * p[0] + m[4] * p[1] + m[8] * p[2] + m[12];
    o[1] = m[1] * p[0] + m[5] * p[1] + m[9] * p[2] + m[13];
    o[2] = m[2] * p[0] + m[6] * p[1] + m[10] * p[2] + m[14];
    o[3] = m[3] * p[0] + m[7] * p[1] + m[11] * p[2] + m[15];
}
static void xvec4x3(const real *p, const real *m, real *o) {
    o[0] = m[0] * p[0] + m[4] * p[1] + m[8] * p[2];
    o[1] = m[1] * p[0] + m[5] * p[1] + m[9] * p[2];
    o[2] = m[2] * p[0] + m[6] * p[1] + m[10] * p[2];
}
static void xvec4x3T(const real *p, const real *m, real *o) {
    o[0] = m[0] * p[0] + m[1] * p[1] + m[2] * p[2];
    o[1] = m[4] * p[0] + m[5] * p[1] + m[6] * p[2];
    o[2] = m[8] * p[0] + m[9] * p[1] + m[10] * p[2];
}
static real rmin(real a, real b) { return a < b ? a : b; }
static real rmax(real a, real b) { return a > b ? a : b; }
static int imin(int a, int b) { return a < b ? a : b; }
static int imax(int a, int b) { return a > b ? a : b; }
/* forward.cu:20-52 */
static int arg_max3(real a, real b, real c) { return (a >= b && a >= c) ? 0 : ((b >= a && b >= c) ? 1 : 2); }
static int arg_min3(real a, real b, real c) { return (a <= b && a <= c) ? 0 : ((b <= a && b <= c) ? 1 : 2); }

/* Rotation matrix from the quaternion AS GIVEN (normalisation is commented out
 * in the reference, forward.cu:57,211). Rm[i][j] is the standard (math)
 * rotation matrix; the reference's glm::mat3 holds its transpose. */
static void quat_to_R(const real *q, real Rm[3][3]) {
    real r = q[0], x = q[1], y = q[2], z = q[3];
    Rm[0][0] = 1 - 2 * (y * y + z * z); Rm[0][1] = 2 * (x * y - r * z); Rm[0][2] = 2 * (x * z + r * y);
    Rm[1][0] = 2 * (x * y + r * z); Rm[1][1] = 1 - 2 * (x * x + z * z); Rm[1][2] = 2 * (y * z - r * x);
    Rm[2][0] = 2 * (x * z - r * y); Rm[2][1] = 2 * (y * z + r * x); Rm[2][2] = 1 - 2 * (x * x + y * y);
}

/* forward.cu:202-235 computeCov3D: Sigma = R S S R^T */
static void cov3d_from(const real *s, real mod, const real *q, real *c6) {
    real Rm[3][3];
    quat_to_R(q, Rm);
    real sx = mod * s[0], sy = mod * s[1], sz = mod * s[2];
    /* M = S * R_glm with R_glm = Rm^T: M[i][j] (math) = s_i * Rm[j][i]; Sigma = M^T M */
    real M[3][3];
    for (int i = 0; i < 3; i++) {
        M[0][i] = sx * Rm[i][0];
        M[1][i] = sy * Rm[i][1];
        M[2][i] = sz * Rm[i][2];
    }
    real S[3][3];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) S[i][j] = M[0][i] * M[0][j] + M[1][i] * M[1][j] + M[2][i] * M[2][j];
    c6[0] = S[0][0]; c6[1] = S[0][1]; c6[2] = S[0][2]; c6[3] = S[1][1]; c6[4] = S[1][2]; c6[5] = S[2][2];
}

/* A = J * Rw (2x3 live rows), with the 1.3*tanfov clamp; forward.cu:158-197, backward.cu:294-322 */
static void ewa_A(const real *mean, const real *view, real fx, real fy, real tanx, real tany, real A[2][3], real t[3],
                  real *txtz_o, real *tytz_o) {
    xform4x3(mean, view, t);
    real limx = (real)1.3f * tanx, limy = (real)1.3f * tany;
    real txtz = t[0] / t[2], tytz = t[1] / t[2];
    t[0] = rmin(limx, rmax(-limx, txtz)) * t[2];
    t[1] = rmin(limy, rmax(-limy, tytz)) * t[2];
    real J00 = fx / t[2], J02 = -(fx * t[0]) / (t[2] * t[2]);
    real J11 = fy / t[2], J12 = -(fy * t[1]) / (t[2] * t[2]);
    /* Rw[i][k] = view[i + 4k] */
    for (int k = 0; k < 3; k++) {
        A[0][k] = J00 * view[0 + 4 * k] + J02 * view[2 + 4 * k];
        A[1][k] = J11 * view[1 + 4 * k] + J12 * view[2 + 4 * k];
    }
    if (txtz_o) *txtz_o = txtz;
    if (tytz_o) *tytz_o = tytz;
}

static void sym6_to_mat(const real *c, real V[3][3]) {
    V[0][0] = c[0]; V[0][1] = c[1]; V[0][2] = c[2];
    V[1][0] = c[1]; V[1][1] = c[3]; V[1][2] = c[4];
    V[2][0] = c[2]; V[2][1] = c[4]; V[2][2] = c[5];
}

/* forward.cu:104-155 */
static void sh_to_rgb(int deg, int M, const real *mean, const real *campos, const real *sh, real *rgb, uint8_t *clamped) {
    real dir[3] = {mean[0] - campos[0], mean[1] - campos[1], mean[2] - campos[2]};
    real len = (real)sqrt((double)(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]));
    if (sizeof(real) == 4) len = sqrtf(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
    real x = dir[0] / len, y = dir[1] / len, z = dir[2] / len;
    (void)M;
    for (int c = 0; c < 3; c++) {
#define S(k) sh[(k) * 3 + c]
        real res = SH_C0 * S(0);
        if (deg > 0) {
            res = res - SH_C1 * y * S(1) + SH_C1 * z * S(2) - SH_C1 * x * S(3);
            if (deg > 1) {
                real xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                res = res + SH_C2[0] * xy * S(4) + SH_C2[1] * yz * S(5) + SH_C2[2] * (2 * zz - xx - yy) * S(6) +
                      SH_C2[3] * xz * S(7) + SH_C2[4] * (xx - yy) * S(8);
                if (deg > 2) {
                    res = res + SH_C3[0] * y * (3 * xx - yy) * S(9) + SH_C3[1] * xy * z * S(10) +
                          SH_C3[2] * y * (4 * zz - xx - yy) * S(11) + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * S(12) +
                          SH_C3[4] * x * (4 * zz - xx - yy) * S(13) + SH_C3[5] * z * (xx - yy) * S(14) +
                          SH_C3[6] * x * (xx - 3 * yy) * S(15);
                }
            }
        }
#undef S
        res += (real)0.5;
        clamped[c] = res < 0;
        rgb[c] = rmax(res, 0);
    }
}

/* auxiliary.h:49-57 getRect */
static void get_rect(real px, real py, int rad, int gx, int gy, int *x0, int *y0, int *x1, int *y1) {
    *x0 = imin(gx, imax(0, (int)((px - rad) / TILE)));
    *y0 = imin(gy, imax(0, (int)((py - rad) / TILE)));
    *x1 = imin(gx, imax(0, (int)((px + rad + TILE - 1) / TILE)));
    *y1 = imin(gy, imax(0, (int)((py + rad + TILE - 1) / TILE)));
}

static int oracle_cmp_pair(const void *a, const void *b) {
    const uint64_t *x = (const uint64_t *)a, *y = (const uint64_t *)b;
    if (x[0] != y[0]) return x[0] < y[0] ? -1 : 1;
    return x[1] < y[1] ? -1 : (x[1] > y[1] ? 1 : 0);
}

static int near_rel(real a, real b, real eps) { return fabs((double)a - (double)b) <= eps * rmax((real)1e-30, (real)fabs((double)b)); }

/* forward.cu:92-100 ndc2ray */
static void pixel_ray(int px, int py, real fx, real fy, real cx, real cy, real *ray) {
    ray[0] = ((real)px - cx) / fx;
    ray[1] = ((real)py - cy) / fy;
    ray[2] = 1;
    real n = sizeof(real) == 4 ? (real)(1 / sqrtf(ray[0] * ray[0] + ray[1] * ray[1] + ray[2] * ray[2]))
                               : (real)(1 / sqrt((double)(ray[0] * ray[0] + ray[1] * ray[1] + ray[2] * ray[2])));
    ray[0] *= n; ray[1] *= n; ray[2] *= n;
}

static real rexp(real x) { return sizeof(real) == 4 ? (real)expf((float)x) : (real)exp((double)x); }

void oracle_free(OracleState *s) {
    if (!s) return;
    free(s->depth); free(s->xy); free(s->conic_o); free(s->rgb); free(s->cov3D); free(s->clamped);
    free(s->radii); free(s->tiles_touched); free(s->keys); free(s->point_list); free(s->ranges);
    free(s->final_T); free(s->hit_normal_c); free(s->hit_point_c); free(s->weight_sum); free(s->n_contrib);
    free(s);
}

int oracle_sizeof_real(void) { return (int)sizeof(real); }

/* ------------------------------------------------------------------ forward
 * Rasterizer::forward, rasterizer_impl.cu:205-437, with the output
 * initialisation of RasterizeGaussiansCUDA (rasterize_points.cu:79-87).
 * `tie` (H*W bytes, may be NULL) is set where a discrete per-pixel decision
 * was within v->tie_eps (relative) of flipping.
 * colors_precomp (P*3, or NULL) replaces the SH colour (forward.cu:330,
 * rasterizer_impl.cu:365): not clamped, clamp flags stay 0. cov3D_precomp
 * (P*6, or NULL) replaces computeCov3D (forward.cu:289-291); scales and rots
 * are then not read. The reference defines no depth side in that mode (its
 * render kernel reads scales[] unconditionally, forward.cu:779, while its
 * Python API forbids passing scales with cov3D_precomp): a hit Gaussian gets
 * no surfel, so its depth is the centre depth.                               */
OracleState *oracle_forward(const OracleView *v, int P, int M, const real *means, const real *shs, const real *opac,
                            const real *scales, const real *rots, const real *colors_precomp, const real *cov3D_precomp,
                            const int32_t *tile_mask, real *out_color,
                            real *out_depth, int32_t *out_hit_color, int32_t *out_hit_depth, real *out_hit_color_w,
                            real *out_hit_depth_w, real *out_T, int32_t *radii_out, uint8_t *tie, int nthreads) {
    const int H = v->H, W = v->W, N = H * W;
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE, T = gx * gy;
    OracleState *s = (OracleState *)calloc(1, sizeof(OracleState));
    s->P = P; s->M = M; s->H = H; s->W = W; s->tiles_x = gx; s->tiles_y = gy; s->v = *v;
    s->means = means; s->shs = shs; s->opac = opac; s->scales = scales; s->rots = rots;
    s->colors_precomp = colors_precomp; s->cov3D_precomp = cov3D_precomp;
    s->depth = (real *)calloc((size_t)P + 1, sizeof(real));
    s->xy = (real *)calloc((size_t)2 * P + 2, sizeof(real));
    s->conic_o = (real *)calloc((size_t)4 * P + 4, sizeof(real));
    s->rgb = (real *)calloc((size_t)3 * P + 3, sizeof(real));
    s->cov3D = (real *)calloc((size_t)6 * P + 6, sizeof(real));
    s->clamped = (uint8_t *)calloc((size_t)3 * P + 3, 1);
    s->radii = (int32_t *)calloc((size_t)P + 1, sizeof(int32_t));
    s->tiles_touched = (int32_t *)calloc((size_t)P + 1, sizeof(int32_t));
    s->ranges = (int64_t *)calloc((size_t)2 * T, sizeof(int64_t));
    s->final_T = (real *)calloc(N, sizeof(real));
    s->n_contrib = (int32_t *)calloc(N, sizeof(int32_t));
    s->hit_normal_c = (real *)calloc((size_t)3 * N, sizeof(real));
    s->hit_point_c = (real *)calloc((size_t)3 * N, sizeof(real));
    s->weight_sum = (real *)calloc(N, sizeof(real));
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#else
    (void)nthreads;
#endif
    /* rasterizer_impl.cu:244-245 */
    const real focal_y = H / (2 * v->tanfovy), focal_x = W / (2 * v->tanfovx);

    /* output initialisation, rasterize_points.cu:79-87 (hit maps start at 0, not -1) */
    for (int i = 0; i < 3 * N; i++) out_color[i] = 0;
    for (int i = 0; i < N; i++) {
        out_depth[i] = 0; out_hit_color[i] = 0; out_hit_depth[i] = 0;
        out_hit_color_w[i] = 0; out_hit_depth_w[i] = 0; out_T[i] = 1;
        if (tie) tie[i] = 0;
    }

    /* ---- preprocessCUDA, forward.cu:238-354 ---- */
#pragma omp parallel for schedule(static)
    for (int idx = 0; idx < P; idx++) {
        s->radii[idx] = 0; s->tiles_touched[idx] = 0;
        const real *p = means + 3 * idx;
        real ph[4], pv[3];
        /* in_frustum, auxiliary.h:139-165 */
        xform4x4(p, v->proj, ph);
        real pw = 1 / (ph[3] + (real)0.0000001f);
        real pp[3] = {ph[0] * pw, ph[1] * pw, ph[2] * pw};
        xform4x3(p, v->view, pv);
        if (pv[2] <= (real)0.2f || pp[0] < -1.3 || pp[0] > 1.3 || pp[1] < -1.3 || pp[1] > 1.3) continue;
        real *c6 = s->cov3D + 6 * idx;
        if (cov3D_precomp) memcpy(c6, cov3D_precomp + 6 * idx, 6 * sizeof(real));
        else cov3d_from(scales + 3 * idx, v->scale_modifier, rots + 4 * idx, c6);
        real A[2][3], t[3], V[3][3];
        ewa_A(p, v->view, focal_x, focal_y, v->tanfovx, v->tanfovy, A, t, NULL, NULL);
        sym6_to_mat(c6, V);
        real AV[2][3];
        for (int i = 0; i < 2; i++)
            for (int j = 0; j < 3; j++) AV[i][j] = A[i][0] * V[0][j] + A[i][1] * V[1][j] + A[i][2] * V[2][j];
        real ca = AV[0][0] * A[0][0] + AV[0][1] * A[0][1] + AV[0][2] * A[0][2] + (real)0.3f;
        real cb = AV[0][0] * A[1][0] + AV[0][1] * A[1][1] + AV[0][2] * A[1][2];
        real cc = AV[1][0] * A[1][0] + AV[1][1] * A[1][1] + AV[1][2] * A[1][2] + (real)0.3f;
        real det = ca * cc - cb * cb;
        if (det == 0) continue;
        real det_inv = 1 / det;
        real conic[3] = {cc * det_inv, -cb * det_inv, ca * det_inv};
        real mid = (real)0.5f * (ca + cc);
        real sq = sizeof(real) == 4 ? (real)sqrtf((float)rmax((real)0.1f, mid * mid - det))
                                    : (real)sqrt((double)rmax((real)0.1f, mid * mid - det));
        real l1 = mid + sq, l2 = mid - sq;
        real lm = rmax(l1, l2);
        real my_radius = sizeof(real) == 4 ? (real)ceilf(v->color_sigma * sqrtf((float)lm))
                                           : (real)ceil((double)(v->color_sigma * sqrt((double)lm)));
        /* ndc2Pix(v, S, c) = v*S*0.5 + c, evaluated in double in the reference (auxiliary.h:44-47) */
        real pix[2] = {(real)((double)(real)(pp[0] * (real)W) * 0.5 + (double)v->cx),
                       (real)((double)(real)(pp[1] * (real)H) * 0.5 + (double)v->cy)};
        int x0, y0, x1, y1;
        get_rect(pix[0], pix[1], (int)my_radius, gx, gy, &x0, &y0, &x1, &y1);
        if ((x1 - x0) * (y1 - y0) == 0) continue;
        if (colors_precomp) memcpy(s->rgb + 3 * idx, colors_precomp + 3 * idx, 3 * sizeof(real));
        else sh_to_rgb(v->sh_degree, M, p, v->campos, shs + (size_t)3 * M * idx, s->rgb + 3 * idx, s->clamped + 3 * idx);
        s->depth[idx] = pv[2];
        s->radii[idx] = (int)my_radius;
        s->xy[2 * idx] = pix[0]; s->xy[2 * idx + 1] = pix[1];
        s->conic_o[4 * idx] = conic[0]; s->conic_o[4 * idx + 1] = conic[1]; s->conic_o[4 * idx + 2] = conic[2];
        s->conic_o[4 * idx + 3] = opac[idx];
        int cnt = 0;
        for (int x = x0; x < x1; x++)
            for (int y = y0; y < y1; y++)
                if (tile_mask[y * gx + x]) cnt++;
        s->tiles_touched[idx] = cnt;
    }
    if (radii_out) memcpy(radii_out, s->radii, sizeof(int32_t) * P);

    /* ---- scan + duplicateWithKeys + stable sort + identifyTileRanges, rasterizer_impl.cu:300-342 ---- */
    int64_t R = 0;
    int64_t *offs = (int64_t *)malloc(sizeof(int64_t) * ((size_t)P + 1));
    for (int i = 0; i < P; i++) { offs[i] = R; R += s->tiles_touched[i]; }
    s->R = R;
    /* key = tile<<32 | depth bits; ties keep Gaussian-index order (stable radix sort). We sort
     * (key, idx) lexicographically, which is the same total order because emission is by ascending idx. */
    uint64_t *pk = (uint64_t *)malloc(sizeof(uint64_t) * 2 * (size_t)(R + 1));
    for (int idx = 0; idx < P; idx++) {
        if (s->radii[idx] <= 0) continue;
        int x0, y0, x1, y1;
        get_rect(s->xy[2 * idx], s->xy[2 * idx + 1], s->radii[idx], gx, gy, &x0, &y0, &x1, &y1);
        int64_t off = offs[idx];
        float df = (float)s->depth[idx];
        uint32_t db;
        memcpy(&db, &df, 4);
        for (int y = y0; y < y1; y++)
            for (int x = x0; x < x1; x++) {
                uint64_t key = (uint64_t)(y * gx + x);
                if (tile_mask[key]) {
                    pk[2 * off] = (key << 32) | db;
                    pk[2 * off + 1] = (uint32_t)idx;
                    off++;
                }
            }
    }
    free(offs);
    /* Stable sort by (tile, depth) == lexicographic sort of (key, idx). Bucket by tile (counting sort on the
     * high word), then sort every bucket independently (parallel over tiles). */
    {
        int64_t *tcount = (int64_t *)calloc((size_t)T + 1, sizeof(int64_t));
        for (int64_t i = 0; i < R; i++) tcount[(pk[2 * i] >> 32) + 1]++;
        for (int t2 = 0; t2 < T; t2++) tcount[t2 + 1] += tcount[t2];
        uint64_t *pk2 = (uint64_t *)malloc(sizeof(uint64_t) * 2 * (size_t)(R + 1));
        int64_t *cur = (int64_t *)malloc(sizeof(int64_t) * ((size_t)T + 1));
        memcpy(cur, tcount, sizeof(int64_t) * ((size_t)T + 1));
        for (int64_t i = 0; i < R; i++) {
            int64_t d = cur[pk[2 * i] >> 32]++;
            pk2[2 * d] = pk[2 * i];
            pk2[2 * d + 1] = pk[2 * i + 1];
        }
#pragma omp parallel for schedule(dynamic, 8)
        for (int t2 = 0; t2 < T; t2++)
            if (tcount[t2 + 1] - tcount[t2] > 1)
                qsort(pk2 + 2 * tcount[t2], (size_t)(tcount[t2 + 1] - tcount[t2]), 2 * sizeof(uint64_t), oracle_cmp_pair);
        free(pk); free(cur); free(tcount);
        pk = pk2;
    }
    s->keys = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)(R + 1));
    s->point_list = (int32_t *)malloc(sizeof(int32_t) * (size_t)(R + 1));
    for (int64_t i = 0; i < R; i++) { s->keys[i] = pk[2 * i]; s->point_list[i] = (int32_t)pk[2 * i + 1]; }
    free(pk);
    for (int64_t i = 0; i < R; i++) {
        uint32_t cur = (uint32_t)(s->keys[i] >> 32);
        if (i == 0) s->ranges[2 * cur] = 0;
        else {
            uint32_t prev = (uint32_t)(s->keys[i - 1] >> 32);
            if (cur != prev) { s->ranges[2 * prev + 1] = i; s->ranges[2 * cur] = i; }
        }
        if (i == R - 1) s->ranges[2 * cur + 1] = R;
    }

    /* ---- renderCUDA_withMask, forward.cu:636-861; one "CTA" per tile with a non-empty range
     *      (rasterizer_impl.cu:345-362) ---- */
    const real eps = v->tie_eps;
#pragma omp parallel for schedule(dynamic, 1)
    for (int tile = 0; tile < T; tile++) {
        int64_t r0 = s->ranges[2 * tile], r1 = s->ranges[2 * tile + 1];
        if (r0 == r1) continue;
        int tx = tile % gx, ty = tile / gx;
        for (int ly = 0; ly < TILE; ly++)
            for (int lx = 0; lx < TILE; lx++) {
                int px = tx * TILE + lx, py = ty * TILE + ly;
                if (px >= W || py >= H) continue;
                int pix_id = W * py + px;
                real ray[3];
                pixel_ray(px, py, focal_x, focal_y, v->cx, v->cy, ray);
                real Tcur = 1, end_T = 1, C[3] = {0, 0, 0}, depth_ = 0, wsum = 0;
                uint32_t contributor = 0, last_contributor = 0;
                int hit = 0, hit_id = -1, hit_color_id = -1, flag = 0;
                real cw_max = -1, hit_cw = 0, hit_dw = 0;
                for (int64_t k = r0; k < r1; k++) {
                    contributor++;
                    int g = s->point_list[k];
                    real dx = s->xy[2 * g] - (real)px, dy = s->xy[2 * g + 1] - (real)py;
                    const real *co = s->conic_o + 4 * g;
                    real power = (real)-0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                    if (power > 0) continue;
                    real alpha = rmin((real)0.99f, co[3] * rexp(power));
                    if (eps > 0 && near_rel(alpha, (real)(1.0f / 255.0f), eps)) flag = 1;
                    if (alpha < (real)(1.0f / 255.0f)) continue;
                    if (!hit && eps > 0 && near_rel(alpha, v->opaque_threshold, eps)) flag = 1;
                    if (!hit && alpha >= v->opaque_threshold && cov3D_precomp) {
                        hit_id = g; /* no surfel: centre depth */
                        hit_dw = alpha * Tcur;
                        depth_ = s->depth[g];
                        hit = 1;
                    } else if (!hit && alpha >= v->opaque_threshold) {
                        /* forward.cu:778-809; computeNormal_ScaleMax :54-74 */
                        real Rm[3][3];
                        const real *sc = scales + 3 * g;
                        quat_to_R(rots + 4 * g, Rm);
                        int na = arg_min3(sc[0], sc[1], sc[2]), ma = arg_max3(sc[0], sc[1], sc[2]);
                        real nw[3] = {Rm[0][na], Rm[1][na], Rm[2][na]};
                        real smax = sc[ma] * v->scale_modifier;
                        real nc[3], pc[3];
                        xvec4x3(nw, v->view, nc);
                        xform4x3(means + 3 * g, v->view, pc);
                        real num = pc[0] * nc[0] + pc[1] * nc[1] + pc[2] * nc[2];
                        real den = ray[0] * nc[0] + ray[1] * nc[1] + ray[2] * nc[2];
                        real t = (real)((double)num / ((double)den + 1e-8)); /* double sub-expression, forward.cu:783-784 */
                        real hp[3] = {t * ray[0], t * ray[1], t * ray[2]};
                        real ang = (real)fabs((double)den);
                        real dd = (real)fabs((double)(hp[2] - pc[2]));
                        hit_id = g;
                        hit_dw = alpha * Tcur;
                        if (eps > 0 && (near_rel(dd, smax * v->depth_threshold, eps) || near_rel(ang, v->normal_threshold, eps))) flag = 1;
                        if (dd <= smax * v->depth_threshold && ang >= v->normal_threshold) depth_ = t * ray[2];
                        else depth_ = s->depth[g];
                        for (int c = 0; c < 3; c++) { s->hit_normal_c[3 * pix_id + c] = nc[c]; s->hit_point_c[3 * pix_id + c] = hp[c]; }
                        hit = 1;
                    }
                    real test_T = Tcur * (1 - alpha);
                    if (eps > 0 && near_rel(test_T, v->T_threshold, eps)) flag = 1;
                    if (test_T < v->T_threshold && hit) break; /* done = true */
                    if (test_T >= v->T_threshold) {
                        real cw = alpha * Tcur;
                        wsum += cw;
                        for (int c = 0; c < 3; c++) C[c] += s->rgb[3 * g + c] * cw;
                        if (eps > 0 && cw_max > 0 && near_rel(cw, cw_max, eps)) flag = 1;
                        if (cw > cw_max) { cw_max = cw; hit_color_id = g; hit_cw = cw_max; }
                        last_contributor = contributor;
                        end_T = test_T;
                    }
                    Tcur = test_T;
                }
                s->final_T[pix_id] = end_T;
                s->n_contrib[pix_id] = (int32_t)last_contributor;
                for (int c = 0; c < 3; c++) out_color[c * N + pix_id] = C[c] + Tcur * v->bg[c];
                out_depth[pix_id] = depth_;
                out_hit_depth[pix_id] = hit_id;
                out_hit_color[pix_id] = hit_color_id;
                out_hit_color_w[pix_id] = hit_cw;
                out_hit_depth_w[pix_id] = hit_dw;
                s->weight_sum[pix_id] = wsum;
                out_T[pix_id] = end_T;
                if (tie) tie[pix_id] = (uint8_t)flag;
            }
    }
    return s;
}

/* accessors for tests */
int64_t oracle_num_rendered(const OracleState *s) { return s->R; }
void oracle_get_geom(const OracleState *s, real *depth, real *xy, real *conic_o, real *rgb, uint8_t *clamped,
                     int32_t *tiles_touched, real *cov3D) {
    int P = s->P;
    if (depth) memcpy(depth, s->depth, sizeof(real) * P);
    if (xy) memcpy(xy, s->xy, sizeof(real) * 2 * P);
    if (conic_o) memcpy(conic_o, s->conic_o, sizeof(real) * 4 * P);
    if (rgb) memcpy(rgb, s->rgb, sizeof(real) * 3 * P);
    if (clamped) memcpy(clamped, s->clamped, 3 * (size_t)P);
    if (tiles_touched) memcpy(tiles_touched, s->tiles_touched, sizeof(int32_t) * P);
    if (cov3D) memcpy(cov3D, s->cov3D, sizeof(real) * 6 * P);
}
void oracle_get_binning(const OracleState *s, int32_t *point_list, int64_t *ranges) {
    if (point_list) memcpy(point_list, s->point_list, sizeof(int32_t) * (size_t)s->R);
    if (ranges) memcpy(ranges, s->ranges, sizeof(int64_t) * 2 * (size_t)(s->tiles_x * s->tiles_y));
}
void oracle_get_image_state(const OracleState *s, real *final_T, int32_t *n_contrib) {
    int N = s->H * s->W;
    if (final_T) memcpy(final_T, s->final_T, sizeof(real) * N);
    if (n_contrib) memcpy(n_contrib, s->n_contrib, sizeof(int32_t) * N);
}

/* ------------------------------------------------------------------ backward
 * Rasterizer::backward, rasterizer_impl.cu:441-560. Gradient buffers are
 * zero-initialised as RasterizeGaussiansBackwardCUDA does
 * (rasterize_points.cu:195-203). Accumulation is sequential per Gaussian
 * (the reference uses fp32 atomics in nondeterministic order).              */
static void add3(real *dst, real a, real b, real c) { dst[0] += a; dst[1] += b; dst[2] += c; }

/* backward.cu:100-148 propagateRotationGrad: d(normal = column `axis` of R(q)) / dq_k, k = w,x,y,z */
static void dnormal_dq(const real *q, int axis, real d[4][3]) {
    real q0 = q[0], q1 = q[1], q2 = q[2], q3 = q[3];
    if (axis == 0) {
        d[0][0] = 0; d[0][1] = 2 * q3; d[0][2] = -2 * q2;
        d[1][0] = 0; d[1][1] = 2 * q2; d[1][2] = 2 * q3;
        d[2][0] = -4 * q2; d[2][1] = 2 * q1; d[2][2] = -2 * q0;
        d[3][0] = -4 * q3; d[3][1] = 2 * q0; d[3][2] = 2 * q1;
    } else if (axis == 1) {
        d[0][0] = -2 * q3; d[0][1] = 0; d[0][2] = 2 * q1;
        d[1][0] = 2 * q2; d[1][1] = -4 * q1; d[1][2] = 2 * q0;
        d[2][0] = 2 * q1; d[2][1] = 0; d[2][2] = 2 * q3;
        d[3][0] = -2 * q0; d[3][1] = -4 * q3; d[3][2] = 2 * q2;
    } else {
        d[0][0] = 2 * q2; d[0][1] = -2 * q1; d[0][2] = 0;
        d[1][0] = 2 * q3; d[1][1] = -2 * q0; d[1][2] = -4 * q1;
        d[2][0] = 2 * q0; d[2][1] = 2 * q3; d[2][2] = -4 * q2;
        d[3][0] = 2 * q1; d[3][1] = 2 * q2; d[3][2] = 0;
    }
}

void oracle_backward(const OracleState *s, const real *dL_dpix, const real *dL_ddepth, const int32_t *hit_image,
                     real *dL_dmeans3D, real *dL_dsh, real *dL_dopacity, real *dL_dscales, real *dL_drot,
                     real *dL_dmean2D /*P*3*/, real *dL_dconic /*P*4*/, real *dL_dcolor /*P*3*/, real *dL_dcov3D /*P*6*/,
                     int nthreads) {
    const OracleView *v = &s->v;
    const int P = s->P, M = s->M, H = s->H, W = s->W, N = H * W, gx = s->tiles_x, T = gx * s->tiles_y;
    const real focal_y = H / (2 * v->tanfovy), focal_x = W / (2 * v->tanfovx);
    memset(dL_dmeans3D, 0, sizeof(real) * 3 * P);
    memset(dL_dsh, 0, sizeof(real) * 3 * (size_t)M * P);
    memset(dL_dopacity, 0, sizeof(real) * P);
    memset(dL_dscales, 0, sizeof(real) * 3 * P);
    memset(dL_drot, 0, sizeof(real) * 4 * P);
    memset(dL_dmean2D, 0, sizeof(real) * 3 * P);
    memset(dL_dconic, 0, sizeof(real) * 4 * P);
    memset(dL_dcolor, 0, sizeof(real) * 3 * P);
    memset(dL_dcov3D, 0, sizeof(real) * 6 * P);

    /* ---- renderCUDA_flat, backward.cu:808-1066 ----
     * The reference accumulates with fp32 atomicAdd; here every thread owns a private
     * accumulator set (thread 0 uses the outputs directly) that is summed afterwards. */
    const real ddelx_dx = (real)(0.5 * W), ddely_dy = (real)(0.5 * H);
    int nt = 1;
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
    nt = omp_get_max_threads();
    if (nt > 16) nt = 16; /* each thread owns an 18*P-float accumulator set: cap the memory / reduction cost */
#endif
    const size_t PP = (size_t)P;
    const size_t priv_stride = 18 * PP; /* color3 mean2D3 conic4 opac1 means3 rot4 */
    real *priv = nt > 1 ? (real *)calloc((size_t)(nt - 1) * priv_stride + 1, sizeof(real)) : NULL;
#pragma omp parallel for schedule(dynamic, 1) num_threads(nt)
    for (int tile = 0; tile < T; tile++) {
        int tid = 0;
#ifdef _OPENMP
        tid = omp_get_thread_num();
#endif
        real *a_color = dL_dcolor, *a_m2 = dL_dmean2D, *a_con = dL_dconic, *a_op = dL_dopacity, *a_m3 = dL_dmeans3D, *a_rot = dL_drot;
        if (tid > 0) {
            real *b = priv + (size_t)(tid - 1) * priv_stride;
            a_color = b; a_m2 = b + 3 * PP; a_con = b + 6 * PP; a_op = b + 10 * PP; a_m3 = b + 11 * PP; a_rot = b + 14 * PP;
        }
        int64_t r0 = s->ranges[2 * tile], r1 = s->ranges[2 * tile + 1];
        if (r0 == r1) continue;
        int tx = tile % gx, ty = tile / gx;
        for (int ly = 0; ly < TILE; ly++)
            for (int lx = 0; lx < TILE; lx++) {
                int px = tx * TILE + lx, py = ty * TILE + ly;
                if (px >= W || py >= H) continue;
                int pix_id = W * py + px;
                const real T_final = s->final_T[pix_id];
                real Tcur = T_final;
                uint32_t contributor = (uint32_t)(r1 - r0);
                const uint32_t last_contributor = (uint32_t)s->n_contrib[pix_id];
                real accum_rec[3] = {0, 0, 0}, last_color[3] = {0, 0, 0}, last_alpha = 0;
                real dLp[3] = {dL_dpix[pix_id], dL_dpix[N + pix_id], dL_dpix[2 * N + pix_id]};
                for (int64_t k = r1 - 1; k >= r0; k--) {
                    contributor--;
                    if (contributor >= last_contributor) continue;
                    int g = s->point_list[k];
                    real dx = s->xy[2 * g] - (real)px, dy = s->xy[2 * g + 1] - (real)py;
                    const real *co = s->conic_o + 4 * g;
                    real power = (real)-0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                    if (power > 0) continue;
                    real G = rexp(power);
                    real alpha = rmin((real)0.99f, co[3] * G);
                    if (alpha < (real)(1.0f / 255.0f)) continue;
                    Tcur = Tcur / (1 - alpha);
                    real dch = alpha * Tcur;
                    real dL_dalpha = 0;
                    for (int c = 0; c < 3; c++) {
                        real col = s->rgb[3 * g + c];
                        accum_rec[c] = last_alpha * last_color[c] + (1 - last_alpha) * accum_rec[c];
                        last_color[c] = col;
                        dL_dalpha += (col - accum_rec[c]) * dLp[c];
                        a_color[3 * g + c] += dch * dLp[c];
                    }
                    dL_dalpha *= Tcur;
                    last_alpha = alpha;
                    real bgdot = v->bg[0] * dLp[0] + v->bg[1] * dLp[1] + v->bg[2] * dLp[2];
                    dL_dalpha += (-T_final / (1 - alpha)) * bgdot;
                    real dL_dG = co[3] * dL_dalpha;
                    real gdx = G * dx, gdy = G * dy;
                    real dG_ddelx = -gdx * co[0] - gdy * co[1];
                    real dG_ddely = -gdy * co[2] - gdx * co[1];
                    a_m2[3 * g] += dL_dG * dG_ddelx * ddelx_dx;
                    a_m2[3 * g + 1] += dL_dG * dG_ddely * ddely_dy;
                    a_con[4 * g] += (real)-0.5f * gdx * dx * dL_dG;
                    a_con[4 * g + 1] += (real)-0.5f * gdx * dy * dL_dG;
                    a_con[4 * g + 3] += (real)-0.5f * gdy * dy * dL_dG;
                    a_op[g] += G * dL_dalpha;
                }
                /* depth-hit gradient, backward.cu:997-1065; without a surfel (cov3D_precomp) the centre depth's */
                if (hit_image[pix_id] >= 0 && s->cov3D_precomp) {
                    int g = hit_image[pix_id];
                    real dLd = dL_ddepth[pix_id];
                    add3(a_m3 + 3 * g, dLd * v->view[2], dLd * v->view[6], dLd * v->view[10]);
                } else if (hit_image[pix_id] >= 0) {
                    int g = hit_image[pix_id];
                    real ray[3];
                    pixel_ray(px, py, focal_x, focal_y, v->cx, v->cy, ray);
                    const real *sc = s->scales + 3 * g;
                    real smax = (real)fmax(fmax((double)sc[0], (double)sc[1]), (double)sc[2]);
                    const real *nc = s->hit_normal_c + 3 * pix_id;
                    const real *hp = s->hit_point_c + 3 * pix_id;
                    real pc[3];
                    xform4x3(s->means + 3 * g, v->view, pc);
                    real ndotr = nc[0] * ray[0] + nc[1] * ray[1] + nc[2] * ray[2];
                    real ang = (real)fabs((double)ndotr);
                    real dd = (real)fabs((double)(hp[2] - pc[2]));
                    real dLd = dL_ddepth[pix_id];
                    if (dd <= v->depth_threshold * smax && ang >= v->normal_threshold) {
                        real nr = (real)((double)ndotr + 1e-8);
                        real inv_nr = 1 / nr, inv_nr2 = inv_nr * inv_nr;
                        real np_ = nc[0] * pc[0] + nc[1] * pc[1] + nc[2] * pc[2];
                        real dpx = ray[2] * nc[0] * inv_nr, dpy = ray[2] * nc[1] * inv_nr, dpz = ray[2] * nc[2] * inv_nr;
                        const real *vm = v->view;
                        add3(a_m3 + 3 * g, dLd * (dpx * vm[0] + dpy * vm[1] + dpz * vm[2]),
                             dLd * (dpx * vm[4] + dpy * vm[5] + dpz * vm[6]), dLd * (dpx * vm[8] + dpy * vm[9] + dpz * vm[10]));
                        int axis = arg_min3(sc[0], sc[1], sc[2]);
                        real n1 = ray[2] * (nr * pc[0] - np_ * ray[0]) * inv_nr2;
                        real n2 = ray[2] * (nr * pc[1] - np_ * ray[1]) * inv_nr2;
                        real n3 = ray[2] * (nr * pc[2] - np_ * ray[2]) * inv_nr2;
                        real w1 = n1 * vm[0] + n2 * vm[1] + n3 * vm[2];
                        real w2 = n1 * vm[4] + n2 * vm[5] + n3 * vm[6];
                        real w3 = n1 * vm[8] + n2 * vm[9] + n3 * vm[10];
                        real d[4][3];
                        dnormal_dq(s->rots + 4 * g, axis, d);
                        for (int k = 0; k < 4; k++) a_rot[4 * g + k] += dLd * (w1 * d[k][0] + w2 * d[k][1] + w3 * d[k][2]);
                    } else {
                        add3(a_m3 + 3 * g, dLd * v->view[2], dLd * v->view[6], dLd * v->view[10]);
                    }
                }
            }
    }
    if (priv) {
#pragma omp parallel for schedule(static)
        for (int g = 0; g < P; g++) {
            for (int t = 0; t < nt - 1; t++) {
                const real *b = priv + (size_t)t * priv_stride;
                for (int c = 0; c < 3; c++) dL_dcolor[3 * g + c] += b[3 * g + c];
                for (int c = 0; c < 3; c++) dL_dmean2D[3 * g + c] += b[3 * PP + 3 * g + c];
                for (int c = 0; c < 4; c++) dL_dconic[4 * g + c] += b[6 * PP + 4 * g + c];
                dL_dopacity[g] += b[10 * PP + g];
                for (int c = 0; c < 3; c++) dL_dmeans3D[3 * g + c] += b[11 * PP + 3 * g + c];
                for (int c = 0; c < 4; c++) dL_drot[4 * g + c] += b[14 * PP + 4 * g + c];
            }
        }
        free(priv);
    }

    /* ---- computeCov2DCUDA (backward.cu:273-422) + preprocessCUDA bwd (:492-548) ---- */
#pragma omp parallel for schedule(static)
    for (int idx = 0; idx < P; idx++) {
        if (!(s->radii[idx] > 0)) continue;
        const real *mean = s->means + 3 * idx;
        const real *c6 = s->cov3D + 6 * idx;
        real dcon[3] = {dL_dconic[4 * idx], dL_dconic[4 * idx + 1], dL_dconic[4 * idx + 3]};
        real A[2][3], t[3], txtz, tytz, V[3][3];
        ewa_A(mean, v->view, focal_x, focal_y, v->tanfovx, v->tanfovy, A, t, &txtz, &tytz);
        const real limx = (real)1.3f * v->tanfovx, limy = (real)1.3f * v->tanfovy;
        const real xg = (txtz < -limx || txtz > limx) ? 0 : 1, yg = (tytz < -limy || tytz > limy) ? 0 : 1;
        sym6_to_mat(c6, V);
        real AV[2][3];
        for (int i = 0; i < 2; i++)
            for (int j = 0; j < 3; j++) AV[i][j] = A[i][0] * V[0][j] + A[i][1] * V[1][j] + A[i][2] * V[2][j];
        real a = AV[0][0] * A[0][0] + AV[0][1] * A[0][1] + AV[0][2] * A[0][2] + (real)0.3f;
        real b = AV[0][0] * A[1][0] + AV[0][1] * A[1][1] + AV[0][2] * A[1][2];
        real c = AV[1][0] * A[1][0] + AV[1][1] * A[1][1] + AV[1][2] * A[1][2] + (real)0.3f;
        real denom = a * c - b * b;
        real da = 0, db = 0, dc = 0;
        real denom2inv = 1 / ((denom * denom) + (real)0.0000001f);
        real *dcov = dL_dcov3D + 6 * idx;
        if (denom2inv != 0) {
            da = denom2inv * (-c * c * dcon[0] + 2 * b * c * dcon[1] + (denom - a * c) * dcon[2]);
            dc = denom2inv * (-a * a * dcon[2] + 2 * a * b * dcon[1] + (denom - a * c) * dcon[0]);
            db = denom2inv * 2 * (b * c * dcon[0] - (denom + 2 * b * b) * dcon[1] + a * b * dcon[2]);
            dcov[0] = A[0][0] * A[0][0] * da + A[0][0] * A[1][0] * db + A[1][0] * A[1][0] * dc;
            dcov[3] = A[0][1] * A[0][1] * da + A[0][1] * A[1][1] * db + A[1][1] * A[1][1] * dc;
            dcov[5] = A[0][2] * A[0][2] * da + A[0][2] * A[1][2] * db + A[1][2] * A[1][2] * dc;
            dcov[1] = 2 * A[0][0] * A[0][1] * da + (A[0][0] * A[1][1] + A[0][1] * A[1][0]) * db + 2 * A[1][0] * A[1][1] * dc;
            dcov[2] = 2 * A[0][0] * A[0][2] * da + (A[0][0] * A[1][2] + A[0][2] * A[1][0]) * db + 2 * A[1][0] * A[1][2] * dc;
            dcov[4] = 2 * A[0][2] * A[0][1] * da + (A[0][1] * A[1][2] + A[0][2] * A[1][1]) * db + 2 * A[1][1] * A[1][2] * dc;
        }
        /* dL/dA (backward.cu:365-376); AV rows are A[i]*Vrk */
        real dA0[3], dA1[3];
        for (int k = 0; k < 3; k++) {
            dA0[k] = 2 * AV[0][k] * da + AV[1][k] * db;
            dA1[k] = 2 * AV[1][k] * dc + AV[0][k] * db;
        }
        const real *vm = v->view; /* Rw[i][k] = vm[i + 4k] */
        real dJ00 = vm[0] * dA0[0] + vm[4] * dA0[1] + vm[8] * dA0[2];
        real dJ02 = vm[2] * dA0[0] + vm[6] * dA0[1] + vm[10] * dA0[2];
        real dJ11 = vm[1] * dA1[0] + vm[5] * dA1[1] + vm[9] * dA1[2];
        real dJ12 = vm[2] * dA1[0] + vm[6] * dA1[1] + vm[10] * dA1[2];
        real tz = 1 / t[2], tz2 = tz * tz, tz3 = tz2 * tz;
        real dt[3];
        dt[0] = xg * -focal_x * tz2 * dJ02;
        dt[1] = yg * -focal_y * tz2 * dJ12;
        dt[2] = -focal_x * tz2 * dJ00 - focal_y * tz2 * dJ11 + (2 * focal_x * t[0]) * tz3 * dJ02 + (2 * focal_y * t[1]) * tz3 * dJ12;
        real dm[3];
        xvec4x3T(dt, vm, dm);
        add3(dL_dmeans3D + 3 * idx, dm[0], dm[1], dm[2]);

        /* preprocessCUDA bwd, backward.cu:516-533 */
        const real *pj = v->proj;
        real mh[4];
        xform4x4(mean, pj, mh);
        real mw = 1 / (mh[3] + (real)0.0000001f);
        real mul1 = (pj[0] * mean[0] + pj[4] * mean[1] + pj[8] * mean[2] + pj[12]) * mw * mw;
        real mul2 = (pj[1] * mean[0] + pj[5] * mean[1] + pj[9] * mean[2] + pj[13]) * mw * mw;
        real g2x = dL_dmean2D[3 * idx], g2y = dL_dmean2D[3 * idx + 1];
        add3(dL_dmeans3D + 3 * idx, (pj[0] * mw - pj[3] * mul1) * g2x + (pj[1] * mw - pj[3] * mul2) * g2y,
             (pj[4] * mw - pj[7] * mul1) * g2x + (pj[5] * mw - pj[7] * mul2) * g2y,
             (pj[8] * mw - pj[11] * mul1) * g2x + (pj[9] * mw - pj[11] * mul2) * g2y);

        /* computeColorFromSH bwd, backward.cu:152-268; skipped for precomputed colours (:539) */
        if (!s->colors_precomp) {
            const real *sh = s->shs + (size_t)3 * M * idx;
            real *dsh = dL_dsh + (size_t)3 * M * idx;
            real dir0[3] = {mean[0] - v->campos[0], mean[1] - v->campos[1], mean[2] - v->campos[2]};
            real len = sizeof(real) == 4 ? (real)sqrtf((float)(dir0[0] * dir0[0] + dir0[1] * dir0[1] + dir0[2] * dir0[2]))
                                         : (real)sqrt((double)(dir0[0] * dir0[0] + dir0[1] * dir0[1] + dir0[2] * dir0[2]));
            real x = dir0[0] / len, y = dir0[1] / len, z = dir0[2] / len;
            real dRGB[3];
            for (int ch = 0; ch < 3; ch++) dRGB[ch] = dL_dcolor[3 * idx + ch] * (s->clamped[3 * idx + ch] ? 0 : 1);
            real ddir[3] = {0, 0, 0};
            int deg = v->sh_degree;
            for (int ch = 0; ch < 3; ch++) {
#define S(k) sh[(k) * 3 + ch]
#define D(k) dsh[(k) * 3 + ch]
                real g = dRGB[ch];
                real rx = 0, ry = 0, rz = 0;
                D(0) = SH_C0 * g;
                if (deg > 0) {
                    D(1) = -SH_C1 * y * g; D(2) = SH_C1 * z * g; D(3) = -SH_C1 * x * g;
                    rx = -SH_C1 * S(3); ry = -SH_C1 * S(1); rz = SH_C1 * S(2);
                    if (deg > 1) {
                        real xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                        D(4) = SH_C2[0] * xy * g; D(5) = SH_C2[1] * yz * g; D(6) = SH_C2[2] * (2 * zz - xx - yy) * g;
                        D(7) = SH_C2[3] * xz * g; D(8) = SH_C2[4] * (xx - yy) * g;
                        rx += SH_C2[0] * y * S(4) + SH_C2[2] * 2 * -x * S(6) + SH_C2[3] * z * S(7) + SH_C2[4] * 2 * x * S(8);
                        ry += SH_C2[0] * x * S(4) + SH_C2[1] * z * S(5) + SH_C2[2] * 2 * -y * S(6) + SH_C2[4] * 2 * -y * S(8);
                        rz += SH_C2[1] * y * S(5) + SH_C2[2] * 2 * 2 * z * S(6) + SH_C2[3] * x * S(7);
                        if (deg > 2) {
                            D(9) = SH_C3[0] * y * (3 * xx - yy) * g; D(10) = SH_C3[1] * xy * z * g;
                            D(11) = SH_C3[2] * y * (4 * zz - xx - yy) * g; D(12) = SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * g;
                            D(13) = SH_C3[4] * x * (4 * zz - xx - yy) * g; D(14) = SH_C3[5] * z * (xx - yy) * g;
                            D(15) = SH_C3[6] * x * (xx - 3 * yy) * g;
                            rx += SH_C3[0] * S(9) * 3 * 2 * xy + SH_C3[1] * S(10) * yz + SH_C3[2] * S(11) * -2 * xy +
                                  SH_C3[3] * S(12) * -3 * 2 * xz + SH_C3[4] * S(13) * (-3 * xx + 4 * zz - yy) +
                                  SH_C3[5] * S(14) * 2 * xz + SH_C3[6] * S(15) * 3 * (xx - yy);
                            ry += SH_C3[0] * S(9) * 3 * (xx - yy) + SH_C3[1] * S(10) * xz + SH_C3[2] * S(11) * (-3 * yy + 4 * zz - xx) +
                                  SH_C3[3] * S(12) * -3 * 2 * yz + SH_C3[4] * S(13) * -2 * xy + SH_C3[5] * S(14) * -2 * yz +
                                  SH_C3[6] * S(15) * -3 * 2 * xy;
                            rz += SH_C3[1] * S(10) * xy + SH_C3[2] * S(11) * 4 * 2 * yz + SH_C3[3] * S(12) * 3 * (2 * zz - xx - yy) +
                                  SH_C3[4] * S(13) * 4 * 2 * xz + SH_C3[5] * S(14) * (xx - yy);
                        }
                    }
                }
#undef S
#undef D
                ddir[0] += rx * g; ddir[1] += ry * g; ddir[2] += rz * g;
            }
            /* dnormvdv, auxiliary.h:107-118 */
            real sum2 = dir0[0] * dir0[0] + dir0[1] * dir0[1] + dir0[2] * dir0[2];
            real inv32 = sizeof(real) == 4 ? (real)(1.0f / sqrtf((float)(sum2 * sum2 * sum2))) : (real)(1.0 / sqrt((double)(sum2 * sum2 * sum2)));
            real dmx = ((+sum2 - dir0[0] * dir0[0]) * ddir[0] - dir0[1] * dir0[0] * ddir[1] - dir0[2] * dir0[0] * ddir[2]) * inv32;
            real dmy = (-dir0[0] * dir0[1] * ddir[0] + (sum2 - dir0[1] * dir0[1]) * ddir[1] - dir0[2] * dir0[1] * ddir[2]) * inv32;
            real dmz = (-dir0[0] * dir0[2] * ddir[0] - dir0[1] * dir0[2] * ddir[1] + (sum2 - dir0[2] * dir0[2]) * ddir[2]) * inv32;
            add3(dL_dmeans3D + 3 * idx, dmx, dmy, dmz);
        }

        /* computeCov3D bwd, backward.cu:426-487; skipped for a precomputed covariance (:546) */
        if (!s->cov3D_precomp) {
            const real *q = s->rots + 4 * idx, *sc = s->scales + 3 * idx;
            real Rm[3][3];
            quat_to_R(q, Rm);
            real sv[3] = {v->scale_modifier * sc[0], v->scale_modifier * sc[1], v->scale_modifier * sc[2]};
            /* M (math) = S * Rm^T : M[i][j] = s_i * Rm[j][i] */
            real Mm[3][3], dS[3][3];
            for (int i = 0; i < 3; i++)
                for (int j = 0; j < 3; j++) Mm[i][j] = sv[i] * Rm[j][i];
            dS[0][0] = dcov[0]; dS[0][1] = (real)0.5f * dcov[1]; dS[0][2] = (real)0.5f * dcov[2];
            dS[1][0] = (real)0.5f * dcov[1]; dS[1][1] = dcov[3]; dS[1][2] = (real)0.5f * dcov[4];
            dS[2][0] = (real)0.5f * dcov[2]; dS[2][1] = (real)0.5f * dcov[4]; dS[2][2] = dcov[5];
            /* Sigma = M^T M  =>  dL/dM = 2 M dSigma (math) */
            real dM[3][3];
            for (int i = 0; i < 3; i++)
                for (int j = 0; j < 3; j++) dM[i][j] = 2 * (Mm[i][0] * dS[0][j] + Mm[i][1] * dS[1][j] + Mm[i][2] * dS[2][j]);
            /* dL/ds_i = sum_j Rm[j][i] * dM[i][j] */
            for (int i = 0; i < 3; i++) dL_dscales[3 * idx + i] = Rm[0][i] * dM[i][0] + Rm[1][i] * dM[i][1] + Rm[2][i] * dM[i][2];
            /* dL/dRm[j][i] = s_i * dM[i][j]  -> G[j][i] */
            real Gm[3][3];
            for (int i = 0; i < 3; i++)
                for (int j = 0; j < 3; j++) Gm[j][i] = sv[i] * dM[i][j];
            real r = q[0], x = q[1], y = q[2], z = q[3];
            real dq[4];
            dq[0] = 2 * z * (Gm[1][0] - Gm[0][1]) + 2 * y * (Gm[0][2] - Gm[2][0]) + 2 * x * (Gm[2][1] - Gm[1][2]);
            dq[1] = 2 * y * (Gm[0][1] + Gm[1][0]) + 2 * z * (Gm[0][2] + Gm[2][0]) + 2 * r * (Gm[2][1] - Gm[1][2]) - 4 * x * (Gm[2][2] + Gm[1][1]);
            dq[2] = 2 * x * (Gm[0][1] + Gm[1][0]) + 2 * r * (Gm[0][2] - Gm[2][0]) + 2 * z * (Gm[2][1] + Gm[1][2]) - 4 * y * (Gm[2][2] + Gm[0][0]);
            dq[3] = 2 * r * (Gm[1][0] - Gm[0][1]) + 2 * x * (Gm[0][2] + Gm[2][0]) + 2 * y * (Gm[2][1] + Gm[1][2]) - 4 * z * (Gm[1][1] + Gm[0][0]);
            /* accumulates ONTO the depth-path value (backward.cu:485-486) */
            for (int k = 0; k < 4; k++) dL_drot[4 * idx + k] += dq[k];
        }
    }
}

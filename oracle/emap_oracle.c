/*
 * oracle/emap_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement (plain C, gcc) of the per-frame elevation-map fusion path of
 * leggedrobotics/elevation_mapping_cupy.  It is the checker the CUDA engine is
 * graded against; nothing in the product path may link, import or call it
 * (only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs do).
 *
 * Every function cites the reference file:line it follows, relative to
 * /root/reference/elevation_mapping_cupy/script/elevation_mapping_cupy/ :
 *   CK.py = kernels/custom_kernels.py,  EM.py = elevation_mapping.py,
 *   TF.py = traversability_filter.py.
 *
 * Arithmetic rules restated here (SURVEY.md section 8(c)):
 *   - every helper parameter the reference types `float16` (CuPy's class
 *     float16 around __half: implicit ctor from float, implicit operator
 *     float) is fp32 -> fp16 (round-nearest-even) -> fp32;  arithmetic between
 *     two such values is fp32;
 *   - an expression containing a substituted literal is evaluated in double
 *     and narrowed on assignment;  `int i = <double>` truncates toward zero
 *     with CUDA's saturating cvt.rzi semantics;
 *   - `float16 s += step` is half(float(double(s) + step));
 *   - sqrt and / are IEEE fp32.  The only places where NVRTC's default
 *     --fmad=true changes a result are marked FMAD: and use the contraction
 *     nvcc 12.9 emits for that source expression (checked against the SASS of
 *     the reference source compiled by oracle/build_ref.py).
 * Build with -ffp-contract=off so that nothing else is contracted.
 *
 * Parity pinning.  PINNED against the reference's own kernel source: oracle/build_ref.py compiles the CUDA-C strings
 * of kernels/custom_kernels.py and plugins/{min,max}_filter.py, robot_centric_elevation.py unmodified for the host
 * (and for sm_90a); tests/test_oracle_cpu.py compares this file with that build through the golden vectors
 * tests/golden/make_golden.py stores from it: bit-identical cell indices, <= 1e-6 on every order-independent cell, for the
 * deployed parameters, the dataclass defaults and four toggle / threshold combinations.  Restated rather than
 * executed (third party, absent here): CuPy's `class float16` (oracle/ref_shim.h), cuDNN's convolution order,
 * cupyx's uniform_filter -- see DESIGN.md section 2.
 *
 * Serialisation.  The reference kernel is racy by construction (SURVEY 3.5).
 * This oracle executes the CANONICAL SERIALISATION of SURVEY 8(c): a legal
 * interleaving of the reference kernel in which (1) the error-count pass runs,
 * (2) drift is applied, (3) all fusion loads happen before all fusion side
 * effects, (4) all ray-cast loads happen after the fusion side effects and
 * before the ray-cast side effects, (5) average_map, (6) overlap clear,
 * dilation, traversability, normals.  Order-dependent float accumulations
 * (sum new_h, sum new_v, sum of validity decrements, sum of drift errors) are
 * made order-INDEPENDENT by accumulating each fp32 term exactly in 2^-32
 * fixed point (int64); repeated additions of the one constant
 * `outlier_variance` are applied as n sequential fp32 adds.  Both choices are
 * within one fp32 rounding of some execution order of the reference atomics.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <limits.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef struct {
    int32_t cell_n;                 /* W: width == height (EM.py:64) */
    int32_t dilation_size;
    int32_t enable_edge_sharpen;
    int32_t enable_drift_compensation;
    int32_t enable_visibility_cleanup;
    int32_t enable_overlap_clearance;
    int32_t cell_min, cell_max;     /* overlap-clear window (EM.py:87-91) */
    double resolution;
    double sensor_noise_factor;
    double mahalanobis_thresh;
    double outlier_variance;
    double drift_compensation_variance_inlier;
    double traversability_inlier;
    double wall_num_thresh;
    double min_height_drift_cnt;
    double max_ray_length;
    double cleanup_step;
    double cleanup_cos_thresh;
    double min_valid_distance;
    double max_height_range;
    double ramped_height_range_a;
    double ramped_height_range_b;
    double ramped_height_range_c;
    double max_variance;
    double initial_variance;
    double max_drift;
    double drift_compensation_alpha;
    double position_noise_thresh;
    double orientation_noise_thresh;
    double overlap_clear_range_z;
} oracle_params;

/* ---- fp16 and conversion helpers --------------------------------------- */

static inline float h16(float x) { return (float)(_Float16)x; }

/* CUDA cvt.rzi.s32.f64: truncate toward zero, saturate, NaN -> 0. */
static inline int cvt_rzi(double d) {
    if (d != d) return 0;
    if (d >= 2147483647.0) return INT_MAX;
    if (d <= -2147483648.0) return INT_MIN;
    return (int)d;
}

/* 2^-32 fixed point of one fp32 term, magnitude saturated at 2^20. */
static inline int64_t fix32(float x) {
    if (x != x) return 0;
    if (x > 1048576.0f) x = 1048576.0f;
    if (x < -1048576.0f) x = -1048576.0f;
    return llrintf(x * 4294967296.0f);
}
static inline double unfix32(int64_t s) { return (double)s * (1.0 / 4294967296.0); }

/* order-preserving uint32 key of a float (for min/max over rays) */
static inline uint32_t fkey(float f) {
    uint32_t u; memcpy(&u, &f, 4);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
static inline float funkey(uint32_t k) {
    uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    float f; memcpy(&f, &u, 4); return f;
}

/* ---- map_utils (CK.py:9-122) -------------------------------------------- */

/* CK.py:22-25 clamp through float16 */
static inline int clamp16(int i, int hi) {
    float c = h16((float)i), lo16 = 0.0f, hi16 = h16((float)hi);
    float r = fmaxf(fminf(c, hi16), lo16);
    return (int)r;
}
/* CK.py:26-33 get_x_idx/get_y_idx with center == 0 (EM.py:337-338,359-360) */
static inline int axis_idx(const oracle_params* p, float c16) {
    return cvt_rzi((double)(c16 - 0.0f) / p->resolution + 0.5 * (double)p->cell_n);
}
/* CK.py:45-49 get_idx: x16,y16 already fp16-valued */
static inline int get_idx(const oracle_params* p, float x16, float y16) {
    int ix = clamp16(axis_idx(p, x16), p->cell_n - 1);
    int iy = clamp16(axis_idx(p, y16), p->cell_n - 1);
    return p->cell_n * ix + iy;
}
/* CK.py:34-44 */
static inline int is_inside(const oracle_params* p, int idx) {
    int W = p->cell_n;
    int ix = idx / W, iy = idx % W;
    if (ix == 0 || ix == W - 1) return 0;
    if (iy == 0 || iy == W - 1) return 0;
    return 1;
}
/* CK.py:408-418 (dilation/normal/min_filter flavour: <= 0, >= W-1, C division) */
static inline int is_inside_rel(int W, int idx) {
    int ix = idx / W, iy = idx % W;
    if (ix <= 0 || ix >= W - 1) return 0;
    if (iy <= 0 || iy >= W - 1) return 0;
    return 1;
}

typedef struct {
    float x, y, z, v;      /* transformed point (fp32) and sensor noise */
    int idx, valid, inside, skip; /* skip: NaN row, dropped at EM.py:458 */
} geom_t;

typedef struct { float R16[9], t16[3], t[3]; } pose_t;

static void make_pose(const float R[9], const float t[3], pose_t* q) {
    for (int i = 0; i < 9; i++) q->R16[i] = h16(R[i]);
    for (int i = 0; i < 3; i++) { q->t16[i] = h16(t[i]); q->t[i] = t[i]; }
}

/* CK.py:68-81 is_valid(x,y,z, sx,sy,sz): all six rounded to fp16 on entry */
static inline int is_valid_pt(const oracle_params* p, float x, float y, float z, const pose_t* q) {
    float X = h16(x), Y = h16(y), Z = h16(z);
    float dx = X - q->t16[0], dy = Y - q->t16[1], dz = Z - q->t16[2];
    /* FMAD: d = dx*dx + dy*dy + dz*dz  ->  fma(dz,dz, fma(dx,dx, dy*dy))  (nvcc 12.9 PTX) */
    float d = dy * dy; d = fmaf(dx, dx, d); d = fmaf(dz, dz, d);
    float sq = sqrtf(X * X + Y * Y);          /* products exact in fp32 */
    float dxy = (float)fmax((double)sq - p->ramped_height_range_b, 0.0);
    if ((double)d < p->min_valid_distance * p->min_valid_distance) return 0;
    float zr = Z - q->t16[2];
    /* FMAD: dxy*a + c in double -> fma */
    if ((double)zr > fma((double)dxy, p->ramped_height_range_a, p->ramped_height_range_c)
        || (double)zr > p->max_height_range) return 0;
    return 1;
}

/* CK.py:160-167,260-262 per-point geometry shared by both point kernels */
static inline void point_geom(const oracle_params* p, const float* pt, const pose_t* q, geom_t* g) {
    if (pt[0] != pt[0] || pt[1] != pt[1] || pt[2] != pt[2]) {   /* EM.py:458 */
        g->skip = 1; g->valid = 0; g->inside = 0; g->idx = -1; g->x = g->y = g->z = g->v = 0; return;
    }
    g->skip = 0;
    float rx = h16(pt[0]), ry = h16(pt[1]), rz = h16(pt[2]);
    /* CK.py:54-57 transform_p: fp16 operands, fp32 products (exact) and sums */
    g->x = ((q->R16[0] * rx + q->R16[1] * ry) + q->R16[2] * rz) + q->t16[0];
    g->y = ((q->R16[3] * rx + q->R16[4] * ry) + q->R16[5] * rz) + q->t16[1];
    g->z = ((q->R16[6] * rx + q->R16[7] * ry) + q->R16[8] * rz) + q->t16[2];
    /* CK.py:58-60 z_noise: double, narrowed to float */
    g->v = (float)((p->sensor_noise_factor * (double)rz) * (double)rz);
    g->idx = get_idx(p, h16(g->x), h16(g->y));
    g->valid = is_valid_pt(p, g->x, g->y, g->z, q);
    g->inside = is_inside(p, g->idx);
}

/* exported: per-point (idx, valid, inside) = the write-back of CK.py:260-262 */
void oracle_point_index(const oracle_params* p, const float* pts, int64_t n, int64_t stride,
                        const float* R, const float* t_rel,
                        int32_t* idx, uint8_t* valid, uint8_t* inside, float* xyzv) {
    pose_t q; make_pose(R, t_rel, &q);
    for (int64_t i = 0; i < n; i++) {
        geom_t g; point_geom(p, pts + i * stride, &q, &g);
        idx[i] = g.idx; valid[i] = (uint8_t)g.valid; inside[i] = (uint8_t)g.inside;
        if (xyzv) { xyzv[4*i] = g.x; xyzv[4*i+1] = g.y; xyzv[4*i+2] = g.z; xyzv[4*i+3] = g.v; }
    }
}

/* ---- per-cell stencil kernels ------------------------------------------ */

/* CK.py:392-449 dilation_filter_kernel (flat-index neighbours, signed dx+dy) */
void oracle_dilation(int W, int k, const float* map, const float* mask, float* newmap, float* newmask) {
    for (int i = 0; i < W * W; i++) {
        float h = map[i], valid = mask[i];
        newmap[i] = h;
        if (valid < 0.5f) {
            float distance = 100.f, near_value = 0.f;
            for (int dy = -k; dy <= k; dy++)
                for (int dx = -k; dx <= k; dx++) {
                    int idx = i + W * dy + dx;
                    if (!is_inside_rel(W, idx)) continue;
                    if (mask[idx] > 0.5f && (float)(dx + dy) < distance) {
                        distance = (float)(dx + dy);
                        near_value = map[idx];
                    }
                }
            if (distance < 100.f) { newmap[i] = near_value; if (newmask) newmask[i] = 1.0f; }
        }
    }
}

/* CK.py:452-506 normal_filter_kernel */
void oracle_normal(int W, double resolution, const float* map, const float* mask, float* normal /*3*W*W, pre-zeroed by caller*/) {
    float res = (float)resolution;           /* CK.py:479-481 returns float */
    int C = W * W;
    for (int i = 0; i < C; i++) {
        float h = map[i];
        if (mask[i] > 0.5f) {
            int ia = i + 1, ib = i + W;
            if (!is_inside_rel(W, ia) || !is_inside_rel(W, ib)) continue;
            float dzdx = map[ia] - h, dzdy = map[ib] - h;
            float nx = -dzdy / res, ny = -dzdx / res, nz = 1.f;
            /* FMAD: (nx*nx) + (ny*ny) + 1 -> fma(nx,nx, ny*ny) + 1 */
            float s = fmaf(nx, nx, ny * ny) + 1.0f;
            float norm = sqrtf(s);
            normal[i] = nx / norm; normal[C + i] = ny / norm; normal[2 * C + i] = nz / norm;
        }
    }
}

/* TF.py:15-42: three dilated 3x3 convs (1->4 ch, dilation 1/2/3, valid), crop
 * to the common (W-6)^2, |.|, 1x1 conv over the 12 channels, exp(-x).
 * Summation order: taps row-major within a channel, channels in order.
 * out is (W-6)*(W-6).  fp32 fused multiply-adds in that order (cuDNN's own order is unspecified). */
void oracle_traversability(int W, const float* in, const float* w1, const float* w2, const float* w3,
                           const float* wout, float* out) {
    int Wo = W - 6;
    const float* ws[3] = {w1, w2, w3};
    for (int r = 0; r < Wo; r++)
        for (int c = 0; c < Wo; c++) {
            int cr = r + 3, cc = c + 3;       /* centre in input coordinates */
            float acc = 0.f;
            for (int l = 0; l < 3; l++) {
                int dil = l + 1;
                for (int ch = 0; ch < 4; ch++) {
                    float s = 0.f;
                    for (int a = 0; a < 3; a++)
                        for (int b = 0; b < 3; b++)
                            s = fmaf(ws[l][ch * 9 + a * 3 + b], in[(cr + (a - 1) * dil) * W + (cc + (b - 1) * dil)], s);
                    acc = fmaf(wout[l * 4 + ch], fabsf(s), acc);
                }
            }
            out[r * Wo + c] = expf(-acc);
        }
}

/* plugins/min_filter.py:57-82,100-118.  The reference kernel updates newmap /
 * newmask in place while other threads read them (SURVEY 3.5, last row); the
 * canonical order here is Jacobi: every iteration reads the previous
 * iteration's planes.  Returns the number of iterations executed. */
int oracle_min_filter(int W, int k, int iteration_n, const float* map, const float* mask, float* out /*NaN where unfilled*/) {
    int C = W * W;
    float* a = (float*)malloc(sizeof(float) * C), *am = (float*)malloc(sizeof(float) * C);
    float* b = (float*)malloc(sizeof(float) * C), *bm = (float*)malloc(sizeof(float) * C);
    memcpy(a, map, sizeof(float) * C); memcpy(am, mask, sizeof(float) * C);
    int it = 0;
    for (; it < iteration_n; it++) {
        memcpy(b, a, sizeof(float) * C); memcpy(bm, am, sizeof(float) * C);
        for (int i = 0; i < C; i++) {
            if (mask[i] < 0.5f) {               /* note: tests the ORIGINAL mask (min_filter.py:61) */
                float mv = 1000000.0f;
                for (int dy = -k; dy <= k; dy++)
                    for (int dx = -k; dx <= k; dx++) {
                        int idx = i + W * dy + dx;
                        if (!is_inside_rel(W, idx)) continue;
                        if (am[idx] > 0.5f && a[idx] < mv) mv = a[idx];
                    }
                if (mv < 1000000.f - 1.f) { b[i] = mv; bm[i] = 0.6f; }
            }
        }
        float* t = a; a = b; b = t; t = am; am = bm; bm = t;
        int all = 1;
        for (int i = 0; i < C; i++) if (!(am[i] > 0.5f)) { all = 0; break; }
        if (all) { it++; break; }
    }
    for (int i = 0; i < C; i++) out[i] = am[i] > 0.5f ? a[i] : NAN;
    free(a); free(am); free(b); free(bm);
    return it;
}

/* plugins/max_filter.py:68-113: Jacobi (the reference copies both arrays before every launch), fill test on
 * the CURRENT mask. */
int oracle_max_filter(int W, int k, int iteration_n, const float* map, const float* mask, float* out) {
    int C = W * W;
    float* a = (float*)malloc(sizeof(float) * C), *am = (float*)malloc(sizeof(float) * C);
    float* b = (float*)malloc(sizeof(float) * C), *bm = (float*)malloc(sizeof(float) * C);
    memcpy(a, map, sizeof(float) * C); memcpy(am, mask, sizeof(float) * C);
    int it = 0;
    for (; it < iteration_n; it++) {
        memcpy(b, a, sizeof(float) * C); memcpy(bm, am, sizeof(float) * C);
        for (int i = 0; i < C; i++) {
            if (am[i] < 0.5f) {
                float mv = -1000000.0f;
                for (int dy = -k; dy <= k; dy++)
                    for (int dx = -k; dx <= k; dx++) {
                        int idx = i + W * dy + dx;
                        if (!is_inside_rel(W, idx)) continue;
                        if (am[idx] > 0.5f && a[idx] > mv) mv = a[idx];
                    }
                if (mv > -1000000.f + 1.f) { b[i] = mv; bm[i] = 0.6f; }
            }
        }
        float* t = a; a = b; b = t; t = am; am = bm; bm = t;
        int all = 1;
        for (int i = 0; i < C; i++) if (!(am[i] > 0.5f)) { all = 0; break; }
        if (all) { it++; break; }
    }
    for (int i = 0; i < C; i++) out[i] = am[i] > 0.5f ? a[i] : NAN;
    free(a); free(am); free(b); free(bm);
    return it;
}

/* plugins/robot_centric_elevation.py:54-83 */
void oracle_robot_centric(int W, double resolution, double threshold, int use_threshold, const float* elev,
                          const float* valid, const float* R, float* out) {
    for (int i = 0; i < W * W; i++) {
        float rz = elev[i];
        out[i] = rz;
        if (valid[i] > 0.5f) {
            float rx = (float)((double)(i / W) * resolution), ry = (float)((double)(i % W) * resolution);
            /* FMAD: r0*x + r1*y + r2*z -> fma(r2,z, fma(r0,x, r1*y)) */
            float zb = fmaf(R[8], rz, fmaf(R[6], rx, R[7] * ry));
            if (use_threshold) out[i] = ((double)zb >= threshold) ? 1.0f : 0.0f;
            else out[i] = zb;
        }
    }
}

/* plugins/smooth_filter.py:57-58: two passes of a 3x3 uniform filter with
 * scipy.ndimage 'reflect' boundary (d c b a | a b c d | d c b a), separable,
 * axis 0 then axis 1; each 1-D pass accumulates in double and stores fp32. */
static inline int reflect_idx(int i, int n) { if (i < 0) return -i - 1; if (i >= n) return 2 * n - 1 - i; return i; }
static void box3_pass(int W, const float* in, float* out) {
    int C = W * W;
    float* tmp = (float*)malloc(sizeof(float) * C);
    const double w = 1.0 / 3.0;     /* cupyx correlate1d weights ones(3)/3 in float64, fp32 output per pass */
    for (int r = 0; r < W; r++)
        for (int c = 0; c < W; c++) {
            double s = ((double)in[reflect_idx(r - 1, W) * W + c] * w + (double)in[r * W + c] * w) + (double)in[reflect_idx(r + 1, W) * W + c] * w;
            tmp[r * W + c] = (float)s;
        }
    for (int r = 0; r < W; r++)
        for (int c = 0; c < W; c++) {
            double s = ((double)tmp[r * W + reflect_idx(c - 1, W)] * w + (double)tmp[r * W + c] * w) + (double)tmp[r * W + reflect_idx(c + 1, W)] * w;
            out[r * W + c] = (float)s;
        }
    free(tmp);
}
void oracle_smooth(int W, const float* in, float* out) {
    float* t = (float*)malloc(sizeof(float) * W * W);
    box3_pass(W, in, t); box3_pass(W, t, out); free(t);
}

/* ---- the frame: EM.py:316-391 under the canonical serialisation -------- */

typedef struct {
    float mean_error;            /* EM.py:354 */
    float additive_mean_error;   /* EM.py:355 */
    float shift_applied;         /* EM.py:357 value added to elevation this frame (0 if none) */
    float error_sum;             /* sum(z-h) over inliers */
    int64_t error_cnt;
    int32_t drift_applied;
    int32_t drift_evaluated;     /* the EM.py:346-353 condition held */
    int64_t ray_visits;          /* cells visited by rays past the same-cell / border skips */
    int64_t ray_steps;           /* total march iterations */
} oracle_frame_stats;

/* Layer order of `map` (7,W,W): elevation, variance, is_valid, traversability,
 * time, upper_bound, is_upper_bound (EM.py:69-77).  `normal` is (3,W,W).
 * `scratch_counts` (optional, 3*W*W floats) returns new_map[3], new_map[4], new_map[2] (fused count). */
void oracle_frame(const oracle_params* p, float* map, float* normal, float* trav_input,
                  const float* w1, const float* w2, const float* w3, const float* wout,
                  const float* pts, int64_t n, int64_t stride,
                  const float* sensor_R, const float* sensor_t_rel, /* per-sensor poses */
                  const int64_t* sensor_offsets, int32_t n_sensors,
                  float position_noise, float orientation_noise,
                  float additive_mean_error_in,
                  int32_t* out_idx, uint8_t* out_valid, uint8_t* out_inside,
                  float* scratch_counts, oracle_frame_stats* st, int nthreads) {
    const int W = p->cell_n, C = W * W;
    float* H = map, *V = map + C, *VALID = map + 2 * C, *TRAV = map + 3 * C, *TIME = map + 4 * C,
          *UPPER = map + 5 * C, *ISUP = map + 6 * C;
    const float c_out = (float)p->outlier_variance;

    uint32_t* cnt_all = (uint32_t*)calloc(C, 4), *cnt_inl = (uint32_t*)calloc(C, 4);
    uint32_t* cnt_fused = (uint32_t*)calloc(C, 4), *n_out = (uint32_t*)calloc(C, 4), *n_ray = (uint32_t*)calloc(C, 4);
    int64_t* SH = (int64_t*)calloc(C, 8), *SV = (int64_t*)calloc(C, 8), *DV = (int64_t*)calloc(C, 8);
    uint64_t* last = (uint64_t*)calloc(C, 8);
    uint32_t* ukey = (uint32_t*)malloc((size_t)C * 4);
    geom_t* G = (geom_t*)malloc(sizeof(geom_t) * (size_t)(n > 0 ? n : 1));
    pose_t* poses = (pose_t*)malloc(sizeof(pose_t) * (size_t)n_sensors);
    int32_t* sensor_of = (int32_t*)malloc(4 * (size_t)(n > 0 ? n : 1));
    for (int s = 0; s < n_sensors; s++) {
        make_pose(sensor_R + 9 * s, sensor_t_rel + 3 * s, &poses[s]);
        for (int64_t i = sensor_offsets[s]; i < sensor_offsets[s + 1]; i++) sensor_of[i] = s;
    }
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#endif

    /* (1) error_counting_kernel CK.py:310-336 against the pre-frame map */
    int64_t E = 0, ecnt = 0;
#pragma omp parallel for schedule(static) reduction(+:E, ecnt)
    for (int64_t i = 0; i < n; i++) {
        geom_t* g = &G[i];
        point_geom(p, pts + i * stride, &poses[sensor_of[i]], g);
        if (out_idx) { out_idx[i] = g->idx; out_valid[i] = (uint8_t)g->valid; out_inside[i] = (uint8_t)g->inside; }
        if (g->skip || !g->valid || !g->inside) continue;
        int idx = g->idx;
        float mh = H[idx], mv = V[idx], mvalid = VALID[idx], mt = TRAV[idx];
        if (mvalid > 0.5f && (double)fabsf(mh - g->z) < (double)mv * p->mahalanobis_thresh
            && (double)mv < p->drift_compensation_variance_inlier / 2.0
            && (double)mt > p->traversability_inlier) {
            E += fix32(g->z - mh); ecnt += 1;
            __atomic_fetch_add(&cnt_inl[idx], 1u, __ATOMIC_RELAXED);
        }
        __atomic_fetch_add(&cnt_all[idx], 1u, __ATOMIC_RELAXED);
    }

    /* (2) drift compensation EM.py:346-357 */
    float error_sum = (float)unfix32(E), shift = 0.f;
    st->error_sum = error_sum; st->error_cnt = ecnt; st->drift_applied = 0; st->drift_evaluated = 0;
    st->mean_error = 0.f; st->additive_mean_error = additive_mean_error_in; st->shift_applied = 0.f;
    if (p->enable_drift_compensation && (double)(float)ecnt > p->min_height_drift_cnt
        && ((double)position_noise > p->position_noise_thresh || (double)orientation_noise > p->orientation_noise_thresh)) {
        float mean = error_sum / (float)ecnt;
        st->mean_error = mean; st->drift_evaluated = 1;
        st->additive_mean_error = additive_mean_error_in + mean;
        if (fabsf(mean) < (float)p->max_drift) {
            shift = mean * (float)p->drift_compensation_alpha;
            st->drift_applied = 1; st->shift_applied = shift;
            for (int i = 0; i < C; i++) H[i] += shift;
        }
    }

    /* (3) fusion half of add_points_kernel CK.py:168-197: all loads (snapshot H,V) ... */
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; i++) {
        const geom_t* g = &G[i];
        if (g->skip || !g->valid || !g->inside) continue;
        int idx = g->idx;
        float mh = H[idx], mv = V[idx], z = g->z, v = g->v;
        float num_points = (float)cnt_all[idx];
        if ((double)fabsf(mh - z) > (double)mv * p->mahalanobis_thresh) {
            __atomic_fetch_add(&n_out[idx], 1u, __ATOMIC_RELAXED);          /* CK.py:174 */
        } else if (p->enable_edge_sharpen && (double)num_points > p->wall_num_thresh
                   && (double)z < (double)mh - (double)mv * p->mahalanobis_thresh / (double)num_points) {
            /* CK.py:177-179: skipped */
        } else {
            /* FMAD: (map_h*v + z*map_v) -> fma(map_h, v, z*map_v) */
            float new_h = fmaf(mh, v, z * mv) / (mv + v);
            float new_v = (mv * v) / (mv + v);
            __atomic_fetch_add(&SH[idx], fix32(new_h), __ATOMIC_RELAXED);
            __atomic_fetch_add(&SV[idx], fix32(new_v), __ATOMIC_RELAXED);
            __atomic_fetch_add(&cnt_fused[idx], 1u, __ATOMIC_RELAXED);
            uint32_t hb; memcpy(&hb, &new_h, 4);
            uint64_t key = ((uint64_t)(uint32_t)i << 32) | hb, cur = __atomic_load_n(&last[idx], __ATOMIC_RELAXED);
            while (key > cur && !__atomic_compare_exchange_n(&last[idx], &cur, key, 1, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
        }
    }
    /* ... then all fusion side effects (CK.py:174,187-192) */
    for (int i = 0; i < C; i++) {
        for (uint32_t k = 0; k < n_out[i]; k++) V[i] += c_out;
        if (cnt_fused[i] > 0) {
            uint32_t hb = (uint32_t)(last[i] & 0xffffffffu); float nh; memcpy(&nh, &hb, 4);
            VALID[i] = 1.f; TIME[i] = 0.f; UPPER[i] = nh; ISUP[i] = 0.f;
        }
        ukey[i] = (ISUP[i] < 0.5f) ? 0xffffffffu : fkey(UPPER[i]);
    }

    /* (4) ray-cast half CK.py:198-259: loads see the state above */
    int64_t visits = 0, steps = 0;
    if (p->enable_visibility_cleanup) {
        const double ray_step = p->resolution / sqrt(2.0);   /* CK.py:268 */
        const float max_len16 = h16((float)p->max_ray_length);
#pragma omp parallel for schedule(dynamic, 256) reduction(+:visits, steps)
        for (int64_t i = 0; i < n; i++) {
            const geom_t* g = &G[i];
            if (g->skip || !g->valid) continue;      /* CK.py:226: every step `continue`s when the point is invalid */
            const pose_t* q = &poses[sensor_of[i]];
            float x = g->x, y = g->y, z = g->z;
            /* ray_vector CK.py:83-101 (all arguments rounded to fp16) */
            float vx = h16(h16(x) - q->t16[0]), vy = h16(h16(y) - q->t16[1]), vz = h16(h16(z) - q->t16[2]);
            float norm = h16(sqrtf((vx * vx + vy * vy) + vz * vz));
            float rx = 0.f, ry = 0.f, rz = 0.f;
            if (norm > 0.f) { rx = h16(vx / norm); ry = h16(vy / norm); rz = h16(vz / norm); }
            float len = fminf(norm, max_len16);                       /* CK.py:201 */
            float dec = (float)(-p->cleanup_step / ((double)len / p->max_ray_length));   /* CK.py:250 */
            int last_nidx = -1;
            for (float s = h16((float)ray_step); s < len; s = h16((float)((double)s + ray_step))) {
                steps++;
                float nx = q->t[0] + rx * s, ny = q->t[1] + ry * s, nz = q->t[2] + rz * s;
                int nidx = get_idx(p, h16(nx), h16(ny));
                if (nidx == last_nidx) continue;
                last_nidx = nidx;
                if (!is_inside(p, nidx)) continue;
                float ddx = x - nx, ddy = y - ny, ddz = z - nz;
                /* FMAD: same contraction as is_valid's d */
                float d = ddy * ddy; d = fmaf(ddx, ddx, d); d = fmaf(ddz, ddz, d); d = h16(d);
                if ((double)d < 0.1) continue;                         /* CK.py:226 */
                visits++;
                float nvalid = VALID[nidx];
                if (nvalid < 0.5f) {                                   /* CK.py:229-235 */
                    uint32_t key = fkey(nz), cur = __atomic_load_n(&ukey[nidx], __ATOMIC_RELAXED);
                    while (key < cur && !__atomic_compare_exchange_n(&ukey[nidx], &cur, key, 1, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
                    continue;
                }
                float ntime = TIME[nidx];
                if (ntime < 0.5f) continue;                            /* CK.py:237 */
                float nh = H[nidx], nv = V[nidx];
                /* FMAD: nz + 0.01 - min(v,1.0)*0.05 in double -> fma(-m, 0.05, nz + 0.01) */
                double rhs = fma(-fmin((double)nv, 1.0), 0.05, (double)nz + 0.01);
                if ((double)nh > rhs) {                                /* CK.py:239 */
                    float n0 = h16(normal[nidx]), n1 = h16(normal[C + nidx]), n2 = h16(normal[2 * C + nidx]);
                    float product = (rx * n0 + ry * n1) + rz * n2;     /* CK.py:103-108, products exact */
                    if ((double)fabsf(product) < p->cleanup_cos_thresh) continue;
                    float npts = (float)cnt_inl[nidx];                 /* newmap[3] CK.py:246 */
                    if ((double)npts > p->wall_num_thresh && (double)ntime < 1.0) continue;
                    __atomic_fetch_add(&DV[nidx], fix32(dec), __ATOMIC_RELAXED);
                    __atomic_fetch_add(&n_ray[nidx], 1u, __ATOMIC_RELAXED);
                    uint32_t key = fkey(nz), cur = __atomic_load_n(&ukey[nidx], __ATOMIC_RELAXED);
                    while (key < cur && !__atomic_compare_exchange_n(&ukey[nidx], &cur, key, 1, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
                }
            }
        }
        /* ray side effects */
        for (int i = 0; i < C; i++) {
            if (n_ray[i] > 0) {
                VALID[i] += (float)unfix32(DV[i]);
                for (uint32_t k = 0; k < n_ray[i]; k++) V[i] += c_out;
            }
            uint32_t key0 = (ISUP[i] < 0.5f) ? 0xffffffffu : fkey(UPPER[i]);
            if (ukey[i] != key0) { UPPER[i] = funkey(ukey[i]); ISUP[i] = 1.0f; }   /* carved by >= 1 ray */
        }
    }
    st->ray_visits = visits; st->ray_steps = steps;

    /* (5) average_map_kernel CK.py:362-384 */
    const float init_var = (float)p->initial_variance;
    for (int i = 0; i < C; i++) {
        float valid = VALID[i];
        if (cnt_fused[i] > 0) {
            double cnt = (double)cnt_fused[i];
            float mean_v = (float)(unfix32(SV[i]) / cnt);
            if ((double)mean_v > p->max_variance) { H[i] = 0.f; V[i] = init_var; VALID[i] = 0.f; }
            else { H[i] = (float)(unfix32(SH[i]) / cnt); V[i] = mean_v; VALID[i] = 1.f; }
        }
        if (valid < 0.5f) { H[i] = 0.f; V[i] = init_var; VALID[i] = 0.f; }
    }

    /* (6a) clear_overlap_map EM.py:393-410 */
    if (p->enable_overlap_clearance) {
        /* height_min/max are fp32 0-d arrays: t[2] -/+ python float (EM.py:400-401) */
        float tz = sensor_t_rel[2];
        float hmin = tz - (float)p->overlap_clear_range_z, hmax = tz + (float)p->overlap_clear_range_z;
        for (int r = p->cell_min; r < p->cell_max; r++)
            for (int c = p->cell_min; c < p->cell_max; c++) {
                int i = r * W + c;
                if (H[i] < hmin || H[i] > hmax) { H[i] = 0.f; V[i] = init_var; VALID[i] = 0.f; }
                if (UPPER[i] < hmin || UPPER[i] > hmax) { UPPER[i] = 0.f; ISUP[i] = 0.f; }
            }
    }

    /* (6b) dilation of upper_bound with mask = is_valid + is_upper_bound EM.py:376-383 */
    float* mask = (float*)malloc(sizeof(float) * C);
    for (int i = 0; i < C; i++) mask[i] = VALID[i] + ISUP[i];
    oracle_dilation(W, p->dilation_size, UPPER, mask, trav_input, NULL);
    free(mask);

    /* (6c) traversability EM.py:385-388 */
    if (W > 6) {
        int Wo = W - 6;
        float* tr = (float*)malloc(sizeof(float) * Wo * Wo);
        oracle_traversability(W, trav_input, w1, w2, w3, wout, tr);
        for (int r = 0; r < Wo; r++) memcpy(TRAV + (r + 3) * W + 3, tr + r * Wo, sizeof(float) * Wo);
        free(tr);
    }

    /* (6d) update_normal EM.py:391,564-577 */
    memset(normal, 0, sizeof(float) * 3 * C);
    oracle_normal(W, p->resolution, trav_input, VALID, normal);

    if (scratch_counts) for (int i = 0; i < C; i++) { scratch_counts[i] = (float)cnt_inl[i]; scratch_counts[C + i] = (float)cnt_all[i]; scratch_counts[2 * C + i] = (float)cnt_fused[i]; }
    free(cnt_all); free(cnt_inl); free(cnt_fused); free(n_out); free(n_ray);
    free(SH); free(SV); free(DV); free(last); free(ukey); free(G); free(poses); free(sensor_of);
}

/* bench.py: torchrun exports OMP_NUM_THREADS=1; the CPU baselines must use every host core */
void oracle_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int oracle_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

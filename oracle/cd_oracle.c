/*
 * TEST INFRASTRUCTURE ONLY (oracle).  Never linked or called by the product path.
 *
 * Plain-C restatement of the third-party arithmetic the reference's hot path
 * calls at lib/decompose.py:449,457 (``Lasso(alpha, warm_start=True,
 * selection='random').fit(Z, reY)``):
 *
 *   scikit-learn (installed and pinned here: 1.9.0)
 *     sklearn/linear_model/_cd_fast.pyx : enet_coordinate_descent (dense, data form)
 *                                         gap_enet, dual_gap_formulation_A
 *     sklearn/utils/_random.pxd         : our_rand_r (32-bit xorshift), rand_int
 *
 * cp_enet_cd_dense  follows enet_coordinate_descent statement by statement
 *                   (including the gap-safe screening rule of 1.9.0).
 * cp_enet_cd_gram   is the same control flow evaluated in Gram arithmetic
 *                   (Q = X'X, q = X'y, |y|^2): the executable, bit-exact specification
 *                   of the CUDA kernel cp_lasso_select (csrc/lasso.cu).
 *
 * Parity is pinned in tests/test_oracle.py against sklearn itself and against
 * golden vectors produced by the reference's own lib/decompose.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define CP_RAND_R_MAX 2147483647u

/* sklearn/utils/_random.pxd:20-34 */
static inline uint32_t our_rand_r(uint32_t *seed) {
    if (*seed == 0) *seed = 1; /* DEFAULT_SEED */
    *seed ^= (uint32_t)(*seed << 13);
    *seed ^= (uint32_t)(*seed >> 17);
    *seed ^= (uint32_t)(*seed << 5);
    return *seed % (CP_RAND_R_MAX + 1u);
}
static inline uint32_t rand_int(uint32_t end, uint32_t *state) { return our_rand_r(state) % end; }

uint32_t cp_our_rand_r(uint32_t *seed) { return our_rand_r(seed); }

static inline double fsign(double f) { return f == 0 ? 0.0 : (f > 0 ? 1.0 : -1.0); }
static inline double dmax(double a, double b) { return a > b ? a : b; }

static double ddot(int n, const double *a, const double *b) {
    double s = 0.0;
    for (int i = 0; i < n; ++i) s += a[i] * b[i];
    return s;
}
static void daxpy(int n, double a, const double *x, double *y) {
    for (int i = 0; i < n; ++i) y[i] += a * x[i];
}

/* _cd_fast.pyx: dual_gap_formulation_A with beta = 0 kept general */
static double gap_formulation_A(double alpha, double beta, double w_l1, double w_l2sq, double R_norm2,
                                double Ry, double dual_norm_XtA) {
    double primal = 0.5 * (R_norm2 + beta * w_l2sq) + alpha * w_l1;
    double scale = dual_norm_XtA > alpha ? alpha / dual_norm_XtA : 1.0;
    double dual = -0.5 * (scale * scale) * (R_norm2 + beta * w_l2sq) + scale * Ry;
    return primal - dual;
}

/* _cd_fast.pyx: gap_enet (alpha > 0 branch; positive=False) */
static double gap_enet_dense(int ns, int nf, const double *w, double alpha, double beta, const double *X,
                             const double *y, const double *R, double *XtA, double *dual_norm_out) {
    double w_l2sq = beta > 0 ? ddot(nf, w, w) : 0.0;
    double R_norm2 = ddot(ns, R, R);
    double Ry = ddot(ns, R, y);
    double dn = 0.0, l1 = 0.0;
    for (int j = 0; j < nf; ++j) {
        XtA[j] = ddot(ns, X + (size_t)j * ns, R) - beta * w[j];
        double a = fabs(XtA[j]);
        if (j == 0 || a > dn) dn = a;
        l1 += fabs(w[j]);
    }
    *dual_norm_out = dn;
    return gap_formulation_A(alpha, beta, l1, w_l2sq, R_norm2, Ry, dn);
}

/*
 * X: column-major (Fortran) ns x nf, already centred; y centred.  alpha = l1_reg = alpha_user*ns.
 * Returns n_iter (sklearn's n_iter + 1 convention), writes gap / tol_scaled.
 */
int cp_enet_cd_dense(double *w, double alpha, double beta, const double *X, const double *y, int ns, int nf,
                     int max_iter, double tol, uint32_t seed, int random, int do_screening, double *gap_out,
                     double *tol_out) {
    double *norm2 = (double *)malloc(sizeof(double) * nf);
    double *R = (double *)malloc(sizeof(double) * ns);
    double *XtA = (double *)malloc(sizeof(double) * nf);
    uint32_t *active = (uint32_t *)malloc(sizeof(uint32_t) * nf);
    uint8_t *excluded = (uint8_t *)malloc(nf);
    for (int j = 0; j < nf; ++j) norm2[j] = ddot(ns, X + (size_t)j * ns, X + (size_t)j * ns);
    uint32_t state = seed;
    double gap = tol + 1.0, d_w_tol = tol, dual_norm = 0.0;
    unsigned n_active = nf;
    int n_iter = 0, ret_iter = 0;
    if (alpha == 0) do_screening = 0;

    memcpy(R, y, sizeof(double) * ns);
    for (int j = 0; j < nf; ++j)
        if (w[j] != 0) daxpy(ns, -w[j], X + (size_t)j * ns, R);
    tol *= ddot(ns, y, y);

    gap = gap_enet_dense(ns, nf, w, alpha, beta, X, y, R, XtA, &dual_norm);
    if (gap <= tol) { ret_iter = 0; goto done; }

    if (do_screening) {
        n_active = 0;
        for (int j = 0; j < nf; ++j) {
            if (norm2[j] == 0) { w[j] = 0; excluded[j] = 1; continue; }
            double Xj_theta = XtA[j] / dmax(alpha, dual_norm);
            double d_j = (1 - fabs(Xj_theta)) / sqrt(norm2[j] + beta);
            if (d_j <= sqrt(2 * gap) / alpha) { active[n_active++] = j; excluded[j] = 0; }
            else {
                if (w[j] != 0) { daxpy(ns, w[j], X + (size_t)j * ns, R); w[j] = 0; }
                excluded[j] = 1;
            }
        }
    }
    int broke = 0;
    for (n_iter = 0; n_iter < max_iter; ++n_iter) {
        double w_max = 0.0, d_w_max = 0.0;
        for (unsigned f = 0; f < n_active; ++f) {
            unsigned j = random ? rand_int(n_active, &state) : f;
            if (do_screening) j = active[j];
            if (norm2[j] == 0.0) continue;
            double w_j = w[j];
            double tmp = ddot(ns, X + (size_t)j * ns, R) + w_j * norm2[j];
            w[j] = fsign(tmp) * dmax(fabs(tmp) - alpha, 0) / (norm2[j] + beta);
            if (w[j] != w_j) daxpy(ns, w_j - w[j], X + (size_t)j * ns, R);
            double d = fabs(w[j] - w_j);
            d_w_max = dmax(d_w_max, d);
            w_max = dmax(w_max, fabs(w[j]));
        }
        if (w_max == 0.0 || d_w_max / w_max <= d_w_tol || n_iter == max_iter - 1) {
            gap = gap_enet_dense(ns, nf, w, alpha, beta, X, y, R, XtA, &dual_norm);
            if (gap <= tol) { broke = 1; break; }
            if (do_screening) {
                n_active = 0;
                for (int j = 0; j < nf; ++j) {
                    if (excluded[j]) continue;
                    double Xj_theta = XtA[j] / dmax(alpha, dual_norm);
                    double d_j = (1 - fabs(Xj_theta)) / sqrt(norm2[j] + beta);
                    if (d_j <= sqrt(2 * gap) / alpha) { active[n_active++] = j; excluded[j] = 0; }
                    else {
                        if (w[j] != 0) { daxpy(ns, w[j], X + (size_t)j * ns, R); w[j] = 0; }
                        excluded[j] = 1;
                    }
                }
            }
        }
    }
    ret_iter = broke ? n_iter + 1 : max_iter; /* python: n_iter + 1 after loop */
done:
    *gap_out = gap;
    *tol_out = tol;
    free(norm2); free(R); free(XtA); free(active); free(excluded);
    return ret_iter;
}

/*
 * Same control flow, Gram arithmetic.  Q (nf x nf, row-major, leading dimension ldq, symmetric up
 * to rounding: the update of coordinate j reads row j only)
 * = X'X, q = X'y, y_norm2 = y'y (all of centred data).  This is, operation for operation, what
 * the CUDA kernel cp_lasso_select (csrc/lasso.cu) executes:
 *   - Qw = Q w is CARRIED between fits (in/out argument; all zeros with w = 0 before the first
 *     fit) instead of being recomputed from w at every fit start as sklearn recomputes R = y - Xw
 *     (a 1e-16-level rounding difference, not an algorithmic one);
 *   - the reductions of the duality-gap check run in "warp order": 32 strided partial sums
 *     combined by a 5-level butterfly, which is how 32 lanes evaluate them;
 *   - every product/sum is rounded separately (no FMA), division is IEEE.
 */
static double wdot(int n, const double *a, const double *b) {
    double p[32], t[32];
    for (int l = 0; l < 32; ++l) {
        double s = 0.0;
        for (int i = l; i < n; i += 32) s += a[i] * b[i];
        p[l] = s;
    }
    for (int off = 16; off; off >>= 1) {
        for (int l = 0; l < 32; ++l) t[l] = p[l] + p[l ^ off];
        memcpy(p, t, sizeof(p));
    }
    return p[0];
}
static double wasum(int n, const double *a) {
    double p[32], t[32];
    for (int l = 0; l < 32; ++l) {
        double s = 0.0;
        for (int i = l; i < n; i += 32) s += fabs(a[i]);
        p[l] = s;
    }
    for (int off = 16; off; off >>= 1) {
        for (int l = 0; l < 32; ++l) t[l] = p[l] + p[l ^ off];
        memcpy(p, t, sizeof(p));
    }
    return p[0];
}

static double gap_enet_gram(int nf, const double *w, double alpha, const double *Qw, const double *q,
                            double y_norm2, double *XtA, double *dual_norm_out) {
    double q_dot_w = wdot(nf, w, q);
    double wQw = wdot(nf, w, Qw);
    double R_norm2 = y_norm2 + wQw - 2.0 * q_dot_w;
    double Ry = y_norm2 - q_dot_w;
    double dn = 0.0;
    for (int j = 0; j < nf; ++j) {
        XtA[j] = q[j] - Qw[j];
        double a = fabs(XtA[j]);
        if (a > dn) dn = a;
    }
    double l1 = wasum(nf, w);
    *dual_norm_out = dn;
    return gap_formulation_A(alpha, 0.0, l1, 0.0, R_norm2, Ry, dn);
}

int cp_enet_cd_gram(double *w, double *Qw, double alpha, const double *Q, int ldq, const double *q, double y_norm2,
                    int nf, int max_iter, double tol, uint32_t seed, int random, int do_screening, double *gap_out,
                    double *tol_out) {
    double *XtA = (double *)malloc(sizeof(double) * nf);
    uint32_t *active = (uint32_t *)malloc(sizeof(uint32_t) * nf);
    uint8_t *excluded = (uint8_t *)malloc(nf);
    uint32_t state = seed;
    double gap = tol + 1.0, d_w_tol = tol, dual_norm = 0.0;
    unsigned n_active = nf;
    int n_iter = 0, ret_iter = 0;
    if (alpha == 0) do_screening = 0;
    tol *= y_norm2;
    gap = gap_enet_gram(nf, w, alpha, Qw, q, y_norm2, XtA, &dual_norm);
    if (gap <= tol) { ret_iter = 0; goto done; }
    if (do_screening) {
        double radius = sqrt(2 * fabs(gap)) / alpha;
        n_active = 0;
        for (int j = 0; j < nf; ++j) {
            double Qjj = Q[(size_t)j * ldq + j];
            if (Qjj == 0) { w[j] = 0; excluded[j] = 1; continue; }
            double Xj_theta = XtA[j] / dmax(alpha, dual_norm);
            double d_j = (1 - fabs(Xj_theta)) / sqrt(Qjj);
            if (d_j <= radius) { active[n_active++] = j; excluded[j] = 0; }
            else {
                if (w[j] != 0) { daxpy(nf, -w[j], Q + (size_t)j * ldq, Qw); w[j] = 0; }
                excluded[j] = 1;
            }
        }
    } else {
        for (int j = 0; j < nf; ++j) active[j] = j;
    }
    int broke = 0;
    for (n_iter = 0; n_iter < max_iter; ++n_iter) {
        double w_max = 0.0, d_w_max = 0.0;
        for (unsigned f = 0; f < n_active; ++f) {
            unsigned j = random ? rand_int(n_active, &state) : f;
            j = active[j];
            double Qjj = Q[(size_t)j * ldq + j];
            if (Qjj == 0.0) continue;
            double w_j = w[j];
            double tmp = q[j] - Qw[j] + w_j * Qjj;
            w[j] = fsign(tmp) * dmax(fabs(tmp) - alpha, 0) / Qjj;
            if (w[j] != w_j) daxpy(nf, w[j] - w_j, Q + (size_t)j * ldq, Qw);
            double d = fabs(w[j] - w_j);
            d_w_max = dmax(d_w_max, d);
            w_max = dmax(w_max, fabs(w[j]));
        }
        if (w_max == 0.0 || d_w_max / w_max <= d_w_tol || n_iter == max_iter - 1) {
            gap = gap_enet_gram(nf, w, alpha, Qw, q, y_norm2, XtA, &dual_norm);
            if (gap <= tol) { broke = 1; break; }
            if (do_screening) {
                double radius = sqrt(2 * fabs(gap)) / alpha;
                n_active = 0;
                for (int j = 0; j < nf; ++j) {
                    if (excluded[j]) continue;
                    double Qjj = Q[(size_t)j * ldq + j];
                    double Xj_theta = XtA[j] / dmax(alpha, dual_norm);
                    double d_j = (1 - fabs(Xj_theta)) / sqrt(Qjj);
                    if (d_j <= radius) { active[n_active++] = j; excluded[j] = 0; }
                    else {
                        if (w[j] != 0) { daxpy(nf, -w[j], Q + (size_t)j * ldq, Qw); w[j] = 0; }
                        excluded[j] = 1;
                    }
                }
            }
        }
    }
    ret_iter = broke ? n_iter + 1 : max_iter;
done:
    *gap_out = gap;
    *tol_out = tol;
    free(XtA); free(active); free(excluded);
    return ret_iter;
}

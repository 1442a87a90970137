/*
 * amg_oracle.c -- TEST INFRASTRUCTURE, never shipped, never on the product path.
 *
 * A plain-C, single-threaded restatement of the AMGCL solve phase that the
 * H100 backend accelerates.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline leg may load this file's library.  Each function
 * cites the reference code (paths relative to /root/reference) it restates.
 *
 * Pinning: tests/test_oracle.py checks every function here against (a) the
 * committed golden vectors in tests/golden/, which were produced by the REAL
 * reference (oracle/_ref/libamgcl_ref.so, built from /root/reference by
 * oracle/Makefile) with tests/golden/make_golden.py, and (b) that library
 * itself whenever it is present.  The reference's own tests only assert a
 * convergence threshold (tests/test_solver.hpp:71,107), so per-primitive
 * goldens had to be generated from the reference run here.
 *
 * Deliberate differences, all within the stated FP64 tolerances:
 *   - inner_product restates the serial Kahan loop (builtin.hpp:1126-1141);
 *     the reference's OpenMP variant applies the same loop per thread chunk.
 *   - the coarsest-level solve is a dense LU without pivoting in natural
 *     ordering; the reference's skyline LU (solver/skyline_lu.hpp:97-200) is
 *     the same factorisation after a Cuthill-McKee permutation.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef int64_t i64;

/* ------------------------------------------------------------------ primitives */

/* y = alpha*A*x + beta*y ; y untouched-on-read when beta == 0
 * (backend/detail/matrix_ops.hpp:47-83) */
void orc_spmv(i64 n, const i64 *ptr, const i64 *col, const double *val, double alpha,
              const double *x, double beta, double *y)
{
    for (i64 i = 0; i < n; ++i) {
        double sum = 0.0;
        for (i64 e = ptr[i]; e < ptr[i + 1]; ++e) sum += val[e] * x[col[e]];
        if (beta != 0.0) y[i] = alpha * sum + beta * y[i];
        else             y[i] = alpha * sum;
    }
}

/* r = f - A*x (backend/detail/matrix_ops.hpp:85-115) */
void orc_residual(i64 n, const i64 *ptr, const i64 *col, const double *val, const double *f,
                  const double *x, double *r)
{
    for (i64 i = 0; i < n; ++i) {
        double sum = 0.0;
        for (i64 e = ptr[i]; e < ptr[i + 1]; ++e) sum += val[e] * x[col[e]];
        r[i] = f[i] - sum;
    }
}

/* x = 0 (backend/builtin.hpp:1081-1097) */
void orc_clear(i64 n, double *x) { for (i64 i = 0; i < n; ++i) x[i] = 0.0; }

/* y = x (backend/builtin.hpp:1304-1321) */
void orc_copy(i64 n, const double *x, double *y) { for (i64 i = 0; i < n; ++i) y[i] = x[i]; }

/* Kahan-compensated inner product (backend/builtin.hpp:1126-1141) */
double orc_inner_product(i64 n, const double *x, const double *y)
{
    double s = 0.0, c = 0.0;
    for (i64 i = 0; i < n; ++i) {
        double d = x[i] * y[i] - c;
        double t = s + d;
        c = (t - s) - d;
        s = t;
    }
    return s;
}

/* y = a*x + b*y ; y not read when b == 0 (backend/builtin.hpp:1185-1209) */
void orc_axpby(i64 n, double a, const double *x, double b, double *y)
{
    if (b != 0.0) for (i64 i = 0; i < n; ++i) y[i] = a * x[i] + b * y[i];
    else          for (i64 i = 0; i < n; ++i) y[i] = a * x[i];
}

/* z = a*x + b*y + c*z ; z not read when c == 0 (backend/builtin.hpp:1211-1236) */
void orc_axpbypcz(i64 n, double a, const double *x, double b, const double *y, double c, double *z)
{
    if (c != 0.0) for (i64 i = 0; i < n; ++i) z[i] = a * x[i] + b * y[i] + c * z[i];
    else          for (i64 i = 0; i < n; ++i) z[i] = a * x[i] + b * y[i];
}

/* z = a*x.*y + b*z ; z not read when b == 0 (backend/builtin.hpp:1238-1265) */
void orc_vmul(i64 n, double a, const double *x, const double *y, double b, double *z)
{
    if (b != 0.0) for (i64 i = 0; i < n; ++i) z[i] = a * x[i] * y[i] + b * z[i];
    else          for (i64 i = 0; i < n; ++i) z[i] = a * x[i] * y[i];
}

/* ------------------------------------------------------------------ smoothers */

/* D^-1 with zero diagonal -> 1 (backend/builtin.hpp:753-773, diagonal(A, invert=true)) */
void orc_jacobi_diag(i64 n, const i64 *ptr, const i64 *col, const double *val, double *d)
{
    for (i64 i = 0; i < n; ++i) {
        for (i64 e = ptr[i]; e < ptr[i + 1]; ++e) {
            if (col[e] == i) {
                double v = val[e];
                d[i] = (v == 0.0) ? 1.0 : 1.0 / v;
                break;
            }
        }
    }
}

/* SPAI-0: M_i = a_ii / sum_j a_ij^2 (relaxation/spai0.hpp:60-82) */
void orc_spai0_diag(i64 n, const i64 *ptr, const i64 *col, const double *val, double *m)
{
    for (i64 i = 0; i < n; ++i) {
        double num = 0.0, den = 0.0;
        for (i64 e = ptr[i]; e < ptr[i + 1]; ++e) {
            double v = val[e];
            double nv = fabs(v);
            den += nv * nv;
            if (col[e] == i) num += v;
        }
        m[i] = (1.0 / den) * num;
    }
}

/* one smoother sweep: tmp = rhs - A x ; x = omega*diag.*tmp + x
 * (relaxation/damped_jacobi.hpp:103-132 with omega = damping;
 *  relaxation/spai0.hpp:86-109 with omega = 1) */
void orc_relax(i64 n, const i64 *ptr, const i64 *col, const double *val, const double *rhs,
               double *x, double *tmp, const double *diag, double omega)
{
    orc_residual(n, ptr, col, val, rhs, x, tmp);
    orc_vmul(n, omega, diag, tmp, 1.0, x);
}

/* ------------------------------------------------------------------ hierarchy */

typedef struct {
    i64 nrows, ncols;
    const i64 *ptr, *col;
    const double *val;
} orc_csr;

typedef struct {
    orc_csr A, P, R;          /* P, R unused on the coarsest level */
    const double *diag;       /* smoother diagonal (D^-1 or M)     */
    double omega;             /* damping (0.72) or 1 for spai0      */
    double *f, *u, *t;        /* level scratch (amg.hpp:317-319)    */
} orc_level;

typedef struct {
    int nlevels;              /* smoothed levels                    */
    orc_level *lv;
    /* coarsest level: dense LU, no pivoting */
    i64 nc;
    double *LU;               /* nc*nc row-major                    */
    double *cf, *cu;          /* coarse rhs / solution scratch      */
    int npre, npost;
} orc_hier;

orc_hier *orc_hier_create(int max_levels)
{
    orc_hier *h = (orc_hier *)calloc(1, sizeof(orc_hier));
    h->lv = (orc_level *)calloc((size_t)max_levels, sizeof(orc_level));
    h->npre = 1;   /* amg.hpp:141 defaults */
    h->npost = 1;
    return h;
}

void orc_hier_destroy(orc_hier *h)
{
    if (!h) return;
    for (int l = 0; l < h->nlevels; ++l) {
        free(h->lv[l].f); free(h->lv[l].u); free(h->lv[l].t);
    }
    free(h->lv); free(h->LU); free(h->cf); free(h->cu);
    free(h);
}

/* Arrays are borrowed: the caller keeps them alive for the hierarchy's life. */
void orc_hier_add_level(orc_hier *h,
                        i64 n, const i64 *aptr, const i64 *acol, const double *aval,
                        i64 nc, const i64 *pptr, const i64 *pcol, const double *pval,
                        const i64 *rptr, const i64 *rcol, const double *rval,
                        const double *diag, double omega)
{
    orc_level *L = &h->lv[h->nlevels++];
    L->A.nrows = n;  L->A.ncols = n;  L->A.ptr = aptr; L->A.col = acol; L->A.val = aval;
    L->P.nrows = n;  L->P.ncols = nc; L->P.ptr = pptr; L->P.col = pcol; L->P.val = pval;
    L->R.nrows = nc; L->R.ncols = n;  L->R.ptr = rptr; L->R.col = rcol; L->R.val = rval;
    L->diag = diag; L->omega = omega;
    L->f = (double *)calloc((size_t)n, sizeof(double));
    L->u = (double *)calloc((size_t)n, sizeof(double));
    L->t = (double *)calloc((size_t)n, sizeof(double));
}

/* Coarsest level: factorise A = L*U once (the role of skyline_lu's constructor,
 * solver/skyline_lu.hpp:97-176). Returns 0, or -1 on a zero pivot. */
int orc_hier_set_coarse(orc_hier *h, i64 n, const i64 *ptr, const i64 *col, const double *val)
{
    h->nc = n;
    h->LU = (double *)calloc((size_t)(n * n), sizeof(double));
    h->cf = (double *)calloc((size_t)n, sizeof(double));
    h->cu = (double *)calloc((size_t)n, sizeof(double));
    double *a = h->LU;
    for (i64 i = 0; i < n; ++i)
        for (i64 e = ptr[i]; e < ptr[i + 1]; ++e) a[i * n + col[e]] += val[e];
    for (i64 k = 0; k < n; ++k) {
        const double piv = a[k * n + k];
        if (piv == 0.0) return -1;
        const double inv = 1.0 / piv;
        for (i64 i = k + 1; i < n; ++i) {
            double l = a[i * n + k];
            if (l == 0.0) continue;
            l *= inv;
            a[i * n + k] = l;
            double *ri = a + i * n;
            const double *rk = a + k * n;
            for (i64 j = k + 1; j < n; ++j) ri[j] -= l * rk[j];
        }
    }
    return 0;
}

/* x = A^-1 rhs by forward / backward substitution
 * (the role of skyline_lu::operator(), solver/skyline_lu.hpp:179-200) */
void orc_coarse_solve(const orc_hier *h, const double *rhs, double *x)
{
    const i64 n = h->nc;
    const double *a = h->LU;
    for (i64 i = 0; i < n; ++i) {
        double s = rhs[i];
        for (i64 j = 0; j < i; ++j) s -= a[i * n + j] * x[j];
        x[i] = s;
    }
    for (i64 i = n - 1; i >= 0; --i) {
        double s = x[i];
        for (i64 j = i + 1; j < n; ++j) s -= a[i * n + j] * x[j];
        x[i] = s / a[i * n + i];
    }
}

/* recursive V-cycle (amg.hpp:514-553), ncycle = 1 */
static void orc_cycle(orc_hier *h, int l, const double *rhs, double *x)
{
    if (l == h->nlevels) {             /* coarsest: direct solve (amg.hpp:521-524) */
        orc_coarse_solve(h, rhs, x);
        return;
    }
    orc_level *L = &h->lv[l];
    const i64 n = L->A.nrows;
    for (int i = 0; i < h->npre; ++i)                                   /* amg.hpp:534-535 */
        orc_relax(n, L->A.ptr, L->A.col, L->A.val, rhs, x, L->t, L->diag, L->omega);
    orc_residual(n, L->A.ptr, L->A.col, L->A.val, rhs, x, L->t);        /* amg.hpp:538 */

    double *fc, *uc;
    i64 nc = L->R.nrows;
    if (l + 1 < h->nlevels) { fc = h->lv[l + 1].f; uc = h->lv[l + 1].u; }
    else                    { fc = h->cf;          uc = h->cu;          }
    orc_spmv(nc, L->R.ptr, L->R.col, L->R.val, 1.0, L->t, 0.0, fc);     /* amg.hpp:540 */
    orc_clear(nc, uc);                                                  /* amg.hpp:542 */
    orc_cycle(h, l + 1, fc, uc);                                        /* amg.hpp:543 */
    orc_spmv(n, L->P.ptr, L->P.col, L->P.val, 1.0, uc, 1.0, x);         /* amg.hpp:545 */
    for (int i = 0; i < h->npost; ++i)                                  /* amg.hpp:548-549 */
        orc_relax(n, L->A.ptr, L->A.col, L->A.val, rhs, x, L->t, L->diag, L->omega);
}

/* preconditioner application: x = 0; one cycle (amg.hpp:289-297, pre_cycles = 1) */
void orc_amg_apply(orc_hier *h, const double *rhs, double *x)
{
    i64 n = h->nlevels ? h->lv[0].A.nrows : h->nc;
    orc_clear(n, x);
    orc_cycle(h, 0, rhs, x);
}

/* ------------------------------------------------------------------ Krylov */

static double orc_norm(i64 n, const double *x) { return sqrt(fabs(orc_inner_product(n, x, x))); }

/* Preconditioned CG (solver/cg.hpp:153-204).  history (may be NULL) receives the
 * relative residual after every iteration (at most maxiter entries). */
int orc_cg(orc_hier *h, const double *rhs, double *x, double tol, int maxiter,
           i64 *iters_out, double *resid_out, double *history)
{
    const orc_csr *A = &h->lv[0].A;
    const i64 n = A->nrows;
    double *r = (double *)calloc((size_t)n, sizeof(double));
    double *s = (double *)calloc((size_t)n, sizeof(double));
    double *p = (double *)calloc((size_t)n, sizeof(double));
    double *q = (double *)calloc((size_t)n, sizeof(double));

    double norm_rhs = orc_norm(n, rhs);                               /* cg.hpp:161 */
    if (norm_rhs < 2.220446049250313e-16) {                           /* cg.hpp:162-169: eps<double>(1) */
        orc_clear(n, x);
        *iters_out = 0; *resid_out = norm_rhs;
        free(r); free(s); free(p); free(q);
        return 0;
    }
    double eps = tol * norm_rhs;                                      /* cg.hpp:171 (abstol = DBL_MIN) */
    if (eps < 2.2250738585072014e-308) eps = 2.2250738585072014e-308;
    double rho1 = 2 * eps, rho2 = 0.0;                                /* cg.hpp:173-174 */

    orc_residual(n, A->ptr, A->col, A->val, rhs, x, r);               /* cg.hpp:176 */
    double res_norm = orc_norm(n, r);                                 /* cg.hpp:177 */

    i64 iter = 0;
    for (; iter < maxiter && res_norm > eps; ++iter) {                /* cg.hpp:180 */
        orc_amg_apply(h, r, s);                                       /* cg.hpp:181 */
        rho2 = rho1;
        rho1 = orc_inner_product(n, r, s);                            /* cg.hpp:184 */
        if (iter) orc_axpby(n, 1.0, s, rho1 / rho2, p);               /* cg.hpp:186-189 */
        else      orc_copy(n, s, p);
        orc_spmv(n, A->ptr, A->col, A->val, 1.0, p, 0.0, q);          /* cg.hpp:191 */
        double alpha = rho1 / orc_inner_product(n, q, p);             /* cg.hpp:193 */
        orc_axpby(n, alpha, p, 1.0, x);                               /* cg.hpp:195 */
        orc_axpby(n, -alpha, q, 1.0, r);                              /* cg.hpp:196 */
        res_norm = orc_norm(n, r);                                    /* cg.hpp:198 */
        if (history) history[iter] = res_norm / norm_rhs;
    }
    *iters_out = iter;
    *resid_out = res_norm / norm_rhs;                                 /* cg.hpp:203 */
    free(r); free(s); free(p); free(q);
    return 0;
}

/* right-preconditioned spmv: T = M^-1 F ; X = A T (solver/precond_side.hpp:78-94) */
static void orc_pspmv(orc_hier *h, const double *F, double *X, double *T)
{
    const orc_csr *A = &h->lv[0].A;
    orc_amg_apply(h, F, T);
    orc_spmv(A->nrows, A->ptr, A->col, A->val, 1.0, T, 0.0, X);
}

/* BiCGStab, right preconditioning, check_after = false (solver/bicgstab.hpp:158-244).
 * Returns -1 on breakdown (zero rho / omega: bicgstab.hpp:204,226). */
int orc_bicgstab(orc_hier *h, const double *rhs, double *x, double tol, int maxiter,
                 i64 *iters_out, double *resid_out, double *history)
{
    const orc_csr *A = &h->lv[0].A;
    const i64 n = A->nrows;
    double *r  = (double *)calloc((size_t)n, sizeof(double));
    double *p  = (double *)calloc((size_t)n, sizeof(double));
    double *v  = (double *)calloc((size_t)n, sizeof(double));
    double *s  = (double *)calloc((size_t)n, sizeof(double));
    double *t  = (double *)calloc((size_t)n, sizeof(double));
    double *rh = (double *)calloc((size_t)n, sizeof(double));
    double *T  = (double *)calloc((size_t)n, sizeof(double));
    int rc = 0;

    double norm_rhs = orc_norm(n, rhs);
    if (norm_rhs < 2.220446049250313e-16) {
        orc_clear(n, x);
        *iters_out = 0; *resid_out = norm_rhs;
        goto done;
    }
    orc_residual(n, A->ptr, A->col, A->val, rhs, x, r);               /* bicgstab.hpp:180 */
    orc_copy(n, r, rh);                                               /* bicgstab.hpp:182 */
    {
        double eps = norm_rhs * tol;
        if (eps < 2.2250738585072014e-308) eps = 2.2250738585072014e-308;
        double res = orc_norm(n, r);                                  /* bicgstab.hpp:185 */
        double rho1 = 0, rho2 = 0, alpha = 0, omega = 0;
        i64 iter = 0;
        int first = 1;
        for (; res > eps && iter < maxiter; ++iter) {                 /* bicgstab.hpp:193 */
            rho2 = rho1;
            rho1 = orc_inner_product(n, r, rh);                       /* bicgstab.hpp:196 */
            if (first) {
                orc_copy(n, r, p);
                first = 0;
            } else {
                if (rho2 == 0.0) { rc = -1; break; }
                double beta = (rho1 * alpha) / (rho2 * omega);        /* bicgstab.hpp:203 */
                orc_axpbypcz(n, 1.0, r, -beta * omega, v, beta, p);   /* bicgstab.hpp:204 */
            }
            orc_pspmv(h, p, v, T);                                    /* bicgstab.hpp:207 */
            alpha = rho1 / orc_inner_product(n, rh, v);               /* bicgstab.hpp:209 */
            orc_axpby(n, alpha, T, 1.0, x);                           /* bicgstab.hpp:214 */
            orc_axpbypcz(n, 1.0, r, -alpha, v, 0.0, s);               /* bicgstab.hpp:217 */
            if ((res = orc_norm(n, s)) > eps) {                       /* bicgstab.hpp:219 */
                orc_pspmv(h, s, t, T);                                /* bicgstab.hpp:220 */
                omega = orc_inner_product(n, t, s) / orc_inner_product(n, t, t);
                if (omega == 0.0) { rc = -1; break; }
                orc_axpby(n, omega, T, 1.0, x);                       /* bicgstab.hpp:229 */
                orc_axpbypcz(n, 1.0, s, -omega, t, 0.0, r);           /* bicgstab.hpp:232 */
                res = orc_norm(n, r);                                 /* bicgstab.hpp:234 */
            }
            if (history) history[iter] = res / norm_rhs;
        }
        *iters_out = iter;
        *resid_out = res / norm_rhs;
    }
done:
    free(r); free(p); free(v); free(s); free(t); free(rh); free(T);
    return rc;
}

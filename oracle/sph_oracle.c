/*
 * oracle/sph_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * fp64 CPU restatement of the PySPH WCSPH hot path.  Every function cites the
 * reference file:line (relative to /root/reference) it restates.  See
 * sph_oracle.h for the scope and oracle/README.md for how the restatement is
 * pinned against the reference.
 *
 * Build:  gcc -O3 -march=x86-64-v3 -fopenmp -shared -fPIC  (oracle/Makefile)
 * With OpenMP the destination loop is `parallel for` -- the same structure as
 * the reference's `prange` over d_idx (acceleration_eval_cython.mako:87-106).
 */
#include "sph_oracle.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_UINT_MAX 0xFFFFFFFFu
#define M_1_PI_ 0.31830988618379067154
#define M_2_SQRTPI_ 1.12837916709551257390

struct orc_ctx {
    int narr;
    int dim;
    double radius_scale;
    orc_array arr[ORC_MAX_ARRAYS];
    /* domain manager state */
    double cell_size, hmin;
    /* NNPS state */
    double xmin[3], xmax[3];
    int nc[3];
    int64_t n_cells;
    uint32_t *head[ORC_MAX_ARRAYS];
    uint32_t *next[ORC_MAX_ARRAYS];
    int64_t head_cap[ORC_MAX_ARRAYS], next_cap[ORC_MAX_ARRAYS];
    double last_domain_size;
};

/* ------------------------------------------------------------------------ */
/* kernels: pysph/base/kernels.py                                            */
/* ------------------------------------------------------------------------ */

/* kernels.py:57-65 (CubicSpline), :291-299 (WendlandQuintic),
 * :1071-1079 (QuinticSpline), :852-858 (Gaussian) */
static double k_fac(int kernel, int dim)
{
    switch (kernel) {
    case ORC_K_CUBIC:
        return dim == 3 ? M_1_PI_ : (dim == 2 ? 10.0 * M_1_PI_ / 7.0 : 2.0 / 3.0);
    case ORC_K_WENDLAND:
        return dim == 2 ? 7.0 * M_1_PI_ / 4.0 : M_1_PI_ * 21.0 / 16.0;
    case ORC_K_QUINTIC:
        return dim == 1 ? 1.0 / 120.0
                        : (dim == 2 ? M_1_PI_ * 7.0 / 478.0 : M_1_PI_ * 1.0 / 120.0);
    case ORC_K_GAUSSIAN: {
        double f = 0.5 * M_2_SQRTPI_;
        if (dim > 1) f *= 0.5 * M_2_SQRTPI_;
        if (dim > 2) f *= 0.5 * M_2_SQRTPI_;
        return f;
    }
    }
    return 0.0;
}

double orc_kernel_radius_scale(int kernel)
{
    /* kernels.py:54, :288, :1067, :850 */
    return (kernel == ORC_K_QUINTIC || kernel == ORC_K_GAUSSIAN) ? 3.0 : 2.0;
}

double orc_kernel_deltap(int kernel)
{
    /* kernels.py:66-67, :301-302, :1081-1085, :860-862 */
    switch (kernel) {
    case ORC_K_CUBIC: return 2. / 3;
    case ORC_K_WENDLAND: return 0.5;
    case ORC_K_QUINTIC: return 0.759298480738450;
    case ORC_K_GAUSSIAN: return 0.70710678118654746;
    }
    return 0.0;
}

static inline double k_norm(double fac, int dim, double h1)
{
    /* kernels.py:73-79 */
    if (dim == 1) return fac * h1;
    if (dim == 2) return fac * h1 * h1;
    return fac * h1 * h1 * h1;
}

/* kernel():  kernels.py:69-92, :304-321, :1087-1117, :864-879 */
static inline double k_w(int kernel, int dim, double kfac, double rij, double h)
{
    double h1 = 1. / h;
    double q = rij * h1;
    double fac = k_norm(kfac, dim, h1);
    double val = 0.0;
    switch (kernel) {
    case ORC_K_CUBIC: {
        double tmp2 = 2. - q;
        if (q > 2.0) val = 0.0;
        else if (q > 1.0) val = 0.25 * tmp2 * tmp2 * tmp2;
        else val = 1 - 1.5 * q * q * (1 - 0.5 * q);
        return val * fac;
    }
    case ORC_K_WENDLAND: {
        double tmp = 1. - 0.5 * q;
        if (q < 2.0) val = tmp * tmp * tmp * tmp * (2.0 * q + 1.0);
        return val * fac;
    }
    case ORC_K_QUINTIC: {
        double tmp3 = 3. - q, tmp2 = 2. - q, tmp1 = 1. - q;
        if (q > 3.0) val = 0.0;
        else if (q > 2.0) val = tmp3 * tmp3 * tmp3 * tmp3 * tmp3;
        else if (q > 1.0) {
            val = tmp3 * tmp3 * tmp3 * tmp3 * tmp3;
            val -= 6.0 * tmp2 * tmp2 * tmp2 * tmp2 * tmp2;
        } else {
            val = tmp3 * tmp3 * tmp3 * tmp3 * tmp3;
            val -= 6.0 * tmp2 * tmp2 * tmp2 * tmp2 * tmp2;
            val += 15. * tmp1 * tmp1 * tmp1 * tmp1 * tmp1;
        }
        return val * fac;
    }
    case ORC_K_GAUSSIAN:
        if (q < 3.0) val = exp(-q * q) * fac;
        return val;
    }
    return 0.0;
}

/* dwdq():  kernels.py:94-124, :323-343, :1119-1153, :881-898 */
static inline double k_dwdq(int kernel, int dim, double kfac, double rij, double h)
{
    double h1 = 1. / h;
    double q = rij * h1;
    double fac = k_norm(kfac, dim, h1);
    double val = 0.0;
    switch (kernel) {
    case ORC_K_CUBIC: {
        double tmp2 = 2. - q;
        if (rij > 1e-12) {
            if (q > 2.0) val = 0.0;
            else if (q > 1.0) val = -0.75 * tmp2 * tmp2;
            else val = -3.0 * q * (1 - 0.75 * q);
        }
        return val * fac;
    }
    case ORC_K_WENDLAND: {
        double tmp = 1.0 - 0.5 * q;
        if (q < 2.0)
            if (rij > 1e-12) val = -5.0 * q * tmp * tmp * tmp;
        return val * fac;
    }
    case ORC_K_QUINTIC: {
        double tmp3 = 3. - q, tmp2 = 2. - q, tmp1 = 1. - q;
        if (rij > 1e-12) {
            if (q > 3.0) val = 0.0;
            else if (q > 2.0) val = -5.0 * tmp3 * tmp3 * tmp3 * tmp3;
            else if (q > 1.0) {
                val = -5.0 * tmp3 * tmp3 * tmp3 * tmp3;
                val += 30.0 * tmp2 * tmp2 * tmp2 * tmp2;
            } else {
                val = -5.0 * tmp3 * tmp3 * tmp3 * tmp3;
                val += 30.0 * tmp2 * tmp2 * tmp2 * tmp2;
                val -= 75.0 * tmp1 * tmp1 * tmp1 * tmp1;
            }
        }
        return val * fac;
    }
    case ORC_K_GAUSSIAN:
        if (q < 3.0)
            if (rij > 1e-12) val = -2.0 * q * exp(-q * q);
        return val * fac;
    }
    return 0.0;
}

/* gradient():  kernels.py:126-136 (same body in every kernel class) */
static inline void k_grad(int kernel, int dim, double kfac, const double xij[3],
                          double rij, double h, double grad[3])
{
    double h1 = 1. / h;
    double tmp;
    if (rij > 1e-12) {
        double wdash = k_dwdq(kernel, dim, kfac, rij, h);
        tmp = wdash * h1 / rij;
    } else {
        tmp = 0.0;
    }
    grad[0] = tmp * xij[0];
    grad[1] = tmp * xij[1];
    grad[2] = tmp * xij[2];
}

double orc_kernel_w(int kernel, int dim, double rij, double h)
{
    return k_w(kernel, dim, k_fac(kernel, dim), rij, h);
}

void orc_kernel_grad(int kernel, int dim, const double xij[3], double rij,
                     double h, double grad[3])
{
    k_grad(kernel, dim, k_fac(kernel, dim), xij, rij, h, grad);
}

/* ------------------------------------------------------------------------ */
/* context                                                                   */
/* ------------------------------------------------------------------------ */

orc_ctx *orc_create(int narrays, int dim, double radius_scale)
{
    if (narrays < 1 || narrays > ORC_MAX_ARRAYS) return NULL;
    orc_ctx *c = (orc_ctx *)calloc(1, sizeof(orc_ctx));
    c->narr = narrays;
    c->dim = dim;
    c->radius_scale = radius_scale;
    c->cell_size = 1.0;
    c->hmin = 1.0;
    c->last_domain_size = 0.0;
    return c;
}

void orc_destroy(orc_ctx *c)
{
    if (!c) return;
    for (int i = 0; i < ORC_MAX_ARRAYS; i++) {
        free(c->head[i]);
        free(c->next[i]);
    }
    free(c);
}

void orc_set_array(orc_ctx *c, int idx, const orc_array *a) { c->arr[idx] = *a; }

void orc_set_num_threads(int n)
{
#ifdef _OPENMP
    omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int orc_get_max_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* ------------------------------------------------------------------------ */
/* domain manager + NNPS                                                     */
/* ------------------------------------------------------------------------ */

/* CPUDomainManager._compute_cell_size_for_binning  nnps_base.pyx:942-978 */
void orc_update_domain(orc_ctx *c)
{
    double hmax = -1.0, hmin = 1.7976931348623157e308;
    for (int a = 0; a < c->narr; a++) {
        const orc_array *pa = &c->arr[a];
        /* BaseArray.update_min_max on an empty array leaves the defaults;
         * an empty array simply does not contribute here */
        for (int64_t i = 0; i < pa->n; i++) {
            double h = pa->h[i];
            if (h > hmax) hmax = h;
            if (h < hmin) hmin = h;
        }
    }
    double cell_size = c->radius_scale * hmax;
    c->hmin = c->radius_scale * hmin;
    if (cell_size < 1e-6) cell_size = 1.0;
    c->cell_size = cell_size;
}

/* NNPS._compute_bounds  nnps_base.pyx:1520-1575 */
static void compute_bounds(orc_ctx *c)
{
    double mx[3] = {-1e100, -1e100, -1e100};
    double mn[3] = {1e100, 1e100, 1e100};
    for (int a = 0; a < c->narr; a++) {
        const orc_array *pa = &c->arr[a];
        for (int64_t i = 0; i < pa->n; i++) {
            double p[3] = {pa->x[i], pa->y[i], pa->z[i]};
            for (int d = 0; d < 3; d++) {
                mx[d] = fmax(p[d], mx[d]);
                mn[d] = fmin(p[d], mn[d]);
            }
        }
    }
    double l[3];
    for (int d = 0; d < 3; d++) l[d] = mx[d] - mn[d];
    for (int d = 0; d < 3; d++) {
        mn[d] -= l[d] * 0.01;
        mx[d] += l[d] * 0.01;
    }
    double domain_size = fmax(fmax(l[0], l[1]), l[2]);
    if (c->last_domain_size > 1e-16 && domain_size > 2.0 * c->last_domain_size) {
        /* nnps_base.pyx:1552-1563: the reference only prints a warning */
        fprintf(stderr, "oracle WARNING: Domain size has increased by a large "
                        "amount. Particles are probably diverging.\n");
    }
    c->last_domain_size = domain_size;
    double eps = 1e-12;
    if (fabs(mx[0] - mn[0]) < eps && fabs(mx[1] - mn[1]) < eps &&
        fabs(mx[2] - mn[2]) < eps) {
        for (int d = 0; d < 3; d++) {
            mn[d] -= 0.5;
            mx[d] += 0.5;
        }
    }
    for (int d = 0; d < 3; d++) {
        c->xmin[d] = mn[d];
        c->xmax[d] = mx[d];
    }
}

/* real_to_int / find_cell_id_raw  nnps_base.pxd:39-80 */
static inline int real_to_int(double v, double step) { return (int)floor(v / step); }

/* flatten_raw  nnps_base.pxd:84-96 */
static inline int64_t flatten_raw(int x, int y, int z, const int *nc)
{
    int64_t ncx = nc[0], ncy = nc[1];
    return (int64_t)x + ncx * y + ncx * ncy * z;
}

/* get_valid_cell_index  nnps_base.pxd:113-135 */
static inline int64_t valid_cell_index(int cx, int cy, int cz, const int *nc,
                                       int64_t n_cells)
{
    int64_t idx = -1;
    int ok = (nc[0] > cx && cx > -1) && (nc[1] > cy && cy > -1) &&
             (nc[2] > cz && cz > -1);
    if (ok) {
        idx = flatten_raw(cx, cy, cz, nc);
        if (!(-1 < idx && idx < n_cells)) idx = -1;
    }
    return idx;
}

int orc_nnps_update(orc_ctx *c)
{
    /* NNPS.update  nnps_base.pyx:1471-1510 (cell_size, hmin come from the
     * domain manager, i.e. the last orc_update_domain call) */
    compute_bounds(c);

    /* LinkedListNNPS._get_number_of_cells  linked_list_nnps.pyx:293-326 */
    double cs1 = 1. / c->cell_size;
    int nc[3];
    for (int d = 0; d < 3; d++) {
        const double extent = cs1 * (c->xmax[d] - c->xmin[d]);
        if (!(extent >= 0.0 && extent < 2147483647.0)) return -3; /* NaN / inf positions: a blown-up run */
        nc[d] = (int)ceil(extent);
        if (nc[d] < 0) return -2;
        if (nc[d] == 0) nc[d] = 1;
        c->nc[d] = nc[d];
    }
    int64_t ncells = nc[0];
    if (c->dim == 2) ncells = (int64_t)nc[0] * nc[1];
    if (c->dim == 3) ncells = (int64_t)nc[0] * nc[1] * nc[2];
    /* _count_occupied_cells  linked_list_nnps.pyx:336-343 */
    if (ncells < 0 || ncells > (1LL << 28)) return -1;
    c->n_cells = ncells;
    /* The reference sizes head[] by the dim-dependent count above but flattens cell ids
     * with all three indices (flatten_raw ignores `dim`, nnps_base.pxd:84-96), so a 1-D /
     * 2-D problem whose particles spread along an unused axis -- e.g. the +-0.5 padding
     * of a degenerate box, nnps_base.pyx:1565-1572 -- writes past its table there.  The
     * oracle keeps the reported n_cells and the lookup bound, but owns enough storage. */
    const int64_t storage = (int64_t)nc[0] * nc[1] * nc[2];
    if (storage < 0 || storage > (1LL << 28)) return -1;
    if (storage > ncells) ncells = storage;

    /* _refresh  linked_list_nnps.pyx:345-382 and _bin :235-286 */
    for (int a = 0; a < c->narr; a++) {
        const orc_array *pa = &c->arr[a];
        if (c->head_cap[a] < ncells) {
            free(c->head[a]);
            c->head[a] = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)ncells);
            c->head_cap[a] = ncells;
        }
        if (c->next_cap[a] < pa->n) {
            free(c->next[a]);
            c->next[a] = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)(pa->n + 1));
            c->next_cap[a] = pa->n;
        }
        uint32_t *head = c->head[a], *next = c->next[a];
        memset(head, 0xFF, sizeof(uint32_t) * (size_t)ncells);
        for (int64_t i = 0; i < pa->n; i++) {
            int cx = real_to_int(pa->x[i] - c->xmin[0], c->cell_size);
            int cy = real_to_int(pa->y[i] - c->xmin[1], c->cell_size);
            int cz = real_to_int(pa->z[i] - c->xmin[2], c->cell_size);
            int64_t cid = flatten_raw(cx, cy, cz, nc);
            if (cid < 0 || cid >= ncells) return -3; /* a non-finite position */
            next[i] = head[cid];
            head[cid] = (uint32_t)i;
        }
    }
    return 0;
}

void orc_get_grid(orc_ctx *c, double *cell_size, double *hmin, double xmin[3],
                  double xmax[3], int ncells[3], int64_t *n_cells)
{
    *cell_size = c->cell_size;
    *hmin = c->hmin;
    for (int d = 0; d < 3; d++) {
        xmin[d] = c->xmin[d];
        xmax[d] = c->xmax[d];
        ncells[d] = c->nc[d];
    }
    *n_cells = c->n_cells;
}

/* Visit every neighbour of (dst, d_idx) in src in the reference's order:
 * 27 cells with ix outermost, iz innermost; shifts = (-1, 0, 1); each cell's
 * linked list front to back.  linked_list_nnps.pyx:92-196 */
#define ORC_FOR_NEIGHBORS(c, dst, src, d_idx, S_IDX, ...)                           \
    do {                                                                            \
        const orc_array *_d = &(c)->arr[dst], *_s = &(c)->arr[src];                 \
        const uint32_t *_head = (c)->head[src], *_next = (c)->next[src];            \
        double _x = _d->x[d_idx], _y = _d->y[d_idx], _z = _d->z[d_idx];             \
        int _cx = real_to_int(_x - (c)->xmin[0], (c)->cell_size);                   \
        int _cy = real_to_int(_y - (c)->xmin[1], (c)->cell_size);                   \
        int _cz = real_to_int(_z - (c)->xmin[2], (c)->cell_size);                   \
        double _hi2 = (c)->radius_scale * _d->h[d_idx];                             \
        _hi2 *= _hi2;                                                               \
        for (int _ix = -1; _ix <= 1; _ix++)                                         \
            for (int _iy = -1; _iy <= 1; _iy++)                                     \
                for (int _iz = -1; _iz <= 1; _iz++) {                               \
                    int64_t _ci = valid_cell_index(_cx + _ix, _cy + _iy, _cz + _iz, \
                                                   (c)->nc, (c)->n_cells);          \
                    if (_ci < 0) continue;                                          \
                    uint32_t _n = _head[_ci];                                       \
                    while (_n != ORC_UINT_MAX) {                                    \
                        double _hj2 = (c)->radius_scale * _s->h[_n];                \
                        _hj2 *= _hj2;                                               \
                        double _dx = _s->x[_n] - _x, _dy = _s->y[_n] - _y,          \
                               _dz = _s->z[_n] - _z;                                \
                        double _r2 = _dx * _dx + _dy * _dy + _dz * _dz;             \
                        if (_r2 < _hi2 || _r2 < _hj2) {                             \
                            int64_t S_IDX = (int64_t)_n;                            \
                            __VA_ARGS__                                             \
                        }                                                           \
                        _n = _next[_n];                                             \
                    }                                                               \
                }                                                                   \
    } while (0)

int64_t orc_find_neighbors(orc_ctx *c, int dst, int src, int64_t d_idx,
                           uint32_t *out, int64_t cap)
{
    int64_t n = 0;
    ORC_FOR_NEIGHBORS(c, dst, src, d_idx, s_idx, {
        if (n < cap) out[n] = (uint32_t)s_idx;
        n++;
    });
    return n;
}

/* NNPS.brute_force_neighbors  nnps_base.pyx:1325-1366 */
int64_t orc_brute_neighbors(orc_ctx *c, int dst, int src, int64_t d_idx,
                            uint32_t *out, int64_t cap)
{
    const orc_array *d = &c->arr[dst], *s = &c->arr[src];
    double xi = d->x[d_idx], yi = d->y[d_idx], zi = d->z[d_idx];
    double hi = d->h[d_idx] * c->radius_scale;
    int64_t n = 0;
    for (int64_t j = 0; j < s->n; j++) {
        double hj = c->radius_scale * s->h[j];
        double dx = xi - s->x[j], dy = yi - s->y[j], dz = zi - s->z[j];
        double r2 = dx * dx + dy * dy + dz * dz;
        if (r2 < hi * hi || r2 < hj * hj) {
            if (n < cap) out[n] = (uint32_t)j;
            n++;
        }
    }
    return n;
}

/* ------------------------------------------------------------------------ */
/* no-source equations                                                       */
/* ------------------------------------------------------------------------ */

/* TaitEOS.loop wc/basic.py:60-65; TaitEOSHGCorrection.loop :118-126 */
void orc_eos(orc_ctx *c, int arr, int hg, double rho0, double c0, double gamma,
             double p0, int real_only)
{
    orc_array *pa = &c->arr[arr];
    int64_t n = real_only ? pa->n_real : pa->n;
    double rho01 = 1.0 / rho0;
    double gamma1 = 0.5 * (gamma - 1.0);
    double B = rho0 * c0 * c0 / gamma;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; i++) {
        if (hg) {
            if (pa->rho[i] < rho0) pa->rho[i] = rho0;
            double ratio = pa->rho[i] * rho01;
            double tmp = pow(ratio, gamma);
            pa->p[i] = B * (tmp - 1.0);
            pa->cs[i] = c0 * pow(ratio, gamma1);
        } else {
            double ratio = pa->rho[i] * rho01;
            double tmp = pow(ratio, gamma);
            pa->p[i] = p0 + B * (tmp - 1.0);
            pa->cs[i] = c0 * pow(ratio, gamma1);
        }
    }
}

/* UpdateSmoothingLengthFerrari.loop  wc/basic.py:458-463 */
void orc_ferrari_h(orc_ctx *c, int arr, double hdx, int dim, int real_only)
{
    orc_array *pa = &c->arr[arr];
    int64_t n = real_only ? pa->n_real : pa->n;
    double dim1 = 1. / dim;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; i++) {
        double Vj = pa->m[i] / pa->rho[i];
        pa->h[i] = hdx * pow(Vj, dim1);
    }
}

/* ------------------------------------------------------------------------ */
/* pair pass: acceleration_eval_cython.mako:10-154                           */
/* ------------------------------------------------------------------------ */

int64_t orc_pair_pass(orc_ctx *c, const orc_pair_program *P)
{
    const int kernel = P->kernel, dim = P->dim;
    const double kfac = k_fac(kernel, dim);
    const double deltap = orc_kernel_deltap(kernel);
    int64_t total_pairs = 0;

    for (int dk = 0; dk < ORC_MAX_ARRAYS && P->dest_order[dk] >= 0; dk++) {
        const int dst = P->dest_order[dk];
        orc_array *D = &c->arr[dst];
        const int64_t np = P->real_only ? D->n_real : D->n;

        uint32_t all_bits = 0;
        for (int s = 0; s < c->narr; s++) all_bits |= P->eqmask[dst][s];
        if (!all_bits) continue;

        /* initialize: every equation of this destination, mako:40-46
         * SummationDensity basic_equations.py:25-26; Continuity :187-188;
         * Momentum wc/basic.py:198-202; XSPH basic_equations.py:285-288;
         * MonaghanArtificialViscosity :235-238 */
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < np; i++) {
            if (all_bits & ORC_EQ_SUMDENS) D->rho[i] = 0.0;
            if (all_bits & ORC_EQ_CONT) D->arho[i] = 0.0;
            if (all_bits & (ORC_EQ_MOM | ORC_EQ_AV)) {
                D->au[i] = 0.0;
                D->av[i] = 0.0;
                D->aw[i] = 0.0;
            }
            if (all_bits & ORC_EQ_MOM) D->dt_cfl[i] = 0.0;
            if (all_bits & ORC_EQ_XSPH) {
                D->ax[i] = 0.0;
                D->ay[i] = 0.0;
                D->az[i] = 0.0;
            }
        }

        /* per-source loops in first-mention order, mako:63-111 */
        for (int sk = 0; sk < ORC_MAX_ARRAYS && P->src_order[dst][sk] >= 0; sk++) {
            const int src = P->src_order[dst][sk];
            const uint32_t bits = P->eqmask[dst][src];
            if (!bits) continue;
            const orc_array *S = &c->arr[src];
            int64_t pairs = 0;

#pragma omp parallel for schedule(dynamic, 256) reduction(+ : pairs)
            for (int64_t d_idx = 0; d_idx < np; d_idx++) {
                ORC_FOR_NEIGHBORS(c, dst, src, d_idx, s_idx, {
                    pairs++;
                    /* precomputed symbols, equation.py:188-297 */
                    double XIJ[3], VIJ[3] = {0, 0, 0}, DWIJ[3] = {0, 0, 0};
                    XIJ[0] = D->x[d_idx] - S->x[s_idx];
                    XIJ[1] = D->y[d_idx] - S->y[s_idx];
                    XIJ[2] = D->z[d_idx] - S->z[s_idx];
                    double R2IJ = XIJ[0] * XIJ[0] + XIJ[1] * XIJ[1] + XIJ[2] * XIJ[2];
                    double RIJ = sqrt(R2IJ);
                    double HIJ = 0.5 * (D->h[d_idx] + S->h[s_idx]);
                    double WIJ = 0.0, RHOIJ1 = 0.0, EPS = 0.01 * HIJ * HIJ;
                    if (bits & (ORC_EQ_CONT | ORC_EQ_MOM | ORC_EQ_XSPH | ORC_EQ_AV | ORC_EQ_LAMINAR)) {
                        VIJ[0] = D->u[d_idx] - S->u[s_idx];
                        VIJ[1] = D->v[d_idx] - S->v[s_idx];
                        VIJ[2] = D->w[d_idx] - S->w[s_idx];
                    }
                    if (bits & (ORC_EQ_MOM | ORC_EQ_XSPH | ORC_EQ_AV)) {
                        double RHOIJ = 0.5 * (D->rho[d_idx] + S->rho[s_idx]);
                        RHOIJ1 = 1.0 / RHOIJ;
                    }
                    if (bits & (ORC_EQ_SUMDENS | ORC_EQ_MOM | ORC_EQ_XSPH))
                        WIJ = k_w(kernel, dim, kfac, RIJ, HIJ);
                    if (bits & (ORC_EQ_CONT | ORC_EQ_MOM | ORC_EQ_AV | ORC_EQ_LAMINAR))
                        k_grad(kernel, dim, kfac, XIJ, RIJ, HIJ, DWIJ);

                    /* equations in user order (scheme.py:452-483: Continuity,
                     * Momentum, XSPH) */
                    if (bits & ORC_EQ_SUMDENS) {
                        /* basic_equations.py:28-29 */
                        D->rho[d_idx] += S->m[s_idx] * WIJ;
                    }
                    if (bits & ORC_EQ_CONT) {
                        /* basic_equations.py:190-192 */
                        double vijdotdwij =
                            DWIJ[0] * VIJ[0] + DWIJ[1] * VIJ[1] + DWIJ[2] * VIJ[2];
                        D->arho[d_idx] += S->m[s_idx] * vijdotdwij;
                    }
                    if (bits & ORC_EQ_MOM) {
                        /* wc/basic.py:204-257 */
                        double rhoi21 = 1.0 / (D->rho[d_idx] * D->rho[d_idx]);
                        double rhoj21 = 1.0 / (S->rho[s_idx] * S->rho[s_idx]);
                        double vijdotxij =
                            VIJ[0] * XIJ[0] + VIJ[1] * XIJ[1] + VIJ[2] * XIJ[2];
                        double piij = 0.0;
                        if (vijdotxij < 0) {
                            double cij = 0.5 * (D->cs[d_idx] + S->cs[s_idx]);
                            double muij = (HIJ * vijdotxij) / (R2IJ + EPS);
                            piij = -P->alpha * cij * muij + P->beta * muij * muij;
                            piij = piij * RHOIJ1;
                        }
                        double _dt_cfl = 0.0;
                        if (R2IJ > 1e-12) {
                            _dt_cfl = fabs(HIJ * vijdotxij / R2IJ) + P->c0;
                            D->dt_cfl[d_idx] = fmax(_dt_cfl, D->dt_cfl[d_idx]);
                        }
                        double tmpi = D->p[d_idx] * rhoi21;
                        double tmpj = S->p[s_idx] * rhoj21;
                        double WDP = k_w(kernel, dim, kfac, deltap * HIJ, HIJ);
                        double fij = WIJ / WDP;
                        double Ri = 0.0, Rj = 0.0;
                        if (P->tensile_correction) {
                            fij = fij * fij;
                            fij = fij * fij;
                            if (D->p[d_idx] > 0) Ri = 0.01 * tmpi;
                            else Ri = 0.2 * fabs(tmpi);
                            if (S->p[s_idx] > 0) Rj = 0.01 * tmpj;
                            else Rj = 0.2 * fabs(tmpj);
                        }
                        double tmp = (tmpi + tmpj) + (Ri + Rj) * fij;
                        D->au[d_idx] += -S->m[s_idx] * (tmp + piij) * DWIJ[0];
                        D->av[d_idx] += -S->m[s_idx] * (tmp + piij) * DWIJ[1];
                        D->aw[d_idx] += -S->m[s_idx] * (tmp + piij) * DWIJ[2];
                    }
                    if (bits & ORC_EQ_AV) {
                        /* basic_equations.py:240-257 */
                        double vijdotxij =
                            VIJ[0] * XIJ[0] + VIJ[1] * XIJ[1] + VIJ[2] * XIJ[2];
                        double piij = 0.0;
                        if (vijdotxij < 0) {
                            double cij = 0.5 * (D->cs[d_idx] + S->cs[s_idx]);
                            double muij = (HIJ * vijdotxij) / (R2IJ + EPS);
                            piij = -P->alpha * cij * muij + P->beta * muij * muij;
                            piij = piij * RHOIJ1;
                        }
                        D->au[d_idx] += -S->m[s_idx] * piij * DWIJ[0];
                        D->av[d_idx] += -S->m[s_idx] * piij * DWIJ[1];
                        D->aw[d_idx] += -S->m[s_idx] * piij * DWIJ[2];
                    }
                    if (bits & ORC_EQ_LAMINAR) {
                        /* wc/viscosity.py:12-27 (inserted before XSPH, scheme.py:496) */
                        const double rhoa = D->rho[d_idx], rhob = S->rho[s_idx];
                        const double Fij = DWIJ[0] * XIJ[0] + DWIJ[1] * XIJ[1] + DWIJ[2] * XIJ[2];
                        const double tmp = S->m[s_idx] * 4 * P->nu * Fij / ((rhoa + rhob) * (R2IJ + P->eta * HIJ * HIJ));
                        D->au[d_idx] += tmp * VIJ[0];
                        D->av[d_idx] += tmp * VIJ[1];
                        D->aw[d_idx] += tmp * VIJ[2];
                    }
                    if (bits & ORC_EQ_XSPH) {
                        /* basic_equations.py:290-295 */
                        double tmp = -P->eps_xsph * S->m[s_idx] * WIJ * RHOIJ1;
                        D->ax[d_idx] += tmp * VIJ[0];
                        D->ay[d_idx] += tmp * VIJ[1];
                        D->az[d_idx] += tmp * VIJ[2];
                    }
                });
            }
            total_pairs += pairs;
        }

        /* post_loop, mako:116-122.  Momentum wc/basic.py:259-269,
         * XSPH basic_equations.py:297-300 */
        if (all_bits & (ORC_EQ_MOM | ORC_EQ_XSPH)) {
#pragma omp parallel for schedule(static)
            for (int64_t i = 0; i < np; i++) {
                if (all_bits & ORC_EQ_MOM) {
                    D->au[i] += P->gx;
                    D->av[i] += P->gy;
                    D->aw[i] += P->gz;
                    double acc2 = D->au[i] * D->au[i] + D->av[i] * D->av[i] +
                                  D->aw[i] * D->aw[i];
                    D->dt_force[i] = acc2;
                }
                if (all_bits & ORC_EQ_XSPH) {
                    D->ax[i] += D->u[i];
                    D->ay[i] += D->v[i];
                    D->az[i] += D->w[i];
                }
            }
        }
    }
    return total_pairs;
}

/* ------------------------------------------------------------------------ */
/* WCSPHStep  integrator_step.py:38-91; loops over real particles only       */
/* (integrator_cython.mako:97-111)                                           */
/* ------------------------------------------------------------------------ */
void orc_stage(orc_ctx *c, int arr, int which, double dt)
{
    orc_array *A = &c->arr[arr];
    const int64_t n = A->n_real;
    if (which == 0) {
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < n; i++) {
            A->x0[i] = A->x[i];
            A->y0[i] = A->y[i];
            A->z0[i] = A->z[i];
            A->u0[i] = A->u[i];
            A->v0[i] = A->v[i];
            A->w0[i] = A->w[i];
            A->rho0[i] = A->rho[i];
        }
    } else {
        const double f = (which == 1) ? 0.5 * dt : dt;
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < n; i++) {
            A->u[i] = A->u0[i] + f * A->au[i];
            A->v[i] = A->v0[i] + f * A->av[i];
            A->w[i] = A->w0[i] + f * A->aw[i];
            A->x[i] = A->x0[i] + f * A->ax[i];
            A->y[i] = A->y0[i] + f * A->ay[i];
            A->z[i] = A->z0[i] + f * A->az[i];
            A->rho[i] = A->rho0[i] + f * A->arho[i];
        }
    }
}

/* Integrator._get_dt_adapt_factors integrator.py:62-81 (np.max over the real
 * particles, -1.0 if empty) and compute_h_minimum :146-159 */
void orc_dt_factors(orc_ctx *c, double out[3])
{
    double f_cfl = -1.0, f_force = -1.0, hmin = 1.0;
    for (int a = 0; a < c->narr; a++) {
        const orc_array *A = &c->arr[a];
        /* pa.get(name) returns the REAL particles only (particle_array.pyx:704-765);
         * get_carray('h').minimum spans all particles */
        for (int64_t i = 0; i < A->n_real; i++) {
            if (A->dt_cfl && A->dt_cfl[i] > f_cfl) f_cfl = A->dt_cfl[i];
            if (A->dt_force && A->dt_force[i] > f_force) f_force = A->dt_force[i];
        }
        for (int64_t i = 0; i < A->n; i++)
            if (A->h[i] < hmin) hmin = A->h[i];
    }
    out[0] = f_cfl;
    out[1] = f_force;
    out[2] = hmin;
}


/* ------------------------------------------------------------------------ */
/* EDAC scheme, transport-velocity branch (fluids only)                       */
/* ------------------------------------------------------------------------ */

int64_t orc_tvf_pass1(orc_ctx *c, const orc_tvf_program *P)
{
    const int kernel = P->kernel, dim = P->dim;
    const double kfac = k_fac(kernel, dim);
    int64_t total = 0;
    for (int dst = 0; dst < c->narr; dst++) {
        if (!(P->fluid_mask >> dst & 1u)) continue;
        orc_array *D = &c->arr[dst];
        const int64_t np = D->n; /* Group(real=False), wc/edac.py:838 */
        /* initialize: transport_velocity.py:52-54, wc/edac.py:69-71 */
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < np; i++) {
            D->V[i] = 0.0;
            D->rho[i] = 0.0;
            if (P->bql) {
                D->pavg[i] = 0.0;
                D->nnbr[i] = 0.0;
            }
        }
        for (int src = 0; src < c->narr; src++) {
            /* SummationDensity(dest=fluid, sources=all), wc/edac.py:806 */
            if (!((P->fluid_mask | P->solid_mask) >> src & 1u)) continue;
            const orc_array *S = &c->arr[src];
            int64_t pairs = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : pairs)
            for (int64_t d_idx = 0; d_idx < np; d_idx++) {
                ORC_FOR_NEIGHBORS(c, dst, src, d_idx, s_idx, {
                    pairs++;
                    double XIJ[3];
                    XIJ[0] = D->x[d_idx] - S->x[s_idx];
                    XIJ[1] = D->y[d_idx] - S->y[s_idx];
                    XIJ[2] = D->z[d_idx] - S->z[s_idx];
                    const double RIJ = sqrt(XIJ[0] * XIJ[0] + XIJ[1] * XIJ[1] + XIJ[2] * XIJ[2]);
                    const double HIJ = 0.5 * (D->h[d_idx] + S->h[s_idx]);
                    const double WIJ = k_w(kernel, dim, kfac, RIJ, HIJ);
                    /* transport_velocity.py:56-58 */
                    D->V[d_idx] += WIJ;
                    D->rho[d_idx] += D->m[d_idx] * WIJ;
                    if (P->bql) { /* wc/edac.py:73-75 */
                        D->pavg[d_idx] += S->p[s_idx];
                        D->nnbr[d_idx] += 1.0;
                    }
                });
            }
            total += pairs;
        }
        if (P->bql) { /* post_loop wc/edac.py:77-79 */
#pragma omp parallel for schedule(static)
            for (int64_t i = 0; i < np; i++)
                if (D->nnbr[i] > 0) D->pavg[i] /= D->nnbr[i];
        }
    }
    return total;
}

int64_t orc_tvf_wall(orc_ctx *c, const orc_tvf_program *P)
{
    const int kernel = P->kernel, dim = P->dim;
    const double kfac = k_fac(kernel, dim);
    int64_t total = 0;
    double damp = 1.0; /* SolidWallPressureBC takes the body force undamped, wc/edac.py:141-161 */
    (void)damp;
    for (int dst = 0; dst < c->narr; dst++) {
        if (!(P->solid_mask >> dst & 1u)) continue;
        orc_array *D = &c->arr[dst];
        const int64_t np = D->n; /* Group(real=False), wc/edac.py:838 */
        /* initialize: wc/edac.py:148-149, :179-180, :203-206; transport_velocity.py:71-72 */
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < np; i++) {
            D->wij[i] = 0.0;
            D->V[i] = 0.0;
            D->p[i] = 0.0;
            D->uf[i] = D->vf[i] = D->wf[i] = 0.0;
        }
        for (int src = 0; src < c->narr; src++) {
            const int is_fluid = (P->fluid_mask >> src) & 1u;
            if (!((P->fluid_mask | P->solid_mask) >> src & 1u)) continue;
            const orc_array *S = &c->arr[src];
            int64_t pairs = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : pairs)
            for (int64_t d_idx = 0; d_idx < np; d_idx++) {
                ORC_FOR_NEIGHBORS(c, dst, src, d_idx, s_idx, {
                    pairs++;
                    double XIJ[3];
                    XIJ[0] = D->x[d_idx] - S->x[s_idx];
                    XIJ[1] = D->y[d_idx] - S->y[s_idx];
                    XIJ[2] = D->z[d_idx] - S->z[s_idx];
                    const double RIJ = sqrt(XIJ[0] * XIJ[0] + XIJ[1] * XIJ[1] + XIJ[2] * XIJ[2]);
                    const double HIJ = 0.5 * (D->h[d_idx] + S->h[s_idx]);
                    const double WIJ = k_w(kernel, dim, kfac, RIJ, HIJ);
                    D->V[d_idx] += WIJ;                 /* VolumeSummation, sources = all */
                    if (is_fluid) {
                        D->wij[d_idx] += WIJ;           /* SourceNumberDensity            */
                        /* SolidWallPressureBC.loop wc/edac.py:151-161 */
                        const double gdotxij = (P->gx - D->au[d_idx]) * XIJ[0] + (P->gy - D->av[d_idx]) * XIJ[1] +
                                               (P->gz - D->aw[d_idx]) * XIJ[2];
                        D->p[d_idx] += S->p[s_idx] * WIJ + S->rho[s_idx] * gdotxij * WIJ;
                        /* SetWallVelocity.loop wc/edac.py:208-214 */
                        D->uf[d_idx] += S->u[s_idx] * WIJ;
                        D->vf[d_idx] += S->v[s_idx] * WIJ;
                        D->wf[d_idx] += S->w[s_idx] * WIJ;
                    }
                });
            }
            total += pairs;
        }
        /* post_loop: wc/edac.py:163-166 and :216-230 */
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < np; i++) {
            if (D->wij[i] > 1e-14) D->p[i] /= D->wij[i];
            if (D->wij[i] > 1e-12) {
                D->uf[i] /= D->wij[i];
                D->vf[i] /= D->wij[i];
                D->wf[i] /= D->wij[i];
            }
            D->ug[i] = 2 * D->u[i] - D->uf[i];
            D->vgw[i] = 2 * D->v[i] - D->vf[i];
            D->wg[i] = 2 * D->w[i] - D->wf[i];
            if (P->clamp_p && D->p[i] < 0.0) D->p[i] = 0.0; /* ClampWallPressure wc/edac.py:172-174 */
        }
    }
    return total;
}

int64_t orc_tvf_avgp(orc_ctx *c, const orc_tvf_program *P)
{
    int64_t total = 0;
    for (int dst = 0; dst < c->narr; dst++) {
        if (!(P->fluid_mask >> dst & 1u)) continue;
        orc_array *D = &c->arr[dst];
        const int64_t np = D->n_real; /* Group(equations=avg_p_group, real=True), wc/edac.py:842 */
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < np; i++) D->pavg[i] = D->nnbr[i] = 0.0;
        for (int src = 0; src < c->narr; src++) {
            if (!((P->fluid_mask | P->solid_mask) >> src & 1u)) continue;
            const orc_array *S = &c->arr[src];
            int64_t pairs = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : pairs)
            for (int64_t d_idx = 0; d_idx < np; d_idx++) {
                ORC_FOR_NEIGHBORS(c, dst, src, d_idx, s_idx, {
                    pairs++;
                    D->pavg[d_idx] += S->p[s_idx]; /* wc/edac.py:73-75 */
                    D->nnbr[d_idx] += 1.0;
                });
            }
            total += pairs;
        }
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < np; i++)
            if (D->nnbr[i] > 0) D->pavg[i] /= D->nnbr[i];
    }
    return total;
}

int64_t orc_tvf_pass2(orc_ctx *c, const orc_tvf_program *P)
{
    const int kernel = P->kernel, dim = P->dim;
    const double kfac = k_fac(kernel, dim);
    const uint32_t bits = P->eqbits;
    int64_t total = 0;
    for (int dst = 0; dst < c->narr; dst++) {
        if (!(P->fluid_mask >> dst & 1u)) continue;
        orc_array *D = &c->arr[dst];
        const int64_t np = D->n_real; /* Group(real=True) default, wc/edac.py:880 */
        /* initialize of every equation: wc/edac.py:362-363, :438-445 */
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < np; i++) {
            D->au[i] = D->av[i] = D->aw[i] = 0.0;
            if (bits & ORC_TVF_PGRAD) D->auhat[i] = D->avhat[i] = D->awhat[i] = 0.0;
            if (bits & ORC_TVF_EDAC) D->ap[i] = 0.0;
            if (bits & ORC_TVF_XSPH) D->ax[i] = D->ay[i] = D->az[i] = 0.0; /* basic_equations.py:280-283 */
        }
        for (int src = 0; src < c->narr; src++) {
            if (!((P->fluid_mask | P->solid_mask) >> src & 1u)) continue;
            /* which equations have this source (wc/edac.py:845-878): a wall is a source of the
             * pressure gradient, the artificial viscosity, the no-slip term and EDAC only */
            const int wall = (P->solid_mask >> src) & 1u;
            uint32_t bits_ = wall ? (P->eqbits & (ORC_TVF_PGRAD | ORC_TVF_MOM | ORC_TVF_AV | ORC_TVF_NOSLIP | ORC_TVF_EDAC))
                                  : (P->eqbits & ~(uint32_t)ORC_TVF_NOSLIP);
            if (src != dst) bits_ &= ~(uint32_t)ORC_TVF_XSPH; /* XSPHCorrection(dest=fluid, sources=[fluid]) */
            const uint32_t bits = bits_;
            const orc_array *S = &c->arr[src];
            int64_t pairs = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : pairs)
            for (int64_t d_idx = 0; d_idx < np; d_idx++) {
                ORC_FOR_NEIGHBORS(c, dst, src, d_idx, s_idx, {
                    pairs++;
                    double XIJ[3], VIJ[3], DWIJ[3] = {0, 0, 0};
                    XIJ[0] = D->x[d_idx] - S->x[s_idx];
                    XIJ[1] = D->y[d_idx] - S->y[s_idx];
                    XIJ[2] = D->z[d_idx] - S->z[s_idx];
                    VIJ[0] = D->u[d_idx] - S->u[s_idx];
                    VIJ[1] = D->v[d_idx] - S->v[s_idx];
                    VIJ[2] = D->w[d_idx] - S->w[s_idx];
                    const double R2IJ = XIJ[0] * XIJ[0] + XIJ[1] * XIJ[1] + XIJ[2] * XIJ[2];
                    const double RIJ = sqrt(R2IJ);
                    const double HIJ = 0.5 * (D->h[d_idx] + S->h[s_idx]);
                    const double EPS = 0.01 * HIJ * HIJ;
                    k_grad(kernel, dim, kfac, XIJ, RIJ, HIJ, DWIJ);
                    const double rhoi = D->rho[d_idx], rhoj = S->rho[s_idx];
                    const double Vi = 1.0 / D->V[d_idx], Vj = 1.0 / S->V[s_idx];
                    const double Vi2 = Vi * Vi, Vj2 = Vj * Vj;
                    const double mi1 = 1.0 / D->m[d_idx];
                    if (bits & ORC_TVF_PGRAD) { /* wc/edac.py:447-481 */
                        const double pavg = D->pavg[d_idx];
                        const double pi = D->p[d_idx], pj = S->p[s_idx];
                        double pij = rhoj * (pi - pavg) + rhoi * (pj - pavg);
                        pij /= (rhoj + rhoi);
                        double tmp = -pij * mi1 * (Vi2 + Vj2);
                        D->au[d_idx] += tmp * DWIJ[0];
                        D->av[d_idx] += tmp * DWIJ[1];
                        D->aw[d_idx] += tmp * DWIJ[2];
                        tmp = -P->pb * mi1 * (Vi2 + Vj2);
                        D->auhat[d_idx] += tmp * DWIJ[0];
                        D->avhat[d_idx] += tmp * DWIJ[1];
                        D->awhat[d_idx] += tmp * DWIJ[2];
                    }
                    if (bits & ORC_TVF_MOM) { /* wc/edac.py:319-341 */
                        const double pi = D->p[d_idx], pj = S->p[s_idx];
                        double pij = rhoj * pi + rhoi * pj;
                        pij /= (rhoj + rhoi);
                        const double tmp = -pij * mi1 * (Vi2 + Vj2);
                        D->au[d_idx] += tmp * DWIJ[0];
                        D->av[d_idx] += tmp * DWIJ[1];
                        D->aw[d_idx] += tmp * DWIJ[2];
                    }
                    if (bits & ORC_TVF_XSPH) { /* basic_equations.py:285-295 */
                        const double WIJ = k_w(kernel, dim, kfac, RIJ, HIJ);
                        const double tmp = -P->eps_xsph * S->m[s_idx] * WIJ / (0.5 * (rhoi + rhoj));
                        D->ax[d_idx] += tmp * VIJ[0];
                        D->ay[d_idx] += tmp * VIJ[1];
                        D->az[d_idx] += tmp * VIJ[2];
                    }
                    if (bits & ORC_TVF_AV) { /* transport_velocity.py:432-448 */
                        const double RHOIJ1 = 1.0 / (0.5 * (rhoi + rhoj));
                        const double vijdotrij = VIJ[0] * XIJ[0] + VIJ[1] * XIJ[1] + VIJ[2] * XIJ[2];
                        double piij = 0.0;
                        if (vijdotrij < 0) {
                            const double muij = (HIJ * vijdotrij) / (R2IJ + EPS);
                            piij = -P->alpha * P->c0 * muij;
                            piij = S->m[s_idx] * piij * RHOIJ1;
                        }
                        D->au[d_idx] += -piij * DWIJ[0];
                        D->av[d_idx] += -piij * DWIJ[1];
                        D->aw[d_idx] += -piij * DWIJ[2];
                    }
                    if (bits & ORC_TVF_VISC) { /* transport_velocity.py:362-386 */
                        const double etai = P->nu * rhoi, etaj = P->nu * rhoj;
                        const double etaij = 2 * (etai * etaj) / (etai + etaj);
                        const double Fij = DWIJ[0] * XIJ[0] + DWIJ[1] * XIJ[1] + DWIJ[2] * XIJ[2];
                        const double tmp = mi1 * (Vi2 + Vj2) * etaij * Fij / (R2IJ + EPS);
                        D->au[d_idx] += tmp * VIJ[0];
                        D->av[d_idx] += tmp * VIJ[1];
                        D->aw[d_idx] += tmp * VIJ[2];
                    }
                    if (bits & ORC_TVF_NOSLIP) { /* transport_velocity.py:611-638 */
                        const double etai = P->nu * rhoi, etaj = P->nu * rhoj;
                        const double etaij = 2 * (etai * etaj) / (etai + etaj);
                        const double Fij = XIJ[0] * DWIJ[0] + XIJ[1] * DWIJ[1] + XIJ[2] * DWIJ[2];
                        const double tmp = mi1 * (Vi2 + Vj2) * (etaij * Fij / (R2IJ + EPS));
                        D->au[d_idx] += tmp * (D->u[d_idx] - S->ug[s_idx]);
                        D->av[d_idx] += tmp * (D->v[d_idx] - S->vgw[s_idx]);
                        D->aw[d_idx] += tmp * (D->w[d_idx] - S->wg[s_idx]);
                    }
                    if (bits & ORC_TVF_ASTRESS) { /* transport_velocity.py:473-545 */
                        const double ui = D->u[d_idx], vi = D->v[d_idx], wi = D->w[d_idx];
                        const double uj = S->u[s_idx], vj = S->v[s_idx], wj = S->w[s_idx];
                        const double dui = D->uhat[d_idx] - ui, dvi = D->vhat[d_idx] - vi, dwi = D->what[d_idx] - wi;
                        const double duj = S->uhat[s_idx] - uj, dvj = S->vhat[s_idx] - vj, dwj = S->what[s_idx] - wj;
                        const double Ax = 0.5 * ((rhoi * ui * dui + rhoj * uj * duj) * DWIJ[0] +
                                                 (rhoi * ui * dvi + rhoj * uj * dvj) * DWIJ[1] +
                                                 (rhoi * ui * dwi + rhoj * uj * dwj) * DWIJ[2]);
                        const double Ay = 0.5 * ((rhoi * vi * dui + rhoj * vj * duj) * DWIJ[0] +
                                                 (rhoi * vi * dvi + rhoj * vj * dvj) * DWIJ[1] +
                                                 (rhoi * vi * dwi + rhoj * vj * dwj) * DWIJ[2]);
                        const double Az = 0.5 * ((rhoi * wi * dui + rhoj * wj * duj) * DWIJ[0] +
                                                 (rhoi * wi * dvi + rhoj * wj * dvj) * DWIJ[1] +
                                                 (rhoi * wi * dwi + rhoj * wj * dwj) * DWIJ[2]);
                        const double tmp = mi1 * (Vi2 + Vj2);
                        D->au[d_idx] += tmp * Ax;
                        D->av[d_idx] += tmp * Ay;
                        D->aw[d_idx] += tmp * Az;
                    }
                    if (bits & ORC_TVF_EDAC) { /* wc/edac.py:365-386 */
                        const double etaij = 2 * P->edac_nu * (rhoi * rhoj) / (rhoi + rhoj);
                        const double vijdotdwij = DWIJ[0] * VIJ[0] + DWIJ[1] * VIJ[1] + DWIJ[2] * VIJ[2];
                        D->ap[d_idx] += rhoi / rhoj * P->c0 * P->c0 * S->m[s_idx] * vijdotdwij;
                        const double xijdotdwij = DWIJ[0] * XIJ[0] + DWIJ[1] * XIJ[1] + DWIJ[2] * XIJ[2];
                        const double tmp = mi1 * (Vi2 + Vj2) * etaij * xijdotdwij / (R2IJ + EPS);
                        D->ap[d_idx] += tmp * (D->p[d_idx] - S->p[s_idx]);
                    }
                });
            }
            total += pairs;
        }
        if (bits & ORC_TVF_XSPH) { /* post_loop basic_equations.py:297-300 */
#pragma omp parallel for schedule(static)
            for (int64_t i = 0; i < np; i++) {
                D->ax[i] += D->u[i];
                D->ay[i] += D->v[i];
                D->az[i] += D->w[i];
            }
        }
        if (bits & (ORC_TVF_PGRAD | ORC_TVF_MOM)) { /* post_loop wc/edac.py:483-488, :343-352 */
            double damp = 1.0;
            if (P->t < P->tdamp) damp = 0.5 * (sin((-0.5 + P->t / P->tdamp) * M_PI) + 1.0);
#pragma omp parallel for schedule(static)
            for (int64_t i = 0; i < np; i++) {
                D->au[i] += P->gx * damp;
                D->av[i] += P->gy * damp;
                D->aw[i] += P->gz * damp;
            }
        }
    }
    return total;
}

/* EDACTVFStep wc/edac.py:491-540 (real particles, integrator_cython.mako:97-111) */
void orc_stage_tvf(orc_ctx *c, int arr, int which, double dt)
{
    orc_array *A = &c->arr[arr];
    const int64_t n = A->n_real;
    if (which == 0) {
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < n; i++) {
            A->x0[i] = A->x[i];
            A->y0[i] = A->y[i];
            A->z0[i] = A->z[i];
            A->u0[i] = A->u[i];
            A->v0[i] = A->v[i];
            A->w0[i] = A->w[i];
            A->p0[i] = A->p[i];
        }
        return;
    }
    const double f = (which == 1) ? 0.5 * dt : dt;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; i++) {
        A->u[i] = A->u0[i] + f * A->au[i];
        A->v[i] = A->v0[i] + f * A->av[i];
        A->w[i] = A->w0[i] + f * A->aw[i];
        A->uhat[i] = A->u[i] + f * A->auhat[i];
        A->vhat[i] = A->v[i] + f * A->avhat[i];
        A->what[i] = A->w[i] + f * A->awhat[i];
        A->x[i] = A->x0[i] + f * A->uhat[i];
        A->y[i] = A->y0[i] + f * A->vhat[i];
        A->z[i] = A->z0[i] + f * A->what[i];
        A->p[i] = A->p0[i] + f * A->ap[i];
    }
}


/* EDACStep wc/edac.py:82-133 (real particles) */
void orc_stage_edac(orc_ctx *c, int arr, int which, double dt)
{
    orc_array *A = &c->arr[arr];
    const int64_t n = A->n_real;
    if (which == 0) {
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < n; i++) {
            A->x0[i] = A->x[i];
            A->y0[i] = A->y[i];
            A->z0[i] = A->z[i];
            A->u0[i] = A->u[i];
            A->v0[i] = A->v[i];
            A->w0[i] = A->w[i];
            A->p0[i] = A->p[i];
        }
        return;
    }
    const double f = (which == 1) ? 0.5 * dt : dt;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; i++) {
        A->u[i] = A->u0[i] + f * A->au[i];
        A->v[i] = A->v0[i] + f * A->av[i];
        A->w[i] = A->w0[i] + f * A->aw[i];
        A->x[i] = A->x0[i] + f * A->ax[i];
        A->y[i] = A->y0[i] + f * A->ay[i];
        A->z[i] = A->z0[i] + f * A->az[i];
        A->p[i] = A->p0[i] + f * A->ap[i];
    }
}

/* ------------------------------------------------------------------------ */
/* elastic dynamics (SURVEY.md 8f-2)                                         */
/* ------------------------------------------------------------------------ */

/* cyclic Jacobi; converges to machine precision in < 10 sweeps for 3x3 */
void orc_eigen_sym3(const double a_in[9], double v[9], double d[3])
{
    double a[3][3];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            a[i][j] = a_in[3 * i + j];
            v[3 * i + j] = (i == j) ? 1.0 : 0.0;
        }
    for (int sweep = 0; sweep < 60; sweep++) {
        const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
        const double diag = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2];
        if (off <= 1e-32 * diag || off == 0.0) break;
        for (int p = 0; p < 2; p++)
            for (int q = p + 1; q < 3; q++) {
                if (a[p][q] == 0.0) continue;
                const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
                for (int k = 0; k < 3; k++) { /* A <- A J */
                    const double akp = a[k][p], akq = a[k][q];
                    a[k][p] = c * akp - sn * akq;
                    a[k][q] = sn * akp + c * akq;
                }
                for (int k = 0; k < 3; k++) { /* A <- J^T A */
                    const double apk = a[p][k], aqk = a[q][k];
                    a[p][k] = c * apk - sn * aqk;
                    a[q][k] = sn * apk + c * aqk;
                }
                for (int k = 0; k < 3; k++) { /* V <- V J */
                    const double vkp = v[3 * k + p], vkq = v[3 * k + q];
                    v[3 * k + p] = c * vkp - sn * vkq;
                    v[3 * k + q] = sn * vkp + c * vkq;
                }
            }
    }
    d[0] = a[0][0];
    d[1] = a[1][1];
    d[2] = a[2][2];
}

static const int VG_I[9] = {0, 0, 0, 1, 1, 1, 2, 2, 2}; /* velocity component of vg[k] */
static const int VG_J[9] = {0, 1, 2, 0, 1, 2, 0, 1, 2}; /* spatial component           */

int64_t orc_solid_group1(orc_ctx *c, const orc_solid_program *P)
{
    const int kernel = P->kernel, dim = P->dim;
    const double kfac = k_fac(kernel, dim);
    int64_t total = 0;
    for (int dst = 0; dst < c->narr; dst++) {
        if (!(P->elastic_mask >> dst & 1u)) continue;
        orc_array *D = &c->arr[dst];
        const int64_t np = D->n_real; /* Group(real=True) default */
        /* initialize: VelocityGradient2D basic_equations.py:82-86 / 3D :115-125 */
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < np; i++)
            for (int k = 0; k < 9; k++)
                if (P->grad3d || (VG_I[k] < 2 && VG_J[k] < 2)) D->vg[k][i] = 0.0;
        /* no-source loops, in the order of the equation list */
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < np; i++) {
            /* IsothermalEOS solid_mech/basic.py:100-101 */
            D->p[i] = P->c0_ref[dst] * P->c0_ref[dst] * (D->rho[i] - P->rho_ref[dst]);
            /* MonaghanArtificialStress :170-242 */
            const double rhoi21 = 1.0 / (D->rho[i] * D->rho[i]);
            double S[9], R[9], V[3], rd[3];
            S[0] = D->s[0][i] - D->p[i];
            S[4] = D->s[3][i] - D->p[i];
            S[8] = D->s[5][i] - D->p[i];
            S[5] = S[7] = D->s[4][i];
            S[2] = S[6] = D->s[2][i];
            S[1] = S[3] = D->s[1][i];
            orc_eigen_sym3(S, R, V);
            for (int k = 0; k < 3; k++) rd[k] = V[k] > 0 ? -P->eps * V[k] * rhoi21 : 0.0;
            /* transform_diag_inv: Rab = R diag(rd) R^T  (linalg3.pyx:220-233) */
            double Rab[9];
            for (int a = 0; a < 3; a++)
                for (int b = 0; b < 3; b++) {
                    double sum = 0.0;
                    for (int k = 0; k < 3; k++) sum += R[3 * a + k] * rd[k] * R[3 * b + k];
                    Rab[3 * a + b] = sum;
                }
            D->r[0][i] = Rab[0];
            D->r[3][i] = Rab[4];
            D->r[5][i] = Rab[8];
            D->r[4][i] = Rab[5];
            D->r[2][i] = Rab[2];
            D->r[1][i] = Rab[1];
        }
        for (int src = 0; src < c->narr; src++) {
            if (!(P->source_mask >> src & 1u)) continue;
            const orc_array *S_ = &c->arr[src];
            int64_t pairs = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : pairs)
            for (int64_t d_idx = 0; d_idx < np; d_idx++) {
                ORC_FOR_NEIGHBORS(c, dst, src, d_idx, s_idx, {
                    pairs++;
                    double XIJ[3], VIJ[3], DWIJ[3] = {0, 0, 0};
                    XIJ[0] = D->x[d_idx] - S_->x[s_idx];
                    XIJ[1] = D->y[d_idx] - S_->y[s_idx];
                    XIJ[2] = D->z[d_idx] - S_->z[s_idx];
                    VIJ[0] = D->u[d_idx] - S_->u[s_idx];
                    VIJ[1] = D->v[d_idx] - S_->v[s_idx];
                    VIJ[2] = D->w[d_idx] - S_->w[s_idx];
                    const double RIJ = sqrt(XIJ[0] * XIJ[0] + XIJ[1] * XIJ[1] + XIJ[2] * XIJ[2]);
                    const double HIJ = 0.5 * (D->h[d_idx] + S_->h[s_idx]);
                    k_grad(kernel, dim, kfac, XIJ, RIJ, HIJ, DWIJ);
                    const double tmp = S_->m[s_idx] / S_->rho[s_idx];
                    for (int k = 0; k < 9; k++)
                        if (P->grad3d || (VG_I[k] < 2 && VG_J[k] < 2))
                            D->vg[k][d_idx] += tmp * -VIJ[VG_I[k]] * DWIJ[VG_J[k]];
                });
            }
            total += pairs;
        }
    }
    return total;
}

int64_t orc_solid_group2(orc_ctx *c, const orc_solid_program *P)
{
    const int kernel = P->kernel, dim = P->dim;
    const double kfac = k_fac(kernel, dim);
    /* symmetric index: (a,b) -> 00 01 02 11 12 22 */
    static const int SYM[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
    int64_t total = 0;
    for (int dst = 0; dst < c->narr; dst++) {
        if (!(P->elastic_mask >> dst & 1u)) continue;
        orc_array *D = &c->arr[dst];
        const int64_t np = D->n_real;
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < np; i++) {
            D->arho[i] = 0.0;
            D->au[i] = D->av[i] = D->aw[i] = 0.0;
            D->ax[i] = D->ay[i] = D->az[i] = 0.0;
            for (int k = 0; k < 6; k++) D->as[k][i] = 0.0;
        }
        /* HookesDeviatoricStressRate (no source) solid_mech/basic.py:420-505 */
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < np; i++) {
            double v[3][3], s[3][3], eps[3][3], om[3][3];
            for (int k = 0; k < 9; k++) v[VG_I[k]][VG_J[k]] = D->vg[k][i];
            for (int a = 0; a < 3; a++)
                for (int b = 0; b < 3; b++) {
                    s[a][b] = D->s[SYM[a][b]][i];
                    eps[a][b] = 0.5 * (v[a][b] + v[b][a]);
                    om[a][b] = 0.5 * (v[a][b] - v[b][a]);
                }
            const double tmp = 2.0 * P->G[dst];
            const double trace = 1.0 / 3.0 * (eps[0][0] + eps[1][1] + eps[2][2]);
            for (int a = 0; a < 3; a++)
                for (int b = a; b < 3; b++) {
                    /* as_ab = 2G (eps_ab - delta_ab trace) + s_ak om_bk + s_kb om_ak
                     * (the reference writes out s_ak*omega_bk + s_kb*omega_ak term by term) */
                    double t1 = 0.0, t2 = 0.0;
                    for (int k = 0; k < 3; k++) {
                        t1 += s[a][k] * om[b][k];
                        t2 += s[k][b] * om[a][k];
                    }
                    D->as[SYM[a][b]][i] = tmp * (eps[a][b] - (a == b ? trace : 0.0)) + t1 + t2;
                }
        }
        for (int src = 0; src < c->narr; src++) {
            if (!(P->source_mask >> src & 1u)) continue;
            const orc_array *S_ = &c->arr[src];
            const int xsph = (src == dst);
            int64_t pairs = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : pairs)
            for (int64_t d_idx = 0; d_idx < np; d_idx++) {
                ORC_FOR_NEIGHBORS(c, dst, src, d_idx, s_idx, {
                    pairs++;
                    double XIJ[3], VIJ[3], DWIJ[3] = {0, 0, 0};
                    XIJ[0] = D->x[d_idx] - S_->x[s_idx];
                    XIJ[1] = D->y[d_idx] - S_->y[s_idx];
                    XIJ[2] = D->z[d_idx] - S_->z[s_idx];
                    VIJ[0] = D->u[d_idx] - S_->u[s_idx];
                    VIJ[1] = D->v[d_idx] - S_->v[s_idx];
                    VIJ[2] = D->w[d_idx] - S_->w[s_idx];
                    const double R2IJ = XIJ[0] * XIJ[0] + XIJ[1] * XIJ[1] + XIJ[2] * XIJ[2];
                    const double RIJ = sqrt(R2IJ);
                    const double HIJ = 0.5 * (D->h[d_idx] + S_->h[s_idx]);
                    const double EPS = 0.01 * HIJ * HIJ;
                    const double WIJ = k_w(kernel, dim, kfac, RIJ, HIJ);
                    k_grad(kernel, dim, kfac, XIJ, RIJ, HIJ, DWIJ);
                    const double mb = S_->m[s_idx];
                    const double rhoa = D->rho[d_idx], rhob = S_->rho[s_idx];
                    const double RHOIJ1 = 1.0 / (0.5 * (rhoa + rhob));
                    /* ContinuityEquation basic_equations.py:190-192 */
                    const double vijdotdwij = DWIJ[0] * VIJ[0] + DWIJ[1] * VIJ[1] + DWIJ[2] * VIJ[2];
                    D->arho[d_idx] += mb * vijdotdwij;
                    /* MomentumEquationWithStress solid_mech/basic.py:267-387 */
                    const double rhoa21 = 1.0 / (rhoa * rhoa), rhob21 = 1.0 / (rhob * rhob);
                    double fab = 0.0;
                    const int art = P->wdeltap[dst] > 0.0;
                    if (art) fab = pow(WIJ / P->wdeltap[dst], P->n[dst]);
                    double acc[3] = {0, 0, 0};
                    for (int a = 0; a < 3; a++)
                        for (int b = 0; b < 3; b++) {
                            const int k = SYM[a][b];
                            double sa = D->s[k][d_idx], sb = S_->s[k][s_idx];
                            if (a == b) {
                                sa -= D->p[d_idx];
                                sb -= S_->p[s_idx];
                            }
                            const double arts = art ? fab * (D->r[k][d_idx] + S_->r[k][s_idx]) : 0.0;
                            acc[a] += mb * (sa * rhoa21 + sb * rhob21 + arts) * DWIJ[b];
                        }
                    D->au[d_idx] += acc[0];
                    D->av[d_idx] += acc[1];
                    D->aw[d_idx] += acc[2];
                    /* MonaghanArtificialViscosity basic_equations.py:240-257 */
                    {
                        const double vijdotxij = VIJ[0] * XIJ[0] + VIJ[1] * XIJ[1] + VIJ[2] * XIJ[2];
                        double piij = 0.0;
                        if (vijdotxij < 0) {
                            const double cij = 0.5 * (D->cs[d_idx] + S_->cs[s_idx]);
                            const double muij = (HIJ * vijdotxij) / (R2IJ + EPS);
                            piij = -P->alpha * cij * muij + P->beta * muij * muij;
                            piij = piij * RHOIJ1;
                        }
                        D->au[d_idx] += -mb * piij * DWIJ[0];
                        D->av[d_idx] += -mb * piij * DWIJ[1];
                        D->aw[d_idx] += -mb * piij * DWIJ[2];
                    }
                    if (xsph) { /* XSPHCorrection(sources=[dest]) basic_equations.py:290-295 */
                        const double tmp = -P->eps_xsph * mb * WIJ * RHOIJ1;
                        D->ax[d_idx] += tmp * VIJ[0];
                        D->ay[d_idx] += tmp * VIJ[1];
                        D->az[d_idx] += tmp * VIJ[2];
                    }
                });
            }
            total += pairs;
        }
        /* XSPHCorrection.post_loop basic_equations.py:297-300 */
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < np; i++) {
            D->ax[i] += D->u[i];
            D->ay[i] += D->v[i];
            D->az[i] += D->w[i];
        }
    }
    return total;
}

/* SolidMechStep integrator_step.py:173-252 */
void orc_stage_solid(orc_ctx *c, int arr, int which, double dt)
{
    orc_array *A = &c->arr[arr];
    const int64_t n = A->n_real;
    if (which == 0) {
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < n; i++) {
            A->x0[i] = A->x[i];
            A->y0[i] = A->y[i];
            A->z0[i] = A->z[i];
            A->u0[i] = A->u[i];
            A->v0[i] = A->v[i];
            A->w0[i] = A->w[i];
            A->rho0[i] = A->rho[i];
            A->e0[i] = A->e[i];
            for (int k = 0; k < 6; k++) A->s0[k][i] = A->s[k][i];
        }
        return;
    }
    const double f = (which == 1) ? 0.5 * dt : dt;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; i++) {
        A->u[i] = A->u0[i] + f * A->au[i];
        A->v[i] = A->v0[i] + f * A->av[i];
        A->w[i] = A->w0[i] + f * A->aw[i];
        A->x[i] = A->x0[i] + f * A->ax[i];
        A->y[i] = A->y0[i] + f * A->ay[i];
        A->z[i] = A->z0[i] + f * A->az[i];
        A->rho[i] = A->rho0[i] + f * A->arho[i];
        A->e[i] = A->e0[i] + f * A->ae[i];
        for (int k = 0; k < 6; k++) A->s[k][i] = A->s0[k][i] + f * A->as[k][i];
    }
}

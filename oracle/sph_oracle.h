/*
 * oracle/sph_oracle.h -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * fp64 CPU restatement of the PySPH WCSPH hot path (LinkedListNNPS + the
 * generated AccelerationEval.compute loop nest + WCSPHStep), used only as the
 * parity checker in tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs.  Nothing under pysph_b200/ may import,
 * link or call this.
 *
 * Parity pinning: see oracle/README.md -- the restatement is checked against
 * (a) the reference's own compiled c_kernels.pyx (built into oracle/_ref),
 * (b) the reference's own Python equation bodies (pysph/sph/wc/basic.py,
 *     pysph/sph/basic_equations.py, pysph/sph/integrator_step.py) driven
 *     pair-by-pair, and (c) the known-answer vectors in the reference tests
 *     (test_acceleration_eval.py, test_nnps.py, test_kernel.py),
 * (d) the reference's own EDACScheme / ElasticSolidsScheme get_equations() and the
 *     bodies of wc/edac.py, wc/transport_velocity.py, solid_mech/basic.py (with the
 *     reference's compiled linalg3.pyx eigen solver), and
 * (e) for periodic domains, the reference's lattice fixtures (test_domain_manager.py).
 */
#ifndef SPH_ORACLE_H
#define SPH_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORC_MAX_ARRAYS 8

/* smoothing kernels -- pysph/base/kernels.py */
enum { ORC_K_CUBIC = 0, ORC_K_WENDLAND = 1, ORC_K_QUINTIC = 2, ORC_K_GAUSSIAN = 3 };

/* pair-equation bits (one nibble+ per (dest, source) entry of the program) */
enum {
    ORC_EQ_SUMDENS = 1,   /* SummationDensity          basic_equations.py:19-29   */
    ORC_EQ_CONT    = 2,   /* ContinuityEquation        basic_equations.py:180-192 */
    ORC_EQ_MOM     = 4,   /* MomentumEquation          wc/basic.py:129-269        */
    ORC_EQ_XSPH    = 8,   /* XSPHCorrection            basic_equations.py:260-300 */
    ORC_EQ_AV      = 16,  /* MonaghanArtificialViscosity basic_equations.py:195-257 */
    ORC_EQ_LAMINAR = 32   /* LaminarViscosity          wc/viscosity.py:5-27 (WCSPHScheme(nu != 0), scheme.py:486-496) */
};

/* borrowed host pointers to one ParticleArray's fp64 SoA properties
 * (pysph/base/utils.py:152-190).  Any pointer an enabled equation does not
 * touch may be NULL. */
typedef struct {
    int64_t n;       /* all particles (real + ghost/remote) */
    int64_t n_real;  /* real particles come first (particle_array.pyx:1092-1172) */
    double *x, *y, *z, *h, *m, *rho, *u, *v, *w, *p, *cs;
    double *arho, *au, *av, *aw, *ax, *ay, *az, *dt_cfl, *dt_force;
    double *x0, *y0, *z0, *u0, *v0, *w0, *rho0;
    /* transport-velocity / EDAC properties (wc/edac.py:724-730); may be NULL */
    double *uhat, *vhat, *what, *V, *pavg, *nnbr, *auhat, *avhat, *awhat, *ap, *p0;
    /* elastic dynamics (solid_mech/basic.py:52-59); may be NULL.  Symmetric tensors
     * are stored as 00 01 02 11 12 22, the velocity gradient as 00 01 02 10 .. 22 */
    double *vg[9], *s[6], *as[6], *r[6], *s0[6], *e, *e0, *ae;
    /* wall arrays of the EDAC scheme (TVF_SOLID_PROPS, wc/edac.py:752-753); may be NULL */
    double *wij, *uf, *vf, *wf, *ug, *vgw, *wg;   /* vgw: the property "vg" (vg[] above is the velocity gradient) */
} orc_array;

typedef struct {
    int kernel;          /* ORC_K_*                                     */
    int dim;             /* 1, 2, 3                                     */
    /* MomentumEquation / MonaghanArtificialViscosity */
    double c0, alpha, beta, gx, gy, gz;
    int tensile_correction;
    /* XSPHCorrection */
    double eps_xsph;
    /* group flag: real=True -> destinations are the real particles only */
    int real_only;
    /* eqmask[d][s]: OR of ORC_EQ_* for dest array d, source array s        */
    uint32_t eqmask[ORC_MAX_ARRAYS][ORC_MAX_ARRAYS];
    /* src_order[d][k]: k-th source array visited for dest d (first-mention
     * order, acceleration_eval.py:139-160); -1 terminates */
    int src_order[ORC_MAX_ARRAYS][ORC_MAX_ARRAYS];
    /* dest_order[k]: k-th destination array; -1 terminates */
    int dest_order[ORC_MAX_ARRAYS];
    /* LaminarViscosity(nu, eta) */
    double nu, eta;
} orc_pair_program;

/* EDAC scheme, internal-flow (transport velocity) branch for fluid arrays without
 * solids: EDACScheme._get_internal_flow_equations wc/edac.py:776-870 */
enum {
    ORC_TVF_PGRAD   = 1,  /* MomentumEquationPressureGradient  wc/edac.py:389-488 */
    ORC_TVF_AV      = 2,  /* MomentumEquationArtificialViscosity transport_velocity.py:389-448 */
    ORC_TVF_VISC    = 4,  /* MomentumEquationViscosity         transport_velocity.py:328-386 */
    ORC_TVF_ASTRESS = 8,  /* MomentumEquationArtificialStress  transport_velocity.py:451-545 */
    ORC_TVF_EDAC    = 16, /* EDACEquation                      wc/edac.py:354-386 */
    ORC_TVF_NOSLIP  = 32, /* SolidWallNoSlipBC                 transport_velocity.py:548-638 */
    /* the external-flow branch (pb == 0), wc/edac.py:882-971 */
    ORC_TVF_MOM     = 64, /* edac.MomentumEquation             wc/edac.py:301-352 */
    ORC_TVF_XSPH    = 128 /* XSPHCorrection(dest=f, sources=[f]) basic_equations.py:260-300 */
};
typedef struct {
    int kernel, dim;
    uint32_t fluid_mask; /* bit a: array a is a fluid; every fluid is a destination and a source */
    int bql;             /* ComputeAveragePressure wc/edac.py:62-79 in the first group */
    uint32_t eqbits;     /* ORC_TVF_* of the second group */
    double pb, nu, edac_nu, c0, rho0, alpha;
    double gx, gy, gz, tdamp, t;
    uint32_t solid_mask; /* bit a: array a is a solid wall (EDACScheme(fluids, solids)): a source of
                          * the pressure gradient, the artificial viscosity, the no-slip term and
                          * the EDAC equation, and a destination of orc_tvf_wall */
    double eps_xsph;     /* XSPHCorrection(eps) of the external-flow branch */
    int clamp_p;         /* ClampWallPressure (wc/edac.py:169-174) behind the wall pressure */
} orc_tvf_program;

/* ElasticSolidsScheme.get_equations, solid_mech/basic.py:604-651 */
typedef struct {
    int kernel, dim;
    uint32_t elastic_mask; /* destinations (elastic solids)                        */
    uint32_t source_mask;  /* sources = solids + elastic solids                    */
    int grad3d;            /* 0: VelocityGradient2D (what the reference scheme emits),
                            * 1: VelocityGradient3D (basic_equations.py:101-148)   */
    double eps;            /* MonaghanArtificialStress(eps)                        */
    double alpha, beta;    /* MonaghanArtificialViscosity                          */
    double eps_xsph;       /* XSPHCorrection                                       */
    /* the array constants of get_particle_array_elastic_dynamics (:61-83) */
    double c0_ref[ORC_MAX_ARRAYS], rho_ref[ORC_MAX_ARRAYS], wdeltap[ORC_MAX_ARRAYS],
        n[ORC_MAX_ARRAYS], G[ORC_MAX_ARRAYS];
} orc_solid_program;

typedef struct orc_ctx orc_ctx;

orc_ctx *orc_create(int narrays, int dim, double radius_scale);
void orc_destroy(orc_ctx *);
void orc_set_array(orc_ctx *, int idx, const orc_array *a);
void orc_set_num_threads(int n);
int orc_get_max_threads(void);

/* a1: CPUDomainManager._compute_cell_size_for_binning  nnps_base.pyx:942-978 */
void orc_update_domain(orc_ctx *);
/* a2-a4: NNPS.update -> _compute_bounds, _refresh, _bin
 * nnps_base.pyx:1471-1575, linked_list_nnps.pyx:235-382.  returns 0, or -1 if
 * the grid needs more than 2^28 cells (linked_list_nnps.pyx:336-343) */
int orc_nnps_update(orc_ctx *);
void orc_get_grid(orc_ctx *, double *cell_size, double *hmin, double xmin[3],
                  double xmax[3], int ncells[3], int64_t *n_cells);

/* a5: LinkedListNNPS.find_nearest_neighbors  linked_list_nnps.pyx:92-196.
 * Writes up to cap indices (linked-list order); returns the full count. */
int64_t orc_find_neighbors(orc_ctx *, int dst, int src, int64_t d_idx,
                           uint32_t *out, int64_t cap);
/* NNPS.brute_force_neighbors  nnps_base.pyx:1325-1366 */
int64_t orc_brute_neighbors(orc_ctx *, int dst, int src, int64_t d_idx,
                            uint32_t *out, int64_t cap);

/* a11: TaitEOS (hg=0) / TaitEOSHGCorrection (hg=1)  wc/basic.py:9-126 */
void orc_eos(orc_ctx *, int arr, int hg, double rho0, double c0, double gamma,
             double p0, int real_only);
/* UpdateSmoothingLengthFerrari  wc/basic.py:417-463 */
void orc_ferrari_h(orc_ctx *, int arr, double hdx, int dim, int real_only);

/* a8-a17: one Group's pair loops (initialize / per-source loop / post_loop)
 * acceleration_eval_cython.mako:10-154.  returns the number of directed pair
 * interactions evaluated (sum of neighbour-list lengths over enabled
 * (dest, source) loops). */
int64_t orc_pair_pass(orc_ctx *, const orc_pair_program *prog);

/* a18: WCSPHStep.initialize (0) / stage1 (1) / stage2 (2) over real particles
 * integrator_step.py:38-91 */
void orc_stage(orc_ctx *, int arr, int which, double dt);

/* a19 inputs: max dt_cfl, max dt_force over real+ghost of all arrays that have
 * them (integrator.py:62-81), raw min h (integrator.py:146-159, start 1.0) */
void orc_dt_factors(orc_ctx *, double out[3]);

/* group 1 (real=False): TVF SummationDensity transport_velocity.py:24-58 and
 * ComputeAveragePressure wc/edac.py:62-79.  Returns the pairs visited. */
int64_t orc_tvf_pass1(orc_ctx *, const orc_tvf_program *);
/* group 2 (real=True): the momentum terms and the EDAC pressure evolution */
int64_t orc_tvf_pass2(orc_ctx *, const orc_tvf_program *);
/* with solid walls (solid_mask != 0), the wall part of the first group, wc/edac.py:815-822:
 * SourceNumberDensity (:177-183), VolumeSummation (transport_velocity.py:61-75),
 * SolidWallPressureBC (wc/edac.py:136-166), SetWallVelocity (:186-230) for every wall array,
 * all particles (real=False); call AFTER orc_tvf_pass1 (it reads the fluids' new rho) */
int64_t orc_tvf_wall(orc_ctx *, const orc_tvf_program *);
/* ComputeAveragePressure as a group of its own, real=True, sources = fluids + walls
 * (wc/edac.py:840-842: "after the wall pressure is set up") */
int64_t orc_tvf_avgp(orc_ctx *, const orc_tvf_program *);
/* EDACTVFStep wc/edac.py:491-540: which = 0 initialize, 1 stage1, 2 stage2 */
void orc_stage_tvf(orc_ctx *, int arr, int which, double dt);
/* EDACStep wc/edac.py:82-133 (the external-flow branch: x moves with the XSPH velocity ax) */
void orc_stage_edac(orc_ctx *, int arr, int which, double dt);

/* elastic dynamics (Gray et al.), SURVEY.md 8f-2; the reference of k_solid_pass1/2 and
 * k_stage_solid (tests/test_gpu_solid_oracle.py).
 * group 1: IsothermalEOS (solid_mech/basic.py:93-101), VelocityGradient2D/3D
 * (basic_equations.py:67-148), MonaghanArtificialStress (:104-242);
 * group 2: ContinuityEquation, MomentumEquationWithStress (:245-387),
 * MonaghanArtificialViscosity, HookesDeviatoricStressRate (:390-505), XSPHCorrection */
int64_t orc_solid_group1(orc_ctx *, const orc_solid_program *);
int64_t orc_solid_group2(orc_ctx *, const orc_solid_program *);
/* SolidMechStep integrator_step.py:173-252 */
void orc_stage_solid(orc_ctx *, int arr, int which, double dt);
/* eigen decomposition of a symmetric 3x3 matrix (row-major a[9]): eigenvalues d[3],
 * eigenvectors as the COLUMNS of v[9] (what pysph/base/linalg3.pyx:503-529 returns;
 * order and signs are not specified and do not matter for R = V diag V^T) */
void orc_eigen_sym3(const double a[9], double v[9], double d[3]);

/* single kernel evaluations for the kernel parity tests */
double orc_kernel_w(int kernel, int dim, double rij, double h);
void orc_kernel_grad(int kernel, int dim, const double xij[3], double rij,
                     double h, double grad[3]);
double orc_kernel_deltap(int kernel);
double orc_kernel_radius_scale(int kernel);

#ifdef __cplusplus
}
#endif
#endif

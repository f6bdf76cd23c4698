/* nlopt_b200.h -- C ABI of the GPU-native (H100, sm_90a) MMA/CCSAQ solver.
 *
 * Drop-in boundary: every `nlopt_*` symbol below has the name, argument list,
 * enum values and error behaviour of NLopt 2.11's public header
 * (reference: src/api/nlopt.h:60-301, soname libnlopt.so.1), so code compiled
 * against the reference header -- including the reference's header-only C++
 * wrapper nlopt.hpp and test/t_tutorial.cxx -- links against libnlopt_b200.so
 * unmodified.  Executable algorithms: NLOPT_LD_MMA and NLOPT_LD_CCSAQ
 * (src/algs/mma/mma.c, ccsa_quadratic.c) and the augmented-Lagrangian family
 * that wraps them (NLOPT_AUGLAG, NLOPT_AUGLAG_EQ, NLOPT_LD_AUGLAG,
 * NLOPT_LD_AUGLAG_EQ, and the LN_ variants when an LD_MMA / LD_CCSAQ local
 * optimizer is set; src/algs/auglag/auglag.c).  nlopt_optimize() on any
 * other algorithm id returns NLOPT_INVALID_ARGS with a message.  All O(n)
 * work of MMA / CCSAQ and the gradient of the augmented Lagrangian run in
 * CUDA kernels on sm_90a; there is no CPU fallback (no device =>
 * NLOPT_FAILURE + message).
 *
 * The AUGLAG family takes device callbacks (objective, inequality and
 * equality constraints, either form) and nlopt_b200_optimize_device as
 * well; host and device callbacks may be mixed.  Such a run keeps x and its
 * best point in HBM and evaluates the outer loop's values on the device
 * (one GPU only; sharded host callbacks are refused).  After any AUGLAG run
 * nlopt_b200_get_stats reports the last sub-optimisation.
 *
 * Maximisation works with every objective form: nlopt_set_max_objective for
 * host callbacks and the nlopt_b200_set_max_objective_* twins of the device
 * and sharded entry points, under LD_MMA, LD_CCSAQ and the AUGLAG family
 * (sharded objectives under LD_MMA / LD_CCSAQ only).
 *
 * Box bounds may live in GPU memory too: nlopt_b200_set_lower_bounds_device /
 * nlopt_b200_set_upper_bounds_device copy n doubles from a device array,
 * snap them as the host setters do, and put the object in device mode (one
 * GPU), where a run checks the start point and detects uniform bounds on the
 * device.
 *
 * So may the per-variable options: nlopt_b200_set_xtol_abs_device,
 * nlopt_b200_set_x_weights_device and nlopt_b200_set_initial_step_device
 * copy n doubles from a device array and check them on the device with
 * the host setters' rule; a run reads them in place.
 *
 * The `nlopt_b200_*` symbols are additive extensions (device-resident
 * callbacks, kernel-level access to the dual evaluation, multi-GPU sharding,
 * statistics).  No torch / CUDA types appear in any signature: device
 * pointers are `double *`, streams are `void *`.
 */
#ifndef NLOPT_B200_H
#define NLOPT_B200_H

#ifndef __CUDACC_RTC__
#include <stddef.h>
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* Under NVRTC (the run-time compile of nlopt_b200_jit_create, which includes nlopt_b200_device_kernels.cuh) only the
 * shard geometry below is seen: NVRTC compiles device code and takes no host declaration. */
#ifndef __CUDACC_RTC__
#define NLOPT_B200 1
#define NLOPT_EXTERN(T) extern T
#define NLOPT_STDCALL

/* ---- callback shapes (reference nlopt.h:60-70) --------------------------- */
typedef double (*nlopt_func)(unsigned n, const double *x, double *gradient, void *func_data);
typedef void (*nlopt_mfunc)(unsigned m, double *result, unsigned n, const double *x,
                            double *gradient, void *func_data);
typedef void (*nlopt_precond)(unsigned n, const double *x, const double *v, double *vpre, void *data);

/* ---- algorithm ids (reference nlopt.h:72-154; values are ABI) ------------- */
typedef enum {
    NLOPT_GN_DIRECT = 0, NLOPT_GN_DIRECT_L = 1, NLOPT_GN_DIRECT_L_RAND = 2,
    NLOPT_GN_DIRECT_NOSCAL = 3, NLOPT_GN_DIRECT_L_NOSCAL = 4, NLOPT_GN_DIRECT_L_RAND_NOSCAL = 5,
    NLOPT_GN_ORIG_DIRECT = 6, NLOPT_GN_ORIG_DIRECT_L = 7,
    NLOPT_GD_STOGO = 8, NLOPT_GD_STOGO_RAND = 9,
    NLOPT_LD_LBFGS_NOCEDAL = 10, NLOPT_LD_LBFGS = 11, NLOPT_LN_PRAXIS = 12,
    NLOPT_LD_VAR1 = 13, NLOPT_LD_VAR2 = 14,
    NLOPT_LD_TNEWTON = 15, NLOPT_LD_TNEWTON_RESTART = 16,
    NLOPT_LD_TNEWTON_PRECOND = 17, NLOPT_LD_TNEWTON_PRECOND_RESTART = 18,
    NLOPT_GN_CRS2_LM = 19,
    NLOPT_GN_MLSL = 20, NLOPT_GD_MLSL = 21, NLOPT_GN_MLSL_LDS = 22, NLOPT_GD_MLSL_LDS = 23,
    NLOPT_LD_MMA = 24,              /* <- built here */
    NLOPT_LN_COBYLA = 25, NLOPT_LN_NEWUOA = 26, NLOPT_LN_NEWUOA_BOUND = 27,
    NLOPT_LN_NELDERMEAD = 28, NLOPT_LN_SBPLX = 29,
    NLOPT_LN_AUGLAG = 30, NLOPT_LD_AUGLAG = 31, NLOPT_LN_AUGLAG_EQ = 32, NLOPT_LD_AUGLAG_EQ = 33,   /* <- built here (over MMA/CCSAQ) */
    NLOPT_LN_BOBYQA = 34, NLOPT_GN_ISRES = 35,
    NLOPT_AUGLAG = 36, NLOPT_AUGLAG_EQ = 37,  /* <- built here */  NLOPT_G_MLSL = 38, NLOPT_G_MLSL_LDS = 39,
    NLOPT_LD_SLSQP = 40,
    NLOPT_LD_CCSAQ = 41,            /* <- built here */
    NLOPT_GN_ESCH = 42, NLOPT_GN_AGS = 43,
    NLOPT_NUM_ALGORITHMS = 44
} nlopt_algorithm;

/* ---- result codes (reference nlopt.h:162-176) ----------------------------- */
typedef enum {
    NLOPT_FAILURE = -1, NLOPT_INVALID_ARGS = -2, NLOPT_OUT_OF_MEMORY = -3,
    NLOPT_ROUNDOFF_LIMITED = -4, NLOPT_FORCED_STOP = -5, NLOPT_NUM_FAILURES = -6,
    NLOPT_SUCCESS = 1, NLOPT_STOPVAL_REACHED = 2, NLOPT_FTOL_REACHED = 3,
    NLOPT_XTOL_REACHED = 4, NLOPT_MAXEVAL_REACHED = 5, NLOPT_MAXTIME_REACHED = 6,
    NLOPT_NUM_RESULTS = 7
} nlopt_result;
#define NLOPT_MINF_MAX_REACHED NLOPT_STOPVAL_REACHED

struct nlopt_opt_s;
typedef struct nlopt_opt_s *nlopt_opt;
typedef void *(*nlopt_munge)(void *p);
typedef void *(*nlopt_munge2)(void *p, void *data);

/* ---- names, version, rng stubs (reference general.c:30-246) --------------- */
const char *nlopt_algorithm_name(nlopt_algorithm a);
const char *nlopt_algorithm_to_string(nlopt_algorithm a);
nlopt_algorithm nlopt_algorithm_from_string(const char *name);
const char *nlopt_result_to_string(nlopt_result r);
nlopt_result nlopt_result_from_string(const char *name);
void nlopt_version(int *major, int *minor, int *bugfix);
void nlopt_srand(unsigned long seed);       /* accepted, no effect: MMA/CCSAQ are deterministic */
void nlopt_srand_time(void);

/* ---- object lifetime (options.c:36-265) ----------------------------------- */
nlopt_opt nlopt_create(nlopt_algorithm algorithm, unsigned n);
void nlopt_destroy(nlopt_opt opt);
nlopt_opt nlopt_copy(const nlopt_opt opt);

/* ---- run (optimize.c:991-1083) --------------------------------------------- */
nlopt_result nlopt_optimize(nlopt_opt opt, double *x, double *opt_f);

/* ---- objective (options.c:322-364) ------------------------------------------ */
nlopt_result nlopt_set_min_objective(nlopt_opt opt, nlopt_func f, void *f_data);
nlopt_result nlopt_set_max_objective(nlopt_opt opt, nlopt_func f, void *f_data);
nlopt_result nlopt_set_precond_min_objective(nlopt_opt opt, nlopt_func f, nlopt_precond pre, void *f_data);
nlopt_result nlopt_set_precond_max_objective(nlopt_opt opt, nlopt_func f, nlopt_precond pre, void *f_data);

nlopt_algorithm nlopt_get_algorithm(const nlopt_opt opt);
unsigned nlopt_get_dimension(const nlopt_opt opt);
const char *nlopt_get_errmsg(nlopt_opt opt);

/* ---- named algorithm parameters (options.c:268-318) -------------------------
 * read by MMA/CCSAQ (optimize.c:798-826): inner_maxeval, verbosity, rho_init, inner_gradients,
 * always_improve, sigma_min, dual_algorithm, dual_ftol_rel, dual_ftol_abs, dual_xtol_rel,
 * dual_xtol_abs, dual_maxeval.  */
nlopt_result nlopt_set_param(nlopt_opt opt, const char *name, double val);
double nlopt_get_param(const nlopt_opt opt, const char *name, double defaultval);
int nlopt_has_param(const nlopt_opt opt, const char *name);
unsigned nlopt_num_params(const nlopt_opt opt);
const char *nlopt_nth_param(const nlopt_opt opt, unsigned n);

/* ---- bounds (options.c:368-474) ---------------------------------------------- */
nlopt_result nlopt_set_lower_bounds(nlopt_opt opt, const double *lb);
nlopt_result nlopt_set_lower_bounds1(nlopt_opt opt, double lb);
nlopt_result nlopt_set_lower_bound(nlopt_opt opt, int i, double lb);
nlopt_result nlopt_get_lower_bounds(const nlopt_opt opt, double *lb);
nlopt_result nlopt_set_upper_bounds(nlopt_opt opt, const double *ub);
nlopt_result nlopt_set_upper_bounds1(nlopt_opt opt, double ub);
nlopt_result nlopt_set_upper_bound(nlopt_opt opt, int i, double ub);
nlopt_result nlopt_get_upper_bounds(const nlopt_opt opt, double *ub);

/* ---- constraints (options.c:476-659) ------------------------------------------ */
nlopt_result nlopt_remove_inequality_constraints(nlopt_opt opt);
nlopt_result nlopt_add_inequality_constraint(nlopt_opt opt, nlopt_func fc, void *fc_data, double tol);
nlopt_result nlopt_add_precond_inequality_constraint(nlopt_opt opt, nlopt_func fc, nlopt_precond pre,
                                                     void *fc_data, double tol);
nlopt_result nlopt_add_inequality_mconstraint(nlopt_opt opt, unsigned m, nlopt_mfunc fc, void *fc_data,
                                              const double *tol);
nlopt_result nlopt_remove_equality_constraints(nlopt_opt opt);
nlopt_result nlopt_add_equality_constraint(nlopt_opt opt, nlopt_func h, void *h_data, double tol);
nlopt_result nlopt_add_precond_equality_constraint(nlopt_opt opt, nlopt_func h, nlopt_precond pre,
                                                   void *h_data, double tol);
nlopt_result nlopt_add_equality_mconstraint(nlopt_opt opt, unsigned m, nlopt_mfunc h, void *h_data,
                                            const double *tol);

/* ---- stopping criteria (options.c:661-816) ------------------------------------- */
nlopt_result nlopt_set_stopval(nlopt_opt opt, double stopval);
double nlopt_get_stopval(const nlopt_opt opt);
nlopt_result nlopt_set_ftol_rel(nlopt_opt opt, double tol);
double nlopt_get_ftol_rel(const nlopt_opt opt);
nlopt_result nlopt_set_ftol_abs(nlopt_opt opt, double tol);
double nlopt_get_ftol_abs(const nlopt_opt opt);
nlopt_result nlopt_set_xtol_rel(nlopt_opt opt, double tol);
double nlopt_get_xtol_rel(const nlopt_opt opt);
nlopt_result nlopt_set_xtol_abs1(nlopt_opt opt, double tol);
nlopt_result nlopt_set_xtol_abs(nlopt_opt opt, const double *tol);
nlopt_result nlopt_get_xtol_abs(const nlopt_opt opt, double *tol);
nlopt_result nlopt_set_x_weights1(nlopt_opt opt, double w);
nlopt_result nlopt_set_x_weights(nlopt_opt opt, const double *w);
nlopt_result nlopt_get_x_weights(const nlopt_opt opt, double *w);
nlopt_result nlopt_set_maxeval(nlopt_opt opt, int maxeval);
int nlopt_get_maxeval(const nlopt_opt opt);
int nlopt_get_numevals(const nlopt_opt opt);
nlopt_result nlopt_set_maxtime(nlopt_opt opt, double maxtime);
double nlopt_get_maxtime(const nlopt_opt opt);
nlopt_result nlopt_force_stop(nlopt_opt opt);
nlopt_result nlopt_set_force_stop(nlopt_opt opt, int val);
int nlopt_get_force_stop(const nlopt_opt opt);

/* ---- algorithm-specific (options.c:818-957) ------------------------------------- */
nlopt_result nlopt_set_local_optimizer(nlopt_opt opt, const nlopt_opt local_opt);
nlopt_result nlopt_set_population(nlopt_opt opt, unsigned pop);
unsigned nlopt_get_population(const nlopt_opt opt);
nlopt_result nlopt_set_vector_storage(nlopt_opt opt, unsigned dim);
unsigned nlopt_get_vector_storage(const nlopt_opt opt);
nlopt_result nlopt_set_default_initial_step(nlopt_opt opt, const double *x);
nlopt_result nlopt_set_initial_step(nlopt_opt opt, const double *dx);   /* = sigma_0 for MMA/CCSAQ */
nlopt_result nlopt_set_initial_step1(nlopt_opt opt, double dx);
nlopt_result nlopt_get_initial_step(const nlopt_opt opt, const double *x, double *dx);

/* ---- wrapper support (options.c:961-981) ------------------------------------------ */
void nlopt_set_munge(nlopt_opt opt, nlopt_munge munge_on_destroy, nlopt_munge munge_on_copy);
void nlopt_munge_data(nlopt_opt opt, nlopt_munge2 munge, void *data);

/* ---- deprecated one-call API (reference nlopt.h:305-343, src/api/deprecated.c): thin wrappers that build an
 * nlopt_opt, set the given options and call nlopt_optimize; kept so that old binaries still link ---- */
typedef double (*nlopt_func_old)(int n, const double *x, double *gradient, void *func_data);
nlopt_result nlopt_minimize(nlopt_algorithm algorithm, int n, nlopt_func_old f, void *f_data, const double *lb,
                            const double *ub, double *x, double *minf, double minf_max, double ftol_rel, double ftol_abs,
                            double xtol_rel, const double *xtol_abs, int maxeval, double maxtime);
nlopt_result nlopt_minimize_constrained(nlopt_algorithm algorithm, int n, nlopt_func_old f, void *f_data, int m,
                                        nlopt_func_old fc, void *fc_data, ptrdiff_t fc_datum_size, const double *lb,
                                        const double *ub, double *x, double *minf, double minf_max, double ftol_rel,
                                        double ftol_abs, double xtol_rel, const double *xtol_abs, int maxeval, double maxtime);
nlopt_result nlopt_minimize_econstrained(nlopt_algorithm algorithm, int n, nlopt_func_old f, void *f_data, int m,
                                         nlopt_func_old fc, void *fc_data, ptrdiff_t fc_datum_size, int p, nlopt_func_old h,
                                         void *h_data, ptrdiff_t h_datum_size, const double *lb, const double *ub, double *x,
                                         double *minf, double minf_max, double ftol_rel, double ftol_abs, double xtol_rel,
                                         const double *xtol_abs, double htol_rel, double htol_abs, int maxeval, double maxtime);
void nlopt_get_local_search_algorithm(nlopt_algorithm *deriv, nlopt_algorithm *nonderiv, int *maxeval);
void nlopt_set_local_search_algorithm(nlopt_algorithm deriv, nlopt_algorithm nonderiv, int maxeval);
int nlopt_get_stochastic_population(void);
void nlopt_set_stochastic_population(int pop);

/* ===========================================================================
 *  Extensions (no reference equivalent)
 * ======================================================================== */

/* Device-resident callbacks.  `x_dev` / `grad_dev` are DEVICE pointers to this rank's shard
 * (n_local contiguous variables starting at global index j0); the callback enqueues its work on
 * `cuda_stream` (a cudaStream_t) and returns the function value.  With more than one rank the
 * callback returns its shard's additive contribution and the library sums over ranks.
 * `grad_dev == NULL` when no gradient is wanted.  These replace the host trip of
 * mma.c:218-229 / :297-311 (x to the user, gradients back) with nothing. */
typedef double (*nlopt_b200_dfunc)(unsigned n_local, unsigned long long j0, const double *x_dev,
                                   double *grad_dev, void *func_data, void *cuda_stream);
nlopt_result nlopt_b200_set_min_objective_device(nlopt_opt opt, nlopt_b200_dfunc f, void *f_data);
/* Maximisation (the device twins of nlopt_set_max_objective, here and for the forms below): the callback returns f and
 * writes grad f of the function to MAXIMISE; the library minimises -f and reports opt_f = f.  The sign flip is exact:
 * the value is negated once it is final (after the sum over ranks and finish) and the gradient by one kernel on the
 * library stream right after the callback, so a maximisation of -F runs through the same points as a minimisation of F,
 * bit for bit (as long as no sum of terms is exactly zero, whose sign may differ).  Argument checks and the stopval handling are those of the _min_ form / nlopt_set_max_objective. */
nlopt_result nlopt_b200_set_max_objective_device(nlopt_opt opt, nlopt_b200_dfunc f, void *f_data);
nlopt_result nlopt_b200_add_inequality_constraint_device(nlopt_opt opt, nlopt_b200_dfunc fc,
                                                         void *fc_data, double tol);
/* h(x) = 0 within tol: accepted by the algorithms that take nlopt_add_equality_constraint (the AUGLAG family here);
 * NLOPT_INVALID_ARGS on LD_MMA / LD_CCSAQ, for a NULL callback or a negative tol */
nlopt_result nlopt_b200_add_equality_constraint_device(nlopt_opt opt, nlopt_b200_dfunc h, void *h_data, double tol);

/* Device callbacks, second form: asynchronous and independent of the number of ranks.
 * The library cuts the n variables into groups and 8 "virtual shards" by a rule that depends on n only (the rule of the
 * dual kernels); a rank owns the virtual shards [vshard0, vshard0 + local_vshards).  The callback enqueues its work on
 * `cuda_stream` and leaves the partial sum of each of ITS virtual shards in vsums_dev[vshard] (8 doubles, zeroed by the
 * library beforehand) -- reduced over the shard's groups in an order that depends on n only.  It does not synchronise
 * and returns nothing: after all callbacks of a point have been enqueued, the library adds the 8 shard sums of all
 * ranks in index order (so the value is bit-identical for 1, 2, 4 and 8 ranks) and calls finish(total, data) on the
 * host for the function value.  One host synchronisation per point instead of one per function.
 * `halo` > 0: the callback also reads x_dev[-halo .. -1] and x_dev[n_local .. n_local + halo - 1] (stencil functions
 * such as the chained Rosenbrock function); the library fills these cells from the neighbouring ranks before the
 * callbacks of a point run.  halo <= 1 in this build. */
#endif  /* __CUDACC_RTC__ */
typedef struct {
    unsigned long long n, n_local, j0;          /* global size; this rank's variables [j0, j0 + n_local)          */
    unsigned long long nchunks, chunk0;         /* 512-variable chunks: all of them / first of this rank           */
    unsigned groups_total, group0, groups_local, groups_per_vshard;   /* group g = chunks [g nchunks / groups_total, ...) */
    unsigned vshard0, local_vshards;
    int rank, world;
} nlopt_b200_shard;
#ifndef __CUDACC_RTC__
void nlopt_b200_shard_geometry(unsigned long long n, int rank, int world, nlopt_b200_shard *out);
typedef void (*nlopt_b200_dfunc2)(const nlopt_b200_shard *shard, const double *x_dev, double *grad_dev, double *vsums_dev,
                                  void *func_data, void *cuda_stream);
typedef double (*nlopt_b200_dfinish)(double total, void *func_data);
nlopt_result nlopt_b200_set_min_objective_device2(nlopt_opt opt, nlopt_b200_dfunc2 f, nlopt_b200_dfinish finish,
                                                  void *f_data, int halo);
/* maximise: finish(total) is the value of the function to maximise (see nlopt_b200_set_max_objective_device) */
nlopt_result nlopt_b200_set_max_objective_device2(nlopt_opt opt, nlopt_b200_dfunc2 f, nlopt_b200_dfinish finish,
                                                  void *f_data, int halo);
nlopt_result nlopt_b200_add_inequality_constraint_device2(nlopt_opt opt, nlopt_b200_dfunc2 fc, nlopt_b200_dfinish finish,
                                                          void *fc_data, double tol, int halo);
/* the equality twin: same argument checks (NULL callback or finish, halo outside {0, 1}, negative tol) and the algorithm
 * check of nlopt_add_equality_constraint */
nlopt_result nlopt_b200_add_equality_constraint_device2(nlopt_opt opt, nlopt_b200_dfunc2 h, nlopt_b200_dfinish finish,
                                                        void *h_data, double tol, int halo);
/* Vector device constraints (the device twin of nlopt_mfunc): one callback produces m constraint rows in one pass over x.
 * The callback enqueues the m components: vsums_dev is an [m][8] block (row i at vsums_dev + 8 i, zeroed by the
 * library); it leaves the sum of component i over each of ITS virtual shards in row i, reduced in an order that depends
 * on n only.  grad_dev: NULL, or row i of the Jacobian at grad_dev + i * grad_ld (this rank's shard).  After all
 * callbacks of a point have been enqueued, the library adds each row's 8 shard sums in index order and calls
 * finish(m, totals, result, data) once on the host: result[i] is constraint i.
 * Argument checks follow nlopt_add_*_mconstraint and the scalar _device2 twins: m == 0 succeeds and registers nothing;
 * NULL callback or finish and halo outside {0, 1} are NLOPT_INVALID_ARGS; tol (m entries) NULL means zeros; the
 * equality form is accepted by the algorithms that take nlopt_add_equality_constraint (the AUGLAG family here). */
typedef void (*nlopt_b200_dmfunc2)(unsigned m, const nlopt_b200_shard *shard, const double *x_dev, double *grad_dev,
                                   unsigned long long grad_ld, double *vsums_dev, void *func_data, void *cuda_stream);
typedef void (*nlopt_b200_dmfinish)(unsigned m, const double *totals, double *result, void *func_data);
nlopt_result nlopt_b200_add_inequality_mconstraint_device2(nlopt_opt opt, unsigned m, nlopt_b200_dmfunc2 fc,
                                                           nlopt_b200_dmfinish finish, void *fc_data, const double *tol,
                                                           int halo);
nlopt_result nlopt_b200_add_equality_mconstraint_device2(nlopt_opt opt, unsigned m, nlopt_b200_dmfunc2 h,
                                                         nlopt_b200_dmfinish finish, void *h_data, const double *tol,
                                                         int halo);
/* Device callbacks, third form: per-variable TERMS, for code that cannot be written as a __device__ functor (its own
 * kernels, cuBLAS / cuSPARSE, a filter, PyTorch).  The callback enqueues on `cuda_stream`, and does not synchronise:
 *     terms_dev[i * ld + jl] = term i of variable j0 + jl          (i < m, jl < shard->n_local)
 * and, when grad_dev != NULL, grad_dev[i * ld + jl] = d c_i / d x_j (m = 1 for a scalar function).  terms_dev is a
 * library-owned buffer of m * ld doubles (ld >= n_local; entries from n_local to ld are never read); it is valid only
 * for the duration of the call and the work the callback enqueues.  The library then reduces row i of the terms on the
 * GPU in exactly the order of the __device__ functors (nlopt_b200_device.cuh: map_group_kernel / map_group_mkernel
 * and the fold of the group sums), adds the 8 virtual-shard sums in index order and calls finish once per point, as
 * for the _device2 forms: finish(total, data) for a scalar function, finish(m, totals, result, data) for m rows.
 * Bit contract: terms bit-equal to a functor's terms give that functor's value bits, so a run matches the functor's run
 * bit for bit (result code, evaluation counts, f*, x*) under LD_MMA, LD_CCSAQ and the AUGLAG family; the value depends
 * on n only, not on the number of ranks.  `halo` as for the _device2 forms (the callback may read x_dev[-1] and
 * x_dev[n_local]).  Argument checks are those of the _device2 / _mconstraint_device2 twins; any m the constraint path
 * accepts (no register-file cap).  Not taken by preconditioned CCSAQ. */
typedef void (*nlopt_b200_dtfunc)(unsigned m, const nlopt_b200_shard *shard, const double *x_dev, double *grad_dev,
                                  unsigned long long ld, double *terms_dev, void *func_data, void *cuda_stream);
nlopt_result nlopt_b200_set_min_objective_terms(nlopt_opt opt, nlopt_b200_dtfunc f, nlopt_b200_dfinish finish,
                                                void *f_data, int halo);
nlopt_result nlopt_b200_set_max_objective_terms(nlopt_opt opt, nlopt_b200_dtfunc f, nlopt_b200_dfinish finish,
                                                void *f_data, int halo);
nlopt_result nlopt_b200_add_inequality_constraint_terms(nlopt_opt opt, nlopt_b200_dtfunc fc, nlopt_b200_dfinish finish,
                                                        void *fc_data, double tol, int halo);
nlopt_result nlopt_b200_add_equality_constraint_terms(nlopt_opt opt, nlopt_b200_dtfunc h, nlopt_b200_dfinish finish,
                                                      void *h_data, double tol, int halo);
nlopt_result nlopt_b200_add_inequality_mconstraint_terms(nlopt_opt opt, unsigned m, nlopt_b200_dtfunc fc,
                                                         nlopt_b200_dmfinish finish, void *fc_data, const double *tol,
                                                         int halo);
nlopt_result nlopt_b200_add_equality_mconstraint_terms(nlopt_opt opt, unsigned m, nlopt_b200_dtfunc h,
                                                       nlopt_b200_dmfinish finish, void *h_data, const double *tol,
                                                       int halo);
/* Device functors given as SOURCE, for callers without nvcc.  nlopt_b200_jit_create compiles `source` with NVRTC
 * (opened at the first call; libnvrtc.so.12 by soname, else from the toolkit the library was built with) for sm_90a,
 * with -std=c++17 --fmad=false and the caller's options, together with the map kernels of
 * include/nlopt_b200_device_kernels.cuh, whose text the library embeds (the source may include nothing else of this
 * library; its functor is a struct of the nlopt_b200_device.cuh concept, named by `name`, with or without namespace).
 * The registrations below launch the header's own map_group_kernel / map_group_mkernel instantiation and the same
 * fold kernels, so values, and whole runs, have the bits of the same functor compiled by nvcc (nlopt_b200_device.cuh).
 * Compiled images are cached per process, keyed by source, name and options.  The handle is returned even when the
 * compile fails: nlopt_b200_jit_errmsg then says why (NULL when compiled), nlopt_b200_jit_log holds the compiler log.
 * A functor must have m (F::m, 0 for a scalar functor) <= 16 and halo <= 1; nlopt_b200_jit_info reports them and
 * sizeof(F) (= param_bytes).  A registration copies the `param_bytes` bytes of the functor object at `params` (its
 * members: scalars, arrays, device pointers) and takes an optional host finish: NULL is the identity, else
 * finish(total, finish_data) / finish(m, totals, result, finish_data) as for the _device2 forms.  NLOPT_INVALID_ARGS,
 * with a message, for a failed handle, param_bytes != sizeof(F), a scalar functor registered with an _mconstraint form
 * or a vector functor with the others, and a negative or NaN tolerance; then the checks of the _device2 twins.  The
 * handle must outlive every opt that uses it (it owns the registrations).  One GPU verified. */
typedef struct nlopt_b200_jit_s *nlopt_b200_jit;
nlopt_b200_jit nlopt_b200_jit_create(const char *source, const char *name, const char *const *options, int noptions);
void nlopt_b200_jit_destroy(nlopt_b200_jit h);
const char *nlopt_b200_jit_errmsg(nlopt_b200_jit h);
const char *nlopt_b200_jit_log(nlopt_b200_jit h);
/* 0, and m / halo / sizeof(F), for a compiled handle; -1 for a failed one */
int nlopt_b200_jit_info(nlopt_b200_jit h, int *m, int *halo, size_t *param_bytes);
/* the compiled sm_90a cubin (NULL for a failed handle) */
const void *nlopt_b200_jit_image(nlopt_b200_jit h, size_t *bytes);
nlopt_result nlopt_b200_jit_set_min_objective(nlopt_opt opt, nlopt_b200_jit f, const void *params, size_t param_bytes,
                                              nlopt_b200_dfinish finish, void *finish_data);
nlopt_result nlopt_b200_jit_set_max_objective(nlopt_opt opt, nlopt_b200_jit f, const void *params, size_t param_bytes,
                                              nlopt_b200_dfinish finish, void *finish_data);
nlopt_result nlopt_b200_jit_add_inequality_constraint(nlopt_opt opt, nlopt_b200_jit fc, const void *params, size_t param_bytes,
                                                      nlopt_b200_dfinish finish, void *finish_data, double tol);
nlopt_result nlopt_b200_jit_add_equality_constraint(nlopt_opt opt, nlopt_b200_jit h, const void *params, size_t param_bytes,
                                                    nlopt_b200_dfinish finish, void *finish_data, double tol);
/* tol: m entries, or NULL for zeros */
nlopt_result nlopt_b200_jit_add_inequality_mconstraint(nlopt_opt opt, nlopt_b200_jit fc, const void *params, size_t param_bytes,
                                                       nlopt_b200_dmfinish finish, void *finish_data, const double *tol);
nlopt_result nlopt_b200_jit_add_equality_mconstraint(nlopt_opt opt, nlopt_b200_jit h, const void *params, size_t param_bytes,
                                                     nlopt_b200_dmfinish finish, void *finish_data, const double *tol);
/* Sharded HOST callbacks (one process per GPU): the callback sees only this rank's variables -- x_shard and grad_shard
 * hold the n_local entries starting at global index j0 -- and returns its ADDITIVE contribution to the function value
 * (a constant term is added by one rank only, e.g. the one with j0 == 0); the library sums the contributions over the
 * ranks.  Compared with a plain nlopt_func on several ranks (every rank receives the full x and uploads its shard of the
 * gradient) each rank moves n_local instead of n doubles per evaluation over PCIe, and the callback's work is divided
 * by the number of ranks.  With one rank this is the plain callback with j0 = 0, n_local = n. */
typedef double (*nlopt_b200_sfunc)(unsigned n_local, unsigned long long j0, unsigned long long n, const double *x_shard,
                                   double *grad_shard, void *func_data);
nlopt_result nlopt_b200_set_min_objective_sharded(nlopt_opt opt, nlopt_b200_sfunc f, void *f_data);
/* maximise (LD_MMA / LD_CCSAQ; see nlopt_b200_set_max_objective_device) */
nlopt_result nlopt_b200_set_max_objective_sharded(nlopt_opt opt, nlopt_b200_sfunc f, void *f_data);
nlopt_result nlopt_b200_add_inequality_constraint_sharded(nlopt_opt opt, nlopt_b200_sfunc fc, void *fc_data, double tol);
/* like nlopt_optimize, but x_dev is a device array of this rank's shard (in/out) */
nlopt_result nlopt_b200_optimize_device(nlopt_opt opt, double *x_dev, double *opt_f);
/* Box bounds from device memory.  The call copies the n doubles at lb_dev / ub_dev into device memory the object owns
 * (on the current device) and returns when the copy is complete, so the buffer may be reused at once; the work that
 * produces it must be complete before the call, as for nlopt_b200_optimize_device.  The copy is snapped on the device
 * as nlopt_set_lower_bounds / nlopt_set_upper_bounds snap (a subnormally thin interval is shut), giving the same bits.
 * The first such call puts the object in device mode for both arrays (the other one is uploaded once); a run then
 * copies them device to device, checks the start point on the device (NLOPT_INVALID_ARGS and the reference's
 * "bounds %d fail" message, no evaluation) and reads each array as one scalar where all its lanes have the bits of
 * lane 0.  Any host bound setter downloads both arrays and leaves device mode; nlopt_get_*_bounds,
 * nlopt_set_local_optimizer and the initial-step heuristics read the device values; nlopt_copy duplicates them.
 * NULL: NLOPT_INVALID_ARGS; n == 0: no-op; no usable device: NLOPT_FAILURE, bounds unchanged; several ranks, a run on
 * another current device, or preconditioned CCSAQ: NLOPT_INVALID_ARGS.  The deprecated nlopt_minimize* API takes host
 * bounds only. */
nlopt_result nlopt_b200_set_lower_bounds_device(nlopt_opt opt, const double *lb_dev);
nlopt_result nlopt_b200_set_upper_bounds_device(nlopt_opt opt, const double *ub_dev);
/* xtol_abs, x_weights and the initial step (MMA / CCSAQ: each variable's first move limit, sigma_0) from device memory.
 * Each call copies the n doubles at its argument into device memory the object owns (on the current device) and returns
 * when the copy and its check are complete, so the buffer may be reused at once; the work that produces it must be
 * complete before the call.  The check is the host setter's, made on the device: a negative weight gives
 * NLOPT_INVALID_ARGS and "invalid negative weight", a zero step (+0.0 or -0.0) NLOPT_INVALID_ARGS and "zero step size"
 * (NaN passes both); xtol_abs is not checked.  The option is then in device mode, independently of the other two and of
 * the bounds: a run reads it in place (no host-to-device copy), and a bitwise uniform step takes the sigma index as
 * nlopt_set_initial_step1 does.  Any host setter of the same option (nlopt_set_xtol_abs / _xtol_abs1, nlopt_set_x_weights
 * / _x_weights1, nlopt_set_initial_step / _initial_step1, nlopt_set_default_initial_step; NULL included) frees the device
 * copy and leaves device mode; nlopt_get_xtol_abs, nlopt_get_x_weights and nlopt_get_initial_step read the device
 * values; nlopt_copy duplicates them; NLOPT_AUGLAG* hands the step (and xtol_abs, to a sub-optimiser it creates) to its
 * sub-optimiser device to device.  NULL: NLOPT_INVALID_ARGS; n == 0: no-op; no usable device: NLOPT_FAILURE; several
 * ranks, or a run on another current device: NLOPT_INVALID_ARGS.  A failed call keeps the previous values. */
nlopt_result nlopt_b200_set_xtol_abs_device(nlopt_opt opt, const double *xtol_abs_dev);
nlopt_result nlopt_b200_set_x_weights_device(nlopt_opt opt, const double *w_dev);
nlopt_result nlopt_b200_set_initial_step_device(nlopt_opt opt, const double *dx_dev);

/* Run statistics of the last nlopt_optimize on this object; after an NLOPT_AUGLAG* run, those of its last
 * sub-optimisation. */
typedef struct {
    long long dual_evals;        /* level-1 dual evaluations (kernel launches of the dual kernel) */
    long long dual_solves;       /* = inner CCSA iterations                                      */
    long long outer_iters;
    double seconds_total;        /* wall time inside nlopt_optimize                               */
    double seconds_callbacks;    /* ... of which inside user callbacks                            */
    double seconds_dual_kernel;  /* device time of the dual kernel (CUDA events), 0 if not timed  */
    long long h2d_bytes, d2h_bytes;
    long long kernel_launches;   /* all kernels of this library                                   */
    double seconds_setup;        /* wall: allocating / uploading the device state                  */
    double seconds_dual_wall;    /* wall: inside dual solves (launch to result, incl. exchange)    */
    double seconds_eval_wall;    /* wall: objective + constraint evaluations (callbacks + copies)  */
    double seconds_glue_wall;    /* wall: sigma init, end-of-outer pass, final copy of x           */
    long long dual_operand_bytes; /* HBM bytes the dual kernels were asked to read on this rank, summed over evaluations,
                                     plus their stores of x*(y): 8 ld (3 + m) per evaluation when both bounds are
                                     uniform (nlopt_set_*_bounds1) and the default kernels run, 8 ld (5 + m) otherwise;
                                     ld = this rank's padded shard length; with the sigma index (below) the default
                                     TMA-staged solve kernel reads 8 ld (2 + m) + 2 ld instead of 8 ld (3 + m) */
    long long sigma_palette;     /* entries of the sigma palette at the end of the run, 0 when the dual kernels no
                                     longer read sigma as a 16-bit index into it (bounds or initial step not uniform,
                                     palette past its 65535-entry cap, or a self-check mismatch)                   */
    long long sigma_index_mismatches;  /* variables whose updated sigma differed from its palette entry (expected 0)  */
} nlopt_b200_stats;
nlopt_result nlopt_b200_get_stats(const nlopt_opt opt, nlopt_b200_stats *out);

/* ---- kernel-level access: one dual evaluation on resident arrays ------------
 * This is the operator the reference implements as the static
 * dual_func(m, y, grad, dual_data*) (mma.c:59-137, ccsa_quadratic.c:79-148).  */
typedef struct nlopt_b200_dual_s *nlopt_b200_dual;
enum { NLOPT_B200_MMA = 0, NLOPT_B200_CCSAQ = 1 };

nlopt_b200_dual nlopt_b200_dual_create(int variant, unsigned n, unsigned m);
void nlopt_b200_dual_destroy(nlopt_b200_dual h);
const char *nlopt_b200_dual_errmsg(nlopt_b200_dual h);
/* host -> device: the arrays of dual_data; grad_c is m*n row-major by constraint */
int nlopt_b200_dual_upload(nlopt_b200_dual h, const double *x, const double *lb, const double *ub,
                           const double *sigma, const double *grad_f, const double *grad_c);
/* fill the resident arrays on the device with the deterministic synthetic instance of
 * SURVEY.md 8(d) (counter-based hash; same generator as tests/synth.py) */
int nlopt_b200_dual_fill_synthetic(nlopt_b200_dual h, unsigned long long seed);
int nlopt_b200_dual_set_scalars(nlopt_b200_dual h, double f0, double rho, const double *c0, const double *rhoc);
/* out[0] = -val (what the dual optimiser minimises), out[1] = g0, out[2] = w, out[3..3+m) = g_i;
 * grad (may be NULL) receives -g_i.  want_xcur != 0 also materialises x*(y) on the device. */
int nlopt_b200_dual_eval(nlopt_b200_dual h, const double *y, int want_xcur, double *out, double *grad);
/* A whole dual solve on the resident arrays -- what mma.c:275-288 does with nlopt_optimize_limited(dual_opt, y, ...) and
 * the final dual_func call: maximise the dual over [lo, hi]^m from the warm start y (in/out) with the level-2/3
 * optimiser of optimize.c:818-826 (ftol_rel, maxeval; the other tolerances 0), then evaluate once more at the solution
 * storing x*(y).  m <= 16 runs as ONE persistent kernel launch; larger m one launch per evaluation.  out[] as for
 * nlopt_b200_dual_eval at the solution; *nevals = dual evaluations performed (the final one included);
 * *kernel_ms = device time of the dual kernels (CUDA events). */
int nlopt_b200_dual_solve(nlopt_b200_dual h, double *y, const double *lo, const double *hi, double ftol_rel, int maxeval,
                          double *out, int *result, long *nevals, double *kernel_ms);
int nlopt_b200_dual_download_xcur(nlopt_b200_dual h, double *xcur_host);
int nlopt_b200_dual_download(nlopt_b200_dual h, const char *which, double *host);  /* "x","sigma","xprev",... */
/* sigma kernels (mma.c:202-210, :431-442) and the fused end-of-outer-iteration pass */
int nlopt_b200_dual_sigma_init(nlopt_b200_dual h, const double *sigma_init_host, double sigma_min);
int nlopt_b200_dual_end_outer(nlopt_b200_dual h, int k, double sigma_min, const double *x_weights_host,
                              const double *xtol_abs_host, double *norms /* [2]: sum w|dx|, sum w|x| */,
                              int *all_below_xtol_abs);
int nlopt_b200_dual_set_prev(nlopt_b200_dual h, const double *xcur, const double *xprev, const double *xprevprev);
/* timing helper: average device milliseconds of `iters` back-to-back evaluations (CUDA events) */
int nlopt_b200_dual_time(nlopt_b200_dual h, const double *y, int want_xcur, int iters, double *ms_avg);
/* tuning knobs for the launch geometry (0 = default); returns 0 on success */
int nlopt_b200_dual_configure(nlopt_b200_dual h, const char *key, long long value);
long long nlopt_b200_dual_query(nlopt_b200_dual h, const char *key);

/* ---- multi-GPU: one process per GPU, variables sharded in contiguous blocks --
 * The host program (torchrun / torch.distributed) creates the 128-byte id on rank 0 with
 * nlopt_b200_comm_unique_id, broadcasts it, and every rank calls nlopt_b200_comm_init.
 * Afterwards objects created in this process shard n over `world` ranks; per dual
 * evaluation one all-gather of (m+3)*8/world doubles crosses NVLink. */
int nlopt_b200_comm_unique_id(unsigned char id128[128]);
int nlopt_b200_comm_init(const unsigned char id128[128], int rank, int world, int device);
int nlopt_b200_comm_finalize(void);
int nlopt_b200_comm_rank(void);
int nlopt_b200_comm_world(void);
/* shard geometry for a problem of n variables: first global index and count owned by `rank` */
void nlopt_b200_shard_range(unsigned long long n, int rank, int world,
                            unsigned long long *j0, unsigned long long *count);

/* nlopt_optimize parks its large device / pinned blocks in a process-wide cache for the next call;
 * this frees them. */
void nlopt_b200_release_cached_memory(void);

/* library / device probe: returns number of visible CUDA devices, <0 on CUDA error */
int nlopt_b200_device_count(void);
const char *nlopt_b200_build_info(void);

#endif  /* __CUDACC_RTC__ */

#ifdef __cplusplus
}
#endif
#endif /* NLOPT_B200_H */

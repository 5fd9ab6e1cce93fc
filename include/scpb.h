/* scpb.h -- C ABI of libscpb (CUDA SCP inner loop for the H100, sm_90a).
 *
 * Drop-in boundary for the hot path of UW-ACL/SCPToolbox.jl (file:line relative to the
 * reference tree):
 *   scpb_discretize*     replaces discretize!(ref, pbm)      src/solvers/discretization.jl:160-217
 *                        (derivs_foh :235-286, set_update_matrices :354-406, rk4 helper.jl:411-501)
 *   scpb_cone_*          replaces solve!(prg)=JuMP.optimize! src/parser/program.jl:419-424
 *                        reached from solve_subproblem!      src/solvers/scp.jl:942-950
 *   scpb_ptr_*           replaces the PTR loop body          src/solvers/ptr.jl:448-532
 *                        (formulate :470-478 + solve :484 + discretize :380) for a batch of seeds
 *
 * Conventions: plain C, every entry point returns int32 status (0 = OK, <0 = error; text via
 * scpb_last_error), never throws or aborts.  Host arrays are caller-owned.  Per-seed blocks use
 * Julia's column-major memory so that a batch of one maps 1:1 onto `ref.dyn.A` etc.
 * A handle is bound to one CUDA device + stream and is not thread-safe; different handles are.
 */
#ifndef SCPB_H
#define SCPB_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct scpb_handle_s *scpb_handle;

/* ---- device model packs (the device-side twin of traj.f/A/B/F, problem.jl:432-450) ---- */
enum {
    SCPB_MODEL_DBLINT = 1,    /* x=[pos,vel] u=[acc] p=[tf];      par: g                          */
    SCPB_MODEL_ROCKET = 2,    /* x=[r3,v3,z] u=[a3,xi] p=[tf];    par: g[3], omega[3], alpha      */
    SCPB_MODEL_STARSHIP = 3,  /* starship_flip/definition.jl:498-637;
                                 par: m, J, lcg, lcp, CD, alpha_e, rate_delay, g0, tau_s           */
    SCPB_MODEL_QUADROTOR = 4, /* quadrotor/definition.jl:140-186; par: g[3]                        */
    SCPB_MODEL_FREEFLYER = 5, /* freeflyer/definition.jl:224-284; par: mass, J[9], Jinv[9] (col-major) */
    SCPB_MODEL_RENDEZVOUS2D = 6, /* rendezvous_planar/definition.jl:147-243 (impulsive RCS thrust): x=[r2,v2,theta,omega],
                                 u[0..2]=(f-,f+,f0) of 12 inputs, p=[tdil]; par: m, J, lu, lv, n.  The only pack with
                                 impulse semantics (the reference's f/B called with a negative segment index).
                                 Its constraint pack (the RCS deadband, definition.jl:337-413: ns = 6, ng = 1) reads
                                 par[5] = f_db, par[6] = f_max, par[7] = kappa, the sharpness of the smooth OR */
    SCPB_MODEL_OSCILLATOR = 7 /* oscillator/definition.jl:161-236 (fixed final time: F = 0, no time-dilation column):
                                 x=[r,v], u=[aa,ar,l1aa,l1adiff], p=[l1r_1..l1r_N] (np must be N); par: zeta, omega0, tf.
                                 Its constraint pack (the input deadband, definition.jl:370-444: ns = 2, ng = 1, the
                                 node's own parameter) reads par[3] = a_db, par[4] = a_max, par[5] = kappa */
};
#define SCPB_MAX_PAR 64

enum { SCPB_FOH = 0, SCPB_IMPULSE = 1 };

/* status codes */
enum {
    SCPB_OK = 0,
    SCPB_ERR_ARG = -1,
    SCPB_ERR_CUDA = -2,
    SCPB_ERR_MODEL = -3,
    SCPB_ERR_UNSUPPORTED = -4,
    SCPB_ERR_STATE = -5
};

/* ---- lifetime ---- */
int32_t scpb_create(int32_t device, scpb_handle *out);
int32_t scpb_destroy(scpb_handle h);
int32_t scpb_last_error(scpb_handle h, char *buf, size_t len);
int32_t scpb_version(void);
/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
int64_t scpb_launch_count(scpb_handle h);
/* CUDA stream the handle launches on (cudaStream_t as void*), for event timing by the caller */
void *scpb_stream(scpb_handle h);
int32_t scpb_sync(scpb_handle h);

/* ---- model selection ---- */
int32_t scpb_model_set(scpb_handle h, int32_t model_id, const double *par, int32_t npar,
                       int32_t nx, int32_t nu, int32_t np);

/* ---- discretize!  (host buffers; H2D + kernel + D2H inside) ----
 * method: SCPB_FOH (discretization.jl:235-286) or SCPB_IMPULSE (:186-193 jump, :304-340 derivs_impulse, :384-390
 * B_k = A_k B(t_k, -k); needs a model pack with impulse semantics).  For IMPULSE dyn.B has ONE block: Bm; Bp (if
 * given) is written as zeros.
 * t_grid[N]; xd[B][N][nx]; ud[B][N][nu]; p[B][np]; iSx_diag[nx];
 * A[B][N-1][nx*nx], Bm/Bp[B][N-1][nx*nu], F[B][N-1][nx*np], r[B][N-1][nx], E[B][N-1][nx*nx],
 * defect[B][N-1][nx], feas[B] (1 = dynamically feasible); *seconds = device time of the kernel. */
int32_t scpb_discretize(scpb_handle h, int32_t method, int32_t B, int32_t N, int32_t Nsub,
                        const double *t_grid, const double *xd, const double *ud, const double *p,
                        const double *iSx_diag, double feas_tol,
                        double *A, double *Bm, double *Bp, double *F, double *r, double *E,
                        double *defect, int32_t *feas, double *seconds);

/* same, all pointers are DEVICE pointers in the same layouts (inputs resident in HBM);
 * asynchronous on the handle's stream. */
int32_t scpb_discretize_dev(scpb_handle h, int32_t method, int32_t B, int32_t N, int32_t Nsub,
                            const double *t_grid, const double *xd, const double *ud, const double *p,
                            const double *iSx_diag, double feas_tol,
                            double *A, double *Bm, double *Bp, double *F, double *r, double *E,
                            double *defect, int32_t *feas);

/* ---- propagate(sol, pbm; res): final continuous-time state trajectory of B converged solutions ----
 * replaces src/solvers/discretization.jl:515-562 (FOH branch), called by SCPSolution (src/solvers/scp.jl:231-232,
 * res = 2*Nsub*(N-1)).  RK4 of the nonlinear dynamics over LinRange(0,1,res) from xd[:,1], the input linearly
 * interpolated over the whole grid, integration actions after every step.
 * xc[B][res][nx]: per seed Julia's column-major nx x res matrix (values of the Trajectory xc).
 * method SCPB_IMPULSE (:539-558): every interval restarts from the impulse-updated node state and coasts; the output
 * has 1 + (N-1)*ceil(res/(N-1)) columns per seed (xd[:,1], then ceil(res/(N-1)) columns per interval), which is what xc
 * must hold. */
int32_t scpb_propagate(scpb_handle h, int32_t method, int32_t B, int32_t N, int32_t res, const double *t_grid,
                       const double *xd, const double *ud, const double *p, double *xc, double *seconds);

/* ---- batched cone solver: replaces solve!(prg) -> JuMP.optimize! -> ECOS (program.jl:419-424) ----
 *   min c'x  s.t.  A x = b,  G x + s = h,  s in K = R+^l x SOC(q_1) x ... x SOC(q_nsoc)
 * (the standard form MathOptInterface hands to ECOS).  The sparsity pattern and the cone partition are
 * shared by the whole batch; values differ per seed.  perm (nullable) is the elimination order of
 * the n variables followed by the p equality rows (perm[k] = node eliminated k-th, variables are
 * 0..n-1, equality rows n..n+p-1); the host template supplies a stage-wise nested dissection. */
/* Host-side helper (no GPU work): a reverse Cuthill-McKee elimination order of the reduced KKT graph for callers that
 * have no stage information (the MathOptInterface shim); writes perm[n + p].  The SCP templates supply a better,
 * stage-wise order themselves. */
int32_t scpb_order_rcm(int32_t n, int32_t p, int32_t m, const int32_t *A_rowptr, const int32_t *A_colind,
                       const int32_t *G_rowptr, const int32_t *G_colind, int32_t l, int32_t nsoc,
                       const int32_t *soc_dims, int32_t *perm);

typedef struct scpb_cone_s *scpb_cone;

typedef struct {
    double feastol, abstol, reltol; /* <=0: ECOS defaults 1e-8                          */
    double delta, delta_dyn;        /* static regularisation of the KKT system: every seed starts from `delta`
                                     * (<=0: 1e-12) and is escalated x1000, up to `delta_dyn` (<=0: 1e-6), whenever a
                                     * factorisation loses its inertia to cancellation (last iterations only)  */
    int32_t maxit;                  /* <=0: 100 ("maxit" of solver_opts)                 */
    int32_t nref;                   /* <0: at most 3 iterative-refinement steps          */
    int32_t verbose;                /* accepted, ignored ("verbose" of solver_opts)      */
    int32_t group;                  /* seeds per CTA (power of two <= 8);  0 = automatic */
    int32_t equil;                  /* Ruiz equilibration passes; <0: default 5, 0: off    */
    int32_t threads;                /* threads per CTA: 1024 (default) or 512              */
    int32_t lanes;                  /* lanes per sparse row in the fallback substitution that is used when the
                                     * vector does not fit shared memory (1,2,4,8); 0: 8   */
} scpb_cone_opts;

/* per-seed status (termination_status, program.jl:427-428): */
enum { SCPB_CONE_OPTIMAL = 0, SCPB_CONE_ITERATION_LIMIT = 1, SCPB_CONE_NUMERICAL_ERROR = 2,
       SCPB_CONE_ALMOST_OPTIMAL = 3, /* best iterate meets ECOS' reduced tolerances (5e-5) */
       SCPB_CONE_INFEASIBLE = 4,      /* certificate (y, z): A'y + G'z ~ 0, b'y + h'z < 0  (MOI INFEASIBLE)          */
       SCPB_CONE_DUAL_INFEASIBLE = 5  /* certificate x: Ax ~ 0, Gx + s ~ 0, c'x < 0, i.e. unbounded (MOI DUAL_INFEASIBLE,
                                         the status compute_scaling tests for, src/solvers/scp.jl:470-473) */ };

int32_t scpb_cone_setup(scpb_handle h, int32_t n, int32_t p, int32_t m,
                        const int32_t *A_rowptr, const int32_t *A_colind,
                        const int32_t *G_rowptr, const int32_t *G_colind,
                        int32_t l, int32_t nsoc, const int32_t *soc_dims, const int32_t *perm,
                        scpb_cone *out);
/* info[24] = {n+p, nnz(L), elimination-tree levels, factor ops, assembly ops, |W^-2|, group, capacity,
 *             8 SM-cycle counters of the last launch (CTA 0): equilibrate, start point, residuals,
 *             scaling+assembly, factorisation, KKT solves, line search+update, total;
 *             forward-substitution cycles, backward-substitution cycles, number of LDL' solves,
 *             number of factorisations (= interior-point iterations of CTA 0);
 *             hybrid program: cut the last launch ran (0 = it ran the scalar / supernodal variant), scalar levels
 *             incl. the bridge level, top supernodal levels, cut it was built with (0 = not built)} */
int32_t scpb_cone_info(scpb_cone c, int64_t *info);
int32_t scpb_cone_free(scpb_cone c);
/* host arrays, seed-major: Avals[B][nnzA], Gvals[B][nnzG], c[B][n], b[B][p], h[B][m];
 * outputs x[B][n], y[B][p], z[B][m], s[B][m], pobj[B], dobj[B], status[B], iters[B] (each nullable). */
int32_t scpb_cone_solve(scpb_cone c, int32_t B, const double *Avals, const double *Gvals,
                        const double *cvec, const double *bvec, const double *hvec,
                        const scpb_cone_opts *opts, double *x, double *y, double *z, double *s,
                        double *pobj, double *dobj, int32_t *status, int32_t *iters, double *seconds);

/* ---- batched PTR loop: replaces the body of PTR.solve (src/solvers/ptr.jl:448-532) for B seeds ----
 * The host template (scptoolbox.jl_b200/ptr.py, mirror of ptr.jl:213-293,565-895 + scp.jl:657-895) supplies
 * the fill matrix W with [Avals; Gvals; c; b; h; c0] = W * src, where src is the per-seed vector of
 * device-computed quantities laid out by the offsets below (source 0 is the constant 1):
 *   oA,oBm,oBp,oF,or_,oE : DLTV blocks per segment (column-major nx*nx, nx*nu, nx*nf, nx) -- discretize!
 *                          (nf = 0 for a model with a fixed final time: the F block is empty)
 *   oC,oD,oG,ors         : ds/dx, ds/du, ds/dp (row-major; ds/dp packed to ng columns, see csrc/constraints.cuh)
 *                          and r = s - Cx - Du - Gp per node (scp.jl:763-773)
 *   oxh,ouh,oph          : scaled reference trajectory (ptr.jl:575-577)
 * vx,vu,vp are the offsets of the scaled x, u, p variable blocks inside the cone program's variables. */
typedef struct scpb_ptr_s *scpb_ptr;

typedef struct {
    int32_t N, Nsub, nx, nu, np, ns, nf;
    int32_t nsrc, oA, oBm, oBp, oF, or_, oE, oC, oD, oG, ors, oxh, ouh, oph;
    int32_t nval, vx, vu, vp;
    int32_t q_exit;          /* stopping-criterion norm: 0 = Inf, 1, 2 (pars.q_exit) */
    int32_t iter_max;
    int32_t ng;              /* packed columns of ds/dp per node (the constraint pack's NG; = np for most packs) */
    double eps_abs, eps_rel, feas_tol;
    int32_t method;          /* SCPB_FOH (0: a zero-initialised descriptor) or SCPB_IMPULSE (a model pack with impulse
                                semantics only; the fill matrix W then references no oBp source, state_update!,
                                discretization.jl:469-494).  scpb_scvx_attach / scpb_gusto_attach refuse IMPULSE. */
} scpb_ptr_desc;

/* scale = [Sx,Su,Sp | cx,cu,cp | iSx] (diagonals, scp.jl:483-516); t_grid[N]. */
int32_t scpb_ptr_setup(scpb_handle h, scpb_cone cone, const scpb_ptr_desc *desc, const int32_t *W_rowptr,
                       const int32_t *W_colind, const double *W_vals, const double *scale, const double *t_grid,
                       scpb_ptr *out);
int32_t scpb_ptr_free(scpb_ptr s);
/* Replace the model parameter block (par[npar], same layout as scpb_model_set) that the problem captured at
 * scpb_ptr_setup; the model, its dimensions and the template stay.  npar must lie between the length of the block given
 * to scpb_model_set before setup and SCPB_MAX_PAR (SCPB_ERR_ARG otherwise): a shorter block would zero trailing entries.  Later solves use the new block,
 * e.g. the next step of a homotopy on a constraint-pack parameter (the reference sets mdl.traj.kappa between two
 * PTR.solve calls on one problem, test/examples/rendezvous_planar/tests.jl:66-78). */
int32_t scpb_ptr_set_par(scpb_ptr s, const double *par, int32_t npar);
/* In-loop homotopy schedule (PTR only): the device twin of a problem_set_callback! that steps a constraint-pack parameter
 * kappa through a grid inside ONE solve (test/examples/rendezvous_3d/definition.jl:96-151, called at ptr.jl:496-506).
 * Every seed keeps its own grid index, kappa, last_update, effective iter_max and update threshold beta.  Right after the
 * stopping rule of iteration `iter`, a seed whose subproblem solved safely updates when
 *   beta >= improv_rel >= worsen_tol  and  its grid index < n_grid - 1   (false for a NaN improv_rel, as at iteration 1):
 * kappa takes the next grid value, iter_max grows by iter - last_update, last_update = iter, and a stop the stopping rule
 * asked for in that iteration is cancelled.  A seed ends with status 1 once iter >= its own iter_max.  Every solve starts
 * every seed from grid[0], last_update = 1 and the descriptor's iter_max (the reference carries the mutated iter_max and
 * kappa over to the next PTR.create on the same parameters).
 * scpb_ptr_set_homotopy attaches the schedule to the homotopy parameter of the problem's constraint pack, which reads it
 * from par[par_index] (the rendezvous pack's kappa, par[7]); par_index = -1 takes the pack's own slot, any other value
 * must name it.  SCPB_ERR_UNSUPPORTED for a pack without a homotopy parameter.  n_grid = 0 detaches the schedule; an
 * unchanged grid is not uploaded again.  A problem with a schedule refuses scpb_scvx_attach / scpb_gusto_attach and
 * vice versa.  Streamed chains (SCPB_PTR_CHUNKS > 1) do not pay off with a schedule: the host polls every chain's
 * progress (one core busy for the whole solve), and on the planar rendezvous beta sweep they ran at about half the
 * lock-step rate.
 * scpb_ptr_set_homotopy_beta sets beta[B] for the next solves, which must have B seeds.
 * scpb_ptr_homotopy_result (after a solve with a schedule, same B): the final grid index hom_index[B], the effective
 * iter_max_eff[B], and per iteration the grid index the subproblem was built with, hist_index[B][cap], and its
 * improv_rel, hist_improv[B][cap]; -1 / NaN after a seed's last iteration.  A seed runs at most
 * iter_max + (n_grid - 1)(iter_max - 1) iterations, so that many columns hold its whole history.  Every pointer is
 * nullable. */
int32_t scpb_ptr_set_homotopy(scpb_ptr s, int32_t par_index, int32_t n_grid, const double *grid, double worsen_tol);
int32_t scpb_ptr_set_homotopy_beta(scpb_ptr s, int32_t B, const double *beta);
int32_t scpb_ptr_homotopy_result(scpb_ptr s, int32_t B, int32_t *hom_index, int32_t *iter_max_eff, int32_t cap,
                                 int32_t *hist_index, double *hist_improv);
/* host arrays: initial guesses xd0[B][N][nx], ud0[B][N][nu], p0[B][np]; outputs the final iterates, per-seed
 * status (0 = stopping criterion met, 1 = iter_max reached [the reference still reports SCP_SOLVED],
 * 2+16*cone_status = SCP_FAILED), iteration counts, J_aug, deviation, dynamic feasibility flags and
 * timing[10] = {discretize, formulate, solve, overhead, total seconds, longest PTR chain (iterations),
 * interior-point iterations summed over seeds and subproblems, number of seed chunks, seconds of the initial
 * full-batch discretize!, 0}.  By default (SCPB_PTR_CHUNKS unset, 0 or 1) one lock-step loop runs over the whole batch.
 * SCPB_PTR_CHUNKS=<n> cuts the batch into n chunks of whole seed groups and every chunk runs its own sequence of PTR
 * iterations on its own CUDA stream (seeds are independent): the four phase times are then those of chunk 0's chain,
 * the total is the whole call. */
int32_t scpb_ptr_solve(scpb_ptr s, int32_t B, const double *xd0, const double *ud0, const double *p0,
                       const scpb_cone_opts *opts, double *xd, double *ud, double *p, int32_t *status,
                       int32_t *iters, double *J, double *deviation, int32_t *feas, double *timing);

/* ---- batched SCvx loop: replaces the body of SCvx.solve (src/solvers/scvx.jl:460-546) for B seeds ----
 * Same template machinery as PTR: scpb_ptr_setup with the SCvx flavour of the subproblem (scptoolbox.jl_b200/scvx.py,
 * mirror of scvx.jl:225-303, 578-701, 804-901): no trust-region variables, the radius eta is the per-seed source
 * `oeta`.  scpb_scvx_attach adds what the ratio test needs: the algorithm constants (scvx.jl:57-81) and the sparse
 * rows Q (over the scaled solver variables of the x, u, p blocks, constants Q_const) of
 *   row 0: original cost L(x,u,p);  rows 1..n_ic: g_ic(x_1,p);  rows n_ic+1..n_ic+n_tc: g_tc(x_N,p)
 * which, with the defects of discretize! and the constraint pack's s, give the nonlinear augmented cost
 * (actual_cost_penalty!, scvx.jl:919-951).  That cost has the penalty of the starship's constraint pack only:
 * scpb_scvx_attach refuses a problem with another pack (SCPB_ERR_UNSUPPORTED).  scpb_scvx_solve returns what
 * SCPSolution keeps of the last subproblem (scp.jl:205-236): trajectory, status (0/1 solved, 2+16*cone status failed),
 * iterations, J_aug, deviation, feas, and the final trust-region radius per seed. */
typedef struct {
    double lam, rho_0, rho_1, rho_2, beta_sh, beta_gr, eta_init, eta_lb, eta_ub;
    int32_t oeta, n_ic, n_tc, reserved;
} scpb_scvx_desc;
int32_t scpb_scvx_attach(scpb_ptr ptr, const scpb_scvx_desc *desc, const int32_t *Q_rowptr, const int32_t *Q_colind,
                         const double *Q_vals, const double *Q_const);
int32_t scpb_scvx_solve(scpb_ptr ptr, int32_t B, const double *xd0, const double *ud0, const double *p0,
                        const scpb_cone_opts *opts, double *xd, double *ud, double *p, int32_t *status,
                        int32_t *iters, double *J, double *deviation, int32_t *feas, double *eta, double *timing);

/* ---- batched GuSTO loop: replaces the body of GuSTO.solve (src/solvers/gusto.jl:425-502, pen = :quad) for B seeds ----
 * Same template machinery: scpb_ptr_setup with the GuSTO flavour of the subproblem (scptoolbox.jl_b200/gusto.py, mirror of
 * gusto.jl:218-287, 534-1190): dynamics and boundary conditions un-relaxed, the nonconvex path constraints and the trust
 * region enter through quadratic soft penalties lambda max(0, .)^2 -- epigraphs q >= v^2 as rotated second-order cones,
 * lambda as a cost coefficient, so the cone entries stay O(1) whatever lambda is -- with the
 * per-seed sources `oeta` (trust-region radius eta) and `olam` (the penalty weight lambda).  scpb_gusto_attach adds the algorithm
 * constants (gusto.jl:58-85) and the sparse rows Q over the scaled solver variables (constants Q_const):
 *   row 0            affine part of the original cost J(x,u,p)            (x, u, p blocks only)
 *   rows 1..nsq      rows r_j whose weighted squares complete it: J = row0 + sum_j Q_weight[j-1] r_j^2   (x, u, p only)
 *   row nsq+1        L_tr / lambda, the soft trust-region cost as the subproblem measures it (any solver variable)
 * With the dynamics / constraint packs these give, per iteration and seed, J, J_st, J_tr, J_aug of the new iterate
 * (gusto.jl:399-418), the convexification error rho (update_trust_region!, :1245-1293), the update rule for the
 * reference, eta and lambda (update_rule!, :1310-1427, incl. the mu-shrink of :268) and the stopping rule (:1203-1231).
 * scpb_gusto_solve returns what SCPSolution keeps of the LAST subproblem (scp.jl:205-236): trajectory, status
 * (0/1 solved, 2+16*cone status failed), iterations, cost = J_aug, deviation, feas, and the final eta and lambda. */
typedef struct {
    double lam_init, lam_max, rho_0, rho_1, beta_sh, beta_gr, gamma_fail, eta_init, eta_lb, eta_ub, mu;
    int32_t iter_mu, q_tr /* 0 = Inf, 1, 2 */, oeta, olam, nsq, reserved;
} scpb_gusto_desc;
int32_t scpb_gusto_attach(scpb_ptr ptr, const scpb_gusto_desc *desc, const int32_t *Q_rowptr, const int32_t *Q_colind,
                          const double *Q_vals, const double *Q_const, const double *Q_weight);
int32_t scpb_gusto_solve(scpb_ptr ptr, int32_t B, const double *xd0, const double *ud0, const double *p0,
                         const scpb_cone_opts *opts, double *xd, double *ud, double *p, int32_t *status,
                         int32_t *iters, double *J, double *deviation, int32_t *feas, double *eta, double *lam,
                         double *timing);

/* Measured fp64 FMA throughput of the handle's device in TFLOP/s (a register-resident FMA microkernel, best of 3
 * timed launches): the denominator of the discretization kernel's roofline in bench.py. */
int32_t scpb_debug_fp64_peak(scpb_handle h, double *tflops);

/* Test hook: the nonconvex-constraint pack of the selected model (scpb_model_set) evaluated on the device at every seed
 * and node, as the PTR loop's linearisation evaluates it: t_grid[N], xd[B][N][nx], ud[B][N][nu], p[B][np] -> s[B][N][ns],
 * C[B][N][ns*nx], D[B][N][ns*nu], G[B][N][ns*ng] (row-major; G packed, see scpb_ptr_desc.ng).  ns / ng must be the pack's. */
int32_t scpb_debug_constraints(scpb_handle h, int32_t B, int32_t N, int32_t ns, int32_t ng, const double *t_grid,
                               const double *xd, const double *ud, const double *p, double *s, double *C, double *D,
                               double *G);

/* Diagnostic: per-level cycle counters of CTA 0 in the last scpb_cone_solve / scpb_ptr_solve launch, recorded
 * only when the environment variable SCPB_LEVEL_PROFILE is set: out[0..L) numeric factorisation, out[L..2L)
 * forward substitution, out[2L..3L) backward substitution (L = info[2] levels); cap >= 3L. */
int32_t scpb_debug_level_profile(scpb_cone cone, int64_t *out, int32_t cap);

/* Diagnostic: with the environment variable SCPB_IPM_TRACE=<seed index> set, the last scpb_cone_solve / scpb_*_solve
 * launch records for that seed one row per interior-point iteration: {iteration, primal residual, dual residual, gap,
 * primal cost, dual cost, previous primal step, previous dual step, static regularisation, sigma*mu}.  Copies up to
 * cap_rows rows of 10 doubles into out; returns the number of rows copied (>= 0) or a negative error code. */
int32_t scpb_debug_ipm_trace(scpb_cone cone, double *out, int32_t cap_rows);

/* ---- test hook: CPU interpreter of the solver's index programs for ONE seed (no GPU needed) ----
 * Assembles M = [dI + G'W^-2 G, A'; A, -dI] from (Av, Gv, wm), factors it with the level-scheduled
 * LDL' program and solves M sol = rhs (natural node order: n variables then p equality rows).
 * Used by the CPU test-suite only; never called by the product path.
 * info[4] = {nnz(L), levels, factor ops, assembly ops}. */
int32_t scpb_debug_kkt_solve(int32_t n, int32_t p, int32_t m, const int32_t *A_rowptr, const int32_t *A_colind,
                             const int32_t *G_rowptr, const int32_t *G_colind, int32_t l, int32_t nsoc,
                             const int32_t *soc_dims, const int32_t *perm, const double *Avals,
                             const double *Gvals, const double *wm, double delta, double delta_dyn,
                             const double *rhs, double *sol, int64_t *info);
/* The same hook for the supernodal program (dense panels, one barrier per supernodal level) that the next kernel
 * generation executes; info[8] = {supernodes, supernodal levels, panel doubles per seed, update scatter entries,
 * max width, max panel rows, scalar levels, nnz(L)}.  The kernels of csrc/conic_sn.cuh execute this program. */
int32_t scpb_debug_kkt_solve_sn(int32_t n, int32_t p, int32_t m, const int32_t *A_rowptr, const int32_t *A_colind,
                             const int32_t *G_rowptr, const int32_t *G_colind, int32_t l, int32_t nsoc,
                             const int32_t *soc_dims, const int32_t *perm, const double *Avals,
                             const double *Gvals, const double *wm, double delta, double delta_dyn,
                             const double *rhs, double *sol, int64_t *info);
/* The same hook for the hybrid program (scalar level-scheduled programs below supernodal level `cut`, register-resident
 * panels addressed in place on the scalar storage above it; SCPB_HYBRID selects it in the solver kernel): info[8] =
 * {scalar levels incl. the bridge level, top supernodal levels, top supernodes, top columns, bridge factor items, bridge
 * factor ops, bridge forward items, scalar levels of the plain program}.  SCPB_ERR_UNSUPPORTED when the split is empty. */
int32_t scpb_debug_kkt_solve_hy(int32_t n, int32_t p, int32_t m, const int32_t *A_rowptr, const int32_t *A_colind,
                             const int32_t *G_rowptr, const int32_t *G_colind, int32_t l, int32_t nsoc,
                             const int32_t *soc_dims, const int32_t *perm, const double *Avals,
                             const double *Gvals, const double *wm, double delta, double delta_dyn, int32_t cut,
                             const double *rhs, double *sol, int64_t *info);
/* The same single KKT solve executed ON THE DEVICE by the code path of the solver kernel (supernodal panels, or the
 * scalar programs with SCPB_SUPERNODAL=0) for B seeds: Avals[B][nnzA], Gvals[B][nnzG], wm[B][|W^-2|] (LP rows one
 * weight, SOC cones dense q x q blocks), rhs / sol [B][n+p] in natural node order; bad[B] (nullable) = 1 when the
 * factorisation flagged lost inertia.  GPU tests compare it with scpb_debug_kkt_solve. */
int32_t scpb_debug_kkt_solve_dev(scpb_cone cone, int32_t B, const double *Avals, const double *Gvals, const double *wm,
                                 double delta, const double *rhs, double *sol, int32_t *bad);
/* Stateful variant of the scalar interpreter for numerics studies on the CPU: symbolic analysis
 * once (scpb_debug_kkt_new), then any number of factorisations and solves.  scpb_debug_kkt_factor applies the kernel's
 * dynamic regularisation (a pivot with sgn*d <= tau becomes sgn*rho) and returns the number of rejected pivots that
 * were NOT small (|d| > bad_abs or non-finite: the inertia was lost to cancellation), or a negative error code;
 * stats[3] = {regularised pivots, max |L|, min |D|}.  info[4] = {nnz(L), levels, factor ops, supernodal levels}. */
int32_t scpb_debug_kkt_new(int32_t n, int32_t p, int32_t m, const int32_t *A_rowptr, const int32_t *A_colind,
                           const int32_t *G_rowptr, const int32_t *G_colind, int32_t l, int32_t nsoc,
                           const int32_t *soc_dims, const int32_t *perm, void **out, int64_t *info);
int32_t scpb_debug_kkt_factor(void *kkt, const double *Avals, const double *Gvals, const double *wm, double delta,
                              double tau, double rho, double bad_abs, double *stats);
int32_t scpb_debug_kkt_resolve(void *kkt, const double *rhs, double *sol);
int32_t scpb_debug_kkt_free(void *kkt);

#ifdef __cplusplus
}
#endif
#endif

// conic_debug.cu -- host-side interpreter of the gather programs built by conic_symbolic.h.
// TEST HOOK ONLY: it executes the assembly / factorisation / substitution programs for ONE seed on
// the CPU so that the index programs can be unit-tested without a GPU (tests/test_conic_symbolic.py).
// It is not reachable from any product entry point (scpb_cone_solve always launches k_ipm_solve).
#include "../../include/scpb.h"
#include "conic_symbolic.h"

// Partial sums of split targets, applied the way k_ipm_solve applies them (conic_symbolic.h: number_pieces,
// combine_in_phase_b); slots are numbered from 0 in every level.
// Substitutions, add(): an item of a split target (.w = 1 + index into info) stores its sum in its slot, and the last
// item of the target subtracts the target's slots in slot order.  add() fails when the info entry belongs to another
// target or its slot lies outside the target's range; level_done() fails when a target of the level did not receive
// all the items its slot range promises.
// Factorisation, store() / take(): phase A stores an item's sum in slot .w - 1, phase B subtracts the slot ranges of
// fb_cmb.  take() fails when a range holds a slot that this level's phase A did not store for that target;
// level_done() fails when a stored slot was not taken exactly once as the entry of a phase-B item.
struct SplitSums {
    std::vector<double> part;
    std::vector<int> cnt, tgt, taken;
    explicit SplitSums(int nslot) : part((size_t)nslot, 0.0), cnt((size_t)nslot, 0), tgt((size_t)nslot, -1), taken((size_t)nslot, 0) {}
    bool add(const int *it, const std::vector<int> &info, double p, double *y)
    {
        if (!it[3]) { y[it[0]] -= p; return true; }
        const size_t q = (size_t)it[3] - 1;
        if (it[3] < 1 || 4 * q + 3 >= info.size()) return false;
        const int *e = &info[4 * q];
        const int sl = e[3];
        if (e[0] != it[0] || e[1] < 0 || e[2] > (int)part.size() || sl < e[1] || sl >= e[2]) return false;
        part[sl] = p;
        if (++cnt[e[1]] == e[2] - e[1]) {
            double acc = y[e[0]];
            for (int k = e[1]; k < e[2]; k++) acc -= part[k];
            y[e[0]] = acc;
            cnt[e[1]] = 0;
        }
        return true;
    }
    bool store(const int *it, double p, double *y)
    {
        if (!it[3]) { y[it[0]] -= p; return true; }
        const int sl = it[3] - 1;
        if (sl < 0 || sl >= (int)part.size() || tgt[sl] >= 0) return false;
        part[sl] = p; tgt[sl] = it[0];
        return true;
    }
    bool take(int t, int s0, int s1, double &acc, bool entry)
    {
        for (int k = s0; k < s1; k++) {
            if (k < 0 || k >= (int)part.size() || tgt[k] != t) return false;
            acc -= part[k];
            taken[k] += entry;
        }
        return true;
    }
    bool level_done()
    {
        bool ok = true;
        for (size_t k = 0; k < cnt.size(); k++) {
            if (cnt[k] || (tgt[k] >= 0 && taken[k] != 1)) ok = false;
            tgt[k] = -1; taken[k] = 0;
        }
        return ok;
    }
};

// Phase B's operands of a factorisation item: its entry and the pivot of its column, each minus the slots of its split
// target.  The entry is written back, because later levels read it; the pivot is not, because the other items of the
// column read it in the same phase (the diagonal item keeps the combined pivot in e).
static bool phase_b_operands(SplitSums &split, const int *it, const int *cm, int nnzL, std::vector<double> &Y, double &e, double &d)
{
    e = Y[it[0]];
    if (!split.take(it[0], cm[0], cm[1], e, true)) return false;
    if (it[3] & 2) { d = e; return true; }
    d = Y[(size_t)nnzL + it[1]];
    if (!split.take(nnzL + it[1], cm[2], cm[3], d, false)) return false;
    Y[it[0]] = e;
    return true;
}

extern "C" int32_t scpb_debug_kkt_solve(int32_t n, int32_t p, int32_t m, const int32_t *A_rp, const int32_t *A_ci,
                                        const int32_t *G_rp, const int32_t *G_ci, int32_t l, int32_t nsoc,
                                        const int32_t *soc_dims, const int32_t *perm, const double *Av,
                                        const double *Gv, const double *wm, double delta, double delta_dyn,
                                        const double *rhs, double *sol, int64_t *info)
{
    ConeSymbolic S;
    static const int zero = 0;
    if (!cone_symbolic_build(S, n, p, m, A_rp, A_ci ? A_ci : &zero, G_rp, G_ci ? G_ci : &zero, l, nsoc, soc_dims, perm))
        return SCPB_ERR_ARG;
    const int nk = S.nk, ntgt = S.nnzL + nk;
    std::vector<double> Y(ntgt), Ls(S.nnzL + 1), invD(nk), v(nk);
    for (int t = 0; t < ntgt; t++) {  // kkt_assemble
        double acc = delta * S.as_sign[t];
        if (S.as_src[t] >= 0) acc += Av[S.as_src[t]];
        for (int k = S.as_ptr[t]; k < S.as_ptr[t + 1]; k++) acc += Gv[S.as_a[k]] * Gv[S.as_b[k]] * wm[S.as_c[k]];
        Y[t] = acc;
    }
    SplitSums split(S.npart);
    int64_t nsplit = 0;
    for (int lv = 0; lv < S.nlevels; lv++) {  // kkt_factor: balanced program (phase A items, then phase B items)
        const int R = S.fa_R[lv];
        for (int w = S.fa_lvl[lv]; w < S.fa_lvl[lv + 1]; w++) {
            const int *it = &S.fa_item[4 * (size_t)w];
            if (it[2] - it[1] > R * CONIC_FACTOR_PF) return SCPB_ERR_ARG;
            double part = 0.0;
            for (int k = it[1]; k < it[2]; k++) part += Y[S.ft_op[2 * (size_t)k]] * Ls[S.Lr_pos[S.ft_op[2 * (size_t)k + 1]]];
            if (!split.store(it, part, Y.data())) return SCPB_ERR_ARG;
            nsplit += it[3] != 0;
        }
        for (int w = S.fb_lvl[lv]; w < S.fb_lvl[lv + 1]; w++) {   // every item regularises its own copy of the pivot
            const int *it = &S.fb_item[4 * (size_t)w];
            double e, d;
            if (!phase_b_operands(split, it, &S.fb_cmb[4 * (size_t)w], S.nnzL, Y, e, d)) return SCPB_ERR_ARG;
            const double sgn = (it[3] & 1) ? 1.0 : -1.0;
            if (!(sgn * d > delta_dyn)) d = sgn * delta_dyn;
            if (it[3] & 2) invD[it[1]] = 1.0 / d;
            else Ls[it[0]] = e * (1.0 / d);
        }
        if (!split.level_done()) return SCPB_ERR_ARG;
    }
    for (int i = 0; i < nk; i++) v[S.iperm[i]] = rhs[i];
    // kkt_ldl_solve_smem: the balanced (split-item) substitution programs, level by level; within a level every
    // item reads v as it was when the level started, except for the target it accumulates into
    std::vector<double> Lrow(S.nnzL + 1);
    for (int k = 0; k < S.nnzL; k++) Lrow[k] = Ls[S.Lr_pos[k]];
    for (int lv = 0; lv < S.nlevels; lv++) {
        const int R = S.fwp_R[lv];
        for (int w = S.fwp_lvl[lv]; w < S.fwp_lvl[lv + 1]; w++) {
            const int *it = &S.fwp_item[4 * (size_t)w];
            if (it[2] - it[1] > R * CONIC_SOLVE_PF) return SCPB_ERR_ARG;
            double part = 0.0;
            for (int k = it[1]; k < it[2]; k++) part += Lrow[k] * v[S.Lr_col[k]];
            if (!split.add(it, S.fwc_item, part, v.data())) return SCPB_ERR_ARG;
            nsplit += it[3] != 0;
        }
        if (!split.level_done()) return SCPB_ERR_ARG;
    }
    for (int i = 0; i < nk; i++) v[i] *= invD[i];
    for (int lv = S.nlevels - 1; lv >= 0; lv--) {
        const int R = S.bwp_R[lv];
        for (int w = S.bwp_lvl[lv]; w < S.bwp_lvl[lv + 1]; w++) {
            const int *it = &S.bwp_item[4 * (size_t)w];
            if (it[2] - it[1] > R * CONIC_SOLVE_PF) return SCPB_ERR_ARG;
            double part = 0.0;
            for (int k = it[1]; k < it[2]; k++) part += Ls[k] * v[S.L_ri[k]];
            if (!split.add(it, S.bwc_item, part, v.data())) return SCPB_ERR_ARG;
            nsplit += it[3] != 0;
        }
        if (!split.level_done()) return SCPB_ERR_ARG;
    }
    for (int i = 0; i < nk; i++) sol[i] = v[S.iperm[i]];
    if (info) { info[0] = S.nnzL; info[1] = S.nlevels; info[2] = S.factor_ops; info[3] = (int64_t)S.as_a.size(); info[4] = nsplit; }
    return SCPB_OK;
}

// Same test hook for the SUPERNODAL program (conic_symbolic.h, "supernodal program"): dense panels, one supernodal
// level at a time, right-looking updates scattered through the precomputed maps.  This is the executable specification
// of the round-2 device kernels; nothing on the product path calls it.
extern "C" int32_t scpb_debug_kkt_solve_sn(int32_t n, int32_t p, int32_t m, const int32_t *A_rp, const int32_t *A_ci,
                                           const int32_t *G_rp, const int32_t *G_ci, int32_t l, int32_t nsoc,
                                           const int32_t *soc_dims, const int32_t *perm, const double *Av,
                                           const double *Gv, const double *wm, double delta, double delta_dyn,
                                           const double *rhs, double *sol, int64_t *info)
{
    ConeSymbolic S;
    static const int zero = 0;
    if (!cone_symbolic_build(S, n, p, m, A_rp, A_ci ? A_ci : &zero, G_rp, G_ci ? G_ci : &zero, l, nsoc, soc_dims, perm))
        return SCPB_ERR_ARG;
    const int nk = S.nk, ntgt = S.nnzL + nk, ns = (int)S.sn_first.size();
    std::vector<double> P((size_t)S.sn_panel_size, 0.0), invD(nk), v(nk);
    for (int t = 0; t < ntgt; t++) {  // assembly straight into the panels
        double acc = delta * S.as_sign[t];
        if (S.as_src[t] >= 0) acc += Av[S.as_src[t]];
        for (int k = S.as_ptr[t]; k < S.as_ptr[t + 1]; k++) acc += Gv[S.as_a[k]] * Gv[S.as_b[k]] * wm[S.as_c[k]];
        P[(size_t)S.sn_pos_of_target[t]] = acc;
    }
    for (int lv = 0; lv < S.sn_nlevels; lv++)
        for (int w_ = S.sn_lvl_ptr[lv]; w_ < S.sn_lvl_ptr[lv + 1]; w_++) {
            const int s = S.sn_lvl_nodes[w_], a = S.sn_first[s], w = S.sn_width[s], R = S.sn_nrows[s];
            double *Q = &P[(size_t)S.sn_panel_off[s]];
            for (int c = 0; c < w; c++) {   // dense LDL' of the panel, right-looking inside the supernode
                double d = Q[c + (size_t)R * c];
                const double sgn = (double)S.as_sign[S.nnzL + a + c];
                if (!(sgn * d > delta_dyn)) d = sgn * delta_dyn;
                Q[c + (size_t)R * c] = d;
                invD[a + c] = 1.0 / d;
                for (int r = c + 1; r < R; r++) Q[r + (size_t)R * c] /= d;
                for (int c2 = c + 1; c2 < w; c2++) {
                    const double f = Q[c2 + (size_t)R * c] * d;
                    for (int r = c2; r < R; r++) Q[r + (size_t)R * c2] -= Q[r + (size_t)R * c] * f;
                }
            }
            int k = S.sn_upd_ptr[s];   // Schur update of the ancestors' panels
            for (int y = 0; y < R - w; y++)
                for (int x = y; x < R - w; x++) {
                    double u = 0.0;
                    for (int c = 0; c < w; c++) u += Q[w + x + (size_t)R * c] * Q[c + (size_t)R * c] * Q[w + y + (size_t)R * c];
                    P[(size_t)S.sn_upd_dst[k++]] -= u;
                }
        }
    for (int i = 0; i < nk; i++) v[S.iperm[i]] = rhs[i];
    for (int lv = 0; lv < S.sn_nlevels; lv++)   // forward: column oriented, updates scattered to the rows below
        for (int w_ = S.sn_lvl_ptr[lv]; w_ < S.sn_lvl_ptr[lv + 1]; w_++) {
            const int s = S.sn_lvl_nodes[w_], w = S.sn_width[s], R = S.sn_nrows[s];
            const double *Q = &P[(size_t)S.sn_panel_off[s]];
            const int *rows = &S.sn_rows[S.sn_rows_ptr[s]];
            for (int c = 0; c < w; c++) {
                const double xc = v[rows[c]];
                for (int r = c + 1; r < R; r++) v[rows[r]] -= Q[r + (size_t)R * c] * xc;
            }
        }
    for (int i = 0; i < nk; i++) v[i] *= invD[i];
    for (int lv = S.sn_nlevels - 1; lv >= 0; lv--)   // backward: gathers from the rows below
        for (int w_ = S.sn_lvl_ptr[lv]; w_ < S.sn_lvl_ptr[lv + 1]; w_++) {
            const int s = S.sn_lvl_nodes[w_], w = S.sn_width[s], R = S.sn_nrows[s];
            const double *Q = &P[(size_t)S.sn_panel_off[s]];
            const int *rows = &S.sn_rows[S.sn_rows_ptr[s]];
            for (int c = w - 1; c >= 0; c--) {
                double acc = v[rows[c]];
                for (int r = c + 1; r < R; r++) acc -= Q[r + (size_t)R * c] * v[rows[r]];
                v[rows[c]] = acc;
            }
        }
    for (int i = 0; i < nk; i++) sol[i] = v[S.iperm[i]];
    if (info) {
        info[0] = ns; info[1] = S.sn_nlevels; info[2] = S.sn_panel_size; info[3] = (int64_t)S.sn_upd_dst.size();
        int wmax = 0, rmax = 0;
        for (int s = 0; s < ns; s++) { wmax = std::max(wmax, S.sn_width[s]); rmax = std::max(rmax, S.sn_nrows[s]); }
        info[4] = wmax; info[5] = rmax; info[6] = S.nlevels; info[7] = S.nnzL;
    }
    (void)ns;
    return SCPB_OK;
}

// Same test hook for the HYBRID program (cone_symbolic_build_hybrid): scalar level-scheduled programs for the low
// columns, one bridge level, then the top supernodes as dense panels addressed in place on the scalar storage -- the
// executable specification of kkt_factor_top / kkt_sweep_top (conic_ipm.cuh).  info[8] = {scalar levels incl. bridge,
// top supernodal levels, top supernodes, top columns, bridge factor items, bridge factor ops, bridge forward items,
// scalar levels of the plain program}.
extern "C" int32_t scpb_debug_kkt_solve_hy(int32_t n, int32_t p, int32_t m, const int32_t *A_rp, const int32_t *A_ci,
                                           const int32_t *G_rp, const int32_t *G_ci, int32_t l, int32_t nsoc,
                                           const int32_t *soc_dims, const int32_t *perm, const double *Av,
                                           const double *Gv, const double *wm, double delta, double delta_dyn,
                                           int32_t cut, const double *rhs, double *sol, int64_t *info)
{
    ConeSymbolic S;
    static const int zero = 0;
    if (!cone_symbolic_build(S, n, p, m, A_rp, A_ci ? A_ci : &zero, G_rp, G_ci ? G_ci : &zero, l, nsoc, soc_dims, perm))
        return SCPB_ERR_ARG;
    if (!cone_symbolic_build_hybrid(S, cut)) return SCPB_ERR_UNSUPPORTED;
    const int nk = S.nk, ntgt = S.nnzL + nk, nl = S.hy_nlevels;
    std::vector<double> Y(ntgt), Ls(S.nnzL + 1), invD(nk), v(nk);
    for (int t = 0; t < ntgt; t++) {  // kkt_assemble
        double acc = delta * S.as_sign[t];
        if (S.as_src[t] >= 0) acc += Av[S.as_src[t]];
        for (int k = S.as_ptr[t]; k < S.as_ptr[t + 1]; k++) acc += Gv[S.as_a[k]] * Gv[S.as_b[k]] * wm[S.as_c[k]];
        Y[t] = acc;
    }
    SplitSums split(S.npart);
    for (int lv = 0; lv < nl; lv++) {  // low columns + bridge level: the scalar balanced programs
        const int R = S.hy_fa_R[lv];
        for (int w = S.hy_fa_lvl[lv]; w < S.hy_fa_lvl[lv + 1]; w++) {
            const int *it = &S.hy_fa_item[4 * (size_t)w];
            if (it[2] - it[1] > R * CONIC_FACTOR_PF) return SCPB_ERR_ARG;
            double part = 0.0;
            for (int k = it[1]; k < it[2]; k++) part += Y[S.hy_ft_op[2 * (size_t)k]] * Ls[S.Lr_pos[S.hy_ft_op[2 * (size_t)k + 1]]];
            if (!split.store(it, part, Y.data())) return SCPB_ERR_ARG;
        }
        for (int w = S.hy_fb_lvl[lv]; w < S.hy_fb_lvl[lv + 1]; w++) {
            const int *it = &S.hy_fb_item[4 * (size_t)w];
            double e, d;
            if (!phase_b_operands(split, it, &S.hy_fb_cmb[4 * (size_t)w], S.nnzL, Y, e, d)) return SCPB_ERR_ARG;
            if (it[3] & 4) continue;   // combine-only item of the bridge level: the top panels finish the target
            const double sgn = (it[3] & 1) ? 1.0 : -1.0;
            if (!(sgn * d > delta_dyn)) d = sgn * delta_dyn;
            if (it[3] & 2) invD[it[1]] = 1.0 / d;
            else Ls[it[0]] = e * (1.0 / d);
        }
        if (!split.level_done()) return SCPB_ERR_ARG;
    }
    // panel entry (r, c) of a top supernode, r >= c, as a target id / L position
    auto ppos = [&](const int *d, int r, int c) { return r == c ? S.nnzL + d[0] + c : d[3] + c * (d[2] - 1) - (c * (c - 1)) / 2 + (r - c - 1); };
    for (int tl = 0; tl < S.hy_ntl; tl++)   // top supernodes: dense LDL' of the panel, Schur complement scattered to the ancestors
        for (int q = S.hy_tl_ptr[tl]; q < S.hy_tl_ptr[tl + 1]; q++) {
            const int *d = &S.hy_desc[8 * (size_t)q];
            const int w = d[1], R = d[2];
            std::vector<double> Q((size_t)R * w, 0.0), dd(w);
            for (int c = 0; c < w; c++)
                for (int r = c; r < R; r++) Q[r + (size_t)R * c] = Y[ppos(d, r, c)];
            for (int c = 0; c < w; c++) {
                double piv = Q[c + (size_t)R * c];
                const double sgn = ((d[6] >> c) & 1) ? 1.0 : -1.0;
                if (!(sgn * piv > delta_dyn)) piv = sgn * delta_dyn;
                dd[c] = piv;
                invD[d[0] + c] = 1.0 / piv;
                for (int r = c + 1; r < R; r++) Q[r + (size_t)R * c] /= piv;
                for (int c2 = c + 1; c2 < w; c2++) {
                    const double f = Q[c2 + (size_t)R * c] * piv;
                    for (int r = c2; r < R; r++) Q[r + (size_t)R * c2] -= Q[r + (size_t)R * c] * f;
                }
            }
            for (int c = 0; c < w; c++)
                for (int r = c + 1; r < R; r++) Ls[ppos(d, r, c)] = Q[r + (size_t)R * c];
            int k = d[5];
            for (int y = 0; y < R - w; y++)
                for (int x = y; x < R - w; x++) {
                    double u = 0.0;
                    for (int c = 0; c < w; c++) u += Q[w + x + (size_t)R * c] * dd[c] * Q[w + y + (size_t)R * c];
                    Y[S.hy_upd_dst[k++]] -= u;
                }
        }
    for (int i = 0; i < nk; i++) v[S.iperm[i]] = rhs[i];
    std::vector<double> Lrow(S.nnzL + 1);
    for (int k = 0; k < S.nnzL; k++) Lrow[k] = Ls[S.Lr_pos[k]];
    for (int lv = 0; lv < nl; lv++) {   // forward: low rows level by level, then the bridge level (top rows, low columns)
        const int R = S.hy_fwp_R[lv];
        for (int w = S.hy_fwp_lvl[lv]; w < S.hy_fwp_lvl[lv + 1]; w++) {
            const int *it = &S.hy_fwp_item[4 * (size_t)w];
            if (it[2] - it[1] > R * CONIC_SOLVE_PF) return SCPB_ERR_ARG;
            double part = 0.0;
            for (int k = it[1]; k < it[2]; k++) part += Lrow[k] * v[S.Lr_col[k]];
            if (!split.add(it, S.hy_fwc_item, part, v.data())) return SCPB_ERR_ARG;
        }
        if (!split.level_done()) return SCPB_ERR_ARG;
    }
    for (int tl = 0; tl < S.hy_ntl; tl++)   // forward through the top panels (column oriented)
        for (int q = S.hy_tl_ptr[tl]; q < S.hy_tl_ptr[tl + 1]; q++) {
            const int *d = &S.hy_desc[8 * (size_t)q];
            const int w = d[1], R = d[2];
            const int *rows = &S.sn_rows[d[4]];
            for (int c = 0; c < w; c++) {
                const double xc = v[rows[c]];
                for (int r = c + 1; r < R; r++) v[rows[r]] -= Ls[ppos(d, r, c)] * xc;
            }
        }
    for (int i = 0; i < nk; i++) v[i] *= invD[i];
    for (int tl = S.hy_ntl - 1; tl >= 0; tl--)   // backward through the top panels
        for (int q = S.hy_tl_ptr[tl]; q < S.hy_tl_ptr[tl + 1]; q++) {
            const int *d = &S.hy_desc[8 * (size_t)q];
            const int w = d[1], R = d[2];
            const int *rows = &S.sn_rows[d[4]];
            for (int c = w - 1; c >= 0; c--) {
                double acc = v[rows[c]];
                for (int r = c + 1; r < R; r++) acc -= Ls[ppos(d, r, c)] * v[rows[r]];
                v[rows[c]] = acc;
            }
        }
    for (int lv = nl - 1; lv >= 0; lv--) {   // backward: low columns
        const int R = S.hy_bwp_R[lv];
        for (int w = S.hy_bwp_lvl[lv]; w < S.hy_bwp_lvl[lv + 1]; w++) {
            const int *it = &S.hy_bwp_item[4 * (size_t)w];
            if (it[2] - it[1] > R * CONIC_SOLVE_PF) return SCPB_ERR_ARG;
            double part = 0.0;
            for (int k = it[1]; k < it[2]; k++) part += Ls[k] * v[S.L_ri[k]];
            if (!split.add(it, S.hy_bwc_item, part, v.data())) return SCPB_ERR_ARG;
        }
        if (!split.level_done()) return SCPB_ERR_ARG;
    }
    for (int i = 0; i < nk; i++) sol[i] = v[S.iperm[i]];
    if (info) {
        int ntopc = 0;
        for (int j = 0; j < nk; j++) ntopc += S.hy_is_top[j];
        info[0] = nl; info[1] = S.hy_ntl; info[2] = S.hy_tl_ptr[S.hy_ntl]; info[3] = ntopc;
        info[4] = S.hy_fa_lvl[nl] - S.hy_fa_lvl[nl - 1];
        info[5] = (int64_t)(S.hy_ft_op.size() - S.ft_op.size()) / 2;
        info[6] = S.hy_fwp_lvl[nl] - S.hy_fwp_lvl[nl - 1];
        info[7] = S.nlevels;
    }
    return SCPB_OK;
}

// ---- stateful variant of the scalar interpreter (numerics studies on the CPU: symbolic analysis once, then any number
// of factor / solve calls).  Dynamic regularisation as in the kernel: a pivot with sgn*d <= tau is replaced by sgn*rho;
// a replaced pivot that is NOT small (|d| > bad_abs, or non-finite) means the inertia was lost to cancellation and is
// counted in the return value of the factor call (the kernel escalates the static regularisation on that signal).
struct scpb_debug_kkt_s {
    ConeSymbolic S;
    std::vector<double> Y, Ls, Lrow, invD, v;
};

extern "C" int32_t scpb_debug_kkt_new(int32_t n, int32_t p, int32_t m, const int32_t *A_rp, const int32_t *A_ci,
                                      const int32_t *G_rp, const int32_t *G_ci, int32_t l, int32_t nsoc,
                                      const int32_t *soc_dims, const int32_t *perm, void **out, int64_t *info)
{
    if (!out) return SCPB_ERR_ARG;
    scpb_debug_kkt_s *k = new scpb_debug_kkt_s();
    static const int zero = 0;
    if (!cone_symbolic_build(k->S, n, p, m, A_rp, A_ci ? A_ci : &zero, G_rp, G_ci ? G_ci : &zero, l, nsoc, soc_dims, perm)) {
        delete k;
        return SCPB_ERR_ARG;
    }
    const ConeSymbolic &S = k->S;
    k->Y.resize((size_t)S.nnzL + S.nk); k->Ls.resize((size_t)S.nnzL + 1); k->Lrow.resize((size_t)S.nnzL + 1);
    k->invD.resize(S.nk); k->v.resize(S.nk);
    if (info) { info[0] = S.nnzL; info[1] = S.nlevels; info[2] = S.factor_ops; info[3] = S.sn_nlevels; }
    *out = k;
    return SCPB_OK;
}

extern "C" int32_t scpb_debug_kkt_free(void *h)
{
    delete (scpb_debug_kkt_s *)h;
    return SCPB_OK;
}

// returns the number of "bad" (large wrong-sign or non-finite) pivots, or a negative error code
extern "C" int32_t scpb_debug_kkt_factor(void *h, const double *Av, const double *Gv, const double *wm, double delta,
                                         double tau, double rho, double bad_abs, double *stats)
{
    scpb_debug_kkt_s *k = (scpb_debug_kkt_s *)h;
    if (!k) return -1;
    const ConeSymbolic &S = k->S;
    const int nk = S.nk, ntgt = S.nnzL + nk;
    std::vector<double> &Y = k->Y, &Ls = k->Ls, &invD = k->invD;
    for (int t = 0; t < ntgt; t++) {
        double acc = delta * S.as_sign[t];
        if (S.as_src[t] >= 0) acc += Av[S.as_src[t]];
        for (int q = S.as_ptr[t]; q < S.as_ptr[t + 1]; q++) acc += Gv[S.as_a[q]] * Gv[S.as_b[q]] * wm[S.as_c[q]];
        Y[t] = acc;
    }
    int nbad = 0, nreg = 0;
    double lmax = 0.0, dmin = 1e300;
    SplitSums split(S.npart);
    for (int lv = 0; lv < S.nlevels; lv++) {
        for (int w = S.fa_lvl[lv]; w < S.fa_lvl[lv + 1]; w++) {
            const int *it = &S.fa_item[4 * (size_t)w];
            double part = 0.0;
            for (int q = it[1]; q < it[2]; q++) part += Y[S.ft_op[2 * (size_t)q]] * Ls[S.Lr_pos[S.ft_op[2 * (size_t)q + 1]]];
            if (!split.store(it, part, Y.data())) return SCPB_ERR_ARG;
        }
        for (int w = S.fb_lvl[lv]; w < S.fb_lvl[lv + 1]; w++) {
            const int *it = &S.fb_item[4 * (size_t)w];
            double e, d;
            if (!phase_b_operands(split, it, &S.fb_cmb[4 * (size_t)w], S.nnzL, Y, e, d)) return SCPB_ERR_ARG;
            const double sgn = (it[3] & 1) ? 1.0 : -1.0;
            if (!(sgn * d > tau)) {
                if (it[3] & 2) { nreg++; if (!(std::abs(d) <= bad_abs)) nbad++; }
                d = sgn * rho;
            }
            if (it[3] & 2) { invD[it[1]] = 1.0 / d; dmin = std::min(dmin, std::abs(d)); }
            else { Ls[it[0]] = e * (1.0 / d); lmax = std::max(lmax, std::abs(Ls[it[0]])); }
        }
        if (!split.level_done()) return SCPB_ERR_ARG;
    }
    for (int q = 0; q < S.nnzL; q++) k->Lrow[q] = Ls[S.Lr_pos[q]];
    if (!(lmax < 1e300)) nbad++;
    if (stats) { stats[0] = nreg; stats[1] = lmax; stats[2] = dmin; }
    return nbad;
}

extern "C" int32_t scpb_debug_kkt_resolve(void *h, const double *rhs, double *sol)
{
    scpb_debug_kkt_s *k = (scpb_debug_kkt_s *)h;
    if (!k) return SCPB_ERR_ARG;
    const ConeSymbolic &S = k->S;
    const int nk = S.nk;
    std::vector<double> &v = k->v;
    for (int i = 0; i < nk; i++) v[S.iperm[i]] = rhs[i];
    for (int i = 0; i < nk; i++) {     // forward, rows in elimination order
        double part = 0.0;
        for (int q = S.Lr_rp[i]; q < S.Lr_rp[i + 1]; q++) part += k->Lrow[q] * v[S.Lr_col[q]];
        v[i] -= part;
    }
    for (int i = 0; i < nk; i++) v[i] *= k->invD[i];
    for (int j = nk - 1; j >= 0; j--) {
        double part = 0.0;
        for (int q = S.L_cp[j]; q < S.L_cp[j + 1]; q++) part += k->Ls[q] * v[S.L_ri[q]];
        v[j] -= part;
    }
    for (int i = 0; i < nk; i++) sol[i] = v[S.iperm[i]];
    return SCPB_OK;
}

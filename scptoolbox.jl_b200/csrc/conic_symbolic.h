// conic_symbolic.h -- host-side (C++) symbolic analysis for the batched interior-point solver.
//
// The cone program   min c'x  s.t.  A x = b,  G x + s = h,  s in K = R+^l x SOC(q_1) x ...
// (the form ECOS receives from JuMP/MOI in the reference: src/parser/program.jl:419-424) has a
// sparsity pattern that is SHARED by every seed of a batch.  Everything that depends only on the
// pattern is computed once here and uploaded as index programs:
//   * the reduced KKT matrix   M = [ dI + G' W^-2 G   A' ; A   -dI ]   in a caller-supplied
//     elimination order (stage-wise nested dissection from the host template),
//   * its elimination tree, the fill pattern of L (M = L D L'), the level schedule (etree height),
//   * gather programs: KKT assembly (triples G*G*W^-2 / direct A entries), numeric factorisation
//     (pairs Y_ik * L_jk per target), forward / backward substitution (row / column lists).
#pragma once
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <string>
#include <vector>

#ifndef CONIC_FACTOR_PF
#define CONIC_FACTOR_PF 4  // factor ops (gather pairs) a lane keeps in flight per item
#endif
#ifndef CONIC_SOLVE_PF
#define CONIC_SOLVE_PF 4   // L entries a lane keeps in flight per substitution item
#endif
// supernodal panels (conic_sn.cuh): a panel is held by a lane group, one lane per row, at most CONIC_SN_WMAX columns
// in registers; wider runs of columns are cut into several supernodes
#define CONIC_SN_WMAX 8
#define CONIC_SN_RMAX 32
#define CONIC_SN_R1MAX 10   // single-column panels up to this height are handled by ONE thread (leaf levels)
// lane-group size of an R x w panel (1, 8, 16 or 32 lanes; 0: the panel does not fit a warp -> scalar programs only)
inline int conic_sn_class(int R, int w)
{
    if (w > CONIC_SN_WMAX || R > CONIC_SN_RMAX) return 0;
    if (w == 1 && R <= CONIC_SN_R1MAX) return 1;
    return R <= 8 ? 8 : (R <= 16 ? 16 : 32);
}

struct ConeSymbolic {
    int n = 0, p = 0, m = 0, l = 0, nsoc = 0;
    int nk = 0;                       // n + p  (KKT dimension)
    std::vector<int> soc_dim, soc_off;   // row offset (within G rows) of each SOC
    std::vector<int> soc_woff;           // offset of each SOC's dense W^-2 block inside the Wm array
    int nwm = 0;                      // l + sum q^2
    // patterns (CSR) and transposes (CSC as CSR of the transpose, with value index map)
    std::vector<int> A_rp, A_ci, G_rp, G_ci;
    std::vector<int> At_rp, At_ri, At_vi, Gt_rp, Gt_ri, Gt_vi;
    // permutation: perm[k] = node eliminated k-th; iperm[node] = k
    std::vector<int> perm, iperm;
    // L pattern: CSC over permuted nodes, strictly lower part; D separate
    std::vector<int> L_cp, L_ri;      // size nk+1, nnzL
    std::vector<int> Lr_rp, Lr_pos, Lr_col;  // CSR view of L: for each row the (position, column) list
    int nnzL = 0;
    // level schedule
    int nlevels = 0;
    std::vector<int> lvl_ptr;         // nlevels+1 -> index into lvl_nodes
    std::vector<int> lvl_nodes;       // nodes (permuted index) sorted by level
    // factor program: targets ordered by level; target t < nk_targets are (pos) ids:
    //   target id = position in L (0..nnzL-1) for off-diagonals, nnzL + j for diagonal of column j
    std::vector<int> ft_lvl_ptr;      // nlevels+1 -> index into ft_target
    std::vector<int> ft_target;       // target ids in level order
    std::vector<int> ft_op_ptr;       // per entry of ft_target: ops range
    std::vector<int> ft_op_a, ft_op_b;   // op: acc -= Y[a] * Ls[b]   (positions in L)
    // per-level list of L positions to scale after the level's targets are final
    std::vector<int> sc_lvl_ptr, sc_pos, sc_col;
    // assembly program over the same target ids: Y[target] = cst + sum G[a]*G[b]*Wm[c] + A[src]
    std::vector<int> as_ptr;          // size nnzL + nk + 1 (targets in natural id order)
    std::vector<int> as_a, as_b, as_c;
    std::vector<int> as_src;          // per target: index into A values or -1
    std::vector<int> as_sign;         // per target: +1 / -1 / 0 times delta (diagonal regularisation)
    // packed work items for the kernels (fewer dependent global loads per level):
    std::vector<int> fw_item, bw_item;   // int4 per level node: {node, start, end, 0} into Lr_pc / (Ls, L_ri)
    std::vector<int> Lr_pc;              // int2 per L entry in row order: {position, column}
    std::vector<int> ft_item;            // int4 per factor target: {target id, op start, op end, sign}
    std::vector<int> ft_op;              // int2 per op: {a, b}
    std::vector<int> sc_item;            // int4 per scaled entry: {position, column, row-order position, 0}
    std::vector<int> lvl_maxlen;         // [3][nlevels]: longest L row / L column / factor op list of each level
    // balanced substitution programs: every item covers at most R*SOLVE_PF entries of one row (forward) / column
    // (backward), R = lanes per item of that level; rows longer than that are split into several items whose partial
    // sums are combined in a fixed order by the last of them to finish (.w = 1 + partial-sum slot, see number_pieces).
    // All loads of an item fit the per-lane register prefetch.
    std::vector<int> fwp_item, bwp_item; // int4 {node, start, end, 0 | 1 + slot}
    std::vector<int> fwp_lvl, bwp_lvl;   // nlevels+1 -> index into the item lists
    std::vector<int> fwp_R, bwp_R;       // lanes per item of each level
    // balanced factorisation program, same idea: phase A items cover at most R*CONIC_FACTOR_PF ops of one target
    // (Y[target] -= sum Y[a]*Ls[b]; split targets are combined like the substitution's; targets without ops have no item), phase B items
    // finish a column: {Y position, column, row-order position, flags}; flags bit0 = expected pivot sign is +,
    // bit1 = the item is the diagonal itself (regularise, write 1/d), otherwise scale the entry by 1/d.
    std::vector<int> fa_item, fa_lvl, fa_R;
    std::vector<int> fb_item, fb_lvl;
    // split targets (number_pieces): int4 per split item {target, first slot, end slot of the target, slot}, slots
    // numbered from 0 in every level.  The substitution items point into these (.w = 1 + index); the factorisation's
    // phase-A items hold their slot itself (.w = 1 + slot), and phase B combines the split targets through fb_cmb.
    std::vector<int> fc_item, fwc_item, bwc_item;
    std::vector<int> fb_cmb;          // int4 per phase-B item: {entry first slot, entry end slot, pivot first slot, pivot end slot}
    int fslots = 0, sslots = 0;       // the most slots of one level: factorisation, substitutions (forward or backward)
    int npart = 0;                    // partial-sum slots per seed: the most any of the programs (hybrid included) uses
    // ---- supernodal program (executed by the kernels of conic_sn.cuh; CPU interpreter scpb_debug_kkt_solve_sn,
    // tests/test_conic_symbolic.py) ----
    // Maximal supernodes: consecutive columns a..b with parent(j) = j+1 and struct(L[:,j]) = {j+1} + struct(L[:,j+1]);
    // each owns a dense column-major R x w panel (rows = its own w columns, then the rows below), D on the panel
    // diagonal, unit-lower L below it (at most CONIC_SN_WMAX columns per supernode).  A supernodal level needs ONE
    // barrier; the bench KKT has 22 such levels against 88 scalar ones (profiles/r1_supernode_study.txt).
    std::vector<int> sn_first, sn_width, sn_nrows;   // per supernode
    std::vector<int> sn_rows_ptr, sn_rows;           // row (node) indices of each panel
    std::vector<int> sn_panel_off;                   // offset of each panel in the per-seed panel array
    std::vector<int> sn_lvl_ptr, sn_lvl_nodes;       // supernodal level schedule (children before parents)
    std::vector<int> sn_pos_of_target;               // target id (L position | nnzL + column) -> panel offset
    std::vector<int> sn_upd_ptr;                     // per supernode: range of its update scatter list
    std::vector<int> sn_upd_dst;                     // lower-triangle pairs (x >= y) of the below rows -> panel offset
    std::vector<int> sn_upd_xy;                      // the pair itself, packed x | y << 16 (indices into the below rows)
    std::vector<int> sn_sign;                        // expected pivot sign of each column (+1 / -1)
    std::vector<int> sn_cls_ptr;                     // [nlevels][5]: level nodes sorted by lane-group size 1 | 8 | 16 | 32 (conic_sn.cuh)
    // ---- hybrid program (cone_symbolic_build_hybrid): the columns of the supernodes at supernodal level >= hy_cut (the
    // "top" of the elimination tree: few, wide, tall panels -- nested-dissection separators and the dense border) are
    // factored and substituted as register-resident panels, one lane per row, straight on the SCALAR storage (a
    // supernode's columns are consecutive in the CSC arrays of L); everything below keeps the scalar level-scheduled
    // gather programs.  hy_nlevels scalar levels: the levels of the low columns plus one "bridge" level in which every
    // top target gathers its contributions from low columns (factorisation) / every top row gathers from low columns
    // (forward substitution) in one wide, barrier-free pass.  Bench KKT: 88 scalar levels -> 20 + 17 supernodal ones.
    int hy_cut = 0, hy_nlevels = 0, hy_ntl = 0;
    std::vector<int> hy_fa_item, hy_fa_lvl, hy_fa_R, hy_fb_item, hy_fb_lvl, hy_ft_op;
    std::vector<int> hy_fwp_item, hy_fwp_lvl, hy_fwp_R, hy_bwp_item, hy_bwp_lvl, hy_bwp_R;
    std::vector<int> hy_fc_item, hy_fwc_item, hy_bwc_item, hy_fb_cmb;
    int hy_fslots = 0, hy_sslots = 0;
    std::vector<int> hy_tl_ptr;     // hy_ntl + 1 -> index into the descriptor list
    std::vector<int> hy_desc;       // 8 ints per top supernode in top-level order: {first column, width, rows, L_cp[first]},
                                    // {offset into sn_rows, offset into hy_upd_dst, pivot signs (bit c: column c expects +), 0}
    std::vector<int> hy_upd_dst;    // below-row pairs (x >= y) of a top supernode -> TARGET id (L position | nnzL + column)
    std::vector<int> hy_is_top;     // per node (tests)
    bool sn_fits = true;                             // every panel fits a warp's scratch
    long long sn_panel_size = 0;
    int sn_nlevels = 0;
    long long factor_ops = 0;
    std::string err;
};

namespace conic_detail {

// Items whose target is split over several items (.w != 0 on input) get a partial-sum slot each.  Slots are numbered
// from 0 in every level, so that the slots of one level fit in shared memory; a target's slots are consecutive, in
// item order.  .w = 1 + index of the split item in info; info[index] = {target, first slot, end slot of the target,
// slot}.  The substitution kernels store an item's partial sum in its slot and count the finished items of the target
// (the counter is numbered by the first slot); the last one subtracts the target's slots from it in slot order, so the
// result does not depend on the order in which the items ran.  nslot: the most slots of one level.
inline void number_pieces(std::vector<int> &item, const std::vector<int> &lvl, std::vector<int> &info, int &nslot)
{
    const int nl = (int)lvl.size() - 1;
    info.clear();
    nslot = 0;
    for (int lv = 0; lv < nl; lv++) {
        std::vector<std::pair<int, int>> sp;   // (target, item) of the split items of the level
        for (int w = lvl[lv]; w < lvl[lv + 1]; w++)
            if (item[4 * (size_t)w + 3]) sp.push_back({item[4 * (size_t)w], w});
        std::stable_sort(sp.begin(), sp.end(), [](const std::pair<int, int> &x, const std::pair<int, int> &y) { return x.first < y.first; });
        int slot = 0;
        for (size_t i = 0; i < sp.size();) {
            size_t j = i;
            while (j < sp.size() && sp[j].first == sp[i].first) j++;
            const int s0 = slot, s1 = slot + (int)(j - i);
            for (; i < j; i++) {
                item[4 * (size_t)sp[i].second + 3] = 1 + (int)(info.size() / 4);
                info.push_back(sp[i].first); info.push_back(s0); info.push_back(s1); info.push_back(slot++);
            }
        }
        nslot = std::max(nslot, slot);
    }
    if (info.empty()) info.assign(4, 0);
}

// The factorisation combines its split targets without counters: phase A only stores the partial sums in their slots
// (.w is rewritten to 1 + slot), and phase B, which follows the level's barrier and reads every target of its level --
// the entry it scales and the pivot of its column -- subtracts their slots in slot order as it reads them.  cmb gets an
// int4 per phase-B item {entry first slot, entry end slot, pivot first slot, pivot end slot} (empty ranges: target not
// split).  Every split target must be the entry of exactly one phase-B item of its level, which writes the combined
// value back to Y for the later levels.  A split target that no phase-B item of its level finishes (the bridge level
// of the hybrid program, whose targets the top panels finish) gets a combine-only phase-B item {target, 0, 0, 4} when
// `extra` is set; otherwise the build fails.  Without `extra` every phase-A target must be an entry of phase B.
inline bool combine_in_phase_b(std::vector<int> &fa, const std::vector<int> &fal, const std::vector<int> &info,
                               std::vector<int> &fb, std::vector<int> &fbl, std::vector<int> &cmb, int ntgt, int nnzL,
                               bool extra)
{
    const int nl = (int)fal.size() - 1;
    std::vector<int> nfb, stamp(ntgt, -1), r0(ntgt, 0), r1(ntgt, 0), used(ntgt, 0), entry(ntgt, -1);
    cmb.clear();
    for (int lv = 0; lv < nl; lv++) {
        for (int w = fal[lv]; w < fal[lv + 1]; w++) {
            int *it = &fa[4 * (size_t)w];
            if (it[0] < 0 || it[0] >= ntgt) return false;
            stamp[it[0]] = lv; used[it[0]] = 0;
            if (!it[3]) { r0[it[0]] = r1[it[0]] = 0; continue; }
            const int *e = &info[4 * (size_t)(it[3] - 1)];
            if (e[0] != it[0]) return false;
            r0[it[0]] = e[1]; r1[it[0]] = e[2];
            it[3] = 1 + e[3];
        }
        for (int w = fbl[lv]; w < fbl[lv + 1]; w++) {
            const int *it = &fb[4 * (size_t)w];
            const int t = it[0], pv = nnzL + it[1];
            const bool te = stamp[t] == lv, tp = stamp[pv] == lv;
            for (int q = 0; q < 4; q++) nfb.push_back(it[q]);
            cmb.push_back(te ? r0[t] : 0); cmb.push_back(te ? r1[t] : 0);
            cmb.push_back(tp ? r0[pv] : 0); cmb.push_back(tp ? r1[pv] : 0);
            if (te) { used[t]++; entry[t] = lv; }
        }
        for (int w = fal[lv]; w < fal[lv + 1]; w++) {
            const int t = fa[4 * (size_t)w];
            if (entry[t] == lv) {
                if (used[t] != 1) return false;   // two phase-B items would write the same target back
                continue;
            }
            if (!extra) return false;             // a target of phase A that phase B of its level does not finish
            if (r1[t] > r0[t]) {
                nfb.push_back(t); nfb.push_back(0); nfb.push_back(0); nfb.push_back(4);
                cmb.push_back(r0[t]); cmb.push_back(r1[t]); cmb.push_back(0); cmb.push_back(0);
                used[t] = 1; entry[t] = lv;
            }
        }
        fbl[lv + 1] = (int)(nfb.size() / 4);
    }
    if (nfb.empty()) nfb.assign(4, 0);
    if (cmb.empty()) cmb.assign(4, 0);
    fb.swap(nfb);
    return true;
}

inline void transpose_pattern(int nrow, int ncol, const std::vector<int> &rp, const std::vector<int> &ci,
                              std::vector<int> &t_rp, std::vector<int> &t_ri, std::vector<int> &t_vi)
{
    t_rp.assign(ncol + 1, 0);
    for (int v : ci) t_rp[v + 1]++;
    for (int j = 0; j < ncol; j++) t_rp[j + 1] += t_rp[j];
    t_ri.resize(ci.size());
    t_vi.resize(ci.size());
    std::vector<int> nxt(t_rp.begin(), t_rp.end() - 1);
    for (int r = 0; r < nrow; r++)
        for (int k = rp[r]; k < rp[r + 1]; k++) {
            int q = nxt[ci[k]]++;
            t_ri[q] = r;
            t_vi[q] = k;
        }
}

}  // namespace conic_detail

// Build everything. Returns false and sets S.err on failure.
inline bool cone_symbolic_build(ConeSymbolic &S, int n, int p, int m, const int *A_rp, const int *A_ci,
                                const int *G_rp, const int *G_ci, int l, int nsoc, const int *soc_dims,
                                const int *perm_in)
{
    using namespace conic_detail;
    S.n = n; S.p = p; S.m = m; S.l = l; S.nsoc = nsoc; S.nk = n + p;
    const int nk = S.nk;
    S.A_rp.assign(A_rp, A_rp + p + 1);
    S.A_ci.assign(A_ci, A_ci + A_rp[p]);
    S.G_rp.assign(G_rp, G_rp + m + 1);
    S.G_ci.assign(G_ci, G_ci + G_rp[m]);
    S.soc_dim.assign(soc_dims, soc_dims + nsoc);
    S.soc_off.resize(nsoc);
    S.soc_woff.resize(nsoc);
    int off = l, woff = l;
    for (int i = 0; i < nsoc; i++) {
        if (soc_dims[i] < 2) { S.err = "SOC dimension < 2"; return false; }
        S.soc_off[i] = off; S.soc_woff[i] = woff;
        off += soc_dims[i]; woff += soc_dims[i] * soc_dims[i];
    }
    if (off != m) { S.err = "cone dimensions do not sum to m"; return false; }
    S.nwm = woff;
    transpose_pattern(p, n, S.A_rp, S.A_ci, S.At_rp, S.At_ri, S.At_vi);
    transpose_pattern(m, n, S.G_rp, S.G_ci, S.Gt_rp, S.Gt_ri, S.Gt_vi);

    // ---- permutation ----
    S.perm.resize(nk);
    if (perm_in) S.perm.assign(perm_in, perm_in + nk);
    else std::iota(S.perm.begin(), S.perm.end(), 0);
    S.iperm.assign(nk, -1);
    for (int k = 0; k < nk; k++) {
        int v = S.perm[k];
        if (v < 0 || v >= nk || S.iperm[v] != -1) { S.err = "perm is not a permutation of 0..n+p-1"; return false; }
        S.iperm[v] = k;
    }

    // ---- KKT entries (lower triangle, permuted): records (col j, row i, a, b, c) ----
    struct Rec { int j, i, a, b, c; };   // a>=0,b>=0: triple; a=-1: direct A source b
    std::vector<Rec> recs;
    auto add_block = [&](int r0, int q, int wbase, bool dense) {
        for (int r1 = r0; r1 < r0 + q; r1++)
            for (int r2 = r0; r2 < r0 + q; r2++) {
                if (!dense && r1 != r2) continue;
                const int c = dense ? wbase + (r1 - r0) * q + (r2 - r0) : wbase;
                for (int ka = S.G_rp[r1]; ka < S.G_rp[r1 + 1]; ka++)
                    for (int kb = S.G_rp[r2]; kb < S.G_rp[r2 + 1]; kb++) {
                        const int pi = S.iperm[S.G_ci[ka]], pj = S.iperm[S.G_ci[kb]];
                        if (pi >= pj) recs.push_back({pj, pi, ka, kb, c});
                    }
            }
    };
    for (int r = 0; r < l; r++) add_block(r, 1, r, false);
    for (int i = 0; i < nsoc; i++) add_block(S.soc_off[i], S.soc_dim[i], S.soc_woff[i], true);
    for (int r = 0; r < p; r++)
        for (int k = S.A_rp[r]; k < S.A_rp[r + 1]; k++) {
            int pi = S.iperm[n + r], pj = S.iperm[S.A_ci[k]];
            if (pi < pj) std::swap(pi, pj);
            recs.push_back({pj, pi, -1, k, 0});
        }
    std::sort(recs.begin(), recs.end(), [](const Rec &x, const Rec &y) {
        return x.j != y.j ? x.j < y.j : x.i < y.i;
    });

    // ---- M pattern (strict lower, CSC) ----
    std::vector<std::vector<int>> mcol(nk);
    for (const Rec &r : recs)
        if (r.i != r.j && (mcol[r.j].empty() || mcol[r.j].back() != r.i)) mcol[r.j].push_back(r.i);

    // ---- elimination tree + column structures of L ----
    std::vector<int> parent(nk, -1);
    std::vector<std::vector<int>> lcol(nk);
    {
        std::vector<std::vector<int>> children(nk);
        std::vector<int> mark(nk, -1);
        for (int j = 0; j < nk; j++) {
            std::vector<int> &s = lcol[j];
            mark[j] = j;
            for (int i : mcol[j])
                if (mark[i] != j) { mark[i] = j; s.push_back(i); }
            for (int c : children[j]) {
                for (int i : lcol[c])
                    if (i != j && mark[i] != j) { mark[i] = j; s.push_back(i); }
            }
            std::sort(s.begin(), s.end());
            if (!s.empty()) {
                parent[j] = s.front();
                children[s.front()].push_back(j);
            }
        }
    }
    S.L_cp.assign(nk + 1, 0);
    for (int j = 0; j < nk; j++) S.L_cp[j + 1] = S.L_cp[j] + (int)lcol[j].size();
    S.nnzL = S.L_cp[nk];
    S.L_ri.resize(S.nnzL);
    for (int j = 0; j < nk; j++) std::copy(lcol[j].begin(), lcol[j].end(), S.L_ri.begin() + S.L_cp[j]);
    auto lpos = [&](int i, int j) -> int {  // position of (i,j), i>j, in L
        auto b = S.L_ri.begin() + S.L_cp[j], e = S.L_ri.begin() + S.L_cp[j + 1];
        auto it = std::lower_bound(b, e, i);
        return (it != e && *it == i) ? (int)(it - S.L_ri.begin()) : -1;
    };

    // ---- levels = etree height ----
    std::vector<int> height(nk, 0);
    for (int j = 0; j < nk; j++)
        if (parent[j] >= 0) height[parent[j]] = std::max(height[parent[j]], height[j] + 1);
    S.nlevels = nk ? *std::max_element(height.begin(), height.end()) + 1 : 0;
    S.lvl_ptr.assign(S.nlevels + 1, 0);
    for (int j = 0; j < nk; j++) S.lvl_ptr[height[j] + 1]++;
    for (int k = 0; k < S.nlevels; k++) S.lvl_ptr[k + 1] += S.lvl_ptr[k];
    S.lvl_nodes.resize(nk);
    {
        std::vector<int> nxt(S.lvl_ptr.begin(), S.lvl_ptr.end() - 1);
        for (int j = 0; j < nk; j++) S.lvl_nodes[nxt[height[j]]++] = j;
    }

    // ---- CSR view of L ----
    S.Lr_rp.assign(nk + 1, 0);
    for (int q = 0; q < S.nnzL; q++) S.Lr_rp[S.L_ri[q] + 1]++;
    for (int i = 0; i < nk; i++) S.Lr_rp[i + 1] += S.Lr_rp[i];
    S.Lr_pos.resize(S.nnzL);
    S.Lr_col.resize(S.nnzL);
    {
        std::vector<int> nxt(S.Lr_rp.begin(), S.Lr_rp.end() - 1);
        for (int j = 0; j < nk; j++)
            for (int q = S.L_cp[j]; q < S.L_cp[j + 1]; q++) {
                int w = nxt[S.L_ri[q]]++;
                S.Lr_pos[w] = q;
                S.Lr_col[w] = j;
            }
    }

    // ---- factor program: per target the (a,b) op pairs, generated column by column ----
    const int ntgt = S.nnzL + nk;
    std::vector<int> cnt(ntgt, 0);
    S.factor_ops = 0;
    for (int k = 0; k < nk; k++) {
        const int b0 = S.L_cp[k], e0 = S.L_cp[k + 1];
        for (int qa = b0; qa < e0; qa++) {
            cnt[S.nnzL + S.L_ri[qa]]++;  // diagonal of row_a
            for (int qb = qa + 1; qb < e0; qb++) {
                int t = lpos(S.L_ri[qb], S.L_ri[qa]);
                if (t < 0) { S.err = "internal: fill entry missing"; return false; }
                cnt[t]++;
            }
        }
    }
    std::vector<long long> optr(ntgt + 1, 0);
    for (int t = 0; t < ntgt; t++) optr[t + 1] = optr[t] + cnt[t];
    S.factor_ops = optr[ntgt];
    if (S.factor_ops > 2000000000LL) { S.err = "factor program too large (bad ordering?)"; return false; }
    std::vector<int> opa(S.factor_ops), opb(S.factor_ops);
    {
        std::vector<long long> nxt(optr.begin(), optr.end() - 1);
        for (int k = 0; k < nk; k++) {
            const int b0 = S.L_cp[k], e0 = S.L_cp[k + 1];
            for (int qa = b0; qa < e0; qa++) {
                long long w = nxt[S.nnzL + S.L_ri[qa]]++;
                opa[w] = qa; opb[w] = qa;
                for (int qb = qa + 1; qb < e0; qb++) {
                    int t = lpos(S.L_ri[qb], S.L_ri[qa]);
                    long long w2 = nxt[t]++;
                    opa[w2] = qb;   // Y_ik  (row_b = i)
                    opb[w2] = qa;   // L_jk  (row_a = j)
                }
            }
        }
    }
    // order targets by level of their column; diagonal target belongs to its own column
    S.ft_lvl_ptr.assign(S.nlevels + 1, 0);
    S.ft_target.clear(); S.ft_op_ptr.clear(); S.ft_op_a.clear(); S.ft_op_b.clear();
    S.ft_target.reserve(ntgt);
    S.ft_op_a.reserve(S.factor_ops); S.ft_op_b.reserve(S.factor_ops);
    S.sc_lvl_ptr.assign(S.nlevels + 1, 0);
    S.sc_pos.clear(); S.sc_col.clear();
    S.ft_op_ptr.push_back(0);
    for (int lv = 0; lv < S.nlevels; lv++) {
        for (int w = S.lvl_ptr[lv]; w < S.lvl_ptr[lv + 1]; w++) {
            const int j = S.lvl_nodes[w];
            auto emit = [&](int t) {
                S.ft_target.push_back(t);
                for (long long o = optr[t]; o < optr[t + 1]; o++) { S.ft_op_a.push_back(opa[o]); S.ft_op_b.push_back(opb[o]); }
                S.ft_op_ptr.push_back((int)S.ft_op_a.size());
            };
            emit(S.nnzL + j);
            for (int q = S.L_cp[j]; q < S.L_cp[j + 1]; q++) { emit(q); S.sc_pos.push_back(q); S.sc_col.push_back(j); }
        }
        S.ft_lvl_ptr[lv + 1] = (int)S.ft_target.size();
        S.sc_lvl_ptr[lv + 1] = (int)S.sc_pos.size();
    }

    // ---- assembly program (targets in natural id order) ----
    S.as_ptr.assign(ntgt + 1, 0);
    S.as_src.assign(ntgt, -1);
    S.as_sign.assign(ntgt, 0);
    std::vector<int> tcount(ntgt, 0);
    auto tid = [&](int i, int j) { return i == j ? S.nnzL + j : lpos(i, j); };
    for (const Rec &r : recs) {
        int t = tid(r.i, r.j);
        if (t < 0) { S.err = "internal: KKT entry outside L pattern"; return false; }
        if (r.a >= 0) tcount[t]++;
    }
    for (int t = 0; t < ntgt; t++) S.as_ptr[t + 1] = S.as_ptr[t] + tcount[t];
    S.as_a.resize(S.as_ptr[ntgt]); S.as_b.resize(S.as_ptr[ntgt]); S.as_c.resize(S.as_ptr[ntgt]);
    {
        std::vector<int> nxt(S.as_ptr.begin(), S.as_ptr.end() - 1);
        for (const Rec &r : recs) {
            int t = tid(r.i, r.j);
            if (r.a >= 0) { int w = nxt[t]++; S.as_a[w] = r.a; S.as_b[w] = r.b; S.as_c[w] = r.c; }
            else S.as_src[t] = r.b;
        }
    }
    for (int k = 0; k < nk; k++) S.as_sign[S.nnzL + k] = (S.perm[k] < n) ? 1 : -1;

    // ---- packed items ----
    S.fw_item.resize(4 * (size_t)nk); S.bw_item.resize(4 * (size_t)nk);
    for (int w = 0; w < nk; w++) {
        const int i = S.lvl_nodes[w];
        S.fw_item[4 * w] = i; S.fw_item[4 * w + 1] = S.Lr_rp[i]; S.fw_item[4 * w + 2] = S.Lr_rp[i + 1]; S.fw_item[4 * w + 3] = 0;
        S.bw_item[4 * w] = i; S.bw_item[4 * w + 1] = S.L_cp[i]; S.bw_item[4 * w + 2] = S.L_cp[i + 1]; S.bw_item[4 * w + 3] = 0;
    }
    S.Lr_pc.resize(2 * (size_t)S.nnzL);
    for (int q = 0; q < S.nnzL; q++) { S.Lr_pc[2 * q] = S.Lr_pos[q]; S.Lr_pc[2 * q + 1] = S.Lr_col[q]; }
    const size_t nft = S.ft_target.size();
    S.ft_item.resize(4 * nft);
    for (size_t w = 0; w < nft; w++) {
        const int t = S.ft_target[w];
        S.ft_item[4 * w] = t; S.ft_item[4 * w + 1] = S.ft_op_ptr[w]; S.ft_item[4 * w + 2] = S.ft_op_ptr[w + 1];
        S.ft_item[4 * w + 3] = S.as_sign[t];
    }
    {
        std::vector<int> rowpos(S.nnzL);
        for (int w = 0; w < S.nnzL; w++) rowpos[S.Lr_pos[w]] = w;
        S.sc_item.resize(4 * S.sc_pos.size());
        for (size_t w = 0; w < S.sc_pos.size(); w++) {
            S.sc_item[4 * w] = S.sc_pos[w]; S.sc_item[4 * w + 1] = S.sc_col[w];
            S.sc_item[4 * w + 2] = rowpos[S.sc_pos[w]]; S.sc_item[4 * w + 3] = 0;
        }
    }
    S.lvl_maxlen.assign(3 * (size_t)S.nlevels, 0);
    for (int lv = 0; lv < S.nlevels; lv++) {
        for (int w = S.lvl_ptr[lv]; w < S.lvl_ptr[lv + 1]; w++) {
            const int i = S.lvl_nodes[w];
            S.lvl_maxlen[lv] = std::max(S.lvl_maxlen[lv], S.Lr_rp[i + 1] - S.Lr_rp[i]);
            S.lvl_maxlen[S.nlevels + lv] = std::max(S.lvl_maxlen[S.nlevels + lv], S.L_cp[i + 1] - S.L_cp[i]);
        }
        for (int w = S.ft_lvl_ptr[lv]; w < S.ft_lvl_ptr[lv + 1]; w++)
            S.lvl_maxlen[2 * S.nlevels + lv] = std::max(S.lvl_maxlen[2 * S.nlevels + lv], S.ft_op_ptr[w + 1] - S.ft_op_ptr[w]);
    }
    // op pairs for the kernel: {Y operand (column-order position), L operand as ROW-order position}.  The ops of a
    // target (i,j) run over all of row j (pattern(row j) is contained in pattern(row i) by the fill rule), so in row
    // order the L operands of an item are consecutive doubles: full 32-byte sectors instead of scattered gathers.
    // (Storing Y in row order as well was measured and is slower: the assembly then scatters its writes.)
    {
        std::vector<int> rowpos(S.nnzL);
        for (int w = 0; w < S.nnzL; w++) rowpos[S.Lr_pos[w]] = w;
        S.ft_op.resize(2 * S.ft_op_a.size());
        for (size_t k = 0; k < S.ft_op_a.size(); k++) { S.ft_op[2 * k] = S.ft_op_a[k]; S.ft_op[2 * k + 1] = rowpos[S.ft_op_b[k]]; }
    }
    // ---- balanced factorisation program ----
    {
        const int PF = CONIC_FACTOR_PF, SLOTS = 512, RMAX = 4;
        S.fa_item.clear(); S.fa_lvl.assign(S.nlevels + 1, 0); S.fa_R.assign(S.nlevels, 1);
        S.fb_item.clear(); S.fb_lvl.assign(S.nlevels + 1, 0);
        std::vector<int> rowpos(S.nnzL);
        for (int w = 0; w < S.nnzL; w++) rowpos[S.Lr_pos[w]] = w;
        for (int lv = 0; lv < S.nlevels; lv++) {
            const int w0 = S.ft_lvl_ptr[lv], w1 = S.ft_lvl_ptr[lv + 1];
            int bestR = 1; long long bestp = -1, bestw = -1;
            for (int R = 1; R <= RMAX; R *= 2) {
                long long items = 0;
                for (int w = w0; w < w1; w++) items += (S.ft_op_ptr[w + 1] - S.ft_op_ptr[w] + R * PF - 1) / (R * PF);
                const long long passes = (items * R + SLOTS - 1) / SLOTS, waste = items * R;
                if (bestp < 0 || passes < bestp || (passes == bestp && waste < bestw)) { bestp = passes; bestw = waste; bestR = R; }
            }
            S.fa_R[lv] = bestR;
            const int cap = bestR * PF;
            for (int w = w0; w < w1; w++) {
                const int k0 = S.ft_op_ptr[w], k1 = S.ft_op_ptr[w + 1], split = (k1 - k0 > cap) ? 1 : 0;
                for (int k = k0; k < k1; k += cap) {
                    S.fa_item.push_back(S.ft_target[w]); S.fa_item.push_back(k);
                    S.fa_item.push_back(std::min(k + cap, k1)); S.fa_item.push_back(split);
                }
            }
            S.fa_lvl[lv + 1] = (int)(S.fa_item.size() / 4);
            for (int w = S.lvl_ptr[lv]; w < S.lvl_ptr[lv + 1]; w++) {
                const int j = S.lvl_nodes[w], pos = (S.as_sign[S.nnzL + j] > 0) ? 1 : 0;
                S.fb_item.push_back(S.nnzL + j); S.fb_item.push_back(j); S.fb_item.push_back(0); S.fb_item.push_back(pos | 2);
                for (int q = S.L_cp[j]; q < S.L_cp[j + 1]; q++) {
                    S.fb_item.push_back(q); S.fb_item.push_back(j); S.fb_item.push_back(rowpos[q]); S.fb_item.push_back(pos);
                }
            }
            S.fb_lvl[lv + 1] = (int)(S.fb_item.size() / 4);
        }
        if (S.fa_item.empty()) S.fa_item.assign(4, 0);
        conic_detail::number_pieces(S.fa_item, S.fa_lvl, S.fc_item, S.fslots);
        if (!conic_detail::combine_in_phase_b(S.fa_item, S.fa_lvl, S.fc_item, S.fb_item, S.fb_lvl, S.fb_cmb, S.nnzL + nk,
                                              S.nnzL, false)) {
            S.err = "internal: a phase-A target of the factorisation is not finished by one phase-B item of its level";
            return false;
        }
    }
    // ---- supernodal program ----
    {
        const int ns_max = nk;
        std::vector<int> sn_of(nk, 0);
        S.sn_first.clear(); S.sn_width.clear(); S.sn_nrows.clear();
        for (int j = 0; j < nk;) {
            int k = j;
            while (k + 1 < nk && (k - j + 1) < CONIC_SN_WMAX && S.L_cp[k + 1] > S.L_cp[k] && S.L_ri[S.L_cp[k]] == k + 1 &&
                   (S.L_cp[k + 1] - S.L_cp[k]) == (S.L_cp[k + 2] - S.L_cp[k + 1]) + 1)
                k++;
            const int sid = (int)S.sn_first.size();
            for (int c = j; c <= k; c++) sn_of[c] = sid;
            S.sn_first.push_back(j); S.sn_width.push_back(k - j + 1);
            S.sn_nrows.push_back((k - j + 1) + (S.L_cp[k + 1] - S.L_cp[k]));
            j = k + 1;
        }
        (void)ns_max;
        const int ns = (int)S.sn_first.size();
        S.sn_rows_ptr.assign(ns + 1, 0); S.sn_panel_off.assign(ns + 1, 0);
        for (int s = 0; s < ns; s++) {
            S.sn_rows_ptr[s + 1] = S.sn_rows_ptr[s] + S.sn_nrows[s];
            const long long nxt_ = (long long)S.sn_panel_off[s] + (long long)S.sn_nrows[s] * S.sn_width[s];
            if (nxt_ > 2000000000LL) { S.err = "supernodal panels too large"; return false; }
            S.sn_panel_off[s + 1] = (int)nxt_;
        }
        S.sn_panel_size = S.sn_panel_off[ns];
        S.sn_rows.resize(S.sn_rows_ptr[ns]);
        for (int s = 0; s < ns; s++) {
            const int a = S.sn_first[s], w = S.sn_width[s], b = a + w - 1;
            int o = S.sn_rows_ptr[s];
            for (int c = 0; c < w; c++) S.sn_rows[o++] = a + c;
            for (int q = S.L_cp[b]; q < S.L_cp[b + 1]; q++) S.sn_rows[o++] = S.L_ri[q];
        }
        // panel position of entry (row i, column j)
        auto panel_pos = [&](int i, int j) -> int {
            const int s = sn_of[j], a = S.sn_first[s], w = S.sn_width[s], R = S.sn_nrows[s], c = j - a;
            int r;
            if (i < a + w) r = i - a;
            else {
                const int *lo = &S.sn_rows[S.sn_rows_ptr[s] + w], *hi = &S.sn_rows[S.sn_rows_ptr[s] + R];
                const int *it = std::lower_bound(lo, hi, i);
                if (it == hi || *it != i) return -1;
                r = w + (int)(it - lo);
            }
            return S.sn_panel_off[s] + r + R * c;
        };
        S.sn_pos_of_target.assign((size_t)S.nnzL + nk, -1);
        for (int j = 0; j < nk; j++) {
            S.sn_pos_of_target[(size_t)S.nnzL + j] = panel_pos(j, j);
            for (int q = S.L_cp[j]; q < S.L_cp[j + 1]; q++) {
                const int pp = panel_pos(S.L_ri[q], j);
                if (pp < 0) { S.err = "internal: supernode panel does not cover an L entry"; return false; }
                S.sn_pos_of_target[q] = pp;
            }
        }
        // update scatter lists
        S.sn_upd_ptr.assign(ns + 1, 0);
        S.sn_upd_dst.clear(); S.sn_upd_xy.clear();
        S.sn_sign.resize(nk);
        for (int j = 0; j < nk; j++) S.sn_sign[j] = S.as_sign[(size_t)S.nnzL + j];
        for (int s = 0; s < ns; s++) {
            const int w = S.sn_width[s], R = S.sn_nrows[s];
            const int *below = &S.sn_rows[S.sn_rows_ptr[s] + w];
            for (int y = 0; y < R - w; y++)
                for (int x = y; x < R - w; x++) {
                    const int pp = panel_pos(below[x], below[y]);
                    if (pp < 0) { S.err = "internal: supernodal update falls outside the L pattern"; return false; }
                    S.sn_upd_dst.push_back(pp);
                    S.sn_upd_xy.push_back(x | (y << 16));
                }
            if (S.sn_upd_dst.size() > 2000000000ULL) { S.err = "supernodal update lists too large"; return false; }
            S.sn_upd_ptr[s + 1] = (int)S.sn_upd_dst.size();
        }
        // level schedule: a supernode follows every supernode whose last column's parent lies inside it
        std::vector<int> slev(ns, 0);
        for (int s = 0; s < ns; s++) {
            const int b = S.sn_first[s] + S.sn_width[s] - 1;
            if (S.L_cp[b + 1] > S.L_cp[b]) {
                const int ps = sn_of[S.L_ri[S.L_cp[b]]];
                slev[ps] = std::max(slev[ps], slev[s] + 1);
            }
        }
        S.sn_nlevels = 0;
        for (int s = 0; s < ns; s++) S.sn_nlevels = std::max(S.sn_nlevels, slev[s] + 1);
        S.sn_lvl_ptr.assign(S.sn_nlevels + 1, 0);
        for (int s = 0; s < ns; s++) S.sn_lvl_ptr[slev[s] + 1]++;
        for (int l2 = 0; l2 < S.sn_nlevels; l2++) S.sn_lvl_ptr[l2 + 1] += S.sn_lvl_ptr[l2];
        S.sn_lvl_nodes.resize(ns);
        {
            std::vector<int> nxt(S.sn_lvl_ptr.begin(), S.sn_lvl_ptr.end() - 1);
            for (int s = 0; s < ns; s++) S.sn_lvl_nodes[nxt[slev[s]]++] = s;
        }
        // inside a level: small panels first (single threads, then lane groups of 8, 16 and 32 lanes)
        auto cls_of = [&](int s) { return conic_sn_class(S.sn_nrows[s], S.sn_width[s]); };
        S.sn_cls_ptr.assign(5 * (size_t)S.sn_nlevels, 0);
        S.sn_fits = true;
        for (int lv = 0; lv < S.sn_nlevels; lv++) {
            int *b = &S.sn_lvl_nodes[S.sn_lvl_ptr[lv]], *e = &S.sn_lvl_nodes[S.sn_lvl_ptr[lv + 1]];
            std::stable_sort(b, e, [&](int x, int y) { int cx = cls_of(x), cy = cls_of(y); return (cx ? cx : 64) < (cy ? cy : 64); });
            int o = S.sn_lvl_ptr[lv];
            S.sn_cls_ptr[5 * lv] = o;
            const int gss[4] = {1, 8, 16, 32};
            for (int q = 0; q < 4; q++) {
                while (o < S.sn_lvl_ptr[lv + 1] && cls_of(S.sn_lvl_nodes[o]) == gss[q]) o++;
                S.sn_cls_ptr[5 * lv + q + 1] = o;
            }
            if (o != S.sn_lvl_ptr[lv + 1]) S.sn_fits = false;   // a panel too large for the warp scratch
        }
    }
    // ---- balanced substitution programs ----
    {
        const int PF = CONIC_SOLVE_PF, SLOTS = 512, RMAX = 4;   // RMAX*IPM_MAXG <= 32 lanes of one warp
        auto build = [&](const std::vector<int> &ptr, std::vector<int> &item, std::vector<int> &lvl, std::vector<int> &Rl) {
            item.clear(); lvl.assign(S.nlevels + 1, 0); Rl.assign(S.nlevels, 1);
            for (int lv = 0; lv < S.nlevels; lv++) {
                int bestR = 1; long long bestp = -1, bestw = -1;
                for (int R = 1; R <= RMAX; R *= 2) {
                    long long items = 0;
                    for (int w = S.lvl_ptr[lv]; w < S.lvl_ptr[lv + 1]; w++) {
                        const int i = S.lvl_nodes[w], len = ptr[i + 1] - ptr[i];
                        items += (len + R * PF - 1) / (R * PF);
                    }
                    const long long passes = (items * R + SLOTS - 1) / SLOTS, waste = items * R;
                    if (bestp < 0 || passes < bestp || (passes == bestp && waste < bestw)) { bestp = passes; bestw = waste; bestR = R; }
                }
                Rl[lv] = bestR;
                const int cap = bestR * PF;
                for (int w = S.lvl_ptr[lv]; w < S.lvl_ptr[lv + 1]; w++) {
                    const int i = S.lvl_nodes[w], k0 = ptr[i], k1 = ptr[i + 1];
                    const int split = (k1 - k0 > cap) ? 1 : 0;
                    for (int k = k0; k < k1; k += cap) {
                        item.push_back(i); item.push_back(k); item.push_back(std::min(k + cap, k1)); item.push_back(split);
                    }
                }
                lvl[lv + 1] = (int)(item.size() / 4);
            }
            if (item.empty()) item.assign(4, 0);
        };
        build(S.Lr_rp, S.fwp_item, S.fwp_lvl, S.fwp_R);
        build(S.L_cp, S.bwp_item, S.bwp_lvl, S.bwp_R);
        int fw_ = 0, bw_ = 0;
        conic_detail::number_pieces(S.fwp_item, S.fwp_lvl, S.fwc_item, fw_);
        conic_detail::number_pieces(S.bwp_item, S.bwp_lvl, S.bwc_item, bw_);
        S.sslots = std::max(fw_, bw_);
    }
    S.npart = std::max(S.fslots, S.sslots);
    return true;
}

// Hybrid program for the supernodes at supernodal level >= cut (see ConeSymbolic::hy_*).  Returns false (and leaves
// hy_cut = 0) when the split is empty on either side or a top panel does not fit a warp.
inline bool cone_symbolic_build_hybrid(ConeSymbolic &S, int cut)
{
    S.hy_cut = 0; S.hy_nlevels = 0; S.hy_ntl = 0;
    const int nk = S.nk, ns = (int)S.sn_first.size();
    if (cut <= 0 || cut >= S.sn_nlevels || nk == 0) return false;
    std::vector<int> slev(ns, 0), sn_of(nk, 0), node_lvl(nk, 0), col_of_pos(S.nnzL, 0);
    for (int lv = 0; lv < S.sn_nlevels; lv++)
        for (int w = S.sn_lvl_ptr[lv]; w < S.sn_lvl_ptr[lv + 1]; w++) slev[S.sn_lvl_nodes[w]] = lv;
    for (int s = 0; s < ns; s++)
        for (int c = 0; c < S.sn_width[s]; c++) sn_of[S.sn_first[s] + c] = s;
    for (int lv = 0; lv < S.nlevels; lv++)
        for (int w = S.lvl_ptr[lv]; w < S.lvl_ptr[lv + 1]; w++) node_lvl[S.lvl_nodes[w]] = lv;
    for (int j = 0; j < nk; j++)
        for (int q = S.L_cp[j]; q < S.L_cp[j + 1]; q++) col_of_pos[q] = j;
    S.hy_is_top.assign(nk, 0);
    int ntop = 0, Lb = 0;
    for (int j = 0; j < nk; j++) {
        S.hy_is_top[j] = slev[sn_of[j]] >= cut ? 1 : 0;
        ntop += S.hy_is_top[j];
        if (!S.hy_is_top[j]) Lb = std::max(Lb, node_lvl[j] + 1);
    }
    if (ntop == 0 || ntop == nk) return false;
    for (int s = 0; s < ns; s++)
        if (slev[s] >= cut && (S.sn_nrows[s] > CONIC_SN_RMAX || S.sn_width[s] > CONIC_SN_WMAX)) return false;
    const std::vector<int> &top = S.hy_is_top;
    const int nl = Lb + 1;   // low levels 0..Lb-1, bridge level Lb
    auto tcol = [&](int t) { return t >= S.nnzL ? t - S.nnzL : col_of_pos[t]; };
    std::vector<int> rowpos(S.nnzL);
    for (int w = 0; w < S.nnzL; w++) rowpos[S.Lr_pos[w]] = w;

    // ---- factorisation: phase A items (target, op range), phase B items, per level ----
    S.hy_ft_op = S.ft_op;
    struct Tgt { int t, k0, k1; };
    std::vector<std::vector<Tgt>> lvl_tgts(nl);
    for (int lv = 0; lv < S.nlevels; lv++)
        for (int w = S.ft_lvl_ptr[lv]; w < S.ft_lvl_ptr[lv + 1]; w++) {
            const int t = S.ft_target[w], j = tcol(t);
            if (!top[j]) { lvl_tgts[lv].push_back({t, S.ft_op_ptr[w], S.ft_op_ptr[w + 1]}); continue; }
            const int k0 = (int)(S.hy_ft_op.size() / 2);
            for (int k = S.ft_op_ptr[w]; k < S.ft_op_ptr[w + 1]; k++)
                if (!top[col_of_pos[S.ft_op_a[k]]]) { S.hy_ft_op.push_back(S.ft_op[2 * (size_t)k]); S.hy_ft_op.push_back(S.ft_op[2 * (size_t)k + 1]); }
            const int k1 = (int)(S.hy_ft_op.size() / 2);
            if (k1 > k0) lvl_tgts[Lb].push_back({t, k0, k1});
        }
    {
        const int PF = CONIC_FACTOR_PF, SLOTS = 512, RMAX = 4;
        S.hy_fa_item.clear(); S.hy_fa_lvl.assign(nl + 1, 0); S.hy_fa_R.assign(nl, 1);
        S.hy_fb_item.clear(); S.hy_fb_lvl.assign(nl + 1, 0);
        for (int lv = 0; lv < nl; lv++) {
            int bestR = 1; long long bestp = -1, bestw = -1;
            for (int R = 1; R <= RMAX; R *= 2) {
                long long items = 0;
                for (const Tgt &g : lvl_tgts[lv]) items += (g.k1 - g.k0 + R * PF - 1) / (R * PF);
                const long long passes = (items * R + SLOTS - 1) / SLOTS, waste = items * R;
                if (bestp < 0 || passes < bestp || (passes == bestp && waste < bestw)) { bestp = passes; bestw = waste; bestR = R; }
            }
            S.hy_fa_R[lv] = bestR;
            const int cap = bestR * PF;
            for (const Tgt &g : lvl_tgts[lv]) {
                const int split = (g.k1 - g.k0 > cap) ? 1 : 0;
                for (int k = g.k0; k < g.k1; k += cap) {
                    S.hy_fa_item.push_back(g.t); S.hy_fa_item.push_back(k);
                    S.hy_fa_item.push_back(std::min(k + cap, g.k1)); S.hy_fa_item.push_back(split);
                }
            }
            S.hy_fa_lvl[lv + 1] = (int)(S.hy_fa_item.size() / 4);
            if (lv < S.nlevels && lv < Lb)
                for (int w = S.lvl_ptr[lv]; w < S.lvl_ptr[lv + 1]; w++) {
                    const int j = S.lvl_nodes[w];
                    if (top[j]) continue;
                    const int pos = (S.as_sign[S.nnzL + j] > 0) ? 1 : 0;
                    S.hy_fb_item.push_back(S.nnzL + j); S.hy_fb_item.push_back(j); S.hy_fb_item.push_back(0); S.hy_fb_item.push_back(pos | 2);
                    for (int q = S.L_cp[j]; q < S.L_cp[j + 1]; q++) {
                        S.hy_fb_item.push_back(q); S.hy_fb_item.push_back(j); S.hy_fb_item.push_back(rowpos[q]); S.hy_fb_item.push_back(pos);
                    }
                }
            S.hy_fb_lvl[lv + 1] = (int)(S.hy_fb_item.size() / 4);
        }
        if (S.hy_fa_item.empty()) S.hy_fa_item.assign(4, 0);
        conic_detail::number_pieces(S.hy_fa_item, S.hy_fa_lvl, S.hy_fc_item, S.hy_fslots);
        if (!conic_detail::combine_in_phase_b(S.hy_fa_item, S.hy_fa_lvl, S.hy_fc_item, S.hy_fb_item, S.hy_fb_lvl, S.hy_fb_cmb,
                                              S.nnzL + nk, S.nnzL, true)) {
            S.err = "internal: a split target of the hybrid factorisation is finished twice";
            return false;
        }
    }
    // ---- substitutions: (node, entry range) runs per level ----
    {
        const int PF = CONIC_SOLVE_PF, SLOTS = 512, RMAX = 4;
        struct Run { int i, k0, k1; };
        auto emit = [&](const std::vector<std::vector<Run>> &runs, std::vector<int> &item, std::vector<int> &lvl, std::vector<int> &Rl) {
            item.clear(); lvl.assign(nl + 1, 0); Rl.assign(nl, 1);
            for (int lv = 0; lv < nl; lv++) {
                int bestR = 1; long long bestp = -1, bestw = -1;
                for (int R = 1; R <= RMAX; R *= 2) {
                    long long items = 0;
                    for (const Run &r : runs[lv]) items += (r.k1 - r.k0 + R * PF - 1) / (R * PF);
                    const long long passes = (items * R + SLOTS - 1) / SLOTS, waste = items * R;
                    if (bestp < 0 || passes < bestp || (passes == bestp && waste < bestw)) { bestp = passes; bestw = waste; bestR = R; }
                }
                Rl[lv] = bestR;
                const int cap = bestR * PF;
                // a node whose entries end up in more than one item (long run, or several runs) is a split target
                std::vector<int> nitems(nk, 0);
                for (const Run &r : runs[lv]) nitems[r.i] += (r.k1 - r.k0 + cap - 1) / cap;
                for (const Run &r : runs[lv])
                    for (int k = r.k0; k < r.k1; k += cap) {
                        item.push_back(r.i); item.push_back(k); item.push_back(std::min(k + cap, r.k1)); item.push_back(nitems[r.i] > 1 ? 1 : 0);
                    }
                lvl[lv + 1] = (int)(item.size() / 4);
            }
            if (item.empty()) item.assign(4, 0);
        };
        std::vector<std::vector<Run>> fr(nl), br(nl);
        for (int i = 0; i < nk; i++) {
            if (!top[i]) {
                if (S.Lr_rp[i + 1] > S.Lr_rp[i]) fr[node_lvl[i]].push_back({i, S.Lr_rp[i], S.Lr_rp[i + 1]});
                if (S.L_cp[i + 1] > S.L_cp[i]) br[node_lvl[i]].push_back({i, S.L_cp[i], S.L_cp[i + 1]});
                continue;
            }
            // top row: the runs of LOW columns (the top columns reach it through the panel sweeps)
            int k = S.Lr_rp[i];
            const int ke = S.Lr_rp[i + 1];
            while (k < ke) {
                while (k < ke && top[S.Lr_col[k]]) k++;
                const int k0 = k;
                while (k < ke && !top[S.Lr_col[k]]) k++;
                if (k > k0) fr[Lb].push_back({i, k0, k});
            }
        }
        emit(fr, S.hy_fwp_item, S.hy_fwp_lvl, S.hy_fwp_R);
        emit(br, S.hy_bwp_item, S.hy_bwp_lvl, S.hy_bwp_R);
        int fw_ = 0, bw_ = 0;
        conic_detail::number_pieces(S.hy_fwp_item, S.hy_fwp_lvl, S.hy_fwc_item, fw_);
        conic_detail::number_pieces(S.hy_bwp_item, S.hy_bwp_lvl, S.hy_bwc_item, bw_);
        S.hy_sslots = std::max(fw_, bw_);
        S.npart = std::max(S.npart, std::max(S.hy_fslots, S.hy_sslots));
    }
    // ---- top supernodes: descriptors in level order, update scatter lists as target ids ----
    {
        auto lpos = [&](int i, int j) -> int {
            auto b = S.L_ri.begin() + S.L_cp[j], e = S.L_ri.begin() + S.L_cp[j + 1];
            auto it = std::lower_bound(b, e, i);
            return (it != e && *it == i) ? (int)(it - S.L_ri.begin()) : -1;
        };
        const int ntl = S.sn_nlevels - cut;
        S.hy_tl_ptr.assign(ntl + 1, 0); S.hy_desc.clear(); S.hy_upd_dst.clear();
        for (int tl = 0; tl < ntl; tl++) {
            for (int w_ = S.sn_lvl_ptr[cut + tl]; w_ < S.sn_lvl_ptr[cut + tl + 1]; w_++) {
                const int s = S.sn_lvl_nodes[w_], a = S.sn_first[s], w = S.sn_width[s], R = S.sn_nrows[s];
                for (int c = 0; c + 1 < w; c++)   // the closed-form panel addressing needs consecutive CSC columns
                    if (S.L_cp[a + c + 1] - S.L_cp[a + c] != R - c - 1) { S.err = "internal: top supernode is not a dense trapezoid"; return false; }
                int sign = 0;
                for (int c = 0; c < w; c++) sign |= (S.as_sign[(size_t)S.nnzL + a + c] > 0 ? 1 : 0) << c;
                const int *below = &S.sn_rows[S.sn_rows_ptr[s] + w];
                const int u0 = (int)S.hy_upd_dst.size();
                for (int y = 0; y < R - w; y++)
                    for (int x = y; x < R - w; x++) {
                        const int t = (x == y) ? S.nnzL + below[y] : lpos(below[x], below[y]);
                        if (t < 0) { S.err = "internal: hybrid update falls outside the L pattern"; return false; }
                        S.hy_upd_dst.push_back(t);
                    }
                const int d[8] = {a, w, R, S.L_cp[a], S.sn_rows_ptr[s], u0, sign, 0};
                S.hy_desc.insert(S.hy_desc.end(), d, d + 8);
            }
            S.hy_tl_ptr[tl + 1] = (int)(S.hy_desc.size() / 8);
        }
        S.hy_desc.resize(S.hy_desc.size() + 8, 0);
        S.hy_ntl = ntl;
    }
    S.hy_nlevels = nl;
    S.hy_cut = cut;
    return true;
}

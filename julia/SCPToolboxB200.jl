#= SCPToolboxB200.jl -- thin ccall glue over libscpb (include/scpb.h).

NOT EXECUTABLE IN THE BUILD IMAGE (no Julia).  Kept mechanically obvious: one wrapper per C entry point, no logic.
See INTEGRATION.md for where each call replaces reference code. =#
module SCPToolboxB200

const libscpb = joinpath(@__DIR__, "..", "scptoolbox.jl_b200", "libscpb.so")

# device model packs, the `id` of model_set! (SCPB_MODEL_*, include/scpb.h)
const MODEL_DBLINT, MODEL_ROCKET, MODEL_STARSHIP, MODEL_QUADROTOR, MODEL_FREEFLYER, MODEL_RENDEZVOUS2D = 1, 2, 3, 4, 5, 6
const MODEL_OSCILLATOR = 7    # fixed final time (no F column); np = N, one l1r slack per node

mutable struct Handle
    ptr::Ptr{Cvoid}
end

function Handle(device::Integer = 0)
    out = Ref{Ptr{Cvoid}}(C_NULL)
    rc = ccall((:scpb_create, libscpb), Int32, (Int32, Ptr{Ptr{Cvoid}}), device, out)
    rc == 0 || error("scpb_create failed ($rc): no usable CUDA device")
    h = Handle(out[])
    finalizer(x -> ccall((:scpb_destroy, libscpb), Int32, (Ptr{Cvoid},), x.ptr), h)
    return h
end

function last_error(h::Handle)
    buf = Vector{UInt8}(undef, 512)
    ccall((:scpb_last_error, libscpb), Int32, (Ptr{Cvoid}, Ptr{UInt8}, Csize_t), h.ptr, buf, 512)
    return unsafe_string(pointer(buf))
end

check(h::Handle, rc::Int32, what) = rc == 0 || error("$what failed ($rc): $(last_error(h))")

model_set!(h::Handle, id::Integer, par::Vector{Float64}, nx, nu, np) = check(h,
    ccall((:scpb_model_set, libscpb), Int32, (Ptr{Cvoid}, Int32, Ptr{Float64}, Int32, Int32, Int32, Int32),
          h.ptr, id, par, length(par), nx, nu, np), "scpb_model_set")

""" discretize!: arrays are Julia column-major `xd[nx,N,B]`, `A[nx,nx,N-1,B]`, ... (B = 1 ⇒ the fields of `ref`). """
function discretize!(h::Handle, t_grid, xd, ud, p, iSx, feas_tol, Nsub, A, Bm, Bp, F, r, E, defect, feas::Vector{Int32})
    N = length(t_grid); B = length(feas); secs = Ref{Float64}(0.0)
    check(h, ccall((:scpb_discretize, libscpb), Int32,
        (Ptr{Cvoid}, Int32, Int32, Int32, Int32, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
         Float64, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
         Ptr{Int32}, Ptr{Float64}),
        h.ptr, 0, B, N, Nsub, t_grid, xd, ud, p, iSx, feas_tol, A, Bm, Bp, F, r, E, defect, feas, secs), "scpb_discretize")
    return secs[]
end

# propagate(sol, pbm; res) (src/solvers/discretization.jl:515-562, FOH): returns the nx x res matrix of xc values
function propagate(h::Handle, N, res, t_grid, xd, ud, p)
    xc = Matrix{Float64}(undef, size(xd, 1), res)
    secs = Ref{Float64}(0.0)
    check(h, ccall((:scpb_propagate, libscpb), Int32,
        (Ptr{Cvoid}, Int32, Int32, Int32, Int32, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
         Ptr{Float64}), h.ptr, 0, 1, N, res, t_grid, xd, ud, p, xc, secs), "scpb_propagate")
    return xc
end

struct ConeOpts
    feastol::Float64; abstol::Float64; reltol::Float64; delta::Float64; delta_dyn::Float64
    maxit::Int32; nref::Int32; verbose::Int32; group::Int32; equil::Int32; threads::Int32; lanes::Int32
end   # field order and types mirror scpb_cone_opts (include/scpb.h)
ConeOpts(; maxit = 0, verbose = 0) = ConeOpts(0, 0, 0, 0, 0, maxit, -1, verbose, 0, -1, 0, 0)

function cone_setup(h::Handle, n, p, m, A_rp, A_ci, G_rp, G_ci, l, soc_dims::Vector{Int32}, perm)
    out = Ref{Ptr{Cvoid}}(C_NULL)
    check(h, ccall((:scpb_cone_setup, libscpb), Int32,
        (Ptr{Cvoid}, Int32, Int32, Int32, Ptr{Int32}, Ptr{Int32}, Ptr{Int32}, Ptr{Int32}, Int32, Int32, Ptr{Int32},
         Ptr{Int32}, Ptr{Ptr{Cvoid}}), h.ptr, n, p, m, A_rp, A_ci, G_rp, G_ci, l, length(soc_dims), soc_dims, perm, out),
        "scpb_cone_setup")
    return out[]
end

function cone_solve(h::Handle, cone, B, Av, Gv, c, b, hh, opts::ConeOpts, x, y, z, s, pobj, dobj, status, iters)
    secs = Ref{Float64}(0.0)
    check(h, ccall((:scpb_cone_solve, libscpb), Int32,
        (Ptr{Cvoid}, Int32, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ref{ConeOpts},
         Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Int32},
         Ptr{Float64}), cone, B, Av, Gv, c, b, hh, opts, x, y, z, s, pobj, dobj, status, iters, secs), "scpb_cone_solve")
    return secs[]
end

cone_free(cone) = ccall((:scpb_cone_free, libscpb), Int32, (Ptr{Cvoid},), cone)

# scpb_scvx_attach / scpb_scvx_solve (SCvx.solve for a batch, src/solvers/scvx.jl:460-546): the descriptor mirrors
# scpb_scvx_desc; Q holds the rows of the original cost and of g_ic / g_tc over the scaled solver variables
struct ScvxDesc
    lam::Float64; rho_0::Float64; rho_1::Float64; rho_2::Float64; beta_sh::Float64; beta_gr::Float64
    eta_init::Float64; eta_lb::Float64; eta_ub::Float64
    oeta::Int32; n_ic::Int32; n_tc::Int32; reserved::Int32
end

function scvx_attach(h::Handle, ptr, desc::ScvxDesc, Q_rp::Vector{Int32}, Q_ci::Vector{Int32}, Q_v::Vector{Float64},
                     Q_c::Vector{Float64})
    check(h, ccall((:scpb_scvx_attach, libscpb), Int32,
        (Ptr{Cvoid}, Ref{ScvxDesc}, Ptr{Int32}, Ptr{Int32}, Ptr{Float64}, Ptr{Float64}), ptr, desc, Q_rp, Q_ci, Q_v, Q_c),
        "scpb_scvx_attach")
end

function scvx_solve(h::Handle, ptr, B, xd0, ud0, p0, opts::ConeOpts, xd, ud, p, status, iters, J, dev, feas, eta, timing)
    check(h, ccall((:scpb_scvx_solve, libscpb), Int32,
        (Ptr{Cvoid}, Int32, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ref{ConeOpts}, Ptr{Float64}, Ptr{Float64},
         Ptr{Float64}, Ptr{Int32}, Ptr{Int32}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Float64}, Ptr{Float64}),
        ptr, B, xd0, ud0, p0, opts, xd, ud, p, status, iters, J, dev, feas, eta, timing), "scpb_scvx_solve")
end

# scpb_ptr_setup / scpb_ptr_solve / scpb_ptr_free (PTR.solve for a batch, src/solvers/ptr.jl:448-532).  The descriptor
# mirrors scpb_ptr_desc field by field (28 Int32 + 3 Float64 + 1 Int32; Julia lays isbits structs out like C).
# method: 0 = FOH, 1 = IMPULSE (PTR only, a model pack with impulse semantics).
struct PtrDesc
    N::Int32; Nsub::Int32; nx::Int32; nu::Int32; np::Int32; ns::Int32; nf::Int32
    nsrc::Int32; oA::Int32; oBm::Int32; oBp::Int32; oF::Int32; or_::Int32; oE::Int32; oC::Int32; oD::Int32; oG::Int32
    ors::Int32; oxh::Int32; ouh::Int32; oph::Int32
    nval::Int32; vx::Int32; vu::Int32; vp::Int32
    q_exit::Int32; iter_max::Int32; ng::Int32
    eps_abs::Float64; eps_rel::Float64; feas_tol::Float64
    method::Int32
end

function ptr_setup(h::Handle, cone, desc::PtrDesc, W_rp::Vector{Int32}, W_ci::Vector{Int32}, W_v::Vector{Float64},
                   scale::Vector{Float64}, t_grid::Vector{Float64})
    out = Ref{Ptr{Cvoid}}(C_NULL)
    check(h, ccall((:scpb_ptr_setup, libscpb), Int32,
        (Ptr{Cvoid}, Ptr{Cvoid}, Ref{PtrDesc}, Ptr{Int32}, Ptr{Int32}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
         Ptr{Ptr{Cvoid}}), h.ptr, cone, desc, W_rp, W_ci, W_v, scale, t_grid, out), "scpb_ptr_setup")
    return out[]
end

# xd0[nx,N,B], ud0[nu,N,B], p0[np,B] in Julia's column-major layout are exactly the (B,N,nx) row-major arrays of the C ABI
function ptr_solve(h::Handle, ptr, B, xd0, ud0, p0, opts::ConeOpts, xd, ud, p, status::Vector{Int32}, iters::Vector{Int32},
                   J::Vector{Float64}, dev::Vector{Float64}, feas::Vector{Int32}, timing::Vector{Float64})
    length(timing) >= 10 || throw(ArgumentError("timing needs 10 entries (include/scpb.h)"))
    check(h, ccall((:scpb_ptr_solve, libscpb), Int32,
        (Ptr{Cvoid}, Int32, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ref{ConeOpts}, Ptr{Float64}, Ptr{Float64},
         Ptr{Float64}, Ptr{Int32}, Ptr{Int32}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Float64}),
        ptr, B, xd0, ud0, p0, opts, xd, ud, p, status, iters, J, dev, feas, timing), "scpb_ptr_solve")
end

ptr_free(ptr) = ccall((:scpb_ptr_free, libscpb), Int32, (Ptr{Cvoid},), ptr)

# scpb_ptr_set_par: the model parameter block for the next ptr_solve calls of this problem, e.g. after
# `mdl.traj.κ = hom_κ(x)` between two solves of a homotopy (test/examples/rendezvous_planar/tests.jl:66-78)
ptr_set_par(h::Handle, ptr, par::Vector{Float64}) =
    check(h, ccall((:scpb_ptr_set_par, libscpb), Int32, (Ptr{Cvoid}, Ptr{Float64}, Int32), ptr, par, length(par)),
          "scpb_ptr_set_par")

# scpb_ptr_set_homotopy / _beta / scpb_ptr_homotopy_result: the in-loop homotopy schedule that replaces a
# problem_set_callback! stepping the pack's kappa through `grid` inside one solve (rendezvous_3d/definition.jl:96-151).
# par_index is 0-based (the rendezvous pack's kappa is par[7]; -1 takes the pack's own slot); an empty grid detaches it.  The history
# matrices are cap x B in Julia's column-major layout (the C ABI's [B][cap]).
ptr_set_homotopy(h::Handle, ptr, par_index::Integer, grid::Vector{Float64}, worsen_tol::Float64 = -1e-3) =
    check(h, ccall((:scpb_ptr_set_homotopy, libscpb), Int32, (Ptr{Cvoid}, Int32, Int32, Ptr{Float64}, Float64),
                   ptr, par_index, length(grid), grid, worsen_tol), "scpb_ptr_set_homotopy")

ptr_set_homotopy_beta(h::Handle, ptr, beta::Vector{Float64}) =
    check(h, ccall((:scpb_ptr_set_homotopy_beta, libscpb), Int32, (Ptr{Cvoid}, Int32, Ptr{Float64}),
                   ptr, length(beta), beta), "scpb_ptr_set_homotopy_beta")

function ptr_homotopy_result(h::Handle, ptr, B::Integer, cap::Integer)
    hom_index = Vector{Int32}(undef, B); iter_max = Vector{Int32}(undef, B)
    hist_index = Matrix{Int32}(undef, cap, B); hist_improv = Matrix{Float64}(undef, cap, B)
    check(h, ccall((:scpb_ptr_homotopy_result, libscpb), Int32,
        (Ptr{Cvoid}, Int32, Ptr{Int32}, Ptr{Int32}, Int32, Ptr{Int32}, Ptr{Float64}),
        ptr, B, hom_index, iter_max, cap, hist_index, hist_improv), "scpb_ptr_homotopy_result")
    return hom_index, iter_max, hist_index, hist_improv
end

# scpb_gusto_attach / scpb_gusto_solve (GuSTO.solve for a batch, src/solvers/gusto.jl:425-502, pen = :quad)
struct GustoDesc
    lam_init::Float64; lam_max::Float64; rho_0::Float64; rho_1::Float64; beta_sh::Float64; beta_gr::Float64
    gamma_fail::Float64; eta_init::Float64; eta_lb::Float64; eta_ub::Float64; mu::Float64
    iter_mu::Int32; q_tr::Int32; oeta::Int32; olam::Int32; nsq::Int32; reserved::Int32
end

function gusto_attach(h::Handle, ptr, desc::GustoDesc, Q_rp::Vector{Int32}, Q_ci::Vector{Int32}, Q_v::Vector{Float64},
                      Q_c::Vector{Float64}, Q_w::Vector{Float64})
    check(h, ccall((:scpb_gusto_attach, libscpb), Int32,
        (Ptr{Cvoid}, Ref{GustoDesc}, Ptr{Int32}, Ptr{Int32}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}),
        ptr, desc, Q_rp, Q_ci, Q_v, Q_c, Q_w), "scpb_gusto_attach")
end

function gusto_solve(h::Handle, ptr, B, xd0, ud0, p0, opts::ConeOpts, xd, ud, p, status, iters, J, dev, feas, eta, lam, timing)
    check(h, ccall((:scpb_gusto_solve, libscpb), Int32,
        (Ptr{Cvoid}, Int32, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ref{ConeOpts}, Ptr{Float64}, Ptr{Float64},
         Ptr{Float64}, Ptr{Int32}, Ptr{Int32}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Float64}, Ptr{Float64},
         Ptr{Float64}), ptr, B, xd0, ud0, p0, opts, xd, ud, p, status, iters, J, dev, feas, eta, lam, timing),
        "scpb_gusto_solve")
end

# ------------------------------------------------------------------------------------------------------------------
# MathOptInterface shim: `solver = SCPToolboxB200` in PTR / SCvx / GuSTO Parameters makes the reference's own
# `set_optimizer(mdl, solver.Optimizer)` (src/parser/program.jl:70-76, 419-424) route every subproblem through
# scpb_cone_solve with B = 1 -- the existing examples run unchanged.  Same cone set as ECOS.jl's wrapper declares
# (Zeros, Nonnegatives, SecondOrderCone over VectorAffineFunction; linear objective); the exponential cone of the
# reference's GEOM / EXP cones (cone.jl:149-165) is not supported and JuMP reports it at model-build time.
# Written against MathOptInterface 1.x (the version ECOS.jl 1.1 of the reference's Manifest pins); not executable in the
# build image (no Julia).
import MathOptInterface
const MOI = MathOptInterface
const MOIU = MOI.Utilities
using SparseArrays

MOIU.@product_of_sets(Cones, MOI.Zeros, MOI.Nonnegatives, MOI.SecondOrderCone)

const OptimizerCache = MOIU.GenericModel{Float64, MOIU.ObjectiveContainer{Float64}, MOIU.VariablesContainer{Float64},
    MOIU.MatrixOfConstraints{Float64, MOIU.MutableSparseMatrixCSC{Float64, Int, MOIU.OneBasedIndexing}, Vector{Float64},
                             Cones{Float64}}}

const _STATUS = Dict{Int32, Tuple{MOI.TerminationStatusCode, MOI.ResultStatusCode, String}}(   # SCPB_CONE_* (include/scpb.h)
    0 => (MOI.OPTIMAL, MOI.FEASIBLE_POINT, "OPTIMAL"),
    1 => (MOI.ITERATION_LIMIT, MOI.UNKNOWN_RESULT_STATUS, "ITERATION_LIMIT"),
    2 => (MOI.NUMERICAL_ERROR, MOI.UNKNOWN_RESULT_STATUS, "NUMERICAL_ERROR"),
    3 => (MOI.ALMOST_OPTIMAL, MOI.NEARLY_FEASIBLE_POINT, "ALMOST_OPTIMAL"),
    4 => (MOI.INFEASIBLE, MOI.NO_SOLUTION, "INFEASIBLE"),
    5 => (MOI.DUAL_INFEASIBLE, MOI.NO_SOLUTION, "DUAL_INFEASIBLE"))

mutable struct Optimizer <: MOI.AbstractOptimizer
    handle::Union{Nothing, Handle}
    cone::Ptr{Cvoid}
    pattern::UInt                      # hash of the (A, G) sparsity pattern the cone object was set up for
    options::Dict{String, Any}
    silent::Bool
    x::Vector{Float64}; pobj::Float64; dobj::Float64; status::Int32; iters::Int32; seconds::Float64
    obj_sign::Float64; obj_const::Float64
    Optimizer() = new(nothing, C_NULL, UInt(0), Dict{String, Any}(), false, Float64[], NaN, NaN, Int32(-1), Int32(0), 0.0, 1.0, 0.0)
end

MOI.get(::Optimizer, ::MOI.SolverName) = "SCPToolboxB200 (libscpb)"
MOI.is_empty(o::Optimizer) = o.status == -1
function MOI.empty!(o::Optimizer)
    o.x = Float64[]; o.status = Int32(-1); o.pobj = NaN; o.dobj = NaN
    return
end
MOI.supports(::Optimizer, ::MOI.Silent) = true
MOI.set(o::Optimizer, ::MOI.Silent, v::Bool) = (o.silent = v)
MOI.get(o::Optimizer, ::MOI.Silent) = o.silent
MOI.supports(::Optimizer, ::MOI.RawOptimizerAttribute) = true      # "maxit", "verbose", "feastol", "abstol", "reltol"
MOI.set(o::Optimizer, a::MOI.RawOptimizerAttribute, v) = (o.options[a.name] = v)
MOI.get(o::Optimizer, a::MOI.RawOptimizerAttribute) = o.options[a.name]
MOI.supports(::Optimizer, ::MOI.ObjectiveSense) = true
MOI.supports(::Optimizer, ::MOI.ObjectiveFunction{MOI.ScalarAffineFunction{Float64}}) = true
MOI.supports_constraint(::Optimizer, ::Type{MOI.VectorAffineFunction{Float64}},
                        ::Type{<:Union{MOI.Zeros, MOI.Nonnegatives, MOI.SecondOrderCone}}) = true

_csr(M::SparseMatrixCSC) = (Mt = sparse(M'); (Int32.(Mt.colptr .- 1), Int32.(Mt.rowval .- 1), Mt.nzval))

function MOI.optimize!(o::Optimizer, src::MOI.ModelLike)
    cache = OptimizerCache()
    index_map = MOI.copy_to(cache, src)
    Ab = cache.constraints
    M = convert(SparseMatrixCSC{Float64, Int}, Ab.coefficients)      # rows in the order Zeros | Nonnegatives | SOC ...
    bconst = Ab.constants
    nz = MOIU.num_rows(Ab.sets, MOI.Zeros)
    nl = MOIU.num_rows(Ab.sets, MOI.Nonnegatives)
    socs = MOI.get(cache, MOI.ListOfConstraintIndices{MOI.VectorAffineFunction{Float64}, MOI.SecondOrderCone}())
    q = Int32[MOI.dimension(MOI.get(cache, MOI.ConstraintSet(), ci)) for ci in socs]
    n = size(M, 2); m = size(M, 1) - nz
    # f(x) = M x + b in K  <=>  A x = -b_zeros ;  G x + s = h with G = -M_cone, h = b_cone, s in K
    A = M[1:nz, :]; G = -M[nz+1:end, :]
    b = -bconst[1:nz]; hv = bconst[nz+1:end]
    sense = MOI.get(cache, MOI.ObjectiveSense())
    o.obj_sign = sense == MOI.MAX_SENSE ? -1.0 : 1.0
    c = zeros(n); o.obj_const = 0.0
    if sense != MOI.FEASIBILITY_SENSE
        f = MOI.get(cache, MOI.ObjectiveFunction{MOI.ScalarAffineFunction{Float64}}())
        for t in f.terms
            c[t.variable.value] += o.obj_sign * t.coefficient
        end
        o.obj_const = f.constant
    end
    o.handle === nothing && (o.handle = Handle(get(o.options, "device", 0)))
    h = o.handle
    A_rp, A_ci, A_v = _csr(A); G_rp, G_ci, G_v = _csr(G)
    pat = hash((A_rp, A_ci, G_rp, G_ci, nl, q))
    if o.cone == C_NULL || pat != o.pattern        # one symbolic analysis per sparsity pattern (the SCP loop reuses it)
        o.cone != C_NULL && cone_free(o.cone)
        perm = zeros(Int32, n + nz)                # no stage information here: reverse Cuthill-McKee (scpb_order_rcm)
        check(h, ccall((:scpb_order_rcm, libscpb), Int32, (Int32, Int32, Int32, Ptr{Int32}, Ptr{Int32}, Ptr{Int32},
              Ptr{Int32}, Int32, Int32, Ptr{Int32}, Ptr{Int32}), n, nz, m, A_rp, A_ci, G_rp, G_ci, nl, length(q), q, perm),
              "scpb_order_rcm")
        o.cone = cone_setup(h, n, nz, m, A_rp, A_ci, G_rp, G_ci, nl, q, perm)
        o.pattern = pat
    end
    opts = ConeOpts(Float64(get(o.options, "feastol", 0.0)), Float64(get(o.options, "abstol", 0.0)),
                    Float64(get(o.options, "reltol", 0.0)), 0.0, 0.0, Int32(get(o.options, "maxit", 0)), Int32(-1),
                    Int32(get(o.options, "verbose", 0)), Int32(1), Int32(-1), Int32(0), Int32(0))
    x = zeros(n); y = zeros(nz); z = zeros(m); s = zeros(m)
    pobj = zeros(1); dobj = zeros(1); st = zeros(Int32, 1); it = zeros(Int32, 1)
    o.seconds = cone_solve(h, o.cone, 1, A_v, G_v, c, b, hv, opts, x, y, z, s, pobj, dobj, st, it)
    o.x = x; o.pobj = pobj[1]; o.dobj = dobj[1]; o.status = st[1]; o.iters = it[1]
    return index_map, false
end

MOI.get(o::Optimizer, ::MOI.TerminationStatus) = o.status < 0 ? MOI.OPTIMIZE_NOT_CALLED : _STATUS[o.status][1]
MOI.get(o::Optimizer, ::MOI.RawStatusString) = o.status < 0 ? "not called" : _STATUS[o.status][3]
MOI.get(o::Optimizer, a::MOI.PrimalStatus) = (a.result_index == 1 && o.status >= 0) ? _STATUS[o.status][2] : MOI.NO_SOLUTION
MOI.get(o::Optimizer, ::MOI.DualStatus) = MOI.NO_SOLUTION          # the SCP loops read primal values only
MOI.get(o::Optimizer, ::MOI.ResultCount) = o.status in (0, 3) ? 1 : 0
MOI.get(o::Optimizer, ::MOI.ObjectiveValue) = o.obj_sign * o.pobj + o.obj_const
MOI.get(o::Optimizer, ::MOI.DualObjectiveValue) = o.obj_sign * o.dobj + o.obj_const
MOI.get(o::Optimizer, ::MOI.SolveTimeSec) = o.seconds
MOI.get(o::Optimizer, ::MOI.BarrierIterations) = Int64(o.iters)
MOI.get(o::Optimizer, ::MOI.VariablePrimal, vi::MOI.VariableIndex) = o.x[vi.value]

end # module

// myo_layout.cuh -- the per-warp shared-memory layout as a function of the model's shape, and the compile-time model shapes of the
// specialised step kernels.  One function decides the layout: the host evaluates it for every batch (fill_devmodel), the compiler for
// every static shape, so that a specialised kernel and the host agree on every offset by construction.
#pragma once
#include "myo_solver.cuh"

__host__ __device__ constexpr int al2(int x) { return (x + 1) & ~1; }
__host__ __device__ constexpr int imax(int a, int b) { return a > b ? a : b; }

// What the layout decided beyond the DevModel offsets (myo_model_layout): the size reserved for every persistent and scratch region
// (slot orders of include/myo_b200.h) and the boundaries and flags of the scratch scheme, the latter relative to the scratch start.
#define LP_ENUM(n) LP_##n,
#define LS_ENUM(n) LS_##n,
enum { MYO_LAYOUT_PERSISTENT(LP_ENUM) LP_N };
enum { MYO_LAYOUT_SCRATCH(LS_ENUM) LS_N };
#undef LP_ENUM
#undef LS_ENUM
struct Layout { int32_t psz[LP_N], ssz[LS_N], head, afterK, extNonSolve, solveEnd, arefInH, qwsInH; };

// Everything the layout depends on: the model's dimensions, the sizes of its kernel program (P_dims), the per-task overrides and the
// requested contact capacity (0: the default).  The field order is that of myosuite_b200/shape.py (MODEL_DIMS), which generates the
// static shapes' initialisers.
struct ModelDims {
  int32_t nq, nv, nu, na, nM, njnt;
  int32_t nbd, nlevel, nsp, nwe, nta, nnz, nlim, neq, npair, npair_an, maxpath, ndepth, eq_tree, ngc, nwz, nlimrow;
  int32_t split_sp, split_we, split_ta, split_nz;      // tendon group A's share of the segments, wrap elements, tendons and moment non-zeros
  int32_t neprm, ovr_geom;                             // per-env model overrides (hold task: 8 values; the geom whose size they give, else -1)
  int32_t maxcon;
};
struct ModelLayout { DevModel d; Layout L; };

// The dimensions and per-warp offsets of a DevModel for shape x (the other fields zero), and the region sizes behind them
__host__ __device__ constexpr ModelLayout model_layout(const ModelDims& x) {
  ModelLayout r{}; DevModel& d = r.d; Layout& L = r.L;
  d.nq = x.nq; d.nv = x.nv; d.nu = x.nu; d.na = x.na; d.nM = x.nM; d.njnt = x.njnt;
  d.nbd = x.nbd; d.nlevel = x.nlevel; d.nsp = x.nsp; d.nwe = x.nwe; d.nta = x.nta; d.nnz = x.nnz; d.nlim = x.nlim; d.neq = x.neq;
  { const int sp_[3] = {0, x.split_sp, d.nsp}, we_[3] = {0, x.split_we, d.nwe}, ta_[3] = {0, x.split_ta, d.nta}, nz_[3] = {0, x.split_nz, d.nnz};
    for (int k = 0; k < 3; k++) { d.tg_sp[k] = sp_[k]; d.tg_we[k] = we_[k]; d.tg_ta[k] = ta_[k]; d.tg_nz[k] = nz_[k]; } }
  d.npair = x.npair; d.npair_an = x.npair_an; d.maxpath = x.maxpath; d.ndepth = x.ndepth; d.eq_tree = x.eq_tree;
  d.ovr_geom = x.ovr_geom;
  int mc = x.maxcon > 0 ? x.maxcon : 32; if (mc > 64) mc = 64; if (mc > 2*d.npair) mc = 2*d.npair; /* (the contact-order merge handles up to 64) */ d.maxcon = mc; d.nlimrow = x.nlimrow > 0 ? x.nlimrow : 2*d.nlim; d.maxefc = d.neq + d.nlimrow + 4*mc;
  int o = 0;
  #define TAKE(field, n) d.o_##field = o; L.psz[LP_##field] = al2(n); o += al2(n)
  // persistent per-env arrays.  ctrl is NOT here: it is written once per control step to a library-owned global row and re-read by the actuation
  // phase of every substep (an L2 hit); the solver's warm start lives in the tail of the Hessian region when that tail is provably idle (below).
  TAKE(qpos, d.nq); TAKE(qvel, d.nv); TAKE(act, d.na); TAKE(dax, 3*d.nv); TAKE(dan, 3*d.nv); TAKE(qM, d.nM); TAKE(fsm, d.nv);
  d.neprm = x.neprm; TAKE(eprm, d.neprm); d.nwz = x.nwz; TAKE(wz, d.nwz); TAKE(cnt, CNT_N/2);
  d.nvp = chol_pad(d.nv); L.psz[LP_qws] = al2(d.nv);
  const int o_qws_persistent = o;          // (claimed only if the warm start cannot alias the Hessian tail)
  // ---- scratch, time-multiplexed by stage (offsets from d.o_scr, fixed up at the end).  Lifetimes:
  //   head: icon (contact / row integer records), con (contact records)     collision .. constraints ; in the solve the con region holds jar, jv
  //   K   (xpos, xmat)                                                      kinematics .. collision              -> right after the head
  //   T   (U, PL, mom, tlen, tvel, tfrc)                                    tendon .. actuation                  -> around K
  //   C   (cin, crb, bf)                                                    body inertia .. bias                 -> around K
  //   G   (gpose, clist)                                                    collision                            -> after K
  //   S   (conJ 48-bit, D, eqJ, a, g|p, Ma, Mp, H | Hs LD Dinv, aref->H)   constraints .. integrate             -> after the head (K is dead)
  const int icon = al2(mc + (mc + 1)/2 + (2*(mc + d.nlimrow + 4) + d.maxefc + 7)/8);       // cmask u64[mc] | crown i32[mc] | cpair i16[mc] | lrow i16[nlimrow+4] | drow u8[maxefc]
  const int rows = al2(d.maxefc), conReg = imax(al2(CON_STRIDE*mc), 2*rows), K = al2(3*d.nbd) + al2(9*d.nbd);
  d.s_icon = 0; d.s_con = icon; d.s_efR = icon; d.s_efV = icon + rows; const int head = icon + conReg;
  L.ssz[LS_icon] = icon; L.ssz[LS_con] = conReg; L.ssz[LS_efR] = rows; L.ssz[LS_efV] = rows;
  d.s_xpos = head; d.s_xmat = head + al2(3*d.nbd); const int afterK = head + K; L.ssz[LS_xpos] = al2(3*d.nbd); L.ssz[LS_xmat] = al2(9*d.nbd);
  int c0 = 0, c1 = 0, ext = 0;      // two cursors: inside [0, head) and after K
  #define PLACE(field, n) { const int n_ = al2(n); L.ssz[LS_##field] = n_; if (c0 + n_ <= head) { d.s_##field = c0; c0 += n_; } else { d.s_##field = c1; c1 += n_; } }
  c0 = 0; c1 = afterK;
  PLACE(mom, d.nnz); PLACE(tlen, d.nta); PLACE(tvel, d.nta); PLACE(tfrc, d.nta); { const int nsA = d.tg_sp[1], nsB = d.nsp - nsA, nwA = d.tg_we[1], nwB = d.nwe - nwA;      // one tendon group at a time lives in U / PL
    PLACE(PL, imax(nsA + nwA, nsB + nwB)); PLACE(U, 3*imax(nsA + 2*nwA, nsB + 2*nwB)); }
  ext = c1;
  c0 = 0; c1 = afterK;
  PLACE(cin, 10*d.nbd); PLACE(crb, 10*d.nbd); PLACE(bf, 6*d.nbd);
  ext = imax(ext, c1);
  d.kcand = d.npair - d.npair_an; d.ngc = x.ngc;
  d.s_gpose = afterK; d.s_clist = afterK + al2(6*d.ngc); ext = imax(ext, d.s_clist + al2((d.kcand + 1)/2)); L.ssz[LS_gpose] = al2(6*d.ngc); L.ssz[LS_clist] = al2((d.kcand + 1)/2);
  ext = imax(ext, d.s_gpose + al2(2*d.njnt));      // the hinge sines / cosines of the kinematics phase (phase_kinematics)
  const int extNonSolve = ext;
  int t = head;
  L.ssz[LS_conJ] = al2(imax((3*d.maxpath*mc*JAC_BYTES + 7)/8, (mc + 1)/2)); L.ssz[LS_efD] = al2(d.neq + d.nlimrow + mc); L.ssz[LS_eqJ] = al2(d.neq);
  d.s_conJ = t; t += L.ssz[LS_conJ]; d.s_efD = t; t += L.ssz[LS_efD]; d.s_eqJ = t; t += L.ssz[LS_eqJ];      /* (the Jacobian region doubles as the int rank keys of the contact ordering) */
  d.s_va = t; t += al2(d.nvp); d.s_vg = t; d.s_vp = t; t += al2(d.nvp); d.s_vMa = t; t += al2(d.nvp); d.s_vMp = t; t += al2(d.nvp);
  L.ssz[LS_va] = L.ssz[LS_vg] = L.ssz[LS_vp] = L.ssz[LS_vMa] = L.ssz[LS_vMp] = al2(d.nvp);
  const int hsize = imax(al2(d.nvp*(d.nvp+1)/2), 2*al2(d.nM) + al2(d.nv)); const bool arefInH = rows <= hsize;
  d.s_efA = t; if (!arefInH) t += rows;      /* aref (constraints -> start of the solve) lives in the Hessian region when it fits: H is first written after its last read */
  d.s_H = t; d.s_Hs = t; d.s_LD = t + al2(d.nM); d.s_Dinv = t + 2*al2(d.nM); if (arefInH) d.s_efA = t; t += hsize;
  L.ssz[LS_efA] = rows; L.ssz[LS_H] = hsize; L.ssz[LS_Hs] = L.ssz[LS_LD] = al2(d.nM); L.ssz[LS_Dinv] = hsize - 2*al2(d.nM);
  // warm start in the last nv slots of the Hessian region: read once at the start of the solve (before any write to H), rewritten at the end
  // of the integrator (after the last read of H).  Requires that no other stage reaches that far and that aref (head of H) does not overlap it.
  int qws = t - al2(d.nv);
  const bool qwsInH = qws >= extNonSolve && (!arefInH || d.s_H + rows <= qws) && d.s_H + al2(d.nvp*(d.nvp+1)/2) <= t;
  ext = imax(ext, t);
  int scratch = ext;
  if (qwsInH) { d.o_scr = o; d.o_qws = o + qws; } else { d.o_qws = o_qws_persistent; o += al2(d.nv); d.o_scr = o; }
  L.psz[LP_scr] = scratch; L.head = head; L.afterK = afterK; L.extNonSolve = extNonSolve; L.solveEnd = t; L.arefInH = arefInH; L.qwsInH = qwsInH;
  #undef PLACE
  #undef TAKE
  // scratch offsets are used relative to the warp base
  #define TO_WARP(n) d.s_##n += d.o_scr;
  MYO_LAYOUT_SCRATCH(TO_WARP)
  #undef TO_WARP
  d.n_per_warp = d.o_scr + scratch;
  return r;
}

// ------------------------------------------------------------------ static shapes
// The DevModel fields a static shape fixes: every one that model_layout sets except the tendon group ranges (below)
#define MYO_SHAPE_FIELDS(X) X(nq) X(nv) X(nu) X(na) X(nM) X(njnt) X(nbd) X(nlevel) X(nsp) X(nwe) X(nta) X(nnz) X(nlim) X(neq) X(npair) X(npair_an) \
  X(maxpath) X(ndepth) X(eq_tree) X(maxcon) X(maxefc) X(nlimrow) X(ovr_geom) X(ngc) X(s_gpose) X(nvp) \
  X(o_qpos) X(o_qvel) X(o_act) X(o_qws) X(o_dax) X(o_dan) X(o_qM) X(o_fsm) X(o_eprm) X(neprm) X(o_wz) X(nwz) X(o_cnt) X(o_scr) X(n_per_warp) \
  X(s_xpos) X(s_xmat) X(s_U) X(s_PL) X(s_mom) X(s_tlen) X(s_tvel) X(s_tfrc) X(s_cin) X(s_crb) X(s_bf) X(s_conJ) X(s_efD) X(s_efA) X(s_eqJ) X(s_icon) X(s_con) \
  X(s_clist) X(kcand) X(s_efR) X(s_efV) X(s_va) X(s_vg) X(s_vp) X(s_vMa) X(s_vMp) X(s_H) X(s_Hs) X(s_LD) X(s_Dinv)
#define MYO_SHAPE_RANGES(X) X(tg_sp) X(tg_we) X(tg_ta) X(tg_nz)

// A three-entry range table whose entries are compile-time constants (indexed like DevModel's int32_t[3]; no storage in device code)
template <int32_t A, int32_t B, int32_t C> struct ConstRange3 { __host__ __device__ constexpr int32_t operator[](int i) const { return i == 0 ? A : (i == 1 ? B : C); } };

// A DevModel whose shape is fixed at compile time: the static members hide DevModel's fields of the same names, so that the phases
// instantiated on it fold their loop bounds, offsets and dead branches (equality rows, the second tendon group, the bordered and n > 36
// dense solves).  Tables, staged sizes and scalars of the model (timestep, gravity, ...) stay kernel-parameter fields.  A batch runs a
// kernel built on a shape only when its own DevModel matches that shape in every fixed field (shape_matches).
template <class Dims> struct StaticShape : DevModel {
  static constexpr ModelLayout lay = model_layout(Dims::value);
  #define SHAPE_FIELD(f) static constexpr int32_t f = lay.d.f;
  MYO_SHAPE_FIELDS(SHAPE_FIELD)
  #undef SHAPE_FIELD
  #define SHAPE_RANGE(f) ConstRange3<lay.d.f[0], lay.d.f[1], lay.d.f[2]> f;
  MYO_SHAPE_RANGES(SHAPE_RANGE)
  #undef SHAPE_RANGE
  static bool matches(const DevModel& d) {
    bool eq = true;
    #define SHAPE_EQ(f) eq = eq && d.f == lay.d.f;
    MYO_SHAPE_FIELDS(SHAPE_EQ)
    #undef SHAPE_EQ
    #define SHAPE_EQ3(f) for (int k = 0; k < 3; k++) eq = eq && d.f[k] == lay.d.f[k];
    MYO_SHAPE_RANGES(SHAPE_EQ3)
    #undef SHAPE_EQ3
    return eq; }
};

// The hand (myohand_pose) at the default contact capacity: the shape of the headline workload and of the hand reach tasks
#include "../../include/myo_hand_shape.h"
struct HandDims { static constexpr ModelDims value = MYO_HAND_SHAPE_DIMS; };
static_assert(sizeof(ModelDims) == MYO_HAND_SHAPE_NDIMS*sizeof(int32_t), "include/myo_hand_shape.h lists every ModelDims field");
// The hand kernel's launch adds one region to the generic launch: the cold f64 tables (blob.py COLD_D), which sit behind the staged
// doubles in the blob.  It passes nD = every hot double, so that the same bulk copy stages them and they land right behind the staged
// tables ([hot f64 | cold f64 | int16 lists | per-warp regions]); GD() / LDC() then read shared memory instead of HBM.  The model layout,
// the DevModel of the batch and every other kernel's launch are those of the generic kernel.
struct HandShape : StaticShape<HandDims> {
  static constexpr bool cold_in_smem = true;
  // bytes of the region for a batch whose blob holds nD_all hot doubles, of which its DevModel d stages d.nD
  static int cold_bytes(const DevModel& d, int nD_all) { return (nD_all - d.nD)*8; }
};

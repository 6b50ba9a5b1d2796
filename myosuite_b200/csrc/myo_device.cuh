// myo_device.cuh -- device-side physics of the B200-native batched musculoskeletal simulator.
//
// One env per warp.  Every phase is a lane-strided loop over a list from the model "program"
// (myosuite_b200/program.py).  Both the per-env working state (f64) AND the model constants the phases
// read (int16 index lists + f64 tables, staged once per CTA with a bulk async copy) live in shared
// memory; HBM is touched only for the per-step state / action / observation rows.
// What is computed is what the reference's mujoco.mj_step computes for these models
// (myosuite/robot/robot.py:856-861; SURVEY.md Appendix A), but the formulation is
// this project's own: origin-centred spatial algebra over dynamic bodies only, compile-time folded
// constant tendon segments, structural-non-zero tendon moments, tree-sparse LDL / dense Newton.
#pragma once
#include <stdint.h>
#include "../../include/myo_blob_layout.h"
#include "../../include/myo_b200.h"

#define MYO_MINVAL 1e-15
#define FULL 0xffffffffu
typedef short idx_t;

// P_dims slots (must match myosuite_b200/program.py)
enum { PD_NBD, PD_NLEVEL, PD_NPT, PD_NSP, PD_NWE, PD_NTA, PD_NNZ, PD_NTERM, PD_NLIM, PD_NEQ, PD_NPAIR, PD_NGC, PD_MAXPATH,
       PD_MAXCHAIN, PD_NSUB, PD_NROW, PD_NCOL, PD_NPIECE, PD_NWE_SPH_OUT, PD_NWE_SPH_IN, PD_NWE_CYL_OUT, PD_NWE_CYL_IN, PD_NDEPTH, PD_EQ_TREE, PD_NPAIR_ANALYTIC, PD_NLIMROW,
       PD_SPLIT_SP, PD_SPLIT_WE, PD_SPLIT_TA, PD_SPLIT_NZ };
#define PB_STRIDE 22      // pos[3] R[9] ipos[3] mass Iloc[6]
#define PWE_STRIDE 16
#define PA_STRIDE 17      // dynprm[3] | gain: range0 range1 lmin lmax vmax fvmax | bias: range0 range1 lmax fpmax | ctrlrange[2] | ctrllimited | pad
#define PAM_STRIDE 6
#define PG_STRIDE 16
#define PPAIR_STRIDE 12
#define PPAIR_ISTRIDE 8     // g1 g2 condim path_adr path_n collider class model-pair-index
#define PLIM_STRIDE 12
#define PEQ_STRIDE 16
#define PEQ_ISTRIDE 6
enum { CT_NONE, CT_CAP_CAP, CT_SPH_SPH, CT_SPH_CAP, CT_PLANE_SPH, CT_PLANE_CAP, CT_PLANE_ELL, CT_CAP_ELL, CT_ELL_ELL };
#define CON_STRIDE 10   // dist, pos[3], normal[3], tangent1[3]  (tangent2 = normal x tangent1 is rebuilt by the constraint phase)

// ------------------------------------------------------------------ device-resident model view (kernel parameter)
struct DevModel {
  const int32_t* gI16; const double* gD;   // hot constant arrays in HBM (source of the per-CTA staging copy)
  double* g_ctrl;                          // [n_env, nu] library-owned: this control step's ctrl rows (written by the prologue, read by every substep)
  int32_t nI16w, nD;                       // sizes of the STAGED arrays: int32 words of packed int16, doubles (gD holds further "cold" tables behind the staged ones: GD())
  int32_t hoff[MYO_NSEC];                  // offset of each hot section (in shorts / doubles), -1 if not staged
  int32_t nq, nv, nu, na, nM, njnt;
  int32_t nbd, nlevel, nsp, nwe, nta, nnz, nlim, neq, npair, npair_an, maxpath, ndepth, eq_tree;
  int32_t tg_sp[3], tg_we[3], tg_ta[3], tg_nz[3];          // tendon groups A / B (two passes through the tendon scratch): ranges of segments, wrap elements, tendons, moment non-zeros
  int32_t maxcon, maxefc, nlimrow, ovr_geom, ngc, s_gpose, solve_sync, nvp;          // ovr_geom: collision geom whose size comes from the per-env overrides (-1: none); nvp: nv padded to the dense solver's order
  double timestep, gx, gy, gz, meaninertia, tolerance;
  // per-warp shared-memory layout, in doubles.  Persistent part:
  int32_t o_qpos, o_qvel, o_act, o_qws, o_dax, o_dan, o_qM, o_fsm, o_eprm, neprm, o_wz, nwz, o_cnt, o_scr, n_per_warp;
  // scratch (time-multiplexed by stage; offsets relative to the warp base, i.e. o_scr included).  See fill_devmodel() for the overlap rules.
  int32_t s_xpos, s_xmat;                                  // K: body poses, alive kinematics .. constraints
  int32_t s_U, s_PL, s_mom, s_tlen, s_tvel, s_tfrc;  // stage 1: tendons + actuation
  int32_t s_cin, s_crb, s_bf;                              // stage 2: CRB / bias
  int32_t s_conJ, s_efD, s_efA, s_eqJ, s_icon, s_con;      // stage 3 -> 4: contacts / constraint rows
  int32_t s_clist, kcand;                                  // collision only: list of the expensive (ellipsoid) candidates that survived the cull
  int32_t s_efR, s_efV, s_va, s_vg, s_vp, s_vMa, s_vMp, s_H, s_Hs, s_LD, s_Dinv;   // stage 4: Newton
};

// The whole dynamic shared-memory window, declared at file scope so that every pointer derived from it is PROVABLY in the
// shared address space: the working-set and constant accesses compile to LDS/STS with 32-bit address arithmetic instead of
// generic 64-bit loads (round 1: 4 048 generic LD.E vs 127 LDS in the kernel's SASS).
// Layout: [hot f64 tables (m.nD)] [hot int16 lists] [per-warp regions of m.n_per_warp doubles]
extern __shared__ __align__(16) double smem[];

struct Warp { int base, lane; };   // by value: offset (doubles) of this warp's region in smem, lane id.  Everything else lives in shared memory.
enum { CNT_ncon, CNT_nefc, CNT_nlimrow, CNT_niter, CNT_overflow, CNT_ncand, CNT_na, CNT_N = 8 };   // per-warp int counters (m.o_cnt)
#define CI(name) ((const idx_t*)(smem + m.nD) + m.hoff[MYO_SEC_##name])
#define CD(name) ((const double*)smem + m.hoff[MYO_SEC_##name])
#ifdef MYO_COLD_L2ONLY
#define LDC(p) __ldcg(p)                                      // (experiment: bypass L1 for the cold tables; the default keeps them in L1)
#else
#define LDC(p) __ldg(p)
#endif
#define GD(name) (m.gD + m.hoff[MYO_SEC_##name])              // cold f64 tables (blob.py COLD_D): read from HBM / L2 through the read-only path (__ldg)
#define W_(f) (smem + w.base + m.o_##f)                       // persistent per-env arrays
#define WI_(f) (((int*)(smem + w.base + m.o_cnt))[CNT_##f])   // per-env counters
#define SCR(field) (smem + w.base + m.field)                  // scratch (m.s_* are offsets from the warp base)
#define S_cpair ((idx_t*)(SCR(s_icon) + m.maxcon + (m.maxcon + 1)/2))   // contact -> program pair index, int16 (after the 64-bit path masks and the row words; see myo_solver.cuh)
#define SHARED_PTR(p) __builtin_assume(__isShared(p))         // for pointer PARAMETERS of functions that may not be inlined

// ------------------------------------------------------------------ small math
__device__ __forceinline__ void cross3(double* r, const double* a, const double* b) {
  double x = a[1]*b[2]-a[2]*b[1], y = a[2]*b[0]-a[0]*b[2], z = a[0]*b[1]-a[1]*b[0]; r[0]=x; r[1]=y; r[2]=z; }
__device__ __forceinline__ double dot3(const double* a, const double* b) { return a[0]*b[0]+a[1]*b[1]+a[2]*b[2]; }
__device__ __forceinline__ void quat2mat(double* m, const double* q) {
  double w=q[0],x=q[1],y=q[2],z=q[3];
  m[0]=w*w+x*x-y*y-z*z; m[1]=2*(x*y-w*z); m[2]=2*(x*z+w*y);
  m[3]=2*(x*y+w*z); m[4]=w*w-x*x+y*y-z*z; m[5]=2*(y*z-w*x);
  m[6]=2*(x*z-w*y); m[7]=2*(y*z+w*x); m[8]=w*w-x*x-y*y+z*z; }
__device__ __forceinline__ void quat_mul(double* r, const double* a, const double* b) {
  double w=a[0]*b[0]-a[1]*b[1]-a[2]*b[2]-a[3]*b[3], x=a[0]*b[1]+a[1]*b[0]+a[2]*b[3]-a[3]*b[2],
         y=a[0]*b[2]-a[1]*b[3]+a[2]*b[0]+a[3]*b[1], z=a[0]*b[3]+a[1]*b[2]-a[2]*b[1]+a[3]*b[0];
  r[0]=w; r[1]=x; r[2]=y; r[3]=z; }
__device__ __forceinline__ void quat_norm(double* q) {
  double n = sqrt(q[0]*q[0]+q[1]*q[1]+q[2]*q[2]+q[3]*q[3]);
  if (n < MYO_MINVAL) { q[0]=1; q[1]=q[2]=q[3]=0; } else { double s=1.0/n; q[0]*=s; q[1]*=s; q[2]*=s; q[3]*=s; } }
__device__ __forceinline__ void mat_vec(double* r, const double* m, const double* v) {
  double x=m[0]*v[0]+m[1]*v[1]+m[2]*v[2], y=m[3]*v[0]+m[4]*v[1]+m[5]*v[2], z=m[6]*v[0]+m[7]*v[1]+m[8]*v[2]; r[0]=x; r[1]=y; r[2]=z; }
__device__ __forceinline__ void matT_vec(double* r, const double* m, const double* v) {
  double x=m[0]*v[0]+m[3]*v[1]+m[6]*v[2], y=m[1]*v[0]+m[4]*v[1]+m[7]*v[2], z=m[2]*v[0]+m[5]*v[1]+m[8]*v[2]; r[0]=x; r[1]=y; r[2]=z; }
__device__ __forceinline__ void mat_mul(double* r, const double* a, const double* b) {   // r = a*b (3x3, row-major), r may not alias
  #pragma unroll
  for (int i = 0; i < 3; i++) { r[3*i] = a[3*i]*b[0]+a[3*i+1]*b[3]+a[3*i+2]*b[6]; r[3*i+1] = a[3*i]*b[1]+a[3*i+1]*b[4]+a[3*i+2]*b[7]; r[3*i+2] = a[3*i]*b[2]+a[3*i+1]*b[5]+a[3*i+2]*b[8]; } }
__device__ __forceinline__ double clipd(double x, double lo, double hi) { return x < lo ? lo : (x > hi ? hi : x); }
__device__ __forceinline__ double warp_sum(double v) {
  #pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v; }

// Reciprocal and square root without libdevice's IEEE special-case paths: MUFU seed (~20 bits) + two Newton steps, 1-2 ulp.  Dependent
// latencies of these and of the libdevice calls they replace: tools/ubench/ubench.cu.  Arguments must be normal numbers; m_sqrt(0) = 0.
// (acos is slower than asin: the wrap arc uses pi/2 - asin.)
__device__ __forceinline__ double m_rcp(double x) { double y; asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x)); double e = fma(-x, y, 1.0); y = fma(y, e, y); e = fma(-x, y, 1.0); return fma(y, e, y); }
__device__ __forceinline__ double m_sqrt(double x) { double y; asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  const double h = 0.5*x; double t = fma(-h*y, y, 0.5); y = fma(y, t, y); t = fma(-h*y, y, 0.5); y = fma(y, t, y);
  double s = x*y; s = fma(fma(-s, s, x), 0.5*y, s); return x > 1e-300 ? s : 0.0; }
#define FDIV(a, b) ((a)*m_rcp(b))

// world position of program point `pt`
__device__ __forceinline__ void world_point(const DevModel& m, const Warp w, int pt, double* out) {
  int b = CI(PPT_body)[pt]; const double* __restrict__ xg = GD(PPT_xyz) + 3*pt; const double x[3] = {LDC(xg), LDC(xg+1), LDC(xg+2)};
  if (b < 0) { out[0]=x[0]; out[1]=x[1]; out[2]=x[2]; }
  else { const double* xp = SCR(s_xpos) + 3*b; mat_vec(out, SCR(s_xmat) + 9*b, x); out[0]+=xp[0]; out[1]+=xp[1]; out[2]+=xp[2]; } }

// spatial motion vector of dof d about the world origin: [omega ; velocity of the point at the origin]
__device__ __forceinline__ void dof_motion(const DevModel& m, const Warp w, int d, double* S) {
  const double* ax = W_(dax) + 3*d;
  if (CI(PD_lin)[d]) { S[0]=S[1]=S[2]=0; S[3]=ax[0]; S[4]=ax[1]; S[5]=ax[2]; }
  else { S[0]=ax[0]; S[1]=ax[1]; S[2]=ax[2]; cross3(S+3, W_(dan) + 3*d, ax); } }
// velocity of world point p due to unit rate of dof d
__device__ __forceinline__ void dof_point_vel(const DevModel& m, const Warp w, int d, const double* p, double* c) {
  const double* ax = W_(dax) + 3*d;
  if (CI(PD_lin)[d]) { c[0]=ax[0]; c[1]=ax[1]; c[2]=ax[2]; }
  else { double r[3] = {p[0]-W_(dan)[3*d], p[1]-W_(dan)[3*d+1], p[2]-W_(dan)[3*d+2]}; cross3(c, ax, r); } }
// f = Ic * S for a spatial inertia about the origin: Ic = (Ixx,Iyy,Izz,Ixy,Ixz,Iyz, m*c[3], m)
__device__ __forceinline__ void inert_mul(double* f, const double* ic, const double* S) {
  const double* wv = S; const double* v = S + 3; const double* mc = ic + 6; double t[3];
  f[0] = ic[0]*wv[0]+ic[3]*wv[1]+ic[4]*wv[2]; f[1] = ic[3]*wv[0]+ic[1]*wv[1]+ic[5]*wv[2]; f[2] = ic[4]*wv[0]+ic[5]*wv[1]+ic[2]*wv[2];
  cross3(t, mc, v); f[0]+=t[0]; f[1]+=t[1]; f[2]+=t[2];
  cross3(t, wv, mc); f[3] = ic[9]*v[0]+t[0]; f[4] = ic[9]*v[1]+t[1]; f[5] = ic[9]*v[2]+t[2]; }

// ------------------------------------------------------------------ phase 1: kinematics (rotation matrices, level by level)
// also writes each dynamic body's spatial inertia about the world origin (cin) into the stage-2 scratch
__device__ void phase_kinematics(const DevModel& m, const Warp w) {
  const idx_t* level = CI(PB_level_adr); const idx_t* par = CI(PB_parent); const idx_t* jadr = CI(PB_jadr); const idx_t* jnum = CI(PB_jnum);
  const double* PB = CD(PB_d);
  const idx_t* jtype = CI(jnt_type); const idx_t* jq = CI(jnt_qposadr); const idx_t* jd = CI(jnt_dofadr);
  const double* jpos = CD(jnt_pos); const double* jaxis = CD(jnt_axis); const double* qpos0 = CD(qpos0);
  double* xpos = SCR(s_xpos); double* xmat = SCR(s_xmat);
  // sin / cos of every hinge angle in ONE lane-parallel pass (the level loop below would otherwise run the sincos code once per tree level with
  // a handful of lanes active).  Parked in the head of the Hessian region, which is idle until the constraint phase (the tail holds the warm start).
  double* sc = SCR(s_H);
  for (int j = w.lane; j < m.njnt; j += 32) { const int t = jtype[j]; if (t != 0 && t != 2) { double s_, c_; sincos(W_(qpos)[jq[j]] - qpos0[jq[j]], &s_, &c_); sc[2*j] = s_; sc[2*j+1] = c_; } }
  __syncwarp();
  for (int L = 0; L < m.nlevel; L++) {
    for (int k = level[L] + w.lane; k < level[L+1]; k += 32) {
      const double* bd = PB + k*PB_STRIDE; int p = par[k]; double pos[3], R[9];
      if (p < 0) { pos[0]=bd[0]; pos[1]=bd[1]; pos[2]=bd[2];
        #pragma unroll
        for (int c = 0; c < 9; c++) R[c] = bd[3+c]; }
      else { mat_vec(pos, xmat + 9*p, bd); pos[0]+=xpos[3*p]; pos[1]+=xpos[3*p+1]; pos[2]+=xpos[3*p+2]; mat_mul(R, xmat + 9*p, bd + 3); }
      for (int j = jadr[k]; j < jadr[k] + jnum[k]; j++) {
        int t = jtype[j], qa = jq[j], da = jd[j];
        if (t == 0) {   // free joint: pose straight from qpos (normalised copy of the quaternion; qpos itself is left untouched)
          const double* qp = W_(qpos) + qa; double qn[4] = {qp[3], qp[4], qp[5], qp[6]}; quat_norm(qn);
          pos[0]=qp[0]; pos[1]=qp[1]; pos[2]=qp[2]; quat2mat(R, qn);
          #pragma unroll
          for (int c = 0; c < 3; c++) {
            W_(dax)[3*(da+c)] = c==0; W_(dax)[3*(da+c)+1] = c==1; W_(dax)[3*(da+c)+2] = c==2;
            W_(dan)[3*(da+c)] = 0; W_(dan)[3*(da+c)+1] = 0; W_(dan)[3*(da+c)+2] = 0;
            W_(dax)[3*(da+3+c)] = R[c]; W_(dax)[3*(da+3+c)+1] = R[3+c]; W_(dax)[3*(da+3+c)+2] = R[6+c];
            W_(dan)[3*(da+3+c)] = pos[0]; W_(dan)[3*(da+3+c)+1] = pos[1]; W_(dan)[3*(da+3+c)+2] = pos[2]; }
        } else {
          const double* al = jaxis + 3*j;
          double ax[3], an[3]; mat_vec(ax, R, al); mat_vec(an, R, jpos + 3*j); an[0]+=pos[0]; an[1]+=pos[1]; an[2]+=pos[2];
          double dq = W_(qpos)[qa] - qpos0[qa];
          if (t == 2) { pos[0]+=ax[0]*dq; pos[1]+=ax[1]*dq; pos[2]+=ax[2]*dq; }
          else {   // hinge: R <- R * Rodrigues(local axis, dq); pos keeps the anchor fixed
            const double s = sc[2*j], c = sc[2*j+1]; double oc = 1-c, x = al[0], y = al[1], z = al[2];
            double Q[9] = {c+oc*x*x, oc*x*y-s*z, oc*x*z+s*y,  oc*x*y+s*z, c+oc*y*y, oc*y*z-s*x,  oc*x*z-s*y, oc*y*z+s*x, c+oc*z*z}, Rn[9];
            mat_mul(Rn, R, Q);
            #pragma unroll
            for (int q = 0; q < 9; q++) R[q] = Rn[q];
            double v[3]; mat_vec(v, R, jpos + 3*j); pos[0]=an[0]-v[0]; pos[1]=an[1]-v[1]; pos[2]=an[2]-v[2]; }
          W_(dax)[3*da]=ax[0]; W_(dax)[3*da+1]=ax[1]; W_(dax)[3*da+2]=ax[2]; W_(dan)[3*da]=an[0]; W_(dan)[3*da+1]=an[1]; W_(dan)[3*da+2]=an[2];
        }
      }
      #pragma unroll
      for (int c = 0; c < 3; c++) xpos[3*k+c] = pos[c];
      #pragma unroll
      for (int c = 0; c < 9; c++) xmat[9*k+c] = R[c];
    }
    __syncwarp();
  }
}

// spatial inertia of every dynamic body about the world origin (needs final poses; writes stage-2 scratch)
__device__ void phase_body_inertia(const DevModel& m, const Warp w) {
  const double* PB = CD(PB_d); const double* xpos = SCR(s_xpos); const double* xmat = SCR(s_xmat); double* cin = SCR(s_cin);
  for (int k = w.lane; k < m.nbd; k += 32) { const double* bd = PB + k*PB_STRIDE; const double* R = xmat + 9*k;
    double c3[3]; mat_vec(c3, R, bd + 12); c3[0]+=xpos[3*k]; c3[1]+=xpos[3*k+1]; c3[2]+=xpos[3*k+2];
    double mass = bd[15]; const double* Il = bd + 16;   // xx yy zz xy xz yz (body frame)
    double A[9] = {Il[0],Il[3],Il[4], Il[3],Il[1],Il[5], Il[4],Il[5],Il[2]}, T[9]; mat_mul(T, R, A);
    double* ci = cin + 10*k; double cc2 = dot3(c3, c3);
    ci[0] = T[0]*R[0]+T[1]*R[1]+T[2]*R[2] + mass*(cc2 - c3[0]*c3[0]);
    ci[1] = T[3]*R[3]+T[4]*R[4]+T[5]*R[5] + mass*(cc2 - c3[1]*c3[1]);
    ci[2] = T[6]*R[6]+T[7]*R[7]+T[8]*R[8] + mass*(cc2 - c3[2]*c3[2]);
    ci[3] = T[0]*R[3]+T[1]*R[4]+T[2]*R[5] - mass*c3[0]*c3[1];
    ci[4] = T[0]*R[6]+T[1]*R[7]+T[2]*R[8] - mass*c3[0]*c3[2];
    ci[5] = T[3]*R[6]+T[4]*R[7]+T[5]*R[8] - mass*c3[1]*c3[2];
    ci[6] = mass*c3[0]; ci[7] = mass*c3[1]; ci[8] = mass*c3[2]; ci[9] = mass; }
  __syncwarp();
}

// ------------------------------------------------------------------ phase 2: spatial tendons
__device__ __forceinline__ bool seg_intersect(const double* p1, const double* p2, const double* p3, const double* p4) {
  double det = (p4[1]-p3[1])*(p2[0]-p1[0]) - (p4[0]-p3[0])*(p2[1]-p1[1]);
  if (fabs(det) < MYO_MINVAL) return false;
  const double id = m_rcp(det);
  double a = ((p4[0]-p3[0])*(p1[1]-p3[1]) - (p4[1]-p3[1])*(p1[0]-p3[0]))*id;
  double b = ((p2[0]-p1[0])*(p1[1]-p3[1]) - (p2[1]-p1[1])*(p1[0]-p3[0]))*id;
  return a >= 0 && a <= 1 && b >= 0 && b <= 1; }

// 2-D tangent wrap of the path d0 -> circle(rad) -> d1 on the outside; returns arc length or -1 (no wrap)
__device__ __forceinline__ double wrap2d_outside(double* pnt, const double* d, const double* sd, bool has_side, double rad) {
  double sq0 = d[0]*d[0]+d[1]*d[1], sq1 = d[2]*d[2]+d[3]*d[3], sqr = rad*rad;
  double dif0 = d[2]-d[0], dif1 = d[3]-d[1], dd = dif0*dif0+dif1*dif1;
  if (sq0 < sqr || sq1 < sqr || rad < MYO_MINVAL || dd < MYO_MINVAL) return -1;
  double a = clipd(-(dif0*d[0]+dif1*d[1])*m_rcp(dd), 0, 1);
  double t0 = a*dif0+d[0], t1 = a*dif1+d[1];
  if (t0*t0+t1*t1 > sqr && (!has_side || t0*sd[0]+t1*sd[1] >= 0)) return -1;
  double s0 = m_sqrt(sq0-sqr), s1 = m_sqrt(sq1-sqr), sol[2][4], good[2], i0 = m_rcp(sq0), i1 = m_rcp(sq1);
  #pragma unroll
  for (int i = 0; i < 2; i++) { double sg = i==0 ? 1.0 : -1.0;
    sol[i][0] = (d[0]*sqr + sg*rad*d[1]*s0)*i0; sol[i][1] = (d[1]*sqr - sg*rad*d[0]*s0)*i0;
    sol[i][2] = (d[2]*sqr - sg*rad*d[3]*s1)*i1; sol[i][3] = (d[3]*sqr + sg*rad*d[2]*s1)*i1;
    if (has_side) { double x = sol[i][0]+sol[i][2], y = sol[i][1]+sol[i][3], n = m_sqrt(x*x+y*y);
      if (n < MYO_MINVAL) { x = 1; y = 0; } else { const double q = m_rcp(n); x *= q; y *= q; } good[i] = x*sd[0]+y*sd[1]; }
    else { double x = sol[i][0]-sol[i][2], y = sol[i][1]-sol[i][3]; good[i] = -(x*x+y*y); }
    if (seg_intersect(d, sol[i], d+2, sol[i]+2)) good[i] = -10000; }
  int i = good[0] > good[1] ? 0 : 1;
  pnt[0]=sol[i][0]; pnt[1]=sol[i][1]; pnt[2]=sol[i][2]; pnt[3]=sol[i][3];
  if (seg_intersect(d, pnt, d+2, pnt+2)) return -1;
  return rad*(1.5707963267948966 - asin(clipd((pnt[0]*pnt[2]+pnt[1]*pnt[3])*m_rcp(sqr), -1, 1))); }

// inverse wrap: the path must pass through the inside of the circle (touches it in one point); returns 0 or -1
__device__ __forceinline__ double wrap2d_inside(double* pnt, const double* d, double rad, double* zwarm) {
  double len0 = m_sqrt(d[0]*d[0]+d[1]*d[1]), len1 = m_sqrt(d[2]*d[2]+d[3]*d[3]);
  if (len0 <= rad || len1 <= rad || rad < MYO_MINVAL || len0 < MYO_MINVAL || len1 < MYO_MINVAL) return -1;
  double dif0 = d[2]-d[0], dif1 = d[3]-d[1], dd = dif0*dif0+dif1*dif1;
  if (dd > MYO_MINVAL) { double a = -(dif0*d[0]+dif1*d[1])*m_rcp(dd);
    if (a > 0 && a < 1) { double x = d[0]+a*dif0, y = d[1]+a*dif1; if (x*x+y*y <= rad*rad) return -1; } }
  { double x = 0.5*(d[0]+d[2]), y = 0.5*(d[1]+d[3]), n = m_sqrt(x*x+y*y); if (n < MYO_MINVAL) { x = 1; y = 0; n = 1; }
    const double q = rad*m_rcp(n); pnt[0]=pnt[2]=x*q; pnt[1]=pnt[3]=y*q; }
  double A = rad*m_rcp(len0), B = rad*m_rcp(len1), cosG = (len0*len0+len1*len1-dd)*m_rcp(2*len0*len1);
  if (cosG < -1+MYO_MINVAL) return -1; else if (cosG > 1-MYO_MINVAL) return 0;
  double G = acos(cosG), z, f; bool solved = false;
  if (*zwarm > 0 && *zwarm < 1-1e-7) {   // warm start from the previous substep's root: a few safeguarded Newton steps, else fall back to the cold start
    z = *zwarm;
    #pragma unroll 1
    for (int it = 0; it < 4; it++) { f = asin(A*z)+asin(B*z)-2*asin(z)+G; if (fabs(f) < 1e-10) { solved = true; break; }
      double df = A*m_rcp(fmax(MYO_MINVAL, m_sqrt(1-z*z*A*A))) + B*m_rcp(fmax(MYO_MINVAL, m_sqrt(1-z*z*B*B))) - 2*m_rcp(fmax(MYO_MINVAL, m_sqrt(1-z*z)));
      if (df > -MYO_MINVAL) break;
      z -= f*m_rcp(df); if (!(z > 0 && z < 1-1e-7)) break; } }
  int it = 0;
  if (!solved) {
  z = 1-1e-7; f = asin(A*z)+asin(B*z)-2*asin(z)+G;
  if (f > 0) { *zwarm = -1; return 0; }
  #pragma unroll 1
  for (; it < 20 && fabs(f) > 1e-6; it++) {
    double df = A*m_rcp(fmax(MYO_MINVAL, m_sqrt(1-z*z*A*A))) + B*m_rcp(fmax(MYO_MINVAL, m_sqrt(1-z*z*B*B))) - 2*m_rcp(fmax(MYO_MINVAL, m_sqrt(1-z*z)));
    if (df > -MYO_MINVAL) return 0;
    double z1 = z - f*m_rcp(df); if (z1 > z) return 0;
    z = z1; f = asin(A*z)+asin(B*z)-2*asin(z)+G;
    if (f > 1e-6) return 0; }
  if (it >= 20) return 0;
  }
  *zwarm = z;
  double vx, vy, ang;
  if (d[0]*d[3]-d[1]*d[2] > 0) { vx = d[0]; vy = d[1]; ang = asin(z)-asin(A*z); } else { vx = d[2]; vy = d[3]; ang = asin(z)-asin(B*z); }
  { const double q = m_rcp(m_sqrt(vx*vx+vy*vy)); vx *= q; vy *= q; } double s, c; sincos(ang, &s, &c);
  pnt[0] = rad*(c*vx - s*vy); pnt[1] = rad*(s*vx + c*vy); pnt[2] = pnt[0]; pnt[3] = pnt[1];
  return 0; }

__device__ void wrap_element(const DevModel& m, const Warp w, int k, int g, double* U, double* PL) {
  const idx_t* we = CI(PWE) + 6*k; const double* __restrict__ wdg = GD(PWE_d) + k*PWE_STRIDE;      // (cold table: 16 independent read-only loads per element)
  double wd[12]; for (int c = 0; c < 12; c++) wd[c] = LDC(wdg + c);
  double x0[3], x1[3]; world_point(m, w, we[0], x0); world_point(m, w, we[1], x1);
  int gb = we[2]; bool cyl = we[3] == 1, has_side = we[4] >= 0, inside = we[5] != 0; const double rad = LDC(wdg + 12);
  const int nspg = m.tg_sp[g+1] - m.tg_sp[g], kl = k - m.tg_we[g];      // slots inside this group's scratch
  double gpos[3], gmat[9];
  if (gb < 0) { for (int c = 0; c < 3; c++) gpos[c] = wd[c]; for (int c = 0; c < 9; c++) gmat[c] = wd[3+c]; }
  else { const double* X = SCR(s_xmat) + 9*gb; const double* xp = SCR(s_xpos) + 3*gb; mat_vec(gpos, X, wd); gpos[0]+=xp[0]; gpos[1]+=xp[1]; gpos[2]+=xp[2]; mat_mul(gmat, X, wd + 3); }
  double t[3], p0[3], p1[3];
  t[0]=x0[0]-gpos[0]; t[1]=x0[1]-gpos[1]; t[2]=x0[2]-gpos[2]; matT_vec(p0, gmat, t);
  t[0]=x1[0]-gpos[0]; t[1]=x1[1]-gpos[1]; t[2]=x1[2]-gpos[2]; matT_vec(p1, gmat, t);
  double wlen = -1, pnt[4], ax0[3] = {1,0,0}, ax1[3] = {0,1,0};
  if (dot3(p0,p0) >= MYO_MINVAL*MYO_MINVAL && dot3(p1,p1) >= MYO_MINVAL*MYO_MINVAL) {
    if (!cyl) {   // plane through p0, p1 and the sphere centre
      double n0 = m_rcp(m_sqrt(dot3(p0,p0))); ax0[0]=p0[0]*n0; ax0[1]=p0[1]*n0; ax0[2]=p0[2]*n0;
      double nrm[3]; cross3(nrm, p0, p1); double nn = m_sqrt(dot3(nrm,nrm));
      if (nn < MYO_MINVAL) { int i = 0; if (fabs(ax0[1]) > fabs(ax0[i])) i = 1; if (fabs(ax0[2]) > fabs(ax0[i])) i = 2;
        double o[3] = {i == 0 ? 0.0 : 1.0, i == 1 ? 0.0 : 1.0, i == 2 ? 0.0 : 1.0}; cross3(nrm, ax0, o); nn = m_sqrt(dot3(nrm,nrm)); }
      { const double q = m_rcp(nn); nrm[0]*=q; nrm[1]*=q; nrm[2]*=q; } cross3(ax1, nrm, ax0); { const double q = m_rcp(m_sqrt(dot3(ax1,ax1))); ax1[0]*=q; ax1[1]*=q; ax1[2]*=q; } }
    double d[4] = {dot3(p0,ax0), dot3(p0,ax1), dot3(p1,ax0), dot3(p1,ax1)}, sd[2] = {0,0};
    if (has_side) { const double s[3] = {LDC(wdg + 13), LDC(wdg + 14), LDC(wdg + 15)}; sd[0] = dot3(s,ax0); sd[1] = dot3(s,ax1); double n = m_sqrt(sd[0]*sd[0]+sd[1]*sd[1]);
      if (n < MYO_MINVAL) { sd[0] = rad; sd[1] = 0; } else { const double q = rad*m_rcp(n); sd[0] *= q; sd[1] *= q; } }
    wlen = inside ? wrap2d_inside(pnt, d, rad, W_(wz) + (we[5] - 1)) : wrap2d_outside(pnt, d, sd, has_side, rad);
  }
  double* u0 = U + 3*(nspg + 2*kl); double* u1 = u0 + 3; double w0[3], w1[3];      // tangent points: only the two straight pieces' directions and the path length leave this function
  if (wlen < 0) {   // straight segment: both "wrap points" sit at x1 (on the line), same direction for both pieces
    double dv[3] = {x1[0]-x0[0], x1[1]-x0[1], x1[2]-x0[2]}, n = m_sqrt(dot3(dv,dv));
    if (n < MYO_MINVAL) { dv[0]=1; dv[1]=0; dv[2]=0; } else { const double q = m_rcp(n); dv[0]*=q; dv[1]*=q; dv[2]*=q; }
    for (int c = 0; c < 3; c++) { u0[c]=dv[c]; u1[c]=dv[c]; }
    PL[nspg + kl] = n; return; }
  double r0[3], r1[3];
  for (int c = 0; c < 3; c++) { r0[c] = ax0[c]*pnt[0]+ax1[c]*pnt[1]; r1[c] = ax0[c]*pnt[2]+ax1[c]*pnt[3]; }
  if (cyl) { double L0 = m_sqrt((p0[0]-pnt[0])*(p0[0]-pnt[0])+(p0[1]-pnt[1])*(p0[1]-pnt[1])), L1 = m_sqrt((p1[0]-pnt[2])*(p1[0]-pnt[2])+(p1[1]-pnt[3])*(p1[1]-pnt[3]));
    double inv = m_rcp(L0+wlen+L1);
    r0[2] = p0[2]+(p1[2]-p0[2])*L0*inv; r1[2] = p0[2]+(p1[2]-p0[2])*(L0+wlen)*inv;
    double h = fabs(r1[2]-r0[2]); wlen = m_sqrt(wlen*wlen+h*h); }
  mat_vec(w0, gmat, r0); mat_vec(w1, gmat, r1);
  for (int c = 0; c < 3; c++) { w0[c]+=gpos[c]; w1[c]+=gpos[c]; }
  double a[3] = {w0[0]-x0[0], w0[1]-x0[1], w0[2]-x0[2]}, b[3] = {x1[0]-w1[0], x1[1]-w1[1], x1[2]-w1[2]};
  double na = m_sqrt(dot3(a,a)), nb = m_sqrt(dot3(b,b));
  if (na < MYO_MINVAL) { u0[0]=1; u0[1]=0; u0[2]=0; } else { double q = m_rcp(na); u0[0]=a[0]*q; u0[1]=a[1]*q; u0[2]=a[2]*q; }
  if (nb < MYO_MINVAL) { u1[0]=1; u1[1]=0; u1[2]=0; } else { double q = m_rcp(nb); u1[0]=b[0]*q; u1[1]=b[1]*q; u1[2]=b[2]*q; }
  PL[nspg + kl] = na + wlen + nb;
}

// One tendon group (pass): straight segments and wrap elements of the group into the group-local unit-vector / piece-length scratch
__device__ void phase_tendon(const DevModel& m, const Warp w, int g) {
  double* U = SCR(s_U); double* PL = SCR(s_PL);
  const idx_t* sp = CI(PSP); const int s0 = m.tg_sp[g], s1 = m.tg_sp[g+1];
  for (int k = s0 + w.lane; k < s1; k += 32) { double a[3], b[3]; world_point(m, w, sp[2*k], a); world_point(m, w, sp[2*k+1], b); const int kl = k - s0;
    double dv[3] = {b[0]-a[0], b[1]-a[1], b[2]-a[2]}, n = m_sqrt(dot3(dv,dv));
    if (n < MYO_MINVAL) { U[3*kl]=1; U[3*kl+1]=0; U[3*kl+2]=0; } else { double q = m_rcp(n); U[3*kl]=dv[0]*q; U[3*kl+1]=dv[1]*q; U[3*kl+2]=dv[2]*q; }
    PL[kl] = n; }
  #pragma unroll 1
  for (int k = m.tg_we[g] + w.lane; k < m.tg_we[g+1]; k += 32) wrap_element(m, w, k, g, U, PL);
  __syncwarp();
}
// second half of a pass: moments per structural non-zero and tendon lengths of the group
__device__ void phase_tendon_moments(const DevModel& m, const Warp w, int g) {
  double* U = SCR(s_U); double* PL = SCR(s_PL); double* mom = SCR(s_mom); double* tlen = SCR(s_tlen);
  const idx_t* nzd = CI(PNZ_dof); const idx_t* tadr = CI(PNZ_term_adr); const idx_t* term = CI(PTERM);
  for (int z = m.tg_nz[g] + w.lane; z < m.tg_nz[g+1]; z += 32) { int d = nzd[z]; double acc = 0;
    #pragma unroll 1
    for (int e = tadr[z]; e < tadr[z+1]; e++) { int ui = term[3*e], pc = term[3*e+1]; double sg = term[3*e+2];
      double pt[3], c[3]; world_point(m, w, pc, pt);
      dof_point_vel(m, w, d, pt, c); acc += sg*dot3(U + 3*ui, c); }
    mom[z] = acc; }
  const idx_t* padr = CI(PT_piece_adr); const idx_t* piece = CI(PT_piece); const double* tconst = CD(PT_const);
  for (int t = m.tg_ta[g] + w.lane; t < m.tg_ta[g+1]; t += 32) { double l = tconst[t];
    #pragma unroll 1
    for (int e = padr[t]; e < padr[t+1]; e++) l += PL[piece[e]];
    tlen[t] = l; }
  __syncwarp();
}
// after both passes: tendon velocities (moment . qvel); tendon forces start at zero
__device__ void phase_tendon_velocity(const DevModel& m, const Warp w) {
  const double* mom = SCR(s_mom); double* tvel = SCR(s_tvel); double* tfrc = SCR(s_tfrc);
  const idx_t* nadr = CI(PT_nz_adr); const idx_t* nzd = CI(PNZ_dof);
  for (int t = w.lane; t < m.nta; t += 32) { double v = 0;
    #pragma unroll 1
    for (int z = nadr[t]; z < nadr[t+1]; z++) v += mom[z]*W_(qvel)[nzd[z]];
    tvel[t] = v; tfrc[t] = 0; }
  __syncwarp();
}
// both passes (groups A, B) + velocities: the whole tendon stage
__device__ __forceinline__ void phase_tendon_all(const DevModel& m, const Warp w) {
  #pragma unroll 1
  for (int g = 0; g < 2; g++) if (m.tg_ta[g+1] > m.tg_ta[g]) { phase_tendon(m, w, g); phase_tendon_moments(m, w, g); }
  phase_tendon_velocity(m, w);
}

// ------------------------------------------------------------------ phase 3: muscle actuation -> qfrc_smooth (passive + actuator); act integration
__device__ __forceinline__ double muscle_FL(double L, double lmin, double lmax) {
  if (lmin <= L && L <= lmax) { double a = 0.5*(lmin+1), b = 0.5*(1+lmax), x;
    if (L <= a) { x = (L-lmin)*m_rcp(fmax(MYO_MINVAL, a-lmin)); return 0.5*x*x; }
    else if (L <= 1) { x = (1-L)*m_rcp(fmax(MYO_MINVAL, 1-a)); return 1-0.5*x*x; }
    else if (L <= b) { x = (L-1)*m_rcp(fmax(MYO_MINVAL, b-1)); return 1-0.5*x*x; }
    else { x = (lmax-L)*m_rcp(fmax(MYO_MINVAL, lmax-b)); return 0.5*x*x; } }
  return 0; }

// tap_force / tap_len: nullable global rows for the parity taps (values before the activation is advanced)
__device__ void phase_actuation(const DevModel& m, const Warp w, bool integrate, const double* ctrl_row, double* tap_force, double* tap_len) {
  const idx_t* atend = CI(PA_tendon); const idx_t* acls = CI(PA_cls); const double* __restrict__ PAc = GD(PA_d); const double* __restrict__ PAm = GD(PAM_d);      // (cold tables: 17 + 5 independent read-only loads per actuator)
  double* tlen = SCR(s_tlen); double* tvel = SCR(s_tvel); double* tfrc = SCR(s_tfrc); double* mom = SCR(s_mom);
  for (int i = w.lane; i < m.nu; i += 32) { double a[PA_STRIDE]; { const double* __restrict__ ag = PAc + acls[i]*PA_STRIDE; for (int c = 0; c < 16; c++) a[c] = LDC(ag + c); } double am[5]; for (int c = 0; c < 5; c++) am[c] = LDC(PAm + i*PAM_STRIDE + c); int t = atend[i];
    const double *dyn = a, *gp = a+3, *bp = a+9, *cr = a+13; double gear = am[4], lr0 = am[2], lr1 = am[3];
    double len = gear*tlen[t], vel = gear*tvel[t], ctrl = ctrl_row[i], act = W_(act)[i];
    if (a[15] != 0) ctrl = clipd(ctrl, cr[0], cr[1]);
    // activation dynamics
    double cc = clipd(ctrl, 0, 1), ac = clipd(act, 0, 1), ta = dyn[0]*(0.5+1.5*ac), td = dyn[1]*m_rcp(0.5+1.5*ac), dctrl = cc - act, tau;
    if (dyn[2] < MYO_MINVAL) tau = dctrl > 0 ? ta : td;
    else { double x = clipd(dctrl/dyn[2]+0.5, 0, 1), s = x*x*x*(3*x*(2*x-5)+10); tau = td+(ta-td)*s; }
    double actdot = dctrl*m_rcp(fmax(MYO_MINVAL, tau));
    // gain (active force-length-velocity) and bias (passive force)
    const double g_lmin = gp[2], g_lmax = gp[3], g_vmax = gp[4], g_fvmax = gp[5], b_lmax = bp[2], b_fpmax = bp[3];
    double F = am[0], L0 = (lr1-lr0)*m_rcp(fmax(MYO_MINVAL, gp[1]-gp[0])), L = gp[0]+(len-lr0)*m_rcp(fmax(MYO_MINVAL, L0)), V = vel*m_rcp(fmax(MYO_MINVAL, L0*g_vmax));
    double FL = muscle_FL(L, g_lmin, g_lmax), y = g_fvmax-1, FV;
    if (V <= -1) FV = 0; else if (V <= 0) FV = (V+1)*(V+1); else if (V <= y) FV = g_fvmax-(y-V)*(y-V)*m_rcp(fmax(MYO_MINVAL, y)); else FV = g_fvmax;
    double gain = -F*FL*FV;
    double Fb = am[1], L0b = (lr1-lr0)*m_rcp(fmax(MYO_MINVAL, bp[1]-bp[0])), Lb = bp[0]+(len-lr0)*m_rcp(fmax(MYO_MINVAL, L0b)), b = 0.5*(1+b_lmax), bias;
    if (Lb <= 1) bias = 0; else if (Lb <= b) { double x = (Lb-1)*m_rcp(fmax(MYO_MINVAL, b-1)); bias = -Fb*b_fpmax*0.5*x*x; }
    else { double x = (Lb-b)*m_rcp(fmax(MYO_MINVAL, b-1)); bias = -Fb*b_fpmax*(0.5+x); }
    double force = gain*act + bias;
    tfrc[t] = gear*force;   // one actuator per tendon (checked on the host)
    if (tap_force) tap_force[i] = force;
    if (tap_len) tap_len[i] = len;
    if (integrate) W_(act)[i] = act + m.timestep*actdot;   // mj_Euler's activation update; act is not read again this substep
  }
  __syncwarp();
  const idx_t* cadr = CI(PCOL_adr); const idx_t* col = CI(PCOL); const idx_t* nzt = CI(PNZ_tendon); const double* dofp = CD(PDOF_d);
  for (int d = w.lane; d < m.nv; d += 32) { double s = -dofp[2*d+1]*W_(qvel)[d];
    #pragma unroll 1
    for (int e = cadr[d]; e < cadr[d+1]; e++) { int z = col[e]; s += mom[z]*tfrc[nzt[z]]; }
    W_(fsm)[d] = s; }
  __syncwarp();
}

// ------------------------------------------------------------------ phase 4: composite inertia -> joint-space mass matrix
__device__ void phase_crb(const DevModel& m, const Warp w) {
  double* crb = SCR(s_crb); const double* cin = SCR(s_cin); const idx_t* sadr = CI(PSUB_adr); const idx_t* sub = CI(PSUB);
  for (int k = w.lane; k < m.nbd; k += 32) { double acc[10] = {0,0,0,0,0,0,0,0,0,0};
    #pragma unroll 1
    for (int e = sadr[k]; e < sadr[k+1]; e++) { const double* c = cin + 10*sub[e];
      #pragma unroll
      for (int q = 0; q < 10; q++) acc[q] += c[q]; }
    #pragma unroll
    for (int q = 0; q < 10; q++) crb[10*k+q] = acc[q]; }
  __syncwarp();
  const idx_t* mi = CI(PM_i); const idx_t* mj = CI(PM_j); const idx_t* dbody = CI(PD_body); const double* dofp = CD(PDOF_d);
  for (int e = w.lane; e < m.nM; e += 32) { int i = mi[e], j = mj[e]; double Si[6], Sj[6], f[6];
    dof_motion(m, w, i, Si); inert_mul(f, crb + 10*dbody[i], Si); dof_motion(m, w, j, Sj);
    double v = Sj[0]*f[0]+Sj[1]*f[1]+Sj[2]*f[2]+Sj[3]*f[3]+Sj[4]*f[4]+Sj[5]*f[5];
    if (i == j) v += dofp[2*i];
    W_(qM)[e] = v; }
  __syncwarp();
}

// ------------------------------------------------------------------ phase 5: Coriolis/centrifugal/gravity bias (subtracts from fsm)
__device__ void phase_bias(const DevModel& m, const Warp w) {
  double* bf = SCR(s_bf); const double* cin = SCR(s_cin); const idx_t* cadr = CI(PCH_adr); const idx_t* ch = CI(PCH);
  for (int k = w.lane; k < m.nbd; k += 32) {
    double v[6] = {0,0,0,0,0,0}, vh[6] = {0,0,0,0,0,0}, a[6] = {0,0,0,-m.gx,-m.gy,-m.gz};
    #pragma unroll 1
    for (int e = cadr[k]; e < cadr[k+1]; e++) { int d = ch[e] >> 1, flag = ch[e] & 1; double S[6], qd = W_(qvel)[d];
      dof_motion(m, w, d, S);
      if (!flag) { for (int c = 0; c < 6; c++) vh[c] = v[c]; }
      double c0[3], c1[3], c2[3]; cross3(c0, vh, S); cross3(c1, vh, S+3); cross3(c2, vh+3, S);   // vh x_m S
      a[0]+=c0[0]*qd; a[1]+=c0[1]*qd; a[2]+=c0[2]*qd; a[3]+=(c1[0]+c2[0])*qd; a[4]+=(c1[1]+c2[1])*qd; a[5]+=(c1[2]+c2[2])*qd;
      for (int c = 0; c < 6; c++) v[c] += S[c]*qd; }
    double Ia[6], Iv[6]; inert_mul(Ia, cin + 10*k, a); inert_mul(Iv, cin + 10*k, v);
    double t0[3], t1[3], t2[3]; cross3(t0, v, Iv); cross3(t1, v+3, Iv+3); cross3(t2, v, Iv+3);   // f = I a + v x_f (I v)
    bf[6*k] = Ia[0]+t0[0]+t1[0]; bf[6*k+1] = Ia[1]+t0[1]+t1[1]; bf[6*k+2] = Ia[2]+t0[2]+t1[2];
    bf[6*k+3] = Ia[3]+t2[0]; bf[6*k+4] = Ia[4]+t2[1]; bf[6*k+5] = Ia[5]+t2[2]; }
  __syncwarp();
  const idx_t* sadr = CI(PSUB_adr); const idx_t* sub = CI(PSUB); const idx_t* dbody = CI(PD_body);
  for (int d = w.lane; d < m.nv; d += 32) { double S[6], tot = 0; dof_motion(m, w, d, S); int b = dbody[d];
    #pragma unroll 1
    for (int e = sadr[b]; e < sadr[b+1]; e++) { const double* f = bf + 6*sub[e]; tot += S[0]*f[0]+S[1]*f[1]+S[2]*f[2]+S[3]*f[3]+S[4]*f[4]+S[5]*f[5]; }
    W_(fsm)[d] -= tot; }
  __syncwarp();
}

// ------------------------------------------------------------------ phase 6: collision (analytic primitives)
// world position and z axis of every collision geom, once per substep (each geom takes part in ~20 pairs)
__device__ __forceinline__ void geom_pose_all(const DevModel& m, const Warp w) {
  double* GP = SCR(s_gpose);
  for (int g = w.lane; g < m.ngc; g += 32) { int b = CI(PG_body)[g]; const double* gd = CD(PG_d) + g*PG_STRIDE; double* o = GP + 6*g;
    if (b < 0) { o[0]=gd[0]; o[1]=gd[1]; o[2]=gd[2]; o[3]=gd[5]; o[4]=gd[8]; o[5]=gd[11]; }
    else { const double* X = SCR(s_xmat) + 9*b; const double* xp = SCR(s_xpos) + 3*b; mat_vec(o, X, gd); o[0]+=xp[0]; o[1]+=xp[1]; o[2]+=xp[2];
      double z[3] = {gd[5], gd[8], gd[11]}; mat_vec(o+3, X, z); } }
  __syncwarp(); }
__device__ __forceinline__ void geom_pose(const DevModel& m, const Warp w, int g, double* pos, double* axis /* z column */) {
  const double* o = SCR(s_gpose) + 6*g; pos[0]=o[0]; pos[1]=o[1]; pos[2]=o[2]; axis[0]=o[3]; axis[1]=o[4]; axis[2]=o[5]; }

__device__ __forceinline__ const double* geom_size(const DevModel& m, const Warp w, int g) { return g == m.ovr_geom ? W_(eprm) + 3 : CD(PG_d) + g*PG_STRIDE + 12; }
// full world rotation of a collision geom (ellipsoids need it)
__device__ __forceinline__ void geom_mat(const DevModel& m, const Warp w, int g, double* mat) {
  int b = CI(PG_body)[g]; const double* gd = CD(PG_d) + g*PG_STRIDE;
  if (b < 0) {
    #pragma unroll
    for (int c = 0; c < 9; c++) mat[c] = gd[3+c]; } else mat_mul(mat, SCR(s_xmat) + 9*b, gd + 3); }

// ---- ellipsoid colliders.  MuJoCo routes ellipsoid-capsule / ellipsoid-ellipsoid through its general convex collider: one
// contact, signed distance = max over unit d of  d.(c2-c1) - h1(d) - h2(-d)  (h = support function), witnesses = support points.
// Here: Newton on the unit sphere for that maximisation (smooth for ellipsoids and points).
// body 1: ellipsoid (R1, s1) or a point (s1 == nullptr); body 2: ellipsoid.  dl = c2 - c1.  d: in = start, out = maximiser.
// p1, p2: support offsets (witness on body 1 = c1 + p1, on body 2 = c2 - p2).
// bound: every iterate's f is a lower bound of the signed distance -> return as soon as f > bound (the pair cannot be in contact).
__device__ __forceinline__ double ell_sd(const double* dl, const double* R1, const double* s1, const double* R2, const double* s2, double* d, double* p1, double* p2, double bound) {
  double f = 0;
  #pragma unroll 1
  for (int it = 0; it < 40; it++) {
    double a[3], u[3], n1 = 0, n2;
    p1[0] = p1[1] = p1[2] = 0;
    if (s1) { matT_vec(a, R1, d); u[0] = s1[0]*s1[0]*a[0]; u[1] = s1[1]*s1[1]*a[1]; u[2] = s1[2]*s1[2]*a[2]; n1 = m_sqrt(dot3(a, u)); mat_vec(p1, R1, u); double q = m_rcp(n1); p1[0]*=q; p1[1]*=q; p1[2]*=q; }
    matT_vec(a, R2, d); u[0] = s2[0]*s2[0]*a[0]; u[1] = s2[1]*s2[1]*a[1]; u[2] = s2[2]*s2[2]*a[2]; n2 = m_sqrt(dot3(a, u)); mat_vec(p2, R2, u); { double q = m_rcp(n2); p2[0]*=q; p2[1]*=q; p2[2]*=q; }
    double g[3] = {dl[0]-p1[0]-p2[0], dl[1]-p1[1]-p2[1], dl[2]-p1[2]-p2[2]};
    f = dot3(d, dl) - n1 - n2;
    if (f > bound) return f;
    // tangent basis
    double e[3]; { int k = fabs(d[0]) < fabs(d[1]) ? (fabs(d[0]) < fabs(d[2]) ? 0 : 2) : (fabs(d[1]) < fabs(d[2]) ? 1 : 2); e[0] = k == 0; e[1] = k == 1; e[2] = k == 2; }
    double t1[3], t2[3]; cross3(t1, d, e); { double q = m_rcp(m_sqrt(dot3(t1,t1))); t1[0]*=q; t1[1]*=q; t1[2]*=q; } cross3(t2, d, t1);
    double g1 = dot3(t1, g), g2 = dot3(t2, g), scale = m_sqrt(dot3(dl,dl)) + n1 + n2;
    if (g1*g1 + g2*g2 < 1e-24*scale*scale) break;      // tangential gradient ~1e-12: direction converged to round-off
    // tangent Hessian of the Lagrangian:  -sum_i (t_k.A_i t_l - (t_k.p_i)(t_l.p_i))/n_i - f delta_kl
    double H11 = -f, H12 = 0, H22 = -f;
    { double b1[3], b2[3], v[3]; matT_vec(b1, R2, t1); matT_vec(b2, R2, t2);
      v[0] = s2[0]*s2[0]; v[1] = s2[1]*s2[1]; v[2] = s2[2]*s2[2];
      double a11 = v[0]*b1[0]*b1[0]+v[1]*b1[1]*b1[1]+v[2]*b1[2]*b1[2], a12 = v[0]*b1[0]*b2[0]+v[1]*b1[1]*b2[1]+v[2]*b1[2]*b2[2], a22 = v[0]*b2[0]*b2[0]+v[1]*b2[1]*b2[1]+v[2]*b2[2]*b2[2];
      double q1 = dot3(t1, p2), q2 = dot3(t2, p2), in = m_rcp(n2); H11 -= (a11-q1*q1)*in; H12 -= (a12-q1*q2)*in; H22 -= (a22-q2*q2)*in;
    }
    if (s1) { double b1[3], b2[3], v[3]; matT_vec(b1, R1, t1); matT_vec(b2, R1, t2);
      v[0] = s1[0]*s1[0]; v[1] = s1[1]*s1[1]; v[2] = s1[2]*s1[2];
      double a11 = v[0]*b1[0]*b1[0]+v[1]*b1[1]*b1[1]+v[2]*b1[2]*b1[2], a12 = v[0]*b1[0]*b2[0]+v[1]*b1[1]*b2[1]+v[2]*b1[2]*b2[2], a22 = v[0]*b2[0]*b2[0]+v[1]*b2[1]*b2[1]+v[2]*b2[2]*b2[2];
      double q1 = dot3(t1, p1), q2 = dot3(t2, p1), in = m_rcp(n1); H11 -= (a11-q1*q1)*in; H12 -= (a12-q1*q2)*in; H22 -= (a22-q2*q2)*in; }
    double det = H11*H22 - H12*H12, dx, dy;
    if (H11 < 0 && det > 1e-200) { double id = m_rcp(det); dx = -(H22*g1 - H12*g2)*id; dy = -(-H12*g1 + H11*g2)*id; }
    else { double L = m_rcp(fabs(H11) + fabs(H22) + fabs(H12) + 1e-12); dx = g1*L; dy = g2*L; }     // safeguarded ascent step
    double nn = m_sqrt(dx*dx + dy*dy); if (nn > 0.5) { const double q = 0.5*m_rcp(nn); dx *= q; dy *= q; }
    bool last = nn < 1e-12;                            // a step this small cannot change the result
    // backtracking: accept the first step that does not decrease f
    #pragma unroll 1
    for (int bt = 0; bt < 12; bt++) { double dn[3] = {d[0]+dx*t1[0]+dy*t2[0], d[1]+dx*t1[1]+dy*t2[1], d[2]+dx*t1[2]+dy*t2[2]}; double q = m_rcp(m_sqrt(dot3(dn,dn))); dn[0]*=q; dn[1]*=q; dn[2]*=q;
      double fn = dot3(dn, dl); { double aa[3]; matT_vec(aa, R2, dn); fn -= m_sqrt(s2[0]*s2[0]*aa[0]*aa[0]+s2[1]*s2[1]*aa[1]*aa[1]+s2[2]*s2[2]*aa[2]*aa[2]); }
      if (s1) { double aa[3]; matT_vec(aa, R1, dn); fn -= m_sqrt(s1[0]*s1[0]*aa[0]*aa[0]+s1[1]*s1[1]*aa[1]*aa[1]+s1[2]*s1[2]*aa[2]*aa[2]); }
      if (fn >= f - 1e-14*scale || bt == 11) { d[0]=dn[0]; d[1]=dn[1]; d[2]=dn[2]; break; }
      dx *= 0.5; dy *= 0.5; }
    if (last) break;
  }
  return f;
}

// up to two contacts of one geom pair, all scalars (arrays here end up in local memory: round 1's kernel carried a 1.3 KB stack frame)
struct Con1 { double dist, px, py, pz, nx, ny, nz; };
struct ConOut { int n; Con1 c0, c1; double yx, yy, yz; bool has_y; };
__device__ __forceinline__ void con_put(ConOut& o, double dist, double px, double py, double pz, double nx, double ny, double nz) {
  if (o.n == 0) { o.c0.dist = dist; o.c0.px = px; o.c0.py = py; o.c0.pz = pz; o.c0.nx = nx; o.c0.ny = ny; o.c0.nz = nz; }
  else { o.c1.dist = dist; o.c1.px = px; o.c1.py = py; o.c1.pz = pz; o.c1.nx = nx; o.c1.ny = ny; o.c1.nz = nz; }
  o.n++; }
__device__ __forceinline__ void sph_sph(ConOut& o, double margin, const double* p1, double r1, const double* p2, double r2) {
  double dv[3] = {p2[0]-p1[0], p2[1]-p1[1], p2[2]-p1[2]}, cd = m_sqrt(dot3(dv,dv)), dist = cd-r1-r2;
  if (dist > margin || o.n >= 2) return;
  double nx, ny, nz; if (cd < MYO_MINVAL) { nx = 1; ny = 0; nz = 0; } else { double q = m_rcp(cd); nx = dv[0]*q; ny = dv[1]*q; nz = dv[2]*q; }
  double off = r1+0.5*dist;
  con_put(o, dist, p1[0]+nx*off, p1[1]+ny*off, p1[2]+nz*off, nx, ny, nz); }
__device__ __forceinline__ void plane_sph(ConOut& o, double margin, const double* pp, const double* pn, const double* sp, double r) {
  double dv[3] = {sp[0]-pp[0], sp[1]-pp[1], sp[2]-pp[2]}, dist = dot3(dv,pn)-r;
  if (dist > margin || o.n >= 2) return;
  double off = r+0.5*dist;
  con_put(o, dist, sp[0]-pn[0]*off, sp[1]-pn[1]*off, sp[2]-pn[2]*off, pn[0], pn[1], pn[2]); }

__device__ __forceinline__ void collide_analytic(const DevModel& m, const Warp w, int p, ConOut& o) {
  const idx_t* pr = CI(PPAIR) + PPAIR_ISTRIDE*p; const double* pd = CD(PPAIR_d) + pr[6]*PPAIR_STRIDE;
  int g1 = pr[0], g2 = pr[1], ct = pr[5]; double margin = pd[0]; o.n = 0; o.has_y = false;
  const double* s1 = geom_size(m, w, g1); const double* s2 = geom_size(m, w, g2);
  double x1[3], a1[3], x2[3], a2[3]; geom_pose(m, w, g1, x1, a1); geom_pose(m, w, g2, x2, a2);
  if (ct == CT_CAP_CAP) {
    double r1 = s1[0], h1 = s1[1], r2 = s2[0], h2 = s2[1];
    double dv[3] = {x1[0]-x2[0], x1[1]-x2[1], x1[2]-x2[2]};
    // cheap reject: the capsules' bounding spheres are farther apart than the margin
    { double rb = r1+h1+r2+h2+margin; if (dot3(dv,dv) > rb*rb) return; }
    double ma = dot3(a1,a1), mb = -dot3(a1,a2), mc = dot3(a2,a2), u = -dot3(a1,dv), v = dot3(a2,dv), det = ma*mc-mb*mb, v1[3], v2[3];
    if (fabs(det) >= MYO_MINVAL) {
      double id = m_rcp(det), t1 = (mc*u-mb*v)*id, t2 = (ma*v-mb*u)*id; const double imc = m_rcp(mc), ima = m_rcp(ma);
      if (t1 > h1) { t1 = h1; t2 = (v-mb*h1)*imc; } else if (t1 < -h1) { t1 = -h1; t2 = (v+mb*h1)*imc; }
      if (t2 > h2) { t2 = h2; t1 = clipd((u-mb*h2)*ima, -h1, h1); } else if (t2 < -h2) { t2 = -h2; t1 = clipd((u+mb*h2)*ima, -h1, h1); }
      for (int k = 0; k < 3; k++) { v1[k] = x1[k]+a1[k]*t1; v2[k] = x2[k]+a2[k]*t2; }
      sph_sph(o, margin, v1, r1, v2, r2);
    } else {   // parallel axes: up to two contacts
      double t;
      for (int k = 0; k < 3; k++) v1[k] = x1[k]+a1[k]*h1; t = clipd((v-mb*h1)/mc, -h2, h2); for (int k = 0; k < 3; k++) v2[k] = x2[k]+a2[k]*t; sph_sph(o, margin, v1, r1, v2, r2);
      for (int k = 0; k < 3; k++) v1[k] = x1[k]-a1[k]*h1; t = clipd((v+mb*h1)/mc, -h2, h2); for (int k = 0; k < 3; k++) v2[k] = x2[k]+a2[k]*t; sph_sph(o, margin, v1, r1, v2, r2);
      if (o.n < 2) { for (int k = 0; k < 3; k++) v2[k] = x2[k]+a2[k]*h2; t = clipd((u-mb*h2)/ma, -h1, h1); for (int k = 0; k < 3; k++) v1[k] = x1[k]+a1[k]*t; sph_sph(o, margin, v1, r1, v2, r2); }
      if (o.n < 2) { for (int k = 0; k < 3; k++) v2[k] = x2[k]-a2[k]*h2; t = clipd((u+mb*h2)/ma, -h1, h1); for (int k = 0; k < 3; k++) v1[k] = x1[k]+a1[k]*t; sph_sph(o, margin, v1, r1, v2, r2); }
    }
  } else if (ct == CT_SPH_SPH) { sph_sph(o, margin, x1, s1[0], x2, s2[0]);
  } else if (ct == CT_SPH_CAP) { double dv[3] = {x1[0]-x2[0], x1[1]-x2[1], x1[2]-x2[2]}, t = clipd(dot3(a2,dv), -s2[1], s2[1]), v2[3];
    for (int k = 0; k < 3; k++) v2[k] = x2[k]+a2[k]*t; sph_sph(o, margin, x1, s1[0], v2, s2[0]);
  } else if (ct == CT_PLANE_SPH) { plane_sph(o, margin, x1, a1, x2, s2[0]);
  } else if (ct == CT_PLANE_CAP) { double e[3];
    for (int k = 0; k < 3; k++) e[k] = x2[k]+a2[k]*s2[1]; plane_sph(o, margin, x1, a1, e, s2[0]);
    for (int k = 0; k < 3; k++) e[k] = x2[k]-a2[k]*s2[1]; plane_sph(o, margin, x1, a1, e, s2[0]);
    o.has_y = true; o.yx = a2[0]; o.yy = a2[1]; o.yz = a2[2];
  } else if (ct == CT_PLANE_ELL) {   // deepest point of the ellipsoid along -normal
    double R2[9], nl[3], u[3], pw[3]; geom_mat(m, w, g2, R2); matT_vec(nl, R2, a1);
    u[0] = s2[0]*s2[0]*nl[0]; u[1] = s2[1]*s2[1]*nl[1]; u[2] = s2[2]*s2[2]*nl[2]; double nn = m_rcp(m_sqrt(dot3(nl, u))); mat_vec(pw, R2, u);
    double pos[3] = {x2[0]-pw[0]*nn, x2[1]-pw[1]*nn, x2[2]-pw[2]*nn}, dv[3] = {pos[0]-x1[0], pos[1]-x1[1], pos[2]-x1[2]}, dist = dot3(dv, a1);
    if (dist <= margin) con_put(o, dist, pos[0]-a1[0]*0.5*dist, pos[1]-a1[1]*0.5*dist, pos[2]-a1[2]*0.5*dist, a1[0], a1[1], a1[2]);
  }
}

__device__ __forceinline__ void collide_ellipsoid(const DevModel& m, const Warp w, int p, ConOut& o) {
  const idx_t* pr = CI(PPAIR) + PPAIR_ISTRIDE*p; const double* pd = CD(PPAIR_d) + pr[6]*PPAIR_STRIDE;
  int g1 = pr[0], g2 = pr[1], ct = pr[5]; double margin = pd[0]; o.n = 0; o.has_y = false;
  const double* s1 = geom_size(m, w, g1); const double* s2 = geom_size(m, w, g2);
  double x1[3], a1[3], x2[3], a2[3]; geom_pose(m, w, g1, x1, a1); geom_pose(m, w, g2, x2, a2);
  if (ct == CT_CAP_ELL) {     // g1 capsule (segment + radius), g2 ellipsoid: min over the segment of the point-ellipsoid distance
    double r = s1[0], h = s1[1], dv[3] = {x2[0]-x1[0], x2[1]-x1[1], x2[2]-x1[2]};
    double R2[9]; geom_mat(m, w, g2, R2);
    // (1) distance to the capsule's whole AXIS LINE = distance, in the plane normal to the axis, from the projected centre to the
    //     ellipsoid's shadow (an ellipse): a 1-D Newton on the unit circle  max_u  c.u - sqrt(u'Au).  Every iterate's value is a
    //     lower bound of the segment distance, so a pair that is provably out of its margin leaves at once.
    double e1[3], e2[3]; { double e[3]; int k = fabs(a1[0]) < fabs(a1[1]) ? (fabs(a1[0]) < fabs(a1[2]) ? 0 : 2) : (fabs(a1[1]) < fabs(a1[2]) ? 1 : 2); e[0] = k == 0; e[1] = k == 1; e[2] = k == 2;
      cross3(e1, a1, e); double q = m_rcp(m_sqrt(dot3(e1,e1))); e1[0]*=q; e1[1]*=q; e1[2]*=q; cross3(e2, a1, e1); }
    double b1[3], b2[3]; matT_vec(b1, R2, e1); matT_vec(b2, R2, e2);
    double v0 = s2[0]*s2[0], v1 = s2[1]*s2[1], v2 = s2[2]*s2[2];
    double A11 = v0*b1[0]*b1[0]+v1*b1[1]*b1[1]+v2*b1[2]*b1[2], A12 = v0*b1[0]*b2[0]+v1*b1[1]*b2[1]+v2*b1[2]*b2[2], A22 = v0*b2[0]*b2[0]+v1*b2[1]*b2[1]+v2*b2[2]*b2[2];
    double c1 = dot3(e1, dv), c2 = dot3(e2, dv), cn = m_sqrt(c1*c1+c2*c2), u1 = 1, u2 = 0, F = 0, scale = cn + m_sqrt(fmax(A11, A22));
    if (cn > MYO_MINVAL) { const double q = m_rcp(cn); u1 = c1*q; u2 = c2*q; }
    #pragma unroll 1
    for (int it = 0; it < 40; it++) {
      double Au1 = A11*u1+A12*u2, Au2 = A12*u1+A22*u2, n2 = u1*Au1+u2*Au2, n = m_sqrt(n2), in = m_rcp(n);
      F = c1*u1+c2*u2 - n;
      if (F - r > margin) return;
      double p1_ = -u2, p2_ = u1;                                  // u_perp
      double uAp = p1_*Au1+p2_*Au2, pAp = A11*p1_*p1_+2*A12*p1_*p2_+A22*p2_*p2_;
      double g = c1*p1_+c2*p2_ - uAp*in, H = -(c1*u1+c2*u2) - ((pAp-n2)*in - uAp*uAp*in*in*in);
      if (fabs(g) < 1e-12*scale) break;
      double dx = H < -1e-200 ? -g*m_rcp(H) : g*m_rcp(fabs(H)+1e-12); if (fabs(dx) > 0.5) dx = dx > 0 ? 0.5 : -0.5;
      bool last = fabs(dx) < 1e-12;
      #pragma unroll 1
      for (int bt = 0; bt < 12; bt++) { double w1 = u1+dx*p1_, w2 = u2+dx*p2_, q = m_rcp(m_sqrt(w1*w1+w2*w2)); w1 *= q; w2 *= q;
        double fn = c1*w1+c2*w2 - m_sqrt(A11*w1*w1+2*A12*w1*w2+A22*w2*w2);
        if (fn >= F - 1e-14*scale || bt == 11) { u1 = w1; u2 = w2; break; }
        dx *= 0.5; }
      if (last) break; }
    double d[3] = {u1*e1[0]+u2*e2[0], u1*e1[1]+u2*e2[1], u1*e1[2]+u2*e2[2]}, p1[3], p2[3], t, sd;
    { double a[3], u[3]; matT_vec(a, R2, d); u[0] = v0*a[0]; u[1] = v1*a[1]; u[2] = v2*a[2]; double nn = m_sqrt(dot3(a, u)); mat_vec(p2, R2, u); double q = m_rcp(nn); p2[0]*=q; p2[1]*=q; p2[2]*=q; }
    t = (dv[0]-p2[0])*a1[0] + (dv[1]-p2[1])*a1[1] + (dv[2]-p2[2])*a1[2];        // axis coordinate of the ellipsoid-side witness
    if (t >= -h && t <= h) sd = F;
    else {   // (2) the line's closest point is beyond a cap: the distance over the segment (convex in t) is attained at that end point
      t = t > h ? h : -h; double dl[3] = {dv[0]-a1[0]*t, dv[1]-a1[1]*t, dv[2]-a1[2]*t};
      sd = ell_sd(dl, nullptr, nullptr, R2, s2, d, p1, p2, margin + r); }
    double dist = sd - r;
    if (dist <= margin) con_put(o, dist, 0.5*((x1[0]+a1[0]*t + d[0]*r) + (x2[0]-p2[0])), 0.5*((x1[1]+a1[1]*t + d[1]*r) + (x2[1]-p2[1])), 0.5*((x1[2]+a1[2]*t + d[2]*r) + (x2[2]-p2[2])), d[0], d[1], d[2]);
  } else if (ct == CT_ELL_ELL) {
    double dl[3] = {x2[0]-x1[0], x2[1]-x1[1], x2[2]-x1[2]}, cd = m_sqrt(dot3(dl,dl));
    if (cd - fmax(s1[0], fmax(s1[1], s1[2])) - fmax(s2[0], fmax(s2[1], s2[2])) > margin) return;
    double R1[9], R2[9], d[3], p1[3], p2[3]; geom_mat(m, w, g1, R1); geom_mat(m, w, g2, R2);
    if (cd < MYO_MINVAL) { d[0]=1; d[1]=0; d[2]=0; } else { const double q = m_rcp(cd); d[0]=dl[0]*q; d[1]=dl[1]*q; d[2]=dl[2]*q; }
    double dist = ell_sd(dl, R1, s1, R2, s2, d, p1, p2, margin);
    if (dist <= margin) con_put(o, dist, 0.5*((x1[0]+p1[0]) + (x2[0]-p2[0])), 0.5*((x1[1]+p1[1]) + (x2[1]-p2[1])), 0.5*((x1[2]+p1[2]) + (x2[2]-p2[2])), d[0], d[1], d[2]);
  }
}

// cheap conservative test for the iterative (ellipsoid) colliders: can this pair be within its margin at all?
__device__ __forceinline__ bool expensive_candidate(const DevModel& m, const Warp w, int p) {
  const idx_t* pr = CI(PPAIR) + PPAIR_ISTRIDE*p; const double* pd = CD(PPAIR_d) + pr[6]*PPAIR_STRIDE;
  int g1 = pr[0], g2 = pr[1]; const double* s1 = geom_size(m, w, g1); const double* s2 = geom_size(m, w, g2); double margin = pd[0];
  double x1[3], a1[3], x2[3], a2[3]; geom_pose(m, w, g1, x1, a1); geom_pose(m, w, g2, x2, a2);
  double dv[3] = {x2[0]-x1[0], x2[1]-x1[1], x2[2]-x1[2]}, rb2 = fmax(s2[0], fmax(s2[1], s2[2]));
  // any unit direction d gives a lower bound  d.(c2-c1) - h1(d) - h2(d)  on the signed distance: use the centre-to-centre
  // (or centre-to-segment) direction -- tight for the flat finger-pad ellipsoids, unlike a bounding sphere
  if (pr[5] == CT_CAP_ELL) { double t = clipd(dot3(dv, a1), -s1[1], s1[1]), q[3] = {dv[0]-a1[0]*t, dv[1]-a1[1]*t, dv[2]-a1[2]*t}, nq = m_sqrt(dot3(q,q));
    if (nq - s1[0] - rb2 > margin) return false;
    if (nq < MYO_MINVAL) return true;
    double R2[9], b[3], iq = m_rcp(nq), d[3] = {q[0]*iq, q[1]*iq, q[2]*iq}; geom_mat(m, w, g2, R2); matT_vec(b, R2, d);
    return nq - m_sqrt(s2[0]*s2[0]*b[0]*b[0]+s2[1]*s2[1]*b[1]*b[1]+s2[2]*s2[2]*b[2]*b[2]) - s1[0] <= margin; }
  double cd = m_sqrt(dot3(dv,dv));
  if (cd - fmax(s1[0], fmax(s1[1], s1[2])) - rb2 > margin) return false;
  if (cd < MYO_MINVAL) return true;
  double R1[9], R2[9], b[3], c[3], icd = m_rcp(cd), d[3] = {dv[0]*icd, dv[1]*icd, dv[2]*icd}; geom_mat(m, w, g1, R1); geom_mat(m, w, g2, R2); matT_vec(b, R1, d); matT_vec(c, R2, d);
  return cd - m_sqrt(s1[0]*s1[0]*b[0]*b[0]+s1[1]*s1[1]*b[1]*b[1]+s1[2]*s1[2]*b[2]*b[2]) - m_sqrt(s2[0]*s2[0]*c[0]*c[0]+s2[1]*s2[1]*c[1]*c[1]+s2[2]*s2[2]*c[2]*c[2]) <= margin; }

__device__ __forceinline__ void store_contact(const DevModel& m, double* con, idx_t* icon, int ci, int p, const Con1& c, const ConOut& o) {
  if (ci >= m.maxcon) return;
  double* cd = con + ci*CON_STRIDE; cd[0] = c.dist; cd[1] = c.px; cd[2] = c.py; cd[3] = c.pz;
  double* f = cd + 4; f[0] = c.nx; f[1] = c.ny; f[2] = c.nz;
  // complete the contact frame (rows: normal, tangent1, tangent2)
  double y0 = 0, y1 = 0, y2 = 0;
  if (o.has_y) { y0 = o.yx; y1 = o.yy; y2 = o.yz; }
  if (y0*y0+y1*y1+y2*y2 < 0.25) { y0 = 0; y1 = 0; y2 = 0; if (c.ny < 0.5 && c.ny > -0.5) y1 = 1; else y2 = 1; }
  double dd = c.nx*y0+c.ny*y1+c.nz*y2; y0 -= dd*c.nx; y1 -= dd*c.ny; y2 -= dd*c.nz; double n = m_rcp(m_sqrt(y0*y0+y1*y1+y2*y2));
  f[3] = y0*n; f[4] = y1*n; f[5] = y2*n;
  icon[ci] = (idx_t)p; }

// Contacts are found by the analytic colliders first ([0, na)), then by the iterative ellipsoid colliders ([na, ncon)), each run in model pair
// order; phase_constraints ranks them into ONE model-pair order (contact reporting, numbering of the constraint rows) without moving records.
// Overflow (more contacts than maxcon, or more surviving ellipsoid candidates than kcand): the extra ones are dropped first-come and
// CNT_overflow is set; the step kernel ORs it into the caller's sticky per-env `overflow` buffer.
__device__ void phase_collision(const DevModel& m, const Warp w) {
  double* con = SCR(s_con); idx_t* icon = S_cpair;
  int ncon = 0, overflow = 0;
  geom_pose_all(m, w);
  // analytic primitives: one pair per lane
  #pragma unroll 1
  for (int base = 0; base < m.npair_an; base += 32) { int p = base + w.lane; ConOut o; o.n = 0; o.has_y = false;
    if (p < m.npair_an) collide_analytic(m, w, p, o);
    unsigned m0 = __ballot_sync(FULL, o.n >= 1), m1 = __ballot_sync(FULL, o.n >= 2), lt = (1u << w.lane) - 1;
    int idx = ncon + __popc(m0 & lt) + __popc(m1 & lt);
    if (o.n >= 1) store_contact(m, con, icon, idx, p, o.c0, o);
    if (o.n >= 2) store_contact(m, con, icon, idx + 1, p, o.c1, o);
    ncon += __popc(m0) + __popc(m1); }
  if (ncon > m.maxcon) { overflow = 1; ncon = m.maxcon; }
  const int na = ncon;
  if (m.npair > m.npair_an) {
    // iterative ellipsoid colliders: rare and expensive -> conservative cull + compaction, then one surviving candidate per lane
    int* clist = (int*)SCR(s_clist); int ncand = 0;
    #pragma unroll 1
    for (int cbase = m.npair_an; cbase < m.npair; cbase += 32) { int p = cbase + w.lane; bool cand = p < m.npair && expensive_candidate(m, w, p);
      unsigned mk = __ballot_sync(FULL, cand); int slot = ncand + __popc(mk & ((1u << w.lane) - 1)); if (cand && slot < m.kcand) clist[slot] = p; ncand += __popc(mk); }
    if (ncand > m.kcand) { ncand = m.kcand; overflow = 1; }   // (kcand = capacity of the candidate list)
    __syncwarp();
    #pragma unroll 1
    for (int kb = 0; kb < ncand; kb += 32) { int k = kb + w.lane; ConOut o; o.n = 0; o.has_y = false; int p = 0;
      if (k < ncand) { p = clist[k]; collide_ellipsoid(m, w, p, o); }
      unsigned m0 = __ballot_sync(FULL, o.n >= 1); int idx = ncon + __popc(m0 & ((1u << w.lane) - 1));
      if (o.n) store_contact(m, con, icon, idx, p, o.c0, o);
      ncon += __popc(m0); }
    if (ncon > m.maxcon) { overflow = 1; ncon = m.maxcon; }
  }
  WI_(ncon) = ncon; WI_(na) = na; WI_(overflow) = overflow;
  __syncwarp();
}

// myo_b200.cu -- kernels + C-ABI of libmyo_b200.so (see include/myo_b200.h for the boundary contract).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -shared -Xcompiler -fPIC
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>

#include "myo_layout.cuh"

// ------------------------------------------------------------------ kernel arguments
#define MYO_BMASK 0x40      /* phases of the product kernels that start with a CTA barrier (bit k = phase k).  0x40: only the solver entry, whose inner
                               barriers need aligned warps anyway; with load-sorted rounds the warps of a CTA stay close without the other phase barriers. */
// Transition-FD kernel (myo_batch_transition_fd): work item k = env * ncol + column; columns [0, nxa) are A's (state), the rest B's (ctrl)
struct FdArgs {
  double* A; double* B;         // the caller's outputs [n, nx, nx] / [n, nx, nu] (nullable)
  const double* nom;            // nominal interval's result: the rollout carry, blocks qpos [n, nq] | qvel [n, nv] | act [n, na]
  double* rows;                 // per-slot rows (slot = CTA * warps + warp): perturbed ctrl [nu], then the + pass's qpos | qvel | act
  double eps, rinv1, rinv2;     // eps, 1 / eps and 1 / (2 eps), IEEE-rounded on the host
  int n_env, ncol, nxa, npass;  // npass: 2 when centered (+ pass, then - pass), else 1
};
struct StepArgs {
  myo_buffers b; myo_task_cfg cfg;
  int n_env, obs_dim, mode;     // mode 0: env step ; 1: debug forward (ctrl verbatim, optional substeps) ; 2: reset only
  int n_substeps;               // mode 1
  int balanced;                 // slot -> env map without perm (slot_env): 1 = e % grid (big models), 0 = contiguous groups of warps (small models)
  const double* dbg_ctrl;       // mode 1
  const uint8_t* reset_mask;    // mode 2 (nullable)
  int* load;                    // mode 0, product kernels (nullable): per-env load key written at the end of the step (mean contacts + Newton iterations per substep)
  const int* perm;              // mode 0, product kernels (nullable): slot -> env, built from last step's load keys by myo_regroup_kernel (-1 = idle slot)
  int perm_rounds;              // rounds of warps each CTA walks when perm is set
  int load_wn, load_wi;         // load key = (load_wn * contacts + load_wi * Newton iterations) averaged over the substeps
  unsigned long long seed; long long env_offset;
  double tol, dt;
  myo_rollout_buffers roll;     // rollout kernels: the caller's ctrl / qfrc_applied and output rows (b points the state at the carry)
  int roll_t, roll_nstep;       // rollout kernels: the interval this launch runs, of how many
  FdArgs fd;                    // transition-FD kernel
};
static const int LOAD_WN = 2, LOAD_WI = 3;      // the load key's weights (StepArgs.load_wn / load_wi) for the product kernels' env steps

// Slot -> env map without load sorting (slot j0 + wid of a CTA: warp wid of the round starting at j0).  Balanced: env e on CTA e % grid, so
// no CTA runs a full extra round while the others idle (4096 envs on 132 SMs at 11 warps: rounds of 11, 11, 9 or 10 everywhere instead of
// 11, 11, 11 on four fifths of the SMs).  Contiguous: each round of a CTA takes nw consecutive envs (neighbouring rows share cache lines).
// SLOTS_PER_CTA is a macro so that the step kernels read gridDim.x inside each branch: as a function argument the read moves ahead of the
// branch and their register allocation changes.
#define SLOTS_PER_CTA(balanced, n_env, grid, nw) ((balanced) ? ((n_env) + (grid) - 1)/(grid) : (((n_env) + (nw) - 1)/(nw) + (grid) - 1)/(grid)*(nw))
__host__ __device__ __forceinline__ int slot_env(int balanced, int cta, int grid, int nw, int j0, int wid) { return balanced ? cta + grid*(j0 + wid) : (cta + grid*(j0/nw))*nw + wid; }

// ------------------------------------------------------------------ Philox4x32-10 (counter-based RNG, one stream per (seed, env, episode))
struct Philox { uint32_t c0, c1, c2, c3, k0, k1, o0, o1, o2, o3; int have; };   // scalars only: indexed arrays would live in local memory
__device__ __forceinline__ void philox_gen(Philox& p) {
  uint32_t c0 = p.c0, c1 = p.c1, c2 = p.c2, c3 = p.c3, k0 = p.k0, k1 = p.k1;
  #pragma unroll
  for (int r = 0; r < 10; r++) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u*c0, hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u*c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0; c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
  p.o0 = c0; p.o1 = c1; p.o2 = c2; p.o3 = c3; p.have = 4; if (++p.c0 == 0) ++p.c1; }
// Stream key (include/myo_b200.h, myo_batch_reset): c1 carries the lane and env bits 20-46, c2 env bits 0-19 and, above them, episode bits
// 0-11, c3 env bits 32-63 and episode bits 12-43.  Injective for env < 2^47, episode < 2^44, lane < 32; c1 == lane for env < 2^20.
__device__ __forceinline__ void philox_init(Philox& p, unsigned long long seed, unsigned long long env, unsigned long long episode, uint32_t lane) {
  p.k0 = (uint32_t)seed; p.k1 = (uint32_t)(seed >> 32); p.c0 = 0; p.c1 = lane | ((uint32_t)(env >> 20) << 5); p.c2 = (uint32_t)env ^ (uint32_t)(episode << 20); p.c3 = (uint32_t)(env >> 32) ^ (uint32_t)(episode >> 12) ^ 0x4D594F42u; p.have = 0; }
__device__ __noinline__ double philox_uniform(Philox& p) {   // [0,1) with 53 random bits; consumes the outputs in pairs (0,1) then (2,3)
  if (p.have < 2) philox_gen(p);
  uint32_t a = p.have == 4 ? p.o0 : p.o2, b = p.have == 4 ? p.o1 : p.o3; p.have -= 2;
  return ((double)(((unsigned long long)(a >> 5) << 26) | (b >> 6))) * (1.0/9007199254740992.0); }

// ------------------------------------------------------------------ parity taps
template <class MD> __device__ void write_taps_solve(const MD& m, const Warp w, const StepArgs& a, int env) {   // after the Newton solve
  const myo_buffers& b = a.b;
  if (b.tap_qacc) for (int i = w.lane; i < m.nv; i += 32) b.tap_qacc[(size_t)env*m.nv+i] = S_a[i];
  if (b.tap_qfrc_smooth) for (int i = w.lane; i < m.nv; i += 32) b.tap_qfrc_smooth[(size_t)env*m.nv+i] = W_(fsm)[i];
  if (b.tap_qM) for (int i = w.lane; i < m.nM; i += 32) b.tap_qM[(size_t)env*m.nM+i] = W_(qM)[i];
  if (b.tap_ncon && w.lane == 0) { int* t = b.tap_ncon + 4*(size_t)env; t[0] = WI_(ncon); t[1] = WI_(nefc); t[2] = WI_(niter); t[3] = WI_(overflow); }
  __syncwarp();
}
template <class MD> __device__ void write_taps_contacts(const MD& m, const Warp w, const StepArgs& a, int env) {   // after constraint assembly (con is overwritten by the solve)
  const myo_buffers& b = a.b; const int ncon = WI_(ncon);
  // reported in model pair order (the rank phase_constraints assigned), -1 / 0 padded
  if (b.tap_contact_pair) for (int c = w.lane; c < m.maxcon; c += 32) if (c >= ncon) b.tap_contact_pair[(size_t)env*m.maxcon+c] = -1;
  if (b.tap_contact_dist) for (int c = w.lane; c < m.maxcon; c += 32) if (c >= ncon) b.tap_contact_dist[(size_t)env*m.maxcon+c] = 0.0;
  for (int c = w.lane; c < ncon; c += 32) { const int r = CRANK(S_crown[c]);
    if (b.tap_contact_pair) b.tap_contact_pair[(size_t)env*m.maxcon+r] = S_cpair[c];
    if (b.tap_contact_dist) b.tap_contact_dist[(size_t)env*m.maxcon+r] = S_con[c*CON_STRIDE]; }
  __syncwarp();
}

// ------------------------------------------------------------------ task logic: pose task (pose_v0.py:100-140,154-170,174-257)
template <class MD> __device__ void env_reset(const MD& m, const Warp w, const StepArgs& a, int env) {
  const myo_buffers& b = a.b; long long ep = b.episode_count ? b.episode_count[env] : 0;
  Philox rng; philox_init(rng, a.seed, (unsigned long long)(a.env_offset + env), (unsigned long long)ep, (uint32_t)w.lane);
  const idx_t* jtype = CI(jnt_type); const idx_t* jq = CI(jnt_qposadr); const double* jrange = CD(jnt_range); const double* qpos0 = CD(qpos0);
  for (int i = w.lane; i < m.nq; i += 32) W_(qpos)[i] = b.init_qpos ? b.init_qpos[i] : qpos0[i];
  int key = 0;                                  // row of init_qpos / init_qvel this episode starts from
  if (a.cfg.task == MYO_TASK_WALK && a.cfg.reset_random && b.init_qpos) {
    // WalkEnvV0.get_randomized_initial_state (walk_v0.py:321-337): keyframe 2 or 3 with probability 1/2 (init_qpos rows 0 / 1), then
    // qpos += N(0, 0.02) on every coordinate except the height qpos[2] (the quaternion "restore" there writes a view back onto
    // itself, so the root quaternion keeps its noise; the kinematics normalise it)
    double u = __shfl_sync(FULL, philox_uniform(rng), 0); key = u < 0.5 ? 0 : 1;
    for (int i = w.lane; i < m.nq; i += 32) { double u1 = philox_uniform(rng), u2 = philox_uniform(rng);
      double z = sqrt(-2.0*log(fmax(u1, 1e-300)))*cos(6.283185307179586*u2), q = b.init_qpos[(size_t)key*m.nq + i];
      W_(qpos)[i] = i == 2 ? q : q + 0.02*z; } }
  __syncwarp();
  if (a.cfg.task == MYO_TASK_POSE) {
    // target_jnt_value ~ U(target_jnt_range) ; reset_type "random": qpos ~ U(jnt_range)
    for (int j = w.lane; j < m.njnt; j += 32) { if (jtype[j] == 0) continue; int qa = jq[j];
      double u0 = philox_uniform(rng), u1 = philox_uniform(rng);
      if (b.target && b.target_range) b.target[(size_t)env*m.nq+qa] = b.target_range[2*qa] + u0*(b.target_range[2*qa+1]-b.target_range[2*qa]);
      if (a.cfg.reset_random) W_(qpos)[qa] = jrange[2*j] + u1*(jrange[2*j+1]-jrange[2*j]); }
  }
  if (a.cfg.task == MYO_TASK_REACH && a.cfg.joint_random[1] > a.cfg.joint_random[0]) {
    // ReachEnvV0.generate_qpos (walk_v0.py:152-167): the first qpos coordinate of EVERY joint (the free root's x included) += U(lo, hi), then
    // clipped to jnt_range whether or not the joint is limited.  Rounded as numpy's uniform (low + (high - low) u) and sum, without FMA.
    const double lo = a.cfg.joint_random[0], span = a.cfg.joint_random[1] - lo;
    for (int j = w.lane; j < m.njnt; j += 32) { const int qa = jq[j];
      const double q = __dadd_rn(W_(qpos)[qa], __dadd_rn(lo, __dmul_rn(span, philox_uniform(rng))));
      W_(qpos)[qa] = fmin(fmax(q, jrange[2*j]), jrange[2*j+1]); }
    __syncwarp(); }
  if (a.cfg.task == MYO_TASK_REACH && b.target && b.target_range) {
    // ReachEnvV0.generate_target_pose (reach_v0.py:163-170): every target site ~ U(span) per coordinate
    for (int k = w.lane; k < 3*a.cfg.task_i[0]; k += 32) { double u = philox_uniform(rng); b.target[(size_t)env*m.nq+k] = b.target_range[2*k] + u*(b.target_range[2*k+1]-b.target_range[2*k]); } }
  if (a.cfg.task == MYO_TASK_HOLD && b.env_prm) {
    // ObjHoldRandomEnvV0.reset (obj_hold_v0.py:126-145): goal = object_init_pos + U(-3cm, 3cm)^3 ; object size ~ U(2cm, 3cm)^3
    // (Fixed variant, reset_random == 0: model values in task_d[6..11])
    if (w.lane < 6) { double u = philox_uniform(rng), v;
      if (w.lane < 3) v = a.cfg.reset_random ? a.cfg.task_d[3+w.lane] + (-0.030 + 0.060*u) : a.cfg.task_d[6+w.lane];
      else v = a.cfg.reset_random ? 0.020 + 0.010*u : a.cfg.task_d[6+w.lane];
      W_(eprm)[w.lane] = v; b.env_prm[(size_t)env*8 + w.lane] = v; } }
  for (int i = w.lane; i < m.nv; i += 32) { W_(qvel)[i] = b.init_qvel ? b.init_qvel[(size_t)key*m.nv + i] : 0.0; W_(qws)[i] = 0; }
  for (int i = w.lane; i < m.na; i += 32) W_(act)[i] = 0;
  if (b.fatigue && a.cfg.muscle_condition == MYO_COND_FATIGUE) for (int i = w.lane; i < m.nu; i += 32) { double* f = b.fatigue + (size_t)env*3*m.nu;      // CumulativeFatigue.reset (fatigue.py:82-99)
    if (a.cfg.fatigue_reset == 1) { const double nf = philox_uniform(rng), ap = philox_uniform(rng); f[i] = nf*ap; f[m.nu+i] = nf*(1-ap); f[2*m.nu+i] = 1-nf; }
    else if (a.cfg.fatigue_reset == 2 && b.fatigue_reset_vec) { const double v = b.fatigue_reset_vec[i]; f[i] = 0; f[m.nu+i] = 1-v; f[2*m.nu+i] = v; }
    else { f[i] = 0; f[m.nu+i] = 1; f[2*m.nu+i] = 0; } }
  if (w.lane == 0) { if (b.time) b.time[env] = 0; if (b.step_count) b.step_count[env] = 0; if (b.episode_count) b.episode_count[env] = ep+1; if (b.ep_return) b.ep_return[env] = 0; }
  __syncwarp();
}

template <class MD> __device__ void write_obs_pose(const MD& m, const Warp w, const StepArgs& a, int env, double* dist_out, double* actmag_out) {
  const myo_buffers& b = a.b; float* o = b.obs ? b.obs + (size_t)env*a.obs_dim : nullptr; double d2 = 0, a2 = 0;
  for (int i = w.lane; i < m.nq; i += 32) { double tgt = b.target ? b.target[(size_t)env*m.nq+i] : 0.0, err = tgt - W_(qpos)[i]; d2 += err*err;
    if (o) { o[i] = (float)W_(qpos)[i]; o[m.nq+m.nv+i] = (float)err; } }
  if (o) for (int i = w.lane; i < m.nv; i += 32) o[m.nq+i] = (float)(W_(qvel)[i]*a.dt);
  for (int i = w.lane; i < m.na; i += 32) { a2 += W_(act)[i]*W_(act)[i]; if (o) o[2*m.nq+m.nv+i] = (float)W_(act)[i]; }
  *dist_out = sqrt(warp_sum(d2)); double am = sqrt(warp_sum(a2)); *actmag_out = m.na ? am/m.na : am;
}

// reward / done of the current state (pose_v0.py:113-140); lane 0 writes
template <class MD> __device__ void pose_reward_done(const MD& m, const Warp w, const StepArgs& a, int env, double* rw_out, bool* done_out) {
  double dist, am; write_obs_pose(m, w, a, env, &dist, &am);
  const double far_th = a.cfg.task_d[0] > 0 ? a.cfg.task_d[0] : 4*3.14159265358979323846/2; double thd = a.cfg.pose_thd;      // PoseEnvV0: 2 pi (pose_v0.py:117); TorsoEnvV0: pi (torso_v0.py:104), passed in task_d[0]
  *rw_out = a.cfg.weights[0]*(-dist) + a.cfg.weights[1]*((dist < thd ? 1.0 : 0.0)+(dist < 1.5*thd ? 1.0 : 0.0)) + a.cfg.weights[2]*(-am) + a.cfg.weights[3]*(dist > far_th ? -1.0 : 0.0);
  *done_out = dist > far_th; }

// spatial velocity [omega; v_origin] of dynamic body k from its dof chain
template <class MD> __device__ __forceinline__ void body_velocity(const MD& m, const Warp w, int k, double* v) {
  const idx_t* cadr = CI(PCH_adr); const idx_t* ch = CI(PCH);
  for (int c = 0; c < 6; c++) v[c] = 0;
  #pragma unroll 1
  for (int e = cadr[k]; e < cadr[k+1]; e++) { int d = ch[e] >> 1; double S[6], qd = W_(qvel)[d]; dof_motion(m, w, d, S); for (int c = 0; c < 6; c++) v[c] += S[c]*qd; } }

// WalkEnvV0 obs / reward / done (walk_v0.py:268-319,358-494) on the post-step state; needs kinematics + tendon + actuation of that
// state in scratch (the reference's extra mj_forward, robot.py:607).  `steps` = WalkEnvV0.steps BEFORE its increment (walk_v0.py:339-342).
template <class MD> __device__ void walk_observe(const MD& m, const Warp w, const StepArgs& a, int env, int steps, double* rw_out, bool* done_out) {
  const myo_buffers& b = a.b; const int* ti = a.cfg.task_i; const double* td = a.cfg.task_d;
  const double* PB = CD(PB_d); const double* xpos = SCR(s_xpos); const double* xmat = SCR(s_xmat);
  double acc[9] = {0,0,0,0,0,0,0,0,0};     // sum m*xipos, sum m*v_origin, sum m*omega
  for (int k = w.lane; k < m.nbd; k += 32) { const double* bd = PB + k*PB_STRIDE; double mass = bd[15], c3[3], v[6];
    mat_vec(c3, xmat + 9*k, bd + 12); body_velocity(m, w, k, v);
    for (int c = 0; c < 3; c++) { acc[c] += mass*(c3[c] + xpos[3*k+c]); acc[3+c] += mass*v[3+c]; acc[6+c] += mass*v[c]; } }
  for (int c = 0; c < 9; c++) acc[c] = warp_sum(acc[c]);
  double M = td[13], com[3] = {acc[0]/M, acc[1]/M, acc[2]/M}, wxc[3]; cross3(wxc, acc + 6, com);
  // _get_com_velocity: -(sum m*cvel)/M, cvel's linear part being the velocity at the root's subtree COM
  double vx = -(acc[3] + wxc[0])/M, vy = -(acc[4] + wxc[1])/M, height = com[2];
  const double* quat = W_(qpos) + 3;
  double tq[4]; quat_mul(tq, quat, td); quat_norm(tq);                                        // torso xquat = root quat (x) constant offset
  const double* pl = xpos + 3*ti[1]; const double* pr_ = xpos + 3*ti[2]; const double* pp = xpos + 3*ti[3];
  double phase = fmod((double)steps/td[6], 1.0);
  float* o = b.obs ? b.obs + (size_t)env*a.obs_dim : nullptr;
  if (o) { int nq2 = m.nq - 2, base = nq2 + m.nv;
    for (int i = w.lane; i < nq2; i += 32) o[i] = (float)W_(qpos)[2+i];
    for (int i = w.lane; i < m.nv; i += 32) o[nq2+i] = (float)(W_(qvel)[i]*a.dt);
    if (w.lane == 0) { o[base] = (float)vx; o[base+1] = (float)vy; for (int c = 0; c < 4; c++) o[base+2+c] = (float)tq[c];
      o[base+6] = (float)pl[2]; o[base+7] = (float)pr_[2]; o[base+8] = (float)height;
      for (int c = 0; c < 3; c++) { o[base+9+c] = (float)(pl[c]-pp[c]); o[base+12+c] = (float)(pr_[c]-pp[c]); }
      o[base+15] = (float)phase; }
    const idx_t* at = CI(PA_tendon); const double* __restrict__ PAm = GD(PAM_d); const double* tlen = SCR(s_tlen); const double* tvel = SCR(s_tvel); const double* tfrc = SCR(s_tfrc);
    int mb = base + 16;
    for (int i = w.lane; i < m.nu; i += 32) { double gear = LDC(PAm + i*PAM_STRIDE + 4); int t = at[i];
      o[mb+i] = (float)(gear*tlen[t]); o[mb+m.nu+i] = (float)clipd(gear*tvel[t], -100, 100); o[mb+2*m.nu+i] = (float)clipd(tfrc[t]/gear/1000.0, -100, 100);
      o[mb+3*m.nu+i] = (float)W_(act)[i]; } }
  // rewards
  double vel_reward = exp(-(td[8]-vy)*(td[8]-vy)) + exp(-(td[7]-vx)*(td[7]-vx));
  const double PI = 3.14159265358979323846;
  double des0 = (double)(float)(0.8*cos(phase*2*PI + PI)), des1 = (double)(float)(0.8*cos(phase*2*PI));
  double e0 = des0 - W_(qpos)[ti[4]], e1 = des1 - W_(qpos)[ti[5]], cyclic = sqrt(e0*e0 + e1*e1);
  double rr = 0; for (int c = 0; c < 4; c++) { double dq = 5.0*(quat[c] - td[9+c]); rr += dq*dq; } double ref_rot = exp(-sqrt(rr));
  double mag = 0.25*(fabs(W_(qpos)[ti[6]]) + fabs(W_(qpos)[ti[7]]) + fabs(W_(qpos)[ti[8]]) + fabs(W_(qpos)[ti[9]])), jrew = exp(-5.0*mag);
  double qn = quat[0]*quat[0]+quat[1]*quat[1]+quat[2]*quat[2]+quat[3]*quat[3], r00 = (quat[0]*quat[0]+quat[1]*quat[1]-quat[2]*quat[2]-quat[3]*quat[3])/qn;
  bool done = height < td[4] || fabs(r00) > td[5];
  *rw_out = a.cfg.weights[0]*vel_reward + a.cfg.weights[1]*(done ? 1.0 : 0.0) + a.cfg.weights[2]*cyclic + a.cfg.weights[3]*ref_rot + a.cfg.weights[4]*jrew;
  *done_out = done;
}

// ObjHold obs / reward / done (obj_hold_v0.py:79-121): needs kinematics of the post-step state in scratch
template <class MD> __device__ void hold_observe(const MD& m, const Warp w, const StepArgs& a, int env, double* rw_out, bool* done_out) {
  const myo_buffers& b = a.b; const int* ti = a.cfg.task_i; const double* td = a.cfg.task_d;
  int ob = ti[0]; const double* xp = SCR(s_xpos) + 3*ob; double op[3]; mat_vec(op, SCR(s_xmat) + 9*ob, td); op[0]+=xp[0]; op[1]+=xp[1]; op[2]+=xp[2];
  double err[3] = {W_(eprm)[0]-op[0], W_(eprm)[1]-op[1], W_(eprm)[2]-op[2]}, dist = sqrt(dot3(err, err));
  float* o = b.obs ? b.obs + (size_t)env*a.obs_dim : nullptr; int nqh = m.nq - 7, nvh = m.nv - 6;
  if (o) { for (int i = w.lane; i < nqh; i += 32) o[i] = (float)W_(qpos)[i];
    for (int i = w.lane; i < nvh; i += 32) o[nqh+i] = (float)(W_(qvel)[i]*a.dt);
    if (w.lane < 3) { const int l = w.lane; o[nqh+nvh+l] = (float)(l == 0 ? op[0] : (l == 1 ? op[1] : op[2])); o[nqh+nvh+3+l] = (float)(l == 0 ? err[0] : (l == 1 ? err[1] : err[2])); }
    for (int i = w.lane; i < m.na; i += 32) o[nqh+nvh+6+i] = (float)W_(act)[i]; }
  bool drop = dist > 0.300;
  *rw_out = a.cfg.weights[0]*(-dist) + a.cfg.weights[1]*((dist < 0.020 ? 1.0 : 0.0) + (dist < 0.010 ? 1.0 : 0.0)) + a.cfg.weights[2]*(drop ? -1.0 : 0.0);
  *done_out = drop;
}

// |qvel dt| of the state in shared memory (the leg stand task's velocity term); out of line, so that the reach epilogue keeps its registers
template <class MD> __device__ __noinline__ double qvel_dt_norm(const MD& m, const Warp w, const StepArgs& a) {
  double v2 = 0; for (int i = w.lane; i < m.nv; i += 32) { const double v = W_(qvel)[i]*a.dt; v2 += v*v; }
  return sqrt(warp_sum(v2)); }

// ReachEnvV0 obs / reward / done (reach_v0.py:98-160): needs kinematics of the post-step state in scratch.  tnow = mjData.time of that state
template <class MD> __device__ void reach_observe(const MD& m, const Warp w, const StepArgs& a, int env, double tnow, double* rw_out, bool* done_out) {
  const myo_buffers& b = a.b; const int* ti = a.cfg.task_i; const double* td = a.cfg.task_d; const int ntip = ti[0];
  float* o = b.obs ? b.obs + (size_t)env*a.obs_dim : nullptr; double d2 = 0, a2 = 0; const int base = m.nq + m.nv;
  if (w.lane < ntip) { int bd = ti[1+w.lane]; const double* lp = td + 3*w.lane; double tip[3] = {lp[0], lp[1], lp[2]};
    if (bd >= 0) { const double* xp = SCR(s_xpos) + 3*bd; mat_vec(tip, SCR(s_xmat) + 9*bd, lp); tip[0]+=xp[0]; tip[1]+=xp[1]; tip[2]+=xp[2]; }
    for (int c = 0; c < 3; c++) { double tgt = b.target ? b.target[(size_t)env*m.nq + 3*w.lane + c] : 0.0, err = tgt - tip[c]; d2 += err*err;
      if (o) { o[base + 3*w.lane + c] = (float)tip[c]; o[base + 3*ntip + 3*w.lane + c] = (float)err; } } }
  if (o) { for (int i = w.lane; i < m.nq; i += 32) o[i] = (float)W_(qpos)[i]; for (int i = w.lane; i < m.nv; i += 32) o[m.nq+i] = (float)(W_(qvel)[i]*a.dt); }
  for (int i = w.lane; i < m.na; i += 32) { a2 += W_(act)[i]*W_(act)[i]; if (o) o[base + 6*ntip + i] = (float)W_(act)[i]; }      // base_v0.py:33-37 appends "act"
  double dist = sqrt(warp_sum(d2)), am = sqrt(warp_sum(a2)); if (m.na) am /= m.na;
  // reward shape: reach_v0.py (all zero) or the leg stand task's 10 - d - 10 |qvel dt|, 100 act_reg and 0.05 near threshold (walk_v0.py:104-140)
  const double* rs = a.cfg.reach_shape;
  double reach = -dist, c_act = 1.0, near_tip = 0.0125;
  if (rs[3] != 0) { reach = rs[0] - dist - (rs[1] != 0 ? rs[1]*qvel_dt_norm(m, w, a) : 0.0); c_act = rs[2]; near_tip = rs[3]; }
  bool armed = tnow > 2*a.dt;                                   // far_th = inf for the first control steps (reach_v0.py:134-138)
  double far_th = td[3*ntip]*ntip, near_th = ntip*near_tip; bool far = armed && dist > far_th;
  *rw_out = a.cfg.weights[0]*reach + a.cfg.weights[1]*((dist < 2*near_th ? 1.0 : 0.0) + (dist < near_th ? 1.0 : 0.0)) + a.cfg.weights[2]*(-c_act*am) + a.cfg.weights[3]*(far ? -1.0 : 0.0);
  *done_out = far;
}

// obs / reward / done of the state held in shared memory, for any task (runs the extra forward stages the task needs)
struct RwDone { double rw; int done; };   // returned by value (registers), not through pointers to the caller's stack
template <class MD> __device__ __noinline__ RwDone task_observe(const MD& m, const Warp w, const StepArgs& a, int env, int steps, double tnow) {
  double rw = 0; bool done = false;
  if (a.cfg.task == MYO_TASK_POSE) pose_reward_done(m, w, a, env, &rw, &done);
  else if (a.cfg.task == MYO_TASK_WALK) { phase_kinematics(m, w); phase_tendon_all(m, w); phase_actuation(m, w, false, m.g_ctrl + (size_t)env*m.nu, nullptr, nullptr); walk_observe(m, w, a, env, steps, &rw, &done); }
  else if (a.cfg.task == MYO_TASK_HOLD) { phase_kinematics(m, w); hold_observe(m, w, a, env, &rw, &done); }
  else if (a.cfg.task == MYO_TASK_REACH) { phase_kinematics(m, w); reach_observe(m, w, a, env, tnow, &rw, &done); }
  __syncwarp();
  RwDone r; r.rw = rw; r.done = done; return r;
}

// barrier among the warps of one lockstep group (named barrier); one group = the whole CTA -> __syncthreads()
__device__ __forceinline__ void group_sync(int ngroups, int gid, int gthreads) {
  if (ngroups <= 1) __syncthreads(); else asm volatile("bar.sync %0, %1;" :: "r"(1 + gid), "r"(gthreads) : "memory"); }

// The model constants into shared memory: bulk async copies (TMA), completion on an mbarrier.  Every thread of the CTA runs it.  A macro,
// not a function: one more call site in env_kernel_body changes the order in which its callees are inlined, and with it the step
// kernels' stack layout and machine code.
#define STAGE_MODEL(m, mbar) { \
  double* s_d = smem; idx_t* s_i = (idx_t*)(smem + m.nD); \
  const unsigned mb = (unsigned)__cvta_generic_to_shared(&mbar); \
  if (threadIdx.x == 0) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(mb)); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); } \
  __syncthreads(); \
  if (threadIdx.x == 0) { \
    const unsigned bytes_d = (unsigned)m.nD*8u, bytes_i = (unsigned)m.nI16w*4u; \
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mb), "r"(bytes_d + bytes_i) : "memory"); \
    const unsigned CH = 32768u;   /* chunked: every piece 16-byte aligned and a multiple of 16 bytes */ \
    for (unsigned o = 0; o < bytes_d; o += CH) { unsigned n = bytes_d - o < CH ? bytes_d - o : CH; \
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" \
                   :: "r"((unsigned)__cvta_generic_to_shared((char*)s_d + o)), "l"((const char*)m.gD + o), "r"(n), "r"(mb) : "memory"); } \
    for (unsigned o = 0; o < bytes_i; o += CH) { unsigned n = bytes_i - o < CH ? bytes_i - o : CH; \
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" \
                   :: "r"((unsigned)__cvta_generic_to_shared((char*)s_i + o)), "l"((const char*)m.gI16 + o), "r"(n), "r"(mb) : "memory"); } \
  } \
  { unsigned done = 0; while (!done) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(mb) : "memory"); } \
}

// The stored state of `env` into this warp's slice (coalesced: one env's row per warp).  The inverse-wrap roots start cold.
template <class MD> __device__ __forceinline__ void load_env_state(const MD& m, const Warp w, const myo_buffers& b, int env) {
  for (int i = w.lane; i < m.nq; i += 32) W_(qpos)[i] = b.qpos[(size_t)env*m.nq+i];
  for (int i = w.lane; i < m.nv; i += 32) { W_(qvel)[i] = b.qvel[(size_t)env*m.nv+i]; W_(qws)[i] = b.qacc_warmstart[(size_t)env*m.nv+i]; }
  for (int i = w.lane; i < m.na; i += 32) W_(act)[i] = b.act[(size_t)env*m.na+i];
  if (w.lane < m.neprm) W_(eprm)[w.lane] = b.env_prm ? b.env_prm[(size_t)env*8 + w.lane] : 0.0;     // per-env model overrides (hold task only)
  for (int i = w.lane; i < m.nwz; i += 32) W_(wz)[i] = -1.0;     // cold start of the inverse-wrap roots at the first substep
  __syncwarp();
}

// ------------------------------------------------------------------ transition FD (myo_batch_transition_fd), per work item
// The sides a column is perturbed to (mjd_stepFD): a state column always goes forward and goes back when centered; a ctrl column of an
// actuator with ctrllimited goes forward when inRange(c, c + eps) and back when (centered || !fwd) && inRange(c - eps, c).
struct FdCol { int col, ctrl; bool fwd, back; };      // ctrl: the actuator of a B column, -1 for an A column
template <class MD> __device__ __forceinline__ FdCol fd_column(const MD& m, const StepArgs& a, int env, int col) {
  const bool centered = a.fd.npass == 2;
  FdCol c; c.col = col; c.ctrl = col < a.fd.nxa ? -1 : col - a.fd.nxa; c.fwd = true; c.back = centered;
  if (c.ctrl >= 0) { const double* __restrict__ pa = GD(PA_d) + CI(PA_cls)[c.ctrl]*PA_STRIDE;
    if (LDC(pa + 15) != 0) { const double lo = LDC(pa + 13), hi = LDC(pa + 14), x = a.roll.ctrl[(size_t)env*m.nu + c.ctrl], e = a.fd.eps;
      c.fwd = x >= lo && x <= hi && x + e >= lo && x + e <= hi;
      c.back = (centered || !c.fwd) && x - e >= lo && x - e <= hi && x >= lo && x <= hi; } }
  return c; }
// Pass p of a column runs the - side when centered and p = 1, or when it cannot go forward; it runs at all when that side is possible
__device__ __forceinline__ bool fd_minus(const StepArgs& a, const FdCol& c, int pass) { return a.fd.npass == 2 ? pass == 1 : !c.fwd; }
__device__ __forceinline__ bool fd_runs(const StepArgs& a, const FdCol& c, int pass) { return fd_minus(a, c, pass) ? c.back : c.fwd; }

// The perturbation of the start state already in the slice (load_env_state); a ctrl column's ctrl row goes to the slot's global row
template <class MD> __device__ void fd_perturb(const MD& m, const Warp w, const StepArgs& a, int env, const FdCol& c, int pass, double* ctrl_row) {
  const double h = fd_minus(a, c, pass) ? -a.fd.eps : a.fd.eps;
  if (c.ctrl >= 0) { const double* src = a.roll.ctrl + (size_t)env*m.nu;
    for (int i = w.lane; i < m.nu; i += 32) ctrl_row[i] = i == c.ctrl ? src[i] + h : src[i]; }
  else if (c.col < m.nv) {      // mj_integratePos(qpos, e_j, h), through the Newton gradient's scratch (dead until the solve)
    for (int i = w.lane; i < m.nv; i += 32) S_g[i] = i == c.col ? 1.0 : 0.0;
    __syncwarp();
    integrate_pos(m, w, W_(qpos), S_g, h); }
  else if (w.lane == 0) { if (c.col < 2*m.nv) W_(qvel)[c.col - m.nv] += h; else W_(act)[c.col - 2*m.nv] += h; }
  __syncwarp();
}

// After a pass: the + pass of a centred column parks its result in the slot's row; the last pass writes the column of A or B
//   both sides (x'+ (-) x'-) * rinv2, forward only (x'+ (-) x'0) * rinv1, back only (x'0 (-) x'-) * rinv1, neither 0
// ((-): differentiate_pos on qpos, subtraction on qvel and act; x'0 from the nominal carry, the last pass's result in the slice).
template <class MD> __device__ void fd_store(const MD& m, const Warp w, const StepArgs& a, int env, const FdCol& c, int pass, bool ran, double* prow) {
  const int nq = m.nq, nv = m.nv, na = m.na, nx = 2*nv + na; const bool centered = a.fd.npass == 2;
  if (centered && pass == 0) {
    if (ran) { for (int i = w.lane; i < nq; i += 32) prow[i] = W_(qpos)[i];
      for (int i = w.lane; i < nv; i += 32) prow[nq+i] = W_(qvel)[i];
      for (int i = w.lane; i < na; i += 32) prow[nq+nv+i] = W_(act)[i]; }
    __syncwarp(); return; }
  const size_t n = a.fd.n_env;
  const double *nq0 = a.fd.nom + (size_t)env*nq, *nv0 = a.fd.nom + n*nq + (size_t)env*nv, *na0 = a.fd.nom + n*(nq + nv) + (size_t)env*na;
  const double *sq = W_(qpos), *sv = W_(qvel), *sa = W_(act);
  const double *pq = centered ? prow : sq, *pv = centered ? prow + nq : sv, *pa = centered ? prow + nq + nv : sa;      // the + result
  const double *q1 = nullptr, *v1 = nullptr, *a1 = nullptr, *q2 = nullptr, *v2 = nullptr, *a2 = nullptr; double r = 0;
  if (c.fwd && c.back) { q1 = sq; v1 = sv; a1 = sa; q2 = pq; v2 = pv; a2 = pa; r = a.fd.rinv2; }      // (both sides only when centered)
  else if (c.fwd) { q1 = nq0; v1 = nv0; a1 = na0; q2 = pq; v2 = pv; a2 = pa; r = a.fd.rinv1; }
  else if (c.back) { q1 = sq; v1 = sv; a1 = sa; q2 = nq0; v2 = nv0; a2 = na0; r = a.fd.rinv1; }
  double* out; size_t st;
  if (c.ctrl < 0) { out = a.fd.A + (size_t)env*nx*nx + c.col; st = nx; } else { out = a.fd.B + (size_t)env*nx*m.nu + c.ctrl; st = m.nu; }
  if (!q1) { for (int i = w.lane; i < nx; i += 32) out[i*st] = 0.0; }
  else { differentiate_pos(m, w, S_g, q1, q2);
    __syncwarp();
    for (int i = w.lane; i < nv; i += 32) out[i*st] = S_g[i]*r;
    for (int i = w.lane; i < nv; i += 32) out[(nv+i)*st] = (v2[i] - v1[i])*r;
    for (int i = w.lane; i < na; i += 32) out[(2*nv+i)*st] = (a2[i] - a1[i])*r; }
  __syncwarp();
}

// ------------------------------------------------------------------ the kernel
// DBG = false: the product step / reset / observe kernel (modes 0, 2, 3): no parity taps, no cycle counters, fixed barrier scheme.
// DBG = true: everything -- forward-debug mode (1), parity taps, per-phase cycle counters, the barrier / lockstep-group tuning knobs.
// ROLL = true: the rollout kernels (myo_batch_rollout), mode 0 only: one interval of a.roll with the caller's ctrl row (m.g_ctrl is neither
// read nor written) and qfrc_applied added to qfrc_smooth; the launch's cfg has no task, fatigue or reafferentation, and its state
// buffers are the library's carry, which is also copied into the output rows of the interval.
// FD = true (with ROLL): the transition-FD kernel (myo_batch_transition_fd).  Its slots are the work items (env, column) of a.fd on the
// contiguous map, so that the warps of a round are neighbouring columns of one env; a.n_env counts the items.  Each item runs a.fd.npass
// consecutive rounds (the + and the - pass when centred), so every warp of every CTA walks the same rounds and solver barriers; a pass
// whose side the column does not take runs as an idle slot (live = false).  A pass loads the env's start state from a.b, perturbs it
// (fd_perturb) and, after the substeps, parks or differences its result (fd_store); no state is stored back.
// MAXT: launch bound (threads per CTA) -> register budget of the instantiation.
template <bool DBG, int MAXT, bool ROLL = false, bool FD = false, class MD>
__device__ __forceinline__ void env_kernel_body(const MD& m, const StepArgs& a) {
  __shared__ __align__(8) unsigned long long mbar;
  const int wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  STAGE_MODEL(m, mbar)
  const Warp w = { m.nD + (m.nI16w + 1)/2 + wid*m.n_per_warp, (int)(threadIdx.x & 31) };
  if (w.lane < CNT_N) ((int*)(smem + w.base + m.o_cnt))[w.lane] = 0;
  __syncwarp();
  const myo_buffers& b = a.b;
  // All warps of a CTA walk the phases in lockstep (CTA barriers between phases) so that they share instruction fetches:
  // the step is a long, mostly straight-line program and the instruction cache, not the data path, is the scarce resource.
  const int nsub = a.mode == 0 ? a.cfg.frame_skip : ((DBG && a.mode == 1) ? (a.n_substeps > 0 ? a.n_substeps : 1) : 0);
  const bool integrate = a.mode == 0 || (DBG && a.mode == 1 && a.n_substeps > 0);
  const bool prof = DBG && b.tap_phase_cycles != nullptr;
  // With a.perm (big models, env steps of the product kernels) the slot -> env map is the load-sorted one: the envs of a round carry
  // similar contact loads, so the lockstep barriers wait for a slowest env that is close to the average one.
  const bool regrouped = !DBG && a.perm != nullptr;
  const int per_cta = regrouped ? a.perm_rounds*nw : SLOTS_PER_CTA(a.balanced, a.n_env, (int)gridDim.x, nw)*(FD ? a.fd.npass : 1);
  for (int j0 = 0; j0 < per_cta; j0 += nw) {
    const int pass = FD ? j0/nw % a.fd.npass : 0;
    const int slot = regrouped ? a.perm[(int)blockIdx.x + (int)gridDim.x*(j0 + wid)] : slot_env(a.balanced, (int)blockIdx.x, (int)gridDim.x, nw, FD ? j0/nw/a.fd.npass*nw : j0, wid);
    const bool item = (j0 + wid) < per_cta && slot >= 0 && slot < a.n_env;
    const int env = FD ? slot/a.fd.ncol : slot;
    const FdCol fc = FD && item ? fd_column(m, a, env, slot - env*a.fd.ncol) : FdCol{};
    double* const fd_row = FD ? a.fd.rows + ((size_t)blockIdx.x*nw + wid)*(m.nu + m.nq + m.nv + m.na) : nullptr;      // this slot's rows
    const bool live = item && (!FD || fd_runs(a, fc, pass)); const long long tstep_ = prof ? clock64() : 0; int load_acc = 0;
    if (live) {
      load_env_state(m, w, b, env);
      if (FD) fd_perturb(m, w, a, env, fc, pass, fd_row);
      if (!ROLL && a.mode == 2) {
        if (!a.reset_mask || a.reset_mask[env]) { env_reset(m, w, a, env);
          task_observe(m, w, a, env, 0, 0.0);
          if (w.lane == 0) { if (b.done) b.done[env] = 0; if (b.truncated) b.truncated[env] = 0; if (b.reward) b.reward[env] = 0; if (b.overflow) b.overflow[env] = 0; } }
      } else if (!ROLL && a.mode == 3) {   // observe: obs/reward/done of the current state, nothing advanced (env.forward(), env_base.py:393-432)
        { const RwDone rd = task_observe(m, w, a, env, b.step_count ? b.step_count[env] : 0, b.time ? b.time[env] : 0.0);
          if (w.lane == 0) { if (b.reward) b.reward[env] = (float)rd.rw; if (b.done) b.done[env] = rd.done != 0; } }
      } else if (DBG && a.mode == 1) {
        for (int i = w.lane; i < m.nu; i += 32) m.g_ctrl[(size_t)env*m.nu+i] = a.dbg_ctrl[(size_t)env*m.nu+i];
      } else if (!ROLL && a.mode == 0) {
        // ---- action -> ctrl  (base_v0.py:83-96); fatigue (fatigue.py:38-76)
        for (int i = w.lane; i < m.nu; i += 32) { double c = (double)b.action[(size_t)env*m.nu+i];
          if (a.cfg.reaf_dst != a.cfg.reaf_src && i == a.cfg.reaf_dst) c = (double)b.action[(size_t)env*m.nu+a.cfg.reaf_src];
          if (a.cfg.normalize_act) c = 1.0/(1.0+exp(-5.0*(c-0.5)));
          if (a.cfg.reaf_dst != a.cfg.reaf_src && i == a.cfg.reaf_src) c = 0.0;
          if (a.cfg.muscle_condition == MYO_COND_FATIGUE && b.fatigue) { double* F = b.fatigue + (size_t)env*3*m.nu; const double* __restrict__ PAg = GD(PA_d) + CI(PA_cls)[i]*PA_STRIDE; const double PA[2] = {LDC(PAg), LDC(PAg + 1)};
            double MA = F[i], MR = F[m.nu+i], MF = F[2*m.nu+i], TL = c, fdt = a.dt, tauact = PA[0], taudeact = PA[1];
            const double r = 10*15, Fc = 0.00912, Rc = 0.1*0.00094;
            double LD = 1.0/tauact*(0.5+1.5*MA), LR = (0.5+1.5*MA)/taudeact, C = 0;
            if (MA < TL && MR > TL-MA) C = LD*(TL-MA);
            if (MA < TL && MR <= TL-MA) C = LD*MR;
            if (MA >= TL) C = LR*(TL-MA);
            double rR = MA >= TL ? r*Rc : Rc;
            double lo = fmax(-MA/fdt + Fc*MA, (MR-1)/fdt + rR*MF), hi = fmin((1-MA)/fdt + Fc*MA, MR/fdt + rR*MF);
            C = fmin(fmax(C, lo), hi);   // np.clip(C, lo, hi) == minimum(maximum(C, lo), hi)
            double dMA = (C-Fc*MA)*fdt, dMR = (-C+rR*MF)*fdt, dMF = (Fc*MA-rR*MF)*fdt;
            MA += dMA; MR += dMR; MF += dMF; F[i] = MA; F[m.nu+i] = MR; F[2*m.nu+i] = MF; c = MA; }
          m.g_ctrl[(size_t)env*m.nu+i] = c; }       // ctrl row in global memory (same lane re-reads it in every substep's actuation phase)
      }
      __syncwarp();
    }
    // ---- physics substeps: forward dynamics + semi-implicit Euler (the only copy of the phase code in the kernel)
    const int ngroups = (DBG && a.cfg.reserved_i > 1) ? (a.cfg.reserved_i < nw ? a.cfg.reserved_i : nw) : 1;
    const int gsz = (nw + ngroups - 1)/ngroups, gid = wid / gsz, gw0 = gid*gsz, gnw = (gw0 + gsz <= nw ? gsz : nw - gw0), gthreads = gnw*32;
    const int bmask = !DBG ? MYO_BMASK : a.cfg.barrier_mode == 0 ? 0xFF : (a.cfg.barrier_mode == 1 ? 0x01 : (a.cfg.barrier_mode == 2 ? 0 : a.cfg.barrier_mode));
    const bool waitprof = DBG && a.cfg.reserved[0] != 0.0;   // profiling: record the barrier wait BEFORE each phase instead of the phase's own cycles
    long long cyc_[DBG ? 20 : 1]; long long* const cyc = DBG ? cyc_ : nullptr; int maxcon_seen = 0, maxefc_seen = 0, overflow_seen = 0;
    if (DBG) for (int k = 0; k < 20; k++) cyc_[DBG ? k : 0] = 0;
    #define PH(k, stmt) { long long tb_ = prof ? clock64() : 0; if (bmask & (1 << k)) group_sync(ngroups, gid, gthreads); long long t0_ = prof ? clock64() : 0; if (live) { stmt; } if (prof) cyc[k] += waitprof ? t0_ - tb_ : clock64() - t0_; }
    #pragma unroll 1
    for (int s = 0; s < nsub; s++) {
      const bool tap = DBG && s == nsub-1;
      PH(0, phase_kinematics(m, w));
      PH(1, phase_tendon_all(m, w); if (tap && b.tap_moment) { const double* mom = SCR(s_mom); for (int i = w.lane; i < m.nnz; i += 32) b.tap_moment[(size_t)env*m.nnz+i] = mom[i]; });
      PH(2, phase_actuation(m, w, integrate, ROLL ? (FD && fc.ctrl >= 0 ? fd_row : a.roll.ctrl + ((size_t)env*a.roll_nstep + a.roll_t)*m.nu) : m.g_ctrl + (size_t)env*m.nu, tap && b.tap_actuator_force ? b.tap_actuator_force + (size_t)env*m.nu : nullptr, tap && b.tap_ten_length ? b.tap_ten_length + (size_t)env*m.nu : nullptr);
            if (ROLL && a.roll.qfrc_applied) { const double* f = a.roll.qfrc_applied + ((size_t)env*a.roll_nstep + a.roll_t)*m.nv;      // mjData.qfrc_applied
              for (int i = w.lane; i < m.nv; i += 32) W_(fsm)[i] += f[i];
              __syncwarp(); });
      PH(3, phase_body_inertia(m, w); phase_crb(m, w); phase_bias(m, w));
      PH(4, phase_collision(m, w); overflow_seen |= WI_(overflow));
      PH(5, phase_constraints(m, w); if (tap) write_taps_contacts(m, w, a, env));
      const bool solver_aligned = ngroups == 1;
      if (solver_aligned) {   // every warp enters the solver: its inner CTA barriers need the idle warps too (lockstep groups run it unaligned)
        long long tb_ = prof ? clock64() : 0; if (bmask & (1 << 6)) __syncthreads(); long long t0_ = prof ? clock64() : 0;
        phase_solve(m, w, a.tol, (prof && live) ? cyc : nullptr, live, true);
        if (prof) cyc[6] += waitprof ? t0_ - tb_ : clock64() - t0_;
      } else PH(6, phase_solve(m, w, a.tol, prof ? cyc : nullptr, true, false));
      PH(7, if (tap) write_taps_solve(m, w, a, env); if (integrate) phase_integrate(m, w, prof ? cyc : nullptr));
      if (DBG && live) { if (WI_(ncon) > maxcon_seen) maxcon_seen = WI_(ncon); if (WI_(nefc) > maxefc_seen) maxefc_seen = WI_(nefc); }
      if (!DBG && live) load_acc += a.load_wn*WI_(ncon) + a.load_wi*WI_(niter);
    }
    #undef PH
    if (prof && live && w.lane == 0) { long long* pc = b.tap_phase_cycles + 20*(size_t)env; for (int k = 0; k < 20; k++) pc[k] = cyc[k]; pc[12] = maxcon_seen; pc[13] = maxefc_seen; pc[17] = clock64() - tstep_; }
    if (FD && item) {
      if (live && overflow_seen && w.lane == 0 && b.overflow) b.overflow[env] = 1;      // (every writer stores 1)
      fd_store(m, w, a, env, fc, pass, live, fd_row + m.nu); }
    if (!FD && live) {
      if (DBG && a.mode == 1) { if (integrate && w.lane == 0 && b.time) b.time[env] += nsub*m.timestep; }
      else if (a.mode == 0) {
        // ---- obs / reward / done / TimeLimit / auto-reset
        // mjData.time advances by one timestep per substep (the accumulated rounding is visible to ReachEnvV0's `time > 2 dt` test)
        double tnow = b.time ? b.time[env] : 0.0; for (int s_ = 0; s_ < a.cfg.frame_skip; s_++) tnow += m.timestep;
        if (overflow_seen && w.lane == 0 && b.overflow) b.overflow[env] |= 1;      // sticky until the next reset of this env
        if (!DBG && a.load && w.lane == 0) a.load[env] = load_acc/(nsub > 0 ? nsub : 1);
        if (!ROLL && a.cfg.task != MYO_TASK_NONE) { const RwDone rd = task_observe(m, w, a, env, b.step_count ? b.step_count[env] : 0, tnow); const double rw = rd.rw; const bool done = rd.done != 0;
          int sc = b.step_count ? b.step_count[env]+1 : 0; bool trunc = a.cfg.max_episode_steps > 0 && sc >= a.cfg.max_episode_steps;
          __syncwarp();
          // truncated follows gym's TimeLimit: set whenever the step budget is reached, also when the episode terminated on the same step
          if (w.lane == 0) { if (b.reward) b.reward[env] = (float)rw; if (b.done) b.done[env] = done; if (b.truncated) b.truncated[env] = trunc;
            if (b.step_count) b.step_count[env] = sc; if (b.time) b.time[env] = tnow;
            if (b.ep_return) { float R = b.ep_return[env] + (float)rw; b.ep_return[env] = R; if ((done || trunc) && b.last_return) b.last_return[env] = R; } }
          __syncwarp();
          // the observation of the state the episode ended in, kept before the auto-reset overwrites obs (the __syncwarp above and the one
          // closing task_observe make every lane's obs stores visible; the one below orders these reads before the reset's obs stores)
          if ((done || trunc) && b.final_obs) { const size_t r = (size_t)env*a.obs_dim;
            for (int i = w.lane; i < a.obs_dim; i += 32) b.final_obs[r+i] = b.obs[r+i];
            __syncwarp(); }
          if ((done || trunc) && a.cfg.auto_reset) { env_reset(m, w, a, env); task_observe(m, w, a, env, 0, 0.0); if (w.lane == 0 && b.overflow) b.overflow[env] = 0; }
        } else if (w.lane == 0 && b.time) b.time[env] = tnow;
      }
      __syncwarp();
      // ---- store state.  A forward pass without substeps runs the solve but not the integrator, so the warm start was not rewritten, and
      // where it lives in the Hessian tail (model_layout) the solve has overwritten it: the caller's warm start stays as it was.
      const bool store_qws = !(DBG && a.mode == 1 && !integrate);
      for (int i = w.lane; i < m.nq; i += 32) b.qpos[(size_t)env*m.nq+i] = W_(qpos)[i];
      for (int i = w.lane; i < m.nv; i += 32) { b.qvel[(size_t)env*m.nv+i] = W_(qvel)[i]; if (store_qws) b.qacc_warmstart[(size_t)env*m.nv+i] = W_(qws)[i]; }
      for (int i = w.lane; i < m.na; i += 32) b.act[(size_t)env*m.na+i] = W_(act)[i];
      if (ROLL) { const myo_rollout_buffers& r = a.roll; const size_t row = (size_t)env*a.roll_nstep + a.roll_t;      // mjData after the interval
        if (r.qpos) for (int i = w.lane; i < m.nq; i += 32) r.qpos[row*m.nq+i] = W_(qpos)[i];
        if (r.qvel) for (int i = w.lane; i < m.nv; i += 32) r.qvel[row*m.nv+i] = W_(qvel)[i];
        if (r.act) for (int i = w.lane; i < m.na; i += 32) r.act[row*m.na+i] = W_(act)[i];
        if (r.qacc) for (int i = w.lane; i < m.nv; i += 32) r.qacc[row*m.nv+i] = W_(qws)[i];
        if (r.time && w.lane == 0) r.time[row] = b.time[env]; }
      __syncwarp();
    }
  }
}
// product kernel: up to 10 env-warps per CTA.  ptxas keeps ~36 registers back for the callees of a kernel that makes ABI calls: the entry
// function gets 168 under launch_bounds(320) and 128 under launch_bounds(448) (14).  __maxnreg__(200) spills a third as much but the kernel
// then launches with at most 8 warps per CTA (measured round 2: "too many resources requested" at 9).
extern "C" __global__ void __launch_bounds__(320) myo_env_kernel(const __grid_constant__ DevModel m, const __grid_constant__ StepArgs a) { env_kernel_body<false, 320>(m, a); }
// the same product body under launch_bounds(448): 128 registers for the entry function, up to 14 env-warps per CTA.  Chosen when the model's
// shared-memory footprint lets that many warps cut the number of rounds (hand, 4096 envs: 2 rounds of 14 instead of 3 of 10).
extern "C" __global__ void __launch_bounds__(448) myo_env_kernel_w14(const __grid_constant__ DevModel m, const __grid_constant__ StepArgs a) { env_kernel_body<false, 448>(m, a); }
// the same product body on the hand's compile-time shape (HandShape), sized for its H100 launch of 11 warps per CTA: 168 registers under launch_bounds(352, 1), and
// the cold tables in shared memory.  Chosen instead of myo_env_kernel_w14 for a batch of that shape whose launch fits its thread limit and shared memory (batch_setup)
extern "C" __global__ void __launch_bounds__(352, 1) myo_env_kernel_w14_hand(const __grid_constant__ HandShape m, const __grid_constant__ StepArgs a) { env_kernel_body<false, 352>(m, a); }
// parity taps / forward-debug / profiling counters / tuning knobs
extern "C" __global__ void __launch_bounds__(320) myo_env_kernel_dbg(const __grid_constant__ DevModel m, const __grid_constant__ StepArgs a) { env_kernel_body<true, 320>(m, a); }
// rollout (myo_batch_rollout): the product body's mode 0 with the caller's ctrl and applied forces, under the two product launch bounds
extern "C" __global__ void __launch_bounds__(320) myo_roll_kernel(const __grid_constant__ DevModel m, const __grid_constant__ StepArgs a) { env_kernel_body<false, 320, true>(m, a); }
extern "C" __global__ void __launch_bounds__(448) myo_roll_kernel_w14(const __grid_constant__ DevModel m, const __grid_constant__ StepArgs a) { env_kernel_body<false, 448, true>(m, a); }
// transition FD (myo_batch_transition_fd): the rollout body over (env, column) work items, under launch_bounds(320)
extern "C" __global__ void __launch_bounds__(320) myo_fd_kernel(const __grid_constant__ DevModel m, const __grid_constant__ StepArgs a) { env_kernel_body<false, 320, true, true>(m, a); }
static_assert(sizeof(HandShape) + sizeof(StepArgs) <= 4096, "the step kernels' arguments fit the 4 KB kernel parameter space");

// ------------------------------------------------------------------ the one-env-per-warp analysis kernels
// Their prologue: the model staged into shared memory when `stage` holds, then this warp's index `wid`, the CTA's warp count `nw` and its
// slice `w`.  Macros for the reason STAGE_MODEL is one: the same statements written out in each kernel give the same machine code.
#define WARP_KERNEL_PROLOGUE(m, stage) \
  __shared__ __align__(8) unsigned long long mbar; \
  const int wid = threadIdx.x >> 5, nw = blockDim.x >> 5; \
  if (stage) STAGE_MODEL(m, mbar) \
  const Warp w = { m.nD + (m.nI16w + 1)/2 + wid*m.n_per_warp, (int)(threadIdx.x & 31) };
// `FOR_EACH_WARP_ENV(env, n_env) body`: this warp's envs on the balanced map (env = CTA + grid * slot), in slot order; the body may
// `continue` to the next env or `break` out of the walk
#define FOR_EACH_WARP_ENV(env, n_env) \
  for (int per_cta_ = SLOTS_PER_CTA(1, (n_env), (int)gridDim.x, nw), j_ = wid; j_ < per_cta_; j_ += nw) \
    if (const int env = slot_env(1, (int)blockIdx.x, (int)gridDim.x, nw, j_ - wid, wid); env >= (n_env)) break; else

// ------------------------------------------------------------------ mjData readout (myo_batch_data)
// One forward pass over the stored state of every env, one env per warp on the balanced map (env = CTA + grid * slot).  Each field is
// written while the scratch region holding it is live; nothing is stored back (the Newton warm start is read, the inverse-wrap roots
// start cold).  The body poses are MuJoCo's quaternion chain over every model body (mj_kinematics), so that xquat carries MuJoCo's
// sign; they come from the model tables in HBM and do not touch shared memory.
enum { DATA_NONE = 0, DATA_ACT = 1, DATA_DYN = 2 };      // how far the shared-memory forward pass runs
struct DataArgs {
  myo_data_buffers d; myo_buffers b;
  int n_env, depth, pose, nbody, nsite, nlevel; double tol;
  const int32_t *lvl, *parent, *jadr, *jnum, *jtype, *jq, *site_body, *pair_geom;   // lvl: level_adr[nlevel + 1], then the bodies in level order
  const double *bpos, *bquat, *jpos, *jaxis, *qpos0, *site_pos;
  double* pose_buf;             // [n_env, 2, nbody, 7] library-owned: pos, quat of every body at qpos (slot 0) and at the target row (slot 1)
};

// mj_kinematics at `qpos` (global row), lanes over the bodies of one tree level at a time: world position and unit quaternion per body
__device__ void data_kinematics(const DataArgs& a, const double* qpos, double* P, int lane) {
  for (int L = 0; L < a.nlevel; L++) {
    for (int k = a.lvl[L] + lane; k < a.lvl[L+1]; k += 32) { const int bd = a.lvl[a.nlevel + 1 + k]; double pos[3] = {0, 0, 0}, quat[4] = {1, 0, 0, 0};
      if (bd > 0) { const int j0 = a.jadr[bd], nj = a.jnum[bd];
        if (nj == 1 && a.jtype[j0] == 0) { const double* qp = qpos + a.jq[j0];      // free joint: pose straight from qpos (normalised copy)
          for (int c = 0; c < 3; c++) pos[c] = qp[c];
          for (int c = 0; c < 4; c++) quat[c] = qp[3+c];
          quat_norm(quat);
        } else { const double* pp = P + 7*a.parent[bd]; double R[9], v[3]; quat2mat(R, pp + 3); mat_vec(v, R, a.bpos + 3*bd);
          for (int c = 0; c < 3; c++) pos[c] = pp[c] + v[c];
          quat_mul(quat, pp + 3, a.bquat + 4*bd);
          for (int j = j0; j < j0 + nj; j++) { const int t = a.jtype[j]; if (t != 2 && t != 3) continue;      // slide, hinge
            const double* al = a.jaxis + 3*j; double ax[3], anc[3]; quat2mat(R, quat); mat_vec(ax, R, al); mat_vec(v, R, a.jpos + 3*j);
            for (int c = 0; c < 3; c++) anc[c] = pos[c] + v[c];
            const double dq = qpos[a.jq[j]] - a.qpos0[a.jq[j]];
            if (t == 2) { for (int c = 0; c < 3; c++) pos[c] += ax[c]*dq; }
            else { double s, co, qn[4]; sincos(0.5*dq, &s, &co); const double ql[4] = {co, al[0]*s, al[1]*s, al[2]*s}; quat_mul(qn, quat, ql);
              for (int c = 0; c < 4; c++) quat[c] = qn[c];
              quat2mat(R, quat); mat_vec(v, R, a.jpos + 3*j); for (int c = 0; c < 3; c++) pos[c] = anc[c] - v[c]; } } }
        quat_norm(quat); }
      double* o = P + 7*bd; for (int c = 0; c < 3; c++) o[c] = pos[c]; for (int c = 0; c < 4; c++) o[3+c] = quat[c]; }
    __syncwarp(); }
}

// world position of local point `loc` on body bd of the pose table P
__device__ __forceinline__ void data_point(const double* P, int bd, const double* loc, double* out) {
  double R[9]; quat2mat(R, P + 7*bd + 3); mat_vec(out, R, loc); for (int c = 0; c < 3; c++) out[c] += P[7*bd + c]; }

__device__ void data_poses(const DevModel& m, const DataArgs& a, int env, int lane) {
  const myo_data_buffers& d = a.d; const int nb = a.nbody;
  double* P = a.pose_buf + (size_t)env*2*nb*7; double* Pt = P + nb*7;
  data_kinematics(a, a.b.qpos + (size_t)env*m.nq, P, lane);
  for (int k = lane; k < nb; k += 32) { const double* p = P + 7*k;
    if (d.xpos) for (int c = 0; c < 3; c++) d.xpos[((size_t)env*nb + k)*3 + c] = p[c];
    if (d.xquat) for (int c = 0; c < 4; c++) d.xquat[((size_t)env*nb + k)*4 + c] = p[3+c];
    if (d.xmat) { double R[9]; quat2mat(R, p + 3); for (int c = 0; c < 9; c++) d.xmat[((size_t)env*nb + k)*9 + c] = R[c]; } }
  if (!d.site_xpos) return;
  const int32_t* src = d.site_source; bool at_target = false;      // a site placed from the kinematics of the target pose
  if (src && a.b.target) for (int s = lane; s < a.nsite; s += 32) at_target |= src[2*s] == 3;
  if (__any_sync(FULL, at_target)) data_kinematics(a, a.b.target + (size_t)env*m.nq, Pt, lane);
  for (int s = lane; s < a.nsite; s += 32) { const int kind = src ? src[2*s] : 0, ix = src ? src[2*s+1] : 0; double loc[3], out[3];
    for (int c = 0; c < 3; c++) loc[c] = a.site_pos[3*s + c];
    if (kind == 1 && a.b.target) { for (int c = 0; c < 3; c++) loc[c] = a.b.target[(size_t)env*m.nq + ix + c]; }
    else if (kind == 2 && a.b.env_prm) { for (int c = 0; c < 3; c++) loc[c] = a.b.env_prm[(size_t)env*8 + ix + c]; }
    else if (kind == 3 && a.b.target) data_point(Pt, a.site_body[ix], a.site_pos + 3*ix, loc);
    data_point(P, a.site_body[s], loc, out);
    for (int c = 0; c < 3; c++) d.site_xpos[((size_t)env*a.nsite + s)*3 + c] = out[c]; }
  __syncwarp();
}

// contact list after constraint assembly (the contact records die in the solve), in model pair order
__device__ void data_contacts(const DevModel& m, const Warp w, const DataArgs& a, int env) {
  const myo_data_buffers& d = a.d; const int ncon = WI_(ncon); const size_t r0 = (size_t)env*m.maxcon;
  for (int c = w.lane; c < m.maxcon; c += 32) { if (c < ncon) continue; const size_t r = r0 + c;
    if (d.contact_geom) { d.contact_geom[2*r] = -1; d.contact_geom[2*r+1] = -1; }
    if (d.contact_dist) d.contact_dist[r] = 0;
    if (d.contact_pos) for (int k = 0; k < 3; k++) d.contact_pos[3*r+k] = 0;
    if (d.contact_frame) for (int k = 0; k < 9; k++) d.contact_frame[9*r+k] = 0; }
  for (int c = w.lane; c < ncon; c += 32) { const size_t r = r0 + CRANK(S_crown[c]); const int p = S_cpair[c]; const double* cd = S_con + c*CON_STRIDE;
    if (d.contact_geom) { d.contact_geom[2*r] = a.pair_geom[2*p]; d.contact_geom[2*r+1] = a.pair_geom[2*p+1]; }
    if (d.contact_dist) d.contact_dist[r] = cd[0];
    if (d.contact_pos) for (int k = 0; k < 3; k++) d.contact_pos[3*r+k] = cd[1+k];
    if (d.contact_frame) { double f[9]; for (int k = 0; k < 6; k++) f[k] = cd[4+k]; cross3(f+6, f, f+3); for (int k = 0; k < 9; k++) d.contact_frame[9*r+k] = f[k]; } }
  __syncwarp();
}

// mj_contactForce of every contact into out [maxcon, 6] (one env's rows), in model pair order, 0 padded: the forces of its rows, -D jar
// where jar = S_jar < 0, decoded from the pyramid (normal = sum of the edges, tangent i = (edge 2i - edge 2i+1) mu_i)
__device__ __forceinline__ void write_contact_force(const DevModel& m, const Warp w, double* out) {
  const int ncon = WI_(ncon);
  for (int c = w.lane; c < m.maxcon; c += 32) if (c >= ncon) for (int k = 0; k < 6; k++) out[6*c + k] = 0;
  const idx_t* pr = CI(PPAIR); const double* pd = CD(PPAIR_d);
  for (int c = w.lane; c < ncon; c += 32) { const int rn = S_crown[c], nr = CNR(rn), rb = CROW(rn); double f[6] = {0, 0, 0, 0, 0, 0};
    if (nr) { const double Dc = S_D[S_DCON(c)]; double q[4] = {0, 0, 0, 0};
      for (int k = 0; k < nr; k++) { const double x = S_jar[rb + k]; q[k] = x < 0 ? -Dc*x : 0.0; }
      if (nr == 1) f[0] = q[0];
      else { const double* P = pd + pr[PPAIR_ISTRIDE*S_cpair[c] + 6]*PPAIR_STRIDE; f[0] = q[0] + q[1] + q[2] + q[3]; f[1] = (q[0] - q[1])*P[2]; f[2] = (q[2] - q[3])*P[3]; } }
    for (int k = 0; k < 6; k++) out[6*CRANK(rn) + k] = f[k]; }
}

// after the Newton solve: qacc, ncon and mj_contactForce of every contact
__device__ void data_solve(const DevModel& m, const Warp w, const DataArgs& a, int env) {
  const myo_data_buffers& d = a.d; const int ncon = WI_(ncon);
  if (d.qacc) for (int i = w.lane; i < m.nv; i += 32) d.qacc[(size_t)env*m.nv + i] = S_a[i];
  if (d.ncon && w.lane == 0) d.ncon[env] = ncon;
  if (d.contact_force) write_contact_force(m, w, d.contact_force + 6*(size_t)env*m.maxcon);
  __syncwarp();
}

extern "C" __global__ void __launch_bounds__(320) myo_data_kernel(const __grid_constant__ DevModel m, const __grid_constant__ DataArgs a) {
  WARP_KERNEL_PROLOGUE(m, a.depth != DATA_NONE)
  const myo_data_buffers& d = a.d; const myo_buffers& b = a.b;
  FOR_EACH_WARP_ENV(env, a.n_env) {
    if (a.pose) data_poses(m, a, env, w.lane);
    if (a.depth == DATA_NONE) continue;
    if (w.lane < CNT_N) ((int*)(smem + w.base + m.o_cnt))[w.lane] = 0;
    load_env_state(m, w, b, env);
    phase_kinematics(m, w); phase_tendon_all(m, w);
    phase_actuation(m, w, false, m.g_ctrl + (size_t)env*m.nu, d.actuator_force ? d.actuator_force + (size_t)env*m.nu : nullptr,
                    d.actuator_length ? d.actuator_length + (size_t)env*m.nu : nullptr);
    if (d.actuator_velocity) { const idx_t* at = CI(PA_tendon); const double* __restrict__ PAm = GD(PAM_d); const double* tvel = SCR(s_tvel);
      for (int i = w.lane; i < m.nu; i += 32) d.actuator_velocity[(size_t)env*m.nu + i] = LDC(PAm + i*PAM_STRIDE + 4)*tvel[at[i]]; }
    if (d.qfrc_actuator) { const idx_t* cadr = CI(PCOL_adr); const idx_t* col = CI(PCOL); const idx_t* nzt = CI(PNZ_tendon); const double* mom = SCR(s_mom); const double* tfrc = SCR(s_tfrc);
      for (int i = w.lane; i < m.nv; i += 32) { double s = 0; for (int e = cadr[i]; e < cadr[i+1]; e++) { const int z = col[e]; s += mom[z]*tfrc[nzt[z]]; }
        d.qfrc_actuator[(size_t)env*m.nv + i] = s; } }
    __syncwarp();
    if (a.depth < DATA_DYN) continue;
    phase_body_inertia(m, w); phase_crb(m, w); phase_bias(m, w);
    phase_collision(m, w); phase_constraints(m, w);
    data_contacts(m, w, a, env);
    phase_solve(m, w, a.tol, nullptr, true, false);
    data_solve(m, w, a, env);
  }
}

// ------------------------------------------------------------------ inverse dynamics (myo_batch_inverse)
// mj_inverse at the stored state of every env, one env per warp on the balanced map: qfrc_inverse = M qacc - qfrc_passive + qfrc_bias -
// J' efc_force with efc_force = -D (J qacc - aref) on equality rows and on the other rows where that is negative.  Nothing is stored back,
// and act, ctrl and the warm start are not read: the passive term goes straight into fsm and no actuation phase runs.
// Scratch lifetimes where they differ from the step's solve stage:
//   T (mom)      the actuator moments leave for HBM right after the tendon phase: C (cin), written next, may overlap T
//   efA / H      aref is copied into efV (con region, dead after the constraint phase) before the discrete conversion writes LD / Dinv in
//                the Hessian region, which holds aref at its head when arefInH
//   vg / vp      vg holds B qacc, then M^-1 B qacc, then qfrc_constraint; vp is not used
//   efR, efV     jar (read again by the contact-force decoding); efV: aref, then the row forces -D jar (folded by rows_applyT_add)
struct InvArgs { myo_inverse_buffers d; myo_buffers b; int n_env, flags; };
// The hooks of inverse_pass: state(m, w) runs on the loaded state before the kinematics, qacc(i, x) gives entry i of the acceleration from
// the caller's x, and where ACT holds the member `actuation` adds the tendon and actuation phases.  NoPerturb (myo_inverse_kernel,
// myo_static_opt_kernel) compiles away: ACT is a compile-time false, so its passes are the same code as before the hooks.
struct NoPerturb { static constexpr bool ACT = false;
  __device__ __forceinline__ void state(const DevModel&, const Warp) const {}
  __device__ __forceinline__ double qacc(int, double x) const { return x; } };
// One env's inverse up to its outputs (myo_inverse_kernel, myo_static_opt_kernel, myo_inverse_fd_kernel): leaves M qacc in S_Ma,
// qfrc_passive - qfrc_bias in fsm and qfrc_constraint in S_g, so that qfrc_inverse = S_Ma - fsm - S_g; qacc and actuator_moment (nullable)
// are the whole batch's rows.  With p.actuation the tendon and actuation phases of the forward pass run after the kinematics and fsm holds
// qfrc_passive + qfrc_actuator - qfrc_bias, so that S_Ma - fsm - S_g = qfrc_inverse - qfrc_actuator (muscle force from act).
template <class P = NoPerturb>
__device__ __forceinline__ void inverse_pass(const DevModel& m, const Warp w, const myo_buffers& b, int env, const double* qacc, double* actuator_moment, bool constraints, bool discrete,
                                             const P& p = P()) {
  if (w.lane < CNT_N) ((int*)(smem + w.base + m.o_cnt))[w.lane] = 0;
  load_env_state(m, w, b, env);
  p.state(m, w);
  phase_kinematics(m, w);
  if (actuator_moment) { phase_tendon_all(m, w);      // dense [nu, nv]: gear x the tendon moment
    const idx_t* at = CI(PA_tendon); const idx_t* nadr = CI(PT_nz_adr); const idx_t* nzd = CI(PNZ_dof); const double* __restrict__ PAm = GD(PAM_d); const double* mom = SCR(s_mom);
    for (int i = w.lane; i < m.nu; i += 32) { double* row = actuator_moment + ((size_t)env*m.nu + i)*m.nv; const double gear = LDC(PAm + i*PAM_STRIDE + 4); const int t = at[i];
      for (int k = 0; k < m.nv; k++) row[k] = 0;
      for (int z = nadr[t]; z < nadr[t+1]; z++) row[nzd[z]] += gear*mom[z]; }
    __syncwarp(); }
  if constexpr (P::ACT) {
    if (p.actuation) { phase_tendon_all(m, w); phase_actuation(m, w, false, W_(act), nullptr, nullptr); }      // (ctrl only enters act_dot, which is not integrated)
    else { const double* dofp = CD(PDOF_d); for (int i = w.lane; i < m.nv; i += 32) W_(fsm)[i] = -dofp[2*i+1]*W_(qvel)[i]; } }
  else { const double* dofp = CD(PDOF_d); for (int i = w.lane; i < m.nv; i += 32) W_(fsm)[i] = -dofp[2*i+1]*W_(qvel)[i]; }
  __syncwarp();
  phase_body_inertia(m, w); phase_crb(m, w); phase_bias(m, w);       // fsm = qfrc_passive - qfrc_bias
  if (constraints) { phase_collision(m, w); phase_constraints(m, w); }
  const int nefc = WI_(nefc);
  for (int r = w.lane; r < nefc; r += 32) S_jv[r] = S_aref[r];
  for (int i = w.lane; i < m.nv; i += 32) S_a[i] = p.qacc(i, qacc[(size_t)env*m.nv + i]);
  __syncwarp();
  if (discrete) {      // (M + h B) qacc = M qacc_c: qacc_c = qacc + h M^-1 B qacc, with the integrator's choice of solver
    const double* dofp = CD(PDOF_d);      // (the program drops the tree-sparse lists where that choice is dense and no Newton step is sparse)
    for (int i = w.lane; i < m.nv; i += 32) S_g[i] = dofp[2*i+1]*S_a[i];
    if (m.nv >= 8 && m.nv <= 36) { load_M_dense(m, w, S_H, 0.0); chol_dense(S_H, m.nv, S_g, w.lane); }
    else { ldl_factor(m, w, W_(qM), S_LD, S_Dinv); ldl_solve(m, w, S_LD, S_Dinv, S_g); }
    for (int i = w.lane; i < m.nv; i += 32) S_a[i] += m.timestep*S_g[i];
    __syncwarp(); }
  mul_M(m, w, S_Ma, S_a);
  for (int i = w.lane; i < m.nv; i += 32) S_g[i] = 0;
  __syncwarp();
  if (constraints) {      // (the row operators walk the equality rows whether or not the constraint phase ran)
    rows_apply(m, w, S_a, S_jar); __syncwarp();
    for (int r = w.lane; r < nefc; r += 32) { const double x = S_jar[r] - S_jv[r]; S_jar[r] = x; S_jv[r] = (r < m.neq || x < 0) ? -S_D[S_drow[r]]*x : 0.0; }
    __syncwarp();
    rows_applyT_add(m, w, S_jv, S_g); }      // qfrc_constraint
}

extern "C" __global__ void __launch_bounds__(320) myo_inverse_kernel(const __grid_constant__ DevModel m, const __grid_constant__ InvArgs a) {
  WARP_KERNEL_PROLOGUE(m, true)
  const myo_inverse_buffers& d = a.d; const bool constraints = !(a.flags & MYO_INV_NOCONSTRAINT), discrete = a.flags & MYO_INV_DISCRETE;
  FOR_EACH_WARP_ENV(env, a.n_env) {
    inverse_pass(m, w, a.b, env, d.qacc, d.actuator_moment, constraints, discrete);
    for (int i = w.lane; i < m.nv; i += 32) { const size_t o = (size_t)env*m.nv + i;
      d.qfrc_inverse[o] = S_Ma[i] - W_(fsm)[i] - S_g[i];
      if (d.qfrc_constraint) d.qfrc_constraint[o] = S_g[i]; }
    if (d.contact_force) write_contact_force(m, w, d.contact_force + 6*(size_t)env*m.maxcon);
    __syncwarp();
  }
}

// ------------------------------------------------------------------ inverse-dynamics FD (myo_batch_inverse_fd)
// f = qfrc_inverse (- qfrc_actuator) of inverse_pass at the start state and at one forward perturbation per work item (include/myo_b200.h
// states the semantics).  Stage 0: one env per warp on the balanced map, the nominal f of every env into the library's rows `nom` (and
// qfrc_inverse).  Stage 1: work item k = env * ncol + column on the contiguous map, so that the warps of a round are neighbouring columns
// of one env; column c perturbs block blk[c / nv] at dof c % nv and writes row c % nv of that block, (f - nom) * rinv.  Nothing is stored
// back; each pass starts from the start state with cold inverse-wrap roots.
struct InvFdArgs { myo_inverse_fd_buffers d; myo_buffers b; double* nom; double eps, rinv; int n_env, ncol, stage, flags, actuation, blk[3]; };
// the perturbation of one column: blk 0 qpos (mj_integratePos(qpos, e_col, eps)), 1 qvel[col] += eps, 2 qacc[col] += eps, -1 none
struct FdPerturb { static constexpr bool ACT = true; int blk, col; double eps; bool actuation;
  __device__ __forceinline__ void state(const DevModel& m, const Warp w) const {
    if (blk == 0) {      // through the Newton gradient's scratch (written again before inverse_pass reads it)
      for (int i = w.lane; i < m.nv; i += 32) S_g[i] = i == col ? 1.0 : 0.0;
      __syncwarp();
      integrate_pos(m, w, W_(qpos), S_g, eps); }
    else if (blk == 1 && w.lane == 0) W_(qvel)[col] += eps;
    __syncwarp(); }
  __device__ __forceinline__ double qacc(int i, double x) const { return blk == 2 && i == col ? x + eps : x; } };

extern "C" __global__ void __launch_bounds__(320) myo_inverse_fd_kernel(const __grid_constant__ DevModel m, const __grid_constant__ InvFdArgs a) {
  WARP_KERNEL_PROLOGUE(m, true)
  const myo_inverse_fd_buffers& d = a.d; const bool constraints = !(a.flags & MYO_INV_NOCONSTRAINT), discrete = a.flags & MYO_INV_DISCRETE;
  const int nv = m.nv, bal = a.stage == 0, n_item = bal ? a.n_env : a.n_env*a.ncol;
  for (int per_cta = SLOTS_PER_CTA(bal, n_item, (int)gridDim.x, nw), j = wid; j < per_cta; j += nw) {
    const int slot = slot_env(bal, (int)blockIdx.x, (int)gridDim.x, nw, j - wid, wid); if (slot >= n_item) break;
    const int env = bal ? slot : slot/a.ncol, c = slot - env*a.ncol;
    const FdPerturb p = {bal ? -1 : a.blk[c/nv], c % nv, a.eps, a.actuation != 0};
    inverse_pass(m, w, a.b, env, d.qacc, nullptr, constraints, discrete, p);
    const double* nom = a.nom + (size_t)env*nv;
    if (bal) for (int i = w.lane; i < nv; i += 32) { const double v = S_Ma[i] - W_(fsm)[i] - S_g[i]; a.nom[(size_t)env*nv + i] = v; if (d.qfrc_inverse) d.qfrc_inverse[(size_t)env*nv + i] = v; }
    else { double* out = (p.blk == 0 ? d.DfDq : p.blk == 1 ? d.DfDv : d.DfDa) + ((size_t)env*nv + p.col)*nv;
      for (int i = w.lane; i < nv; i += 32) out[i] = (S_Ma[i] - W_(fsm)[i] - S_g[i] - nom[i])*a.rinv; }
    if (d.overflow && w.lane == 0) { if (bal) d.overflow[env] = WI_(overflow); else if (WI_(overflow)) d.overflow[env] = 1; }      // (every stage-1 writer stores 1)
    __syncwarp();
  }
}
static_assert(sizeof(DevModel) + sizeof(InvFdArgs) <= 4096, "myo_inverse_fd_kernel's arguments fit the 4 KB kernel parameter space");

// ------------------------------------------------------------------ inverse kinematics (myo_batch_ik)
// Damped least squares to site targets (include/myo_b200.h: myo_ik_buffers), one env per warp on the balanced map.  Each warp runs its own
// iterations and leaves on its own stop test; nothing is stored back.  Lane s < ns holds site s: its pose and errors stay in registers,
// and the normal equations are summed site by site, so the per-env slice is the step kernels' whatever ns is.  Lane l owns rows l and
// l + 32 of the packed H (the dense solver's padded order, identity padding) and the same entries of g.
// Scratch lifetimes within one iteration:
//   K (xpos, xmat)   written by the kinematics, read once into the site lanes' registers; dead before H is touched (H may overlap it)
//   va, vMa, vMp     one site's three Jacobian rows at a time (position, then rotation), read by every lane's rows of H
//   vg, H            g and H from the first site to the solve; vg then holds the step dq until the joint update
struct IkArgs {
  myo_ik_buffers d; myo_ik_params p; const double* bound_qpos; int n_env;
  int site_body[MYO_IK_MAXSITE];                    // program body of each site, -1 for a static body (site_frame is then in world coordinates)
  unsigned long long site_dofs[MYO_IK_MAXSITE];     // bit i: dof i moves the site's body (the ancestor dofs; the host checks nv <= 64)
  double site_frame[MYO_IK_MAXSITE][12];            // site position in its program body; for a static body: world position, world body rotation
};

// log(Q R'): world-frame rotation vector from the site rotation R to the unit target quaternion Q, angle in [0, pi]
__device__ __forceinline__ void ik_rotvec(const double* Q, const double* R, double* out) {
  double T[9], E[9]; quat2mat(T, Q);
  #pragma unroll
  for (int i = 0; i < 3; i++)
    #pragma unroll
    for (int j = 0; j < 3; j++) E[3*i+j] = T[3*i]*R[3*j] + T[3*i+1]*R[3*j+1] + T[3*i+2]*R[3*j+2];
  double q[4]; const double tr = E[0] + E[4] + E[8];      // rotation matrix -> quaternion, largest pivot first
  if (tr > 0) { const double s = 2*sqrt(tr + 1); q[0] = 0.25*s; q[1] = (E[7] - E[5])/s; q[2] = (E[2] - E[6])/s; q[3] = (E[3] - E[1])/s; }
  else if (E[0] > E[4] && E[0] > E[8]) { const double s = 2*sqrt(1 + E[0] - E[4] - E[8]); q[0] = (E[7] - E[5])/s; q[1] = 0.25*s; q[2] = (E[1] + E[3])/s; q[3] = (E[2] + E[6])/s; }
  else if (E[4] > E[8]) { const double s = 2*sqrt(1 + E[4] - E[0] - E[8]); q[0] = (E[2] - E[6])/s; q[1] = (E[1] + E[3])/s; q[2] = 0.25*s; q[3] = (E[5] + E[7])/s; }
  else { const double s = 2*sqrt(1 + E[8] - E[0] - E[4]); q[0] = (E[3] - E[1])/s; q[1] = (E[2] + E[6])/s; q[2] = (E[5] + E[7])/s; q[3] = 0.25*s; }
  if (q[0] < 0) { q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3]; }
  const double sn = sqrt(q[1]*q[1] + q[2]*q[2] + q[3]*q[3]), f = sn > 0 ? 2*atan2(sn, q[0])/sn : 2/q[0];
  out[0] = f*q[1]; out[1] = f*q[2]; out[2] = f*q[3];
}

extern "C" __global__ void __launch_bounds__(320) myo_ik_kernel(const __grid_constant__ DevModel m, const __grid_constant__ IkArgs a) {
  WARP_KERNEL_PROLOGUE(m, true)
  const myo_ik_buffers& d = a.d; const int ns = a.p.nsite, nv = m.nv, np = m.nvp, lane = w.lane; const bool rot = d.target_quat != nullptr;
  unsigned long long keep = ~0ull;      // dofs that may move
  if (d.dof_mask) keep = (unsigned long long)__ballot_sync(FULL, lane < nv && d.dof_mask[lane]) | (unsigned long long)__ballot_sync(FULL, lane + 32 < nv && d.dof_mask[lane + 32]) << 32;
  double* H = S_H; double* g = S_g; double* bx = S_a; double* by = S_Ma; double* bz = S_Mp;
  const idx_t* jtype = CI(jnt_type); const idx_t* jq = CI(jnt_qposadr); const idx_t* jd = CI(jnt_dofadr); const idx_t* lin = CI(PD_lin);
  FOR_EACH_WARP_ENV(env, a.n_env) {
    const double* q0 = (d.qpos0 ? d.qpos0 : a.bound_qpos) + (size_t)env*m.nq; const double* ref = d.qpos_ref ? d.qpos_ref + (size_t)env*m.nq : q0;
    for (int i = lane; i < m.nq; i += 32) W_(qpos)[i] = q0[i];
    __syncwarp();
    for (int it = 0; ; it++) {
      phase_kinematics(m, w);
      // site pose and errors (lane s)
      double p[3] = {0, 0, 0}, R[9], e[3] = {0, 0, 0}, wv[3] = {0, 0, 0}, ep = 0, er = 0;
      if (lane < ns) { const int k = a.site_body[lane]; const double* f = a.site_frame[lane]; double Rb[9];
        if (k < 0) { for (int c = 0; c < 3; c++) p[c] = f[c]; for (int c = 0; c < 9; c++) Rb[c] = f[3+c]; }
        else { const double* X = SCR(s_xmat) + 9*k; mat_vec(p, X, f); for (int c = 0; c < 3; c++) p[c] += SCR(s_xpos)[3*k+c]; for (int c = 0; c < 9; c++) Rb[c] = X[c]; }
        { double S[9]; quat2mat(S, d.site_quat + 4*lane); mat_mul(R, Rb, S); }
        const double* t = d.target_pos + ((size_t)env*ns + lane)*3;
        for (int c = 0; c < 3; c++) e[c] = t[c] - p[c];
        ep = sqrt(dot3(e, e));
        if (rot) { const double* tq = d.target_quat + ((size_t)env*ns + lane)*4; double Q[4] = {tq[0], tq[1], tq[2], tq[3]}; quat_norm(Q); ik_rotvec(Q, R, wv); er = sqrt(dot3(wv, wv)); } }
      const bool conv = __all_sync(FULL, lane >= ns || (ep <= a.p.tol && (!rot || er <= a.p.tol)));
      if (conv || it == a.p.max_iter) {      // outputs at the returned q
        for (int i = lane; i < m.nq; i += 32) d.qpos[(size_t)env*m.nq + i] = W_(qpos)[i];
        if (lane == 0) { if (d.niter) d.niter[env] = it; if (d.converged) d.converged[env] = conv; }
        if (lane < ns) { const size_t r = (size_t)env*ns + lane;
          if (d.err) { d.err[2*r] = ep; d.err[2*r+1] = er; }
          if (d.site_xpos) for (int c = 0; c < 3; c++) d.site_xpos[3*r + c] = p[c];
          if (d.site_xmat) for (int c = 0; c < 9; c++) d.site_xmat[9*r + c] = R[c]; }
        if (d.jacp || d.jacr) for (int s = 0; s < ns; s++) { const double ps[3] = {__shfl_sync(FULL, p[0], s), __shfl_sync(FULL, p[1], s), __shfl_sync(FULL, p[2], s)};
          const size_t r = ((size_t)env*ns + s)*3;
          for (int i = lane; i < nv; i += 32) { double jp[3] = {0, 0, 0}, jr[3] = {0, 0, 0};
            if ((a.site_dofs[s] >> i) & 1) { dof_point_vel(m, w, i, ps, jp); if (!lin[i]) for (int c = 0; c < 3; c++) jr[c] = W_(dax)[3*i + c]; }
            for (int c = 0; c < 3; c++) { if (d.jacp) d.jacp[(r + c)*nv + i] = jp[c]; if (d.jacr) d.jacr[(r + c)*nv + i] = jr[c]; } } }
        __syncwarp();
        break; }
      // normal equations, site by site
      double gi[2] = {0, 0};
      #pragma unroll
      for (int c = 0; c < 2; c++) { const int i = lane + 32*c; if (i < np) { for (int j = 0; j <= i; j++) H[TRI(i,j)] = 0; if (i >= nv) H[TRI(i,i)] = 1; } }
      for (int s = 0; s < ns; s++) {
        const double ps[3] = {__shfl_sync(FULL, p[0], s), __shfl_sync(FULL, p[1], s), __shfl_sync(FULL, p[2], s)};
        const double es[3] = {__shfl_sync(FULL, e[0], s), __shfl_sync(FULL, e[1], s), __shfl_sync(FULL, e[2], s)};
        const double ws[3] = {__shfl_sync(FULL, wv[0], s), __shfl_sync(FULL, wv[1], s), __shfl_sync(FULL, wv[2], s)};
        const double wp = d.site_weight ? d.site_weight[2*s] : 1.0, wr = d.site_weight ? d.site_weight[2*s+1] : 1.0;
        const unsigned long long mk = a.site_dofs[s];
        double jp[2][3], jr[2][3];
        #pragma unroll
        for (int c = 0; c < 2; c++) { const int i = lane + 32*c; for (int k = 0; k < 3; k++) jp[c][k] = jr[c][k] = 0;
          if (i < nv && ((mk >> i) & 1)) { dof_point_vel(m, w, i, ps, jp[c]); if (!lin[i]) for (int k = 0; k < 3; k++) jr[c][k] = W_(dax)[3*i + k]; }
          gi[c] += wp*dot3(jp[c], es) + (rot ? wr*dot3(jr[c], ws) : 0.0); }
        #pragma unroll 1
        for (int pass = 0; pass < (rot ? 2 : 1); pass++) { const double wt = pass ? wr : wp;
          #pragma unroll
          for (int c = 0; c < 2; c++) { const int i = lane + 32*c; if (i < nv) { const double* J = pass ? jr[c] : jp[c]; bx[i] = J[0]; by[i] = J[1]; bz[i] = J[2]; } }
          __syncwarp();
          #pragma unroll
          for (int c = 0; c < 2; c++) { const int i = lane + 32*c; if (i >= nv || !((mk >> i) & 1)) continue; const double* J = pass ? jr[c] : jp[c];
            for (unsigned long long bits = mk & ((2ull << i) - 1); bits; bits &= bits - 1) { const int j = __ffsll((long long)bits) - 1;
              H[TRI(i,j)] += wt*(J[0]*bx[j] + J[1]*by[j] + J[2]*bz[j]); } }
          __syncwarp(); } }
      #pragma unroll
      for (int c = 0; c < 2; c++) { const int i = lane + 32*c; if (i < np) g[i] = i < nv ? gi[c] : 0.0; }
      __syncwarp();
      if (a.p.eq_weight != 0 && lane == 0) {      // joint equalities: row 1 at d1, -deriv at d2
        const idx_t* eq = CI(PEQ); const double* eqd = CD(PEQ_d); const double we = a.p.eq_weight;
        for (int k = 0; k < m.neq; k++) { const int q1 = eq[PEQ_ISTRIDE*k], d1 = eq[PEQ_ISTRIDE*k+1], q2 = eq[PEQ_ISTRIDE*k+2], d2 = eq[PEQ_ISTRIDE*k+3]; double deriv;
          const double cpos = eq_residual(eqd + k*PEQ_STRIDE, W_(qpos), q1, q2, deriv);
          H[TRI(d1,d1)] += we; g[d1] -= we*cpos;
          if (q2 >= 0) { const double j2 = -deriv; H[TRI(d2,d2)] += we*j2*j2; H[d1 > d2 ? TRI(d1,d2) : TRI(d2,d1)] += we*j2; g[d2] -= we*j2*cpos; } } }
      __syncwarp();
      if (a.p.posture_weight != 0) { const double rho = a.p.posture_weight;      // hinge and slide dofs toward the reference
        for (int j = lane; j < m.njnt; j += 32) if (jtype[j] == 2 || jtype[j] == 3) { const int da = jd[j], qa = jq[j]; H[TRI(da,da)] += rho; g[da] += rho*(ref[qa] - W_(qpos)[qa]); } }
      __syncwarp();
      #pragma unroll
      for (int c = 0; c < 2; c++) { const int i = lane + 32*c; if (i >= nv) continue;
        H[TRI(i,i)] += a.p.damping;
        if (!((keep >> i) & 1)) { for (int j = 0; j < i; j++) H[TRI(i,j)] = 0; H[TRI(i,i)] = 1; g[i] = 0; }
        else if (~keep) for (int j = 0; j < i; j++) if (!((keep >> j) & 1)) H[TRI(i,j)] = 0; }
      __syncwarp();
      chol_dense(H, nv, g, lane);
      __syncwarp();
      double ss = 0;
      for (int i = lane; i < nv; i += 32) ss += g[i]*g[i];
      const double nrm = sqrt(warp_sum(ss));
      if (nrm > a.p.max_step) { const double sc = a.p.max_step/nrm; for (int i = lane; i < nv; i += 32) g[i] *= sc; }
      __syncwarp();
      integrate_pos(m, w, W_(qpos), g, 1.0);
      __syncwarp();
      { const idx_t* lim = CI(PLIM); const double* __restrict__ limd = GD(PLIM_d);
        for (int l = lane; l < m.nlim; l += 32) { double* q = W_(qpos) + lim[2*l+1]; *q = clipd(*q, LDC(limd + l*PLIM_STRIDE), LDC(limd + l*PLIM_STRIDE + 1)); } }
      __syncwarp();
    }
  }
}

// ------------------------------------------------------------------ muscle static optimisation (myo_batch_static_opt)
// The dual Newton of include/myo_b200.h (myo_static_opt_buffers), one env per warp on the balanced map; each warp leaves on its own stop test
// and nothing is stored back.  The inverse pass gives t; a second kinematics and tendon pass gives the moments, lengths and velocities (the
// inverse's CRB stage overwrites them).  G is never formed: (G' l)_m = gear g (mom . l) over the muscle's moment non-zeros, and (G a)_i sums
// mom x (gear g a) of its tendon over dof i's column list, as phase_actuation sums the tendon forces.  Lane i owns rows i and i + 32 of the
// packed H (the dense solver's padded order, identity padding) and adds each free muscle's outer product from its non-zeros: no atomics,
// one summation order whatever the batch.  Scratch lifetimes:
//   everything      the inverse pass (its own lifetimes, above), then the kinematics and tendon passes, as in a forward pass
//   fsm             qfrc_passive - qfrc_bias, then t from the end of the inverse pass to the last iteration
//   T (mom)         from the tendon pass to the end: read by every product with G; T (tlen, tvel): read by the gain and bias only
//   gm, bm          gain and bias per muscle, from the gain pass to the outputs; placed outside mom, tlen and tvel
//   H, x, l, cg, tf, s   written after the gain pass, so they may overlap tlen, tvel, the rest of the scratch and the dead persistent
//                   dof axes and mass matrix (dax, dan, qM); cg: gear g per tendon, tf: gear b, then gear g a per tendon; s: (G' l)_m
//   F               in registers (lane i: F_i and F_{i+32})
// The host places the arrays (so_plan), first fit by decreasing size, and refuses a model whose slice has no room.
struct SoArgs { myo_static_opt_buffers d; myo_static_opt_params p; myo_buffers b; int n_env, flags;
  int o_H, o_x, o_l, o_cg, o_tf, o_s, o_gm, o_bm; };      // offsets from the warp base (doubles)

// phi(s + ds) - phi(s) of a muscle's conjugate term phi(s) = max_{a in [0, 1]} (a s - w a^2 / 2), without cancellation inside one piece
__device__ __forceinline__ double so_phi_diff(double s, double ds, double wm) {
  const double s1 = s + ds; const int k0 = s <= 0 ? 0 : (s < wm ? 1 : 2), k1 = s1 <= 0 ? 0 : (s1 < wm ? 1 : 2);
  if (k0 == k1) return k0 == 0 ? 0.0 : (k0 == 1 ? ds*(s + 0.5*ds)/wm : ds);
  const double p0 = k0 == 0 ? 0.0 : (k0 == 1 ? 0.5*s*s/wm : s - 0.5*wm), p1 = k1 == 0 ? 0.0 : (k1 == 1 ? 0.5*s1*s1/wm : s1 - 0.5*wm);
  return p1 - p0;
}

// act after one mj_step of the activation dynamics with ctrl c (phase_actuation's update; c already inside ctrlrange)
__device__ __forceinline__ double so_act_next(const double* dyn, double c, double act, double h) {
  const double dctrl = clipd(c, 0, 1) - act; return act + h*(dctrl*m_rcp(fmax(MYO_MINVAL, muscle_tau(dyn, dctrl, act)))); }

// the excitation that, held for k mj_steps, takes act to a, inside [lo, hi]: in one step without smooth activation (dyn[2]) the closed
// form of that step, otherwise bisection over the k-step map
__device__ __forceinline__ double excitation(const double* dyn, double act, double a, double h, int k, double lo, double hi) {
  if (k == 1 && dyn[2] < MYO_MINVAL) { const double dd = a - act; return clipd(act + dd*muscle_tau(dyn, dd, act)/h, lo, hi); }
  const auto after = [&](double c) { double x = act; for (int j = 0; j < k; j++) x = so_act_next(dyn, c, x, h); return x; };
  if (after(hi) <= a) return hi;
  if (after(lo) >= a) return lo;
  for (int it = 0; it < 200; it++) { const double mid = 0.5*(lo + hi); if (!(mid > lo && mid < hi)) break;
    if (after(mid) < a) lo = mid; else hi = mid; }
  return fabs(after(lo) - a) <= fabs(after(hi) - a) ? lo : hi;
}

// the range an excitation is clipped to, from the muscle's PA_d row ag: ctrlrange inside [0, 1] when ctrllimited, else [0, 1]
__device__ __forceinline__ void excitation_range(const DevModel& m, const double* __restrict__ ag, double& lo, double& hi) {
  const bool lim = LDC(ag + 15) != 0; lo = lim ? fmax(LDC(ag + 13), 0.0) : 0.0; hi = lim ? fmin(LDC(ag + 14), 1.0) : 1.0; }

extern "C" __global__ void __launch_bounds__(320) myo_static_opt_kernel(const __grid_constant__ DevModel m, const __grid_constant__ SoArgs a) {
  WARP_KERNEL_PROLOGUE(m, true)
  const myo_static_opt_buffers& d = a.d; const bool constraints = !(a.flags & MYO_INV_NOCONSTRAINT), discrete = a.flags & MYO_INV_DISCRETE;
  const int nv = m.nv, nu = m.nu, np = m.nvp, lane = w.lane;
  double* t = W_(fsm); double* H = smem + w.base + a.o_H; double* x = smem + w.base + a.o_x; double* lam = smem + w.base + a.o_l;
  double* cg = smem + w.base + a.o_cg; double* tf = smem + w.base + a.o_tf; double* sm = smem + w.base + a.o_s;
  double* gm = smem + w.base + a.o_gm; double* bm = smem + w.base + a.o_bm; const double* mom = SCR(s_mom);
  const idx_t* at = CI(PA_tendon); const idx_t* acls = CI(PA_cls); const idx_t* nadr = CI(PT_nz_adr); const idx_t* nzd = CI(PNZ_dof);
  const idx_t* cadr = CI(PCOL_adr); const idx_t* col = CI(PCOL); const idx_t* nzt = CI(PNZ_tendon);
  const double* __restrict__ PAc = GD(PA_d); const double* __restrict__ PAm = GD(PAM_d);
  FOR_EACH_WARP_ENV(env, a.n_env) {
    inverse_pass(m, w, a.b, env, d.qacc, nullptr, constraints, discrete);
    for (int i = lane; i < nv; i += 32) { const double v = S_Ma[i] - W_(fsm)[i] - S_g[i]; t[i] = v; if (d.qfrc_inverse) d.qfrc_inverse[(size_t)env*nv + i] = v; }
    __syncwarp();
    phase_kinematics(m, w); phase_tendon_all(m, w);
    // gain and bias of every muscle (phase_actuation's), then gear g and gear b per tendon (0 on tendons without a muscle)
    for (int i = lane; i < nu; i += 32) { double ag[16], am[5]; for (int c = 0; c < 16; c++) ag[c] = LDC(PAc + acls[i]*PA_STRIDE + c); for (int c = 0; c < 5; c++) am[c] = LDC(PAm + i*PAM_STRIDE + c);
      const int tt = at[i]; double g, b; muscle_gain_bias(ag + 3, ag + 9, am, am[4]*SCR(s_tlen)[tt], am[4]*SCR(s_tvel)[tt], g, b); gm[i] = g; bm[i] = b;
      if (d.muscle_gain) d.muscle_gain[(size_t)env*nu + i] = g;
      if (d.muscle_bias) d.muscle_bias[(size_t)env*nu + i] = b; }
    __syncwarp();
    for (int k = lane; k < m.nta; k += 32) { cg[k] = 0; tf[k] = 0; }
    __syncwarp();
    for (int i = lane; i < nu; i += 32) { const double gear = LDC(PAm + i*PAM_STRIDE + 4); cg[at[i]] = gear*gm[i]; tf[at[i]] = gear*bm[i]; }
    __syncwarp();
    double tmax = 0;      // t = tau - AM' b
    for (int i = lane; i < nv; i += 32) { double s = 0; for (int e = cadr[i]; e < cadr[i+1]; e++) { const int z = col[e]; s += mom[z]*tf[nzt[z]]; }
      t[i] -= s; tmax = fmax(tmax, fabs(t[i])); lam[i] = d.lambda0 ? d.lambda0[(size_t)env*nv + i] : 0.0; }
    for (int o = 16; o > 0; o >>= 1) tmax = fmax(tmax, __shfl_xor_sync(FULL, tmax, o));
    const double thr = a.p.tol*fmax(1.0, tmax);
    __syncwarp();
    int it = 0; bool conv = false; double fnorm = 0, F[2] = {0, 0};
    for (;; it++) {
      // muscle duals s = G' l, the activations a(l) and gear g a per tendon
      for (int i = lane; i < nu; i += 32) { const int tt = at[i]; double acc = 0; for (int z = nadr[tt]; z < nadr[tt+1]; z++) acc += mom[z]*lam[nzd[z]];
        const double s = cg[tt]*acc, wm = d.weight ? d.weight[i] : 1.0; sm[i] = s; tf[tt] = cg[tt]*clipd(s/wm, 0, 1); }
      __syncwarp();
      fnorm = 0;      // F = G a + rho^2 l - t
      #pragma unroll
      for (int c = 0; c < 2; c++) { const int i = lane + 32*c; F[c] = 0; if (i >= nv) continue;
        double s = 0; for (int e = cadr[i]; e < cadr[i+1]; e++) { const int z = col[e]; s += mom[z]*tf[nzt[z]]; }
        const double rho = d.reserve[i]; F[c] = s + rho*rho*lam[i] - t[i]; fnorm = fmax(fnorm, fabs(F[c])); }
      for (int o = 16; o > 0; o >>= 1) fnorm = fmax(fnorm, __shfl_xor_sync(FULL, fnorm, o));
      conv = fnorm <= thr;
      if (conv || it >= a.p.max_iter) break;
      // H = G_F W_F^-1 G_F' + diag rho^2 over the free muscles and those at the kink s = 0 (every muscle at l = 0), rows owned by lanes
      #pragma unroll
      for (int c = 0; c < 2; c++) { const int i = lane + 32*c; if (i < np) { for (int k = 0; k < i; k++) H[TRI(i,k)] = 0; H[TRI(i,i)] = i < nv ? d.reserve[i]*d.reserve[i] : 1.0; } }
      for (int mu = 0; mu < nu; mu++) { const double wm = d.weight ? d.weight[mu] : 1.0, q = sm[mu]/wm; if (!((q > 0 || sm[mu] == 0) && q < 1)) continue;
        const int tt = at[mu], z0 = nadr[tt], z1 = nadr[tt+1]; const double c = cg[tt];
        #pragma unroll
        for (int cc = 0; cc < 2; cc++) { const int i = lane + 32*cc; if (i >= nv) continue;
          double gi = 0; for (int z = z0; z < z1; z++) if (nzd[z] == i) gi += mom[z];
          if (gi == 0) continue;
          gi *= c*c/wm;
          for (int z = z0; z < z1; z++) { const int k = nzd[z]; if (k <= i) H[TRI(i,k)] += gi*mom[z]; } } }
      #pragma unroll
      for (int c = 0; c < 2; c++) { const int i = lane + 32*c; if (i < np) x[i] = -F[c]; }      // (F = 0 on the padding rows)
      __syncwarp();
      chol_dense(H, nv, x, lane);
      __syncwarp();
      // Armijo backtracking on psi along x: psi(l + al x) - psi(l) = al x'(t - rho^2 l) - al^2/2 x' rho^2 x - sum_m [phi_m(s + al sd) - phi_m(s)]
      // with sd = G' x, and slope x' grad psi = -F' x
      double A1 = 0, A2 = 0, slope = 0;
      #pragma unroll
      for (int c = 0; c < 2; c++) { const int i = lane + 32*c; if (i >= nv) continue; const double r2 = d.reserve[i]*d.reserve[i];
        A1 += x[i]*(t[i] - r2*lam[i]); A2 += r2*x[i]*x[i]; slope -= F[c]*x[i]; }
      A1 = warp_sum(A1); A2 = warp_sum(A2); slope = warp_sum(slope);
      double al = 1;
      for (int ls = 0; ls < 60; ls++) { double ph = 0;
        for (int i = lane; i < nu; i += 32) { const int tt = at[i]; double acc = 0; for (int z = nadr[tt]; z < nadr[tt+1]; z++) acc += mom[z]*x[nzd[z]];
          ph += so_phi_diff(sm[i], al*(cg[tt]*acc), d.weight ? d.weight[i] : 1.0); }
        const double dpsi = al*A1 - 0.5*al*al*A2 - warp_sum(ph);
        if (dpsi >= 1e-4*al*slope) break;
        al *= 0.5; }
      for (int i = lane; i < nv; i += 32) lam[i] += al*x[i];
      __syncwarp();
    }
    // outputs at the returned l: a(l), r, the excitation, the forces
    if (lane == 0) { if (d.niter) d.niter[env] = it; if (d.converged) d.converged[env] = conv; if (d.residual) d.residual[env] = fnorm; }
    for (int i = lane; i < nv; i += 32) { const size_t o = (size_t)env*nv + i; const double rho = d.reserve[i];
      if (d.reserve_force) d.reserve_force[o] = rho*rho*lam[i];
      if (d.lambda) d.lambda[o] = lam[i]; }
    for (int i = lane; i < nu; i += 32) { const size_t o = (size_t)env*nu + i; const double act = clipd(sm[i]/(d.weight ? d.weight[i] : 1.0), 0, 1);
      d.act[o] = act;
      if (d.actuator_force) d.actuator_force[o] = gm[i]*act + bm[i];
      if (d.ctrl) { const double* __restrict__ ag = PAc + acls[i]*PA_STRIDE; const double dyn[3] = {LDC(ag), LDC(ag + 1), LDC(ag + 2)};
        double lo, hi; excitation_range(m, ag, lo, hi);
        d.ctrl[o] = excitation(dyn, W_(act)[i], act, m.timestep, 1, lo, hi); } }
    __syncwarp();
  }
}

// ================================================================== host side (C-ABI)
static thread_local std::string g_err;
static int fail(const std::string& s) { g_err = s; return -1; }
#define CUDA_OK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return fail(std::string(#x) + ": " + cudaGetErrorString(e_)); } while (0)

struct myo_model { std::vector<int32_t> I; std::vector<double> D; };
// Counting sort of the envs by last step's load key (descending), then groups of `nw` consecutive envs -> one round of one CTA, the rounds
// filled boustrophedon (round 0: CTA 0 .. grid-1 takes the heaviest groups in order, round 1 runs back) so that every CTA's rounds add up to
// about the same work.  One CTA; the order inside a bucket is whatever the atomics give (results do not depend on the grouping).
__global__ void __launch_bounds__(1024) myo_regroup_kernel(const int* __restrict__ load, int* __restrict__ perm, int n, int grid, int nw, int nslots) {
  __shared__ int cnt[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) cnt[i] = 0;
  for (int i = threadIdx.x; i < nslots; i += blockDim.x) perm[i] = -1;
  __syncthreads();
  for (int e = threadIdx.x; e < n; e += blockDim.x) { int k = load[e]; k = k < 0 ? 0 : (k > 255 ? 255 : k); atomicAdd(&cnt[255 - k], 1); }
  __syncthreads();
  if (threadIdx.x == 0) { int run = 0; for (int i = 0; i < 256; i++) { int c = cnt[i]; cnt[i] = run; run += c; } }
  __syncthreads();
  for (int e = threadIdx.x; e < n; e += blockDim.x) { int k = load[e]; k = k < 0 ? 0 : (k > 255 ? 255 : k);
    const int p = atomicAdd(&cnt[255 - k], 1), g = p / nw, u = p % nw, r = g / grid; int c = g % grid; if (r & 1) c = grid - 1 - c;
    perm[c + grid*(r*nw + u)] = e; }
}

struct LaunchShape { int warps, smem, grid; };      // env-warps per CTA, dynamic shared memory (bytes), CTAs
struct LazyShape { LaunchShape s; bool ready; };    // a launch shape sized by the first call that launches its kernel
// Zero-initialised by myo_batch_create (new myo_batch()), so that myo_batch_destroy can free a partly built batch.
struct myo_batch { const myo_model* model; int device, n_env; myo_task_cfg cfg; double tol; myo_buffers bufs; bool bound; DevModel dm; int32_t* dI; double* dD; double* dCtrl; int const_bytes, cold_bytes;
  LaunchShape prod, dbg; int balanced, dbg_balanced, obs_dim; bool use_w14, use_hand; bool regroup; int* dLoad; int* dPerm; int perm_rounds, perm_slots; bool perm_built; long long launches; unsigned long long seed; long long env_offset;
  // mjData readout (myo_batch_data), set up by its first call: model tables in HBM, the pose scratch and the launch shape of myo_data_kernel
  int32_t* dRI; double* dRD; double* dPose; DataArgs data; LazyShape data_shape;
  LazyShape inv_shape, ik_shape;      // launch shapes of myo_inverse_kernel and myo_ik_kernel
  // rollout (myo_batch_rollout), set up by its first call: carry state [n, nq + 2 nv + na + 1] (qpos | qvel | act | warm start | time)
  bool big; double* dCarry; LazyShape roll_shape; bool roll_regroup, roll_balanced;
  // transition FD (myo_batch_transition_fd): launch shape of myo_fd_kernel for fd_items work items, and its per-slot rows
  LaunchShape fd_shape; long long fd_items; double* dFdRows; size_t fd_rows_bytes;
  LazyShape so_shape; int so_off[8]; LazyShape cmc_shape; double* dCmc;      // myo_static_opt_kernel's launch shape and scratch placement (so_plan), set by the first myo_batch_static_opt or myo_batch_cmc; myo_cmc_kernel's launch shape and the per-frame rows (cmc_rows), set by the first myo_batch_cmc
  // inverse-dynamics FD (myo_batch_inverse_fd): launch shapes of myo_inverse_fd_kernel's stage 0 (per env) and stage 1 (ifd_items work
  // items), and the nominal rows [n, nv], allocated by the first call
  LazyShape ifd_shape; LaunchShape ifd_item_shape; long long ifd_items; double* dIfdNom; };

extern "C" const char* myo_last_error(void) { return g_err.c_str(); }
extern "C" int myo_version(void) { return 2; }     // 2: myo_buffers.final_obs appended

extern "C" int myo_model_from_blob(const int32_t* I, int64_t nI, const double* D, int64_t nD, myo_model** out) {
  if (!I || !out || nI < MYO_BLOB_HDR + MYO_NDIM + 3*MYO_NSEC) return fail("myo_model_from_blob: bad arguments");
  if (I[0] != MYO_BLOB_MAGIC || I[1] != MYO_BLOB_VERSION || I[2] != MYO_NDIM || I[3] != MYO_NSEC) return fail("myo_model_from_blob: blob magic/version/layout mismatch");
  for (int s = 0; s < MYO_NSEC; s++) { long long off = MYO_SEC_OFF(I, s), len = MYO_SEC_LEN(I, s); int kind = I[MYO_BLOB_HDR+MYO_NDIM+3*s];
    if (off < 0 || len < 0 || off + len > (kind ? nD : nI)) return fail("myo_model_from_blob: section out of range"); }
  if (MYO_SEC_LEN(I, MYO_SEC_P_dims) < 30 || MYO_SEC_LEN(I, MYO_SEC_HOT_off) != MYO_NSEC + 1) return fail("myo_model_from_blob: blob carries no kernel program (pack with program=build_program(m))");
  myo_model* m = new myo_model(); m->I.assign(I, I+nI); m->D.assign(D, D+nD); *out = m; return 0;
}
extern "C" void myo_model_destroy(myo_model* m) { delete m; }

// The DevModel of a model under a task configuration: its shape's dimensions and layout (model_layout), the staged tables and the scalars
static void fill_devmodel(const myo_model* mm, const myo_task_cfg* cfg, DevModel& d, Layout* lay = nullptr) {
  const int32_t* I = mm->I.data(); const double* D = mm->D.data(); const int32_t* P = MYO_ISEC(I, MYO_SEC_P_dims);
  const bool hold = cfg && cfg->task == MYO_TASK_HOLD;
  const ModelDims x = {MYO_DIM(I, MYO_DIM_nq), MYO_DIM(I, MYO_DIM_nv), MYO_DIM(I, MYO_DIM_nu), MYO_DIM(I, MYO_DIM_na), MYO_DIM(I, MYO_DIM_nM), MYO_DIM(I, MYO_DIM_njnt),
    P[PD_NBD], P[PD_NLEVEL], P[PD_NSP], P[PD_NWE], P[PD_NTA], P[PD_NNZ], P[PD_NLIM], P[PD_NEQ], P[PD_NPAIR], P[PD_NPAIR_ANALYTIC], P[PD_MAXPATH], P[PD_NDEPTH],
    P[PD_EQ_TREE], P[PD_NGC], P[PD_NWE_SPH_IN] + P[PD_NWE_CYL_IN], P[PD_NLIMROW], P[PD_SPLIT_SP], P[PD_SPLIT_WE], P[PD_SPLIT_TA], P[PD_SPLIT_NZ],
    hold ? 8 : 0, hold ? cfg->task_i[1] : -1, cfg ? cfg->maxcon : 0};
  const ModelLayout ml = model_layout(x); d = ml.d; if (lay) *lay = ml.L;
  const int32_t* hoff = MYO_ISEC(I, MYO_SEC_HOT_off);
  for (int s = 0; s < MYO_NSEC; s++) d.hoff[s] = hoff[s];
  d.nI16w = MYO_SEC_LEN(I, MYO_SEC_HOT_I16); d.nD = hoff[MYO_NSEC] >= 0 ? hoff[MYO_NSEC] : MYO_SEC_LEN(I, MYO_SEC_HOT_D);      // doubles staged to shared memory (the cold tables behind them stay in HBM)
  const double* opt = MYO_DSEC(I, D, MYO_SEC_opt); d.timestep = opt[0]; d.gx = opt[1]; d.gy = opt[2]; d.gz = opt[3]; d.tolerance = opt[4]; d.meaninertia = opt[6];
}

extern "C" int myo_model_dims(const myo_model* m, const myo_task_cfg* cfg, myo_dims* out) {
  if (!m || !out) return fail("myo_model_dims: null"); DevModel d; fill_devmodel(m, cfg, d); const int32_t* I = m->I.data();
  memset(out, 0, sizeof(*out)); out->nq = d.nq; out->nv = d.nv; out->nu = d.nu; out->na = d.na; out->nbody = MYO_DIM(I, MYO_DIM_nbody); out->njnt = d.njnt; out->ntendon = MYO_DIM(I, MYO_DIM_ntendon);
  out->nM = d.nM; out->npair = d.npair; out->nta = d.nta; out->maxcon = d.maxcon; out->maxefc = d.maxefc; out->smem_bytes_per_env = d.n_per_warp*8; out->reserved[0] = d.nnz; out->reserved[1] = d.nD*8 + ((d.nI16w + 1)/2)*8; return 0;
}

extern "C" int myo_model_layout(const myo_model* m, const myo_task_cfg* cfg, int32_t* out, int cap) {
  if (!m || !out || cap < 1) return fail("myo_model_layout: bad arguments");
  DevModel d; Layout L; fill_devmodel(m, cfg, d, &L);
  #define P_OFF(n) d.o_##n,
  #define S_OFF(n) d.s_##n,
  const int32_t po[LP_N] = {MYO_LAYOUT_PERSISTENT(P_OFF)};
  const int32_t so[LS_N] = {MYO_LAYOUT_SCRATCH(S_OFF)};
  #undef P_OFF
  #undef S_OFF
  int32_t v[MYO_LAYOUT_N]; int k = 0;
  for (int i = 0; i < LP_N; i++) v[k++] = po[i];
  for (int i = 0; i < LP_N; i++) v[k++] = L.psz[i];
  for (int i = 0; i < LS_N; i++) v[k++] = so[i];
  for (int i = 0; i < LS_N; i++) v[k++] = L.ssz[i];
  const int32_t tail[] = {d.o_scr + L.head, d.o_scr + L.afterK, d.o_scr + L.extNonSolve, d.o_scr + L.solveEnd, L.arefInH, L.qwsInH, d.n_per_warp, d.maxcon, d.maxefc};
  static_assert(2*LP_N + 2*LS_N + sizeof(tail)/sizeof(tail[0]) == MYO_LAYOUT_N, "MYO_LAYOUT_N counts the region lists of include/myo_b200.h");
  for (int32_t x : tail) v[k++] = x;
  for (int i = 0; i < cap && i < MYO_LAYOUT_N; i++) out[i] = v[i];
  return 0;
}

static int warps_that_fit(const cudaDeviceProp& prop, int per_env_bytes, int const_bytes) { return ((int)prop.sharedMemPerBlockOptin - const_bytes - 64)/per_env_bytes; }
// Launch shape of kernel `fn`: as many env-warps per CTA as its thread limit and shared memory allow, at most one per env.  min_rounds (one
// CTA per SM): the batch takes ceil(n_env / (SMs * warps)) rounds; among the warp counts that reach the minimal number of rounds take the
// SMALLEST (same rounds, less issue contention and less lockstep imbalance per round).  want (tuning override, 0 = none) wins where it fits.
// The dynamic shared-memory limit is an attribute of the kernel in the device context, shared by every batch: it is set to the most the
// device allows that kernel, the same value from every batch and host thread, so that no batch's set-up can lower another batch's limit.
static int launch_shape(const void* fn, const cudaDeviceProp& prop, int per_env_bytes, int const_bytes, int n_env, bool min_rounds, int want, LaunchShape& s) {
  cudaFuncAttributes fa; CUDA_OK(cudaFuncGetAttributes(&fa, fn));
  const int smem_max = (int)prop.sharedMemPerBlockOptin - (int)fa.sharedSizeBytes;
  const int sms = prop.multiProcessorCount, fit = warps_that_fit(prop, per_env_bytes, const_bytes), maxw = fa.maxThreadsPerBlock/32;
  int wpc = fit < maxw ? fit : maxw; if (n_env < wpc) wpc = n_env;
  if (wpc < 1) return fail("model working set exceeds shared memory of one CTA");
  if (min_rounds) { int best = wpc, rounds = (n_env + sms*wpc - 1)/(sms*wpc); for (int q = wpc - 1; q >= 1; q--) if ((n_env + sms*q - 1)/(sms*q) == rounds) best = q;
    if ((size_t)per_env_bytes*best + const_bytes > 100*1024) wpc = best; }
  if (want >= 1 && want <= (maxw < fit ? maxw : fit)) wpc = want;
  s.warps = wpc; s.smem = const_bytes + wpc*per_env_bytes;
  if (s.smem > smem_max) return fail("launch shape needs more dynamic shared memory than the device allows the kernel");
  CUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
  int c = 1; CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, fn, wpc*32, s.smem)); if (c < 1) c = 1;
  const int need = (n_env + wpc - 1)/wpc, cap = sms*c; s.grid = need < cap ? need : cap;
  return 0;
}
// The launch shape of a one-env-per-warp analysis kernel `fn` over the batch, sized from the kernel's own register and thread limits at
// the first call that launches it
static int analysis_shape(const myo_batch* b, const void* fn, LazyShape& l) {
  if (l.ready) return 0;
  cudaDeviceProp prop; CUDA_OK(cudaGetDeviceProperties(&prop, b->device));
  if (launch_shape(fn, prop, b->dm.n_per_warp*8, b->const_bytes, b->n_env, false, 0, l.s)) return -1;
  l.ready = true; return 0;
}

// Everything myo_batch_create does after allocating the batch; on failure the caller destroys the partly built batch.
static int batch_setup(myo_batch* b, const myo_model* m, const myo_task_cfg* cfg) {
  const int n_env = b->n_env;
  fill_devmodel(m, cfg, b->dm);
  if (b->cfg.frame_skip <= 0) b->cfg.frame_skip = 1;
  b->tol = cfg->solver_tolerance > 0 ? cfg->solver_tolerance : 1e-10;
  if (cfg->task == MYO_TASK_POSE && b->dm.nq != b->dm.nv) return fail("pose task needs nq == nv");
  if (cfg->task == MYO_TASK_POSE) b->obs_dim = 2*b->dm.nq + b->dm.nv + b->dm.na;
  else if (cfg->task == MYO_TASK_WALK) b->obs_dim = (b->dm.nq - 2) + b->dm.nv + 16 + 4*b->dm.nu;
  else if (cfg->task == MYO_TASK_HOLD) b->obs_dim = (b->dm.nq - 7) + (b->dm.nv - 6) + 6 + b->dm.na;
  else if (cfg->task == MYO_TASK_REACH) { if (cfg->task_i[0] < 1 || cfg->task_i[0] > 7 || 3*cfg->task_i[0] > b->dm.nq) return fail("reach task: 1..7 tips and 3*ntip <= nq");
    b->obs_dim = b->dm.nq + b->dm.nv + 6*cfg->task_i[0] + b->dm.na; }
  cudaDeviceProp prop; CUDA_OK(cudaGetDeviceProperties(&prop, b->device));
  b->const_bytes = b->dm.nD*8 + ((b->dm.nI16w + 1)/2)*8;
  const int per = b->dm.n_per_warp*8, fit = warps_that_fit(prop, per, b->const_bytes);
  if (b->dm.neq + b->dm.nlimrow + b->dm.maxcon > 255) return fail("equality + limit rows + contact capacity exceed the 255 regulariser slots of the row map");
  // Launch configurations.  Product: the launch_bounds(320) kernel (168 registers, <= 10 warps) unless more warps fit in shared memory AND cut the
  // number of rounds, then the launch_bounds(448) kernel (128 registers, <= 14 warps).  Debug kernel: its own configuration (<= 10 warps).
  cudaFuncAttributes fa_p, fa_w, fa_h, fa_d; CUDA_OK(cudaFuncGetAttributes(&fa_p, myo_env_kernel)); CUDA_OK(cudaFuncGetAttributes(&fa_w, myo_env_kernel_w14));
  CUDA_OK(cudaFuncGetAttributes(&fa_h, myo_env_kernel_w14_hand)); CUDA_OK(cudaFuncGetAttributes(&fa_d, myo_env_kernel_dbg));
  const bool big = (size_t)per*(fit < 4 ? fit : 4) + b->const_bytes > 50*1024;      // a 4-warp CTA already takes > 50 KB: one CTA per SM, sized by the round count (small models run several CTAs per SM instead)
  auto rounds_of = [&](const LaunchShape& s) { const int sms = prop.multiProcessorCount; return (n_env + sms*s.warps - 1)/(sms*s.warps); }; LaunchShape sp, sw;
  if (launch_shape((const void*)myo_env_kernel, prop, per, b->const_bytes, n_env, big, 0, sp) || launch_shape((const void*)myo_env_kernel_w14, prop, per, b->const_bytes, n_env, big, 0, sw)) return -1;
  b->use_w14 = sw.warps > sp.warps && rounds_of(sw) < rounds_of(sp);      // (small models too: the elbow runs 4096 envs in 2 rounds of 14 warps instead of 3 of 10 -- registers, not shared memory, keep it at one CTA per SM)
  if (const char* e = getenv("MYO_B200_W14")) b->use_w14 = atoi(e) != 0 && fa_w.maxThreadsPerBlock > fa_p.maxThreadsPerBlock;      // tuning override
  const void* prod_fn = b->use_w14 ? (const void*)myo_env_kernel_w14 : (const void*)myo_env_kernel;
  const char* want_env = getenv("MYO_B200_WARPS_PER_CTA"); const int want = want_env ? atoi(want_env) : 0;      // tuning override (never above what fits)
  if (launch_shape(prod_fn, prop, per, b->const_bytes, n_env, big, want, b->prod) ||
      launch_shape((const void*)myo_env_kernel_dbg, prop, per, b->const_bytes, n_env, big, want, b->dbg)) return -1;
  b->balanced = b->prod.smem > 100*1024; b->dbg_balanced = b->dbg.smem > 100*1024;      // the balanced slot map for CTAs that fill an SM
  // The w14 launch on the kernel compiled for this batch's shape, where that launch fits it: the same warps per CTA within its thread
  // limit and, with its cold-table region, within the device's shared memory.  It then runs the same grid and slot map.
  if (b->use_w14 && HandShape::matches(b->dm)) {
    const int cold = HandShape::cold_bytes(b->dm, MYO_SEC_LEN(m->I.data(), MYO_SEC_HOT_D)); LaunchShape sh;
    if (b->prod.warps <= fa_h.maxThreadsPerBlock/32 && b->prod.warps <= warps_that_fit(prop, per, b->const_bytes + cold)) {
      if (launch_shape((const void*)myo_env_kernel_w14_hand, prop, per, b->const_bytes + cold, n_env, big, b->prod.warps, sh)) return -1;
      if (sh.warps == b->prod.warps && sh.grid == b->prod.grid) { b->use_hand = true; b->cold_bytes = cold; b->prod = sh; } } }
  // load-sorted env -> round map (one-CTA-per-SM models only; MYO_B200_REGROUP=0 switches it off)
  b->big = big; b->regroup = big; if (const char* e = getenv("MYO_B200_REGROUP")) b->regroup = big && atoi(e) != 0;
  if (b->regroup) { b->perm_rounds = (SLOTS_PER_CTA(1, n_env, b->prod.grid, b->prod.warps) + b->prod.warps - 1)/b->prod.warps; b->perm_slots = b->prod.grid*b->prod.warps*b->perm_rounds; }
  // device memory, after every check
  { const int32_t* I = m->I.data(); const double* D = m->D.data();
    size_t nI = (size_t)b->dm.nI16w*4, nD = (size_t)MYO_SEC_LEN(I, MYO_SEC_HOT_D)*8;      /* ALL hot doubles go to HBM; the first dm.nD of them are staged per CTA */
    CUDA_OK(cudaMalloc(&b->dI, nI ? nI : 16)); CUDA_OK(cudaMalloc(&b->dD, nD ? nD : 16));
    CUDA_OK(cudaMemcpy(b->dI, MYO_ISEC(I, MYO_SEC_HOT_I16), nI, cudaMemcpyHostToDevice)); CUDA_OK(cudaMemcpy(b->dD, MYO_DSEC(I, D, MYO_SEC_HOT_D), nD, cudaMemcpyHostToDevice)); }
  CUDA_OK(cudaMalloc(&b->dCtrl, (size_t)n_env*imax(b->dm.nu, 1)*8)); CUDA_OK(cudaMemset(b->dCtrl, 0, (size_t)n_env*imax(b->dm.nu, 1)*8));
  b->dm.gI16 = b->dI; b->dm.gD = b->dD; b->dm.g_ctrl = b->dCtrl;
  if (b->regroup) { CUDA_OK(cudaMalloc(&b->dLoad, (size_t)n_env*4)); CUDA_OK(cudaMemset(b->dLoad, 0, (size_t)n_env*4)); CUDA_OK(cudaMalloc(&b->dPerm, (size_t)b->perm_slots*4)); }
  // the uploads and memsets above run on the legacy stream (a pageable upload may return before its DMA lands): complete them here, so
  // that a caller whose first launch goes to a non-blocking stream finds the model and the zeroed rows in place
  CUDA_OK(cudaStreamSynchronize(cudaStreamLegacy));
  if (getenv("MYO_B200_VERBOSE")) fprintf(stderr, "[myo_b200] n_env %d: %s kernel, %d warps/CTA, grid %d, smem %d B (const %d + cold tables %d + %d/env, %d fit); debug kernel %d warps, grid %d; max threads / regs: product %d / %d, w14 %d / %d, w14_hand %d / %d, debug %d / %d\n",
    n_env, b->use_hand ? "myo_env_kernel_w14_hand" : b->use_w14 ? "myo_env_kernel_w14" : "myo_env_kernel", b->prod.warps, b->prod.grid, b->prod.smem, b->const_bytes, b->cold_bytes, per, fit, b->dbg.warps, b->dbg.grid, fa_p.maxThreadsPerBlock, fa_p.numRegs, fa_w.maxThreadsPerBlock, fa_w.numRegs, fa_h.maxThreadsPerBlock, fa_h.numRegs, fa_d.maxThreadsPerBlock, fa_d.numRegs);
  return 0;
}

extern "C" int myo_batch_create(const myo_model* m, int device, int n_env, const myo_task_cfg* cfg, myo_batch** out) {
  if (!m || !cfg || !out || n_env <= 0) return fail("myo_batch_create: bad arguments");
  int ndev = 0; cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) return fail("myo_batch_create: no CUDA device available (this library has no CPU fallback)");
  if (device < 0 || device >= ndev) return fail("myo_batch_create: bad device index");
  CUDA_OK(cudaSetDevice(device));
  myo_batch* b = new myo_batch(); b->model = m; b->device = device; b->n_env = n_env; b->cfg = *cfg;
  if (const int rc = batch_setup(b, m, cfg)) { myo_batch_destroy(b); return rc; }
  *out = b; return 0;
}
// The readout's device memory and set-up (also on a failed data_setup, which leaves the batch as if it had not run)
static void data_release(myo_batch* b) {
  cudaFree(b->dRI); cudaFree(b->dRD); cudaFree(b->dPose); b->dRI = nullptr; b->dRD = nullptr; b->dPose = nullptr;
  memset(&b->data, 0, sizeof(b->data)); b->data_shape = LazyShape(); }
extern "C" void myo_batch_destroy(myo_batch* b) { if (!b) return; cudaSetDevice(b->device); cudaFree(b->dI); cudaFree(b->dD); cudaFree(b->dCtrl); cudaFree(b->dLoad); cudaFree(b->dPerm);
  cudaFree(b->dCarry); cudaFree(b->dFdRows); cudaFree(b->dCmc); cudaFree(b->dIfdNom); data_release(b); delete b; }
extern "C" int myo_batch_obs_dim(const myo_batch* b) { return b ? b->obs_dim : -1; }
extern "C" int64_t myo_batch_launch_count(const myo_batch* b) { return b ? b->launches : -1; }
// Launch shape of the product kernels' env steps, as launch() and env_kernel_body use it.  Fields (first min(n, 9) written):
// use_w14, warps_per_cta, grid, rounds per CTA, regroup, balanced, smem_bytes, perm_slots, hand_shape (1: the launch_bounds(448) kernel is
// myo_env_kernel_w14_hand, compiled for the hand's shape).
extern "C" int myo_batch_launch_info(const myo_batch* b, int32_t* out, int n) {
  if (!b || !out || n < 1) return fail("myo_batch_launch_info: bad arguments");
  const int nw = b->prod.warps, grid = b->prod.grid;
  // per_cta and the round loop of env_kernel_body (for j0 = 0; j0 < per_cta; j0 += nw)
  const int per_cta = b->regroup ? b->perm_rounds*nw : SLOTS_PER_CTA(b->balanced, b->n_env, grid, nw);
  const int32_t v[9] = {b->use_w14 ? 1 : 0, nw, grid, (per_cta + nw - 1)/nw, b->regroup ? 1 : 0, b->balanced, b->prod.smem, b->perm_slots, b->use_hand ? 1 : 0};
  for (int i = 0; i < n && i < 9; i++) out[i] = v[i];
  return 0;
}
// Slot -> env map (-1 = idle slot) the last env step ran with: slot blockIdx.x + grid*(round*warps_per_cta + warp).  Synchronises the device.
extern "C" int myo_batch_debug_perm(const myo_batch* b, int32_t* host_out, int n) {
  if (!b || !host_out) return fail("myo_batch_debug_perm: null");
  if (!b->regroup) return fail("myo_batch_debug_perm: this batch runs without the load-sorted map (regroup off)");
  if (!b->perm_built) return fail("myo_batch_debug_perm: no env step has run yet");
  if (n < b->perm_slots) return fail("myo_batch_debug_perm: output holds fewer entries than the map's perm_slots");
  CUDA_OK(cudaSetDevice(b->device)); CUDA_OK(cudaDeviceSynchronize());
  CUDA_OK(cudaMemcpy(host_out, b->dPerm, (size_t)b->perm_slots*4, cudaMemcpyDeviceToHost));
  return 0;
}

// ---- unit-test hook: the dense solver on caller-supplied systems (one warp per system, shared-memory staging like the step kernel)
__global__ void myo_chol_test_kernel(const double* H, double* x, int n, int count) {
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31, sys = blockIdx.x*(blockDim.x >> 5) + wid, nt = n*(n+1)/2, np = chol_pad(n), ntp = np*(np+1)/2;
  double* h = smem + (size_t)wid*(ntp + np + 2); double* v = h + ntp;
  if (sys < count) { for (int i = lane; i < ntp; i += 32) h[i] = i < nt ? H[(size_t)sys*nt + i] : 0.0; for (int i = lane; i < np; i += 32) v[i] = i < n ? x[(size_t)sys*n + i] : 0.0; }
  __syncwarp();
  if (sys < count) { for (int i = n + lane; i < np; i += 32) h[TRI(i,i)] = 1.0; __syncwarp();      // identity padding, as load_M_dense does
    chol_dense(h, n, v, lane); for (int i = lane; i < n; i += 32) x[(size_t)sys*n + i] = v[i]; }
}
extern "C" int myo_debug_chol_solve(int device, const double* H_host, double* x_host, int n, int count, int mode) {
  if (!H_host || !x_host || n < 1 || n > 64 || count < 1) return fail("myo_debug_chol_solve: bad arguments");
  int ndev = 0; if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return fail("myo_debug_chol_solve: no such CUDA device");
  CUDA_OK(cudaSetDevice(device));
  const size_t nt = (size_t)n*(n+1)/2; double *dH = nullptr, *dx = nullptr;
  CUDA_OK(cudaMalloc(&dH, nt*count*8)); CUDA_OK(cudaMalloc(&dx, (size_t)n*count*8));
  CUDA_OK(cudaMemcpy(dH, H_host, nt*count*8, cudaMemcpyHostToDevice)); CUDA_OK(cudaMemcpy(dx, x_host, (size_t)n*count*8, cudaMemcpyHostToDevice));
  const int wpb = 4, np = chol_pad(n); size_t smem = (size_t)wpb*((size_t)np*(np+1)/2 + np + 2)*8; (void)nt;
  CUDA_OK(cudaFuncSetAttribute(myo_chol_test_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  myo_chol_test_kernel<<<(count + wpb - 1)/wpb, wpb*32, smem>>>(dH, dx, n, count); (void)mode;
  CUDA_OK(cudaGetLastError()); CUDA_OK(cudaDeviceSynchronize());
  CUDA_OK(cudaMemcpy(x_host, dx, (size_t)n*count*8, cudaMemcpyDeviceToHost));
  cudaFree(dH); cudaFree(dx); return 0;
}

static int require_bound(const myo_batch* b) { return b->bound ? 0 : fail("batch has no bound buffers (call myo_batch_bind)"); }
static int require_64_dofs(const myo_batch* b, const std::string& call) {      // the IK and static-optimisation kernels: two dofs per lane
  return b->dm.nv > 64 ? fail(call + ": models with more than 64 dofs are not supported") : 0; }

extern "C" int myo_batch_bind(myo_batch* b, const myo_buffers* bufs) {
  if (!b || !bufs) return fail("myo_batch_bind: null");
  if (!bufs->qpos || !bufs->qvel || !bufs->qacc_warmstart || (b->dm.na && !bufs->act)) return fail("myo_batch_bind: qpos/qvel/act/qacc_warmstart are required");
  if (b->cfg.muscle_condition == MYO_COND_FATIGUE && !bufs->fatigue) return fail("myo_batch_bind: fatigue buffer required for MYO_COND_FATIGUE");
  if (b->cfg.muscle_condition == MYO_COND_FATIGUE && b->cfg.fatigue_reset == 2 && !bufs->fatigue_reset_vec) return fail("myo_batch_bind: fatigue_reset_vec buffer required for fatigue_reset = 2");
  if (b->cfg.task == MYO_TASK_HOLD && !bufs->env_prm) return fail("myo_batch_bind: env_prm buffer required for MYO_TASK_HOLD");
  if (bufs->final_obs && !bufs->obs) return fail("myo_batch_bind: final_obs is a copy of obs and needs the obs buffer");
  b->bufs = *bufs; b->bound = true; return 0;
}

static int launch(myo_batch* b, StepArgs& a, void* stream) {
  if (const int rc = require_bound(b)) return rc;
  CUDA_OK(cudaSetDevice(b->device));
  a.b = b->bufs; a.cfg = b->cfg; a.n_env = b->n_env; a.obs_dim = b->obs_dim; a.dt = b->dm.timestep*b->cfg.frame_skip;
  a.seed = b->seed; a.env_offset = b->env_offset;
  a.tol = b->tol;
  // the debug instantiation serves forward-debug calls, bound parity taps / cycle counters and the barrier / lockstep tuning knobs
  const myo_buffers& q = b->bufs;
  const bool dbg = a.mode == 1 || b->cfg.barrier_mode != 0 || b->cfg.reserved_i > 1 || q.tap_qacc || q.tap_actuator_force || q.tap_ten_length || q.tap_qfrc_smooth ||
                   q.tap_ncon || q.tap_contact_pair || q.tap_contact_dist || q.tap_moment || q.tap_qM || q.tap_phase_cycles;
  if (dbg) { a.balanced = b->dbg_balanced; myo_env_kernel_dbg<<<b->dbg.grid, b->dbg.warps*32, b->dbg.smem, (cudaStream_t)stream>>>(b->dm, a); }
  else { const LaunchShape& s = b->prod; a.balanced = b->balanced;
    if (a.mode == 0 && b->regroup) {      // env steps: regroup by last step's load first (same stream), then step through the permutation
      myo_regroup_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(b->dLoad, b->dPerm, b->n_env, s.grid, s.warps, b->perm_slots);
      a.load = b->dLoad; a.perm = b->dPerm; a.perm_rounds = b->perm_rounds; a.load_wn = LOAD_WN; a.load_wi = LOAD_WI; b->perm_built = true; b->launches++; }
    if (b->use_hand) { HandShape hm; static_cast<DevModel&>(hm) = b->dm; hm.nD += b->cold_bytes/8;      // the cold tables staged too
      myo_env_kernel_w14_hand<<<s.grid, s.warps*32, s.smem, (cudaStream_t)stream>>>(hm, a); }
    else if (b->use_w14) myo_env_kernel_w14<<<s.grid, s.warps*32, s.smem, (cudaStream_t)stream>>>(b->dm, a);
    else myo_env_kernel<<<s.grid, s.warps*32, s.smem, (cudaStream_t)stream>>>(b->dm, a); }
  CUDA_OK(cudaGetLastError()); b->launches++; return 0;
}
extern "C" int myo_batch_step(myo_batch* b, void* stream) {
  if (!b) return fail("null batch"); if (!b->bufs.action) return fail("myo_batch_step: action buffer not bound");
  StepArgs a; memset(&a, 0, sizeof(a)); a.mode = 0; return launch(b, a, stream);
}
extern "C" int myo_batch_reset(myo_batch* b, const uint8_t* mask, uint64_t seed, int64_t env_offset, void* stream) {
  if (!b) return fail("null batch");
  if (env_offset < 0 || env_offset > MYO_RESET_ENV_LIMIT - b->n_env) return fail("myo_batch_reset: env_offset must be in [0, 2^47 - n_env] (global env ids key the reset streams)");
  StepArgs a; memset(&a, 0, sizeof(a)); a.mode = 2; a.reset_mask = mask; b->seed = seed; b->env_offset = env_offset;
  return launch(b, a, stream);
}
extern "C" int myo_batch_observe(myo_batch* b, void* stream) {
  if (!b) return fail("null batch");
  StepArgs a; memset(&a, 0, sizeof(a)); a.mode = 3; return launch(b, a, stream);
}
extern "C" int myo_batch_forward_debug(myo_batch* b, const double* ctrl, int n_substeps, void* stream) {
  if (!b || !ctrl) return fail("myo_batch_forward_debug: null");
  StepArgs a; memset(&a, 0, sizeof(a)); a.mode = 1; a.dbg_ctrl = ctrl; a.n_substeps = n_substeps; return launch(b, a, stream);
}

// First readout of a batch: the model tables of mj_kinematics (every body, in tree-level order), the sites and the geoms of every program
// pair go to HBM; the pose scratch is allocated; the launch shape of myo_data_kernel follows from its own register and thread limits.
static int data_setup(myo_batch* b) {
  const int32_t* I = b->model->I.data(); const double* D = b->model->D.data(); DataArgs& a = b->data;
  const int nb = MYO_DIM(I, MYO_DIM_nbody), nj = MYO_DIM(I, MYO_DIM_njnt), ns = MYO_DIM(I, MYO_DIM_nsite), nq = MYO_DIM(I, MYO_DIM_nq), np = b->dm.npair;
  const int32_t* parent = MYO_ISEC(I, MYO_SEC_body_parentid); const int32_t* ppair = MYO_ISEC(I, MYO_SEC_PPAIR);
  std::vector<int> depth(nb, 0); int nlevel = 1;
  for (int k = 1; k < nb; k++) { depth[k] = depth[parent[k]] + 1; nlevel = imax(nlevel, depth[k] + 1); }      // (parents precede children)
  std::vector<int32_t> ri(nlevel + 1, 0);
  for (int k = 0; k < nb; k++) ri[depth[k] + 1]++;
  for (int L = 0; L < nlevel; L++) ri[L + 1] += ri[L];
  for (int L = 0; L < nlevel; L++) for (int k = 0; k < nb; k++) if (depth[k] == L) ri.push_back(k);
  size_t o_parent = ri.size(); ri.insert(ri.end(), parent, parent + nb);
  size_t o_jadr = ri.size(); ri.insert(ri.end(), MYO_ISEC(I, MYO_SEC_body_jntadr), MYO_ISEC(I, MYO_SEC_body_jntadr) + nb);
  size_t o_jnum = ri.size(); ri.insert(ri.end(), MYO_ISEC(I, MYO_SEC_body_jntnum), MYO_ISEC(I, MYO_SEC_body_jntnum) + nb);
  size_t o_jtype = ri.size(); ri.insert(ri.end(), MYO_ISEC(I, MYO_SEC_jnt_type), MYO_ISEC(I, MYO_SEC_jnt_type) + nj);
  size_t o_jq = ri.size(); ri.insert(ri.end(), MYO_ISEC(I, MYO_SEC_jnt_qposadr), MYO_ISEC(I, MYO_SEC_jnt_qposadr) + nj);
  size_t o_sb = ri.size(); ri.insert(ri.end(), MYO_ISEC(I, MYO_SEC_site_bodyid), MYO_ISEC(I, MYO_SEC_site_bodyid) + ns);
  size_t o_pg = ri.size();
  for (int p = 0; p < np; p++) { const int mp = ppair[PPAIR_ISTRIDE*p + 7]; ri.push_back(MYO_ISEC(I, MYO_SEC_pair_geom1)[mp]); ri.push_back(MYO_ISEC(I, MYO_SEC_pair_geom2)[mp]); }
  std::vector<double> rd;
  const int sec[6] = {MYO_SEC_body_pos, MYO_SEC_body_quat, MYO_SEC_jnt_pos, MYO_SEC_jnt_axis, MYO_SEC_qpos0, MYO_SEC_site_pos};
  const int len[6] = {3*nb, 4*nb, 3*nj, 3*nj, nq, 3*ns}; size_t od[6];
  for (int s = 0; s < 6; s++) { if (MYO_SEC_LEN(I, sec[s]) != len[s]) return fail("myo_batch_data: model blob section of unexpected size");
    od[s] = rd.size(); rd.insert(rd.end(), MYO_DSEC(I, D, sec[s]), MYO_DSEC(I, D, sec[s]) + len[s]); }
  CUDA_OK(cudaMalloc(&b->dRI, ri.size()*4)); CUDA_OK(cudaMemcpy(b->dRI, ri.data(), ri.size()*4, cudaMemcpyHostToDevice));
  CUDA_OK(cudaMalloc(&b->dRD, imax((int)rd.size(), 1)*8)); CUDA_OK(cudaMemcpy(b->dRD, rd.data(), rd.size()*8, cudaMemcpyHostToDevice));
  CUDA_OK(cudaMalloc(&b->dPose, (size_t)b->n_env*2*nb*7*8));
  CUDA_OK(cudaStreamSynchronize(cudaStreamLegacy));      // the tables are in place before a launch on any stream reads them (as batch_setup)
  a.nbody = nb; a.nsite = ns; a.nlevel = nlevel; a.lvl = b->dRI; a.parent = b->dRI + o_parent; a.jadr = b->dRI + o_jadr; a.jnum = b->dRI + o_jnum;
  a.jtype = b->dRI + o_jtype; a.jq = b->dRI + o_jq; a.site_body = b->dRI + o_sb; a.pair_geom = b->dRI + o_pg;
  a.bpos = b->dRD + od[0]; a.bquat = b->dRD + od[1]; a.jpos = b->dRD + od[2]; a.jaxis = b->dRD + od[3]; a.qpos0 = b->dRD + od[4]; a.site_pos = b->dRD + od[5];
  a.pose_buf = b->dPose; a.n_env = b->n_env; a.tol = b->tol;
  return analysis_shape(b, (const void*)myo_data_kernel, b->data_shape);
}

extern "C" int myo_batch_data(myo_batch* b, const myo_data_buffers* d, void* stream) {
  if (!b || !d) return fail("myo_batch_data: null");
  if (const int rc = require_bound(b)) return rc;
  const bool pose = d->xpos || d->xquat || d->xmat || d->site_xpos;
  const bool act = d->actuator_length || d->actuator_velocity || d->actuator_force || d->qfrc_actuator;
  const bool dyn = d->qacc || d->ncon || d->contact_geom || d->contact_dist || d->contact_pos || d->contact_frame || d->contact_force;
  if (!pose && !act && !dyn) return 0;
  CUDA_OK(cudaSetDevice(b->device));
  if (!b->data_shape.ready) { if (const int rc = data_setup(b)) { data_release(b); return rc; } }
  DataArgs a = b->data; a.d = *d; a.b = b->bufs; a.pose = pose; a.depth = dyn ? DATA_DYN : (act ? DATA_ACT : DATA_NONE); const LaunchShape& s = b->data_shape.s;
  myo_data_kernel<<<s.grid, s.warps*32, a.depth == DATA_NONE ? 0 : s.smem, (cudaStream_t)stream>>>(b->dm, a);
  CUDA_OK(cudaGetLastError()); b->launches++; return 0;
}

extern "C" int myo_batch_inverse(myo_batch* b, const myo_inverse_buffers* d, int flags, void* stream) {
  if (!b || !d) return fail("myo_batch_inverse: null");
  if (!d->qacc || !d->qfrc_inverse) return fail("myo_batch_inverse: qacc and qfrc_inverse are required");
  if (flags & ~(MYO_INV_NOCONSTRAINT | MYO_INV_DISCRETE)) return fail("myo_batch_inverse: unknown flag bits");
  if (const int rc = require_bound(b)) return rc;
  CUDA_OK(cudaSetDevice(b->device));
  if (analysis_shape(b, (const void*)myo_inverse_kernel, b->inv_shape)) return -1;
  InvArgs a; a.d = *d; a.b = b->bufs; a.n_env = b->n_env; a.flags = flags; const LaunchShape& s = b->inv_shape.s;
  myo_inverse_kernel<<<s.grid, s.warps*32, s.smem, (cudaStream_t)stream>>>(b->dm, a);
  CUDA_OK(cudaGetLastError()); b->launches++; return 0;
}

// Inverse-dynamics FD: stage 0 (the nominal f per env, on the balanced map), then stage 1 (one warp per (env, column) of the requested blocks,
// on the contiguous map), both on `stream`; the start state is the caller's rows or the bound buffers, read only.
extern "C" int myo_batch_inverse_fd(myo_batch* b, const myo_inverse_fd_buffers* d, const myo_inverse_fd_params* p, int flags, void* stream) {
  if (!b || !d || !p) return fail("myo_batch_inverse_fd: null");
  if (!d->qacc) return fail("myo_batch_inverse_fd: qacc is required");
  if (!d->DfDq && !d->DfDv && !d->DfDa) return fail("myo_batch_inverse_fd: at least one of DfDq, DfDv and DfDa is required");
  if (const int rc = require_bound(b)) return rc;
  if (flags & ~(MYO_INV_NOCONSTRAINT | MYO_INV_DISCRETE)) return fail("myo_batch_inverse_fd: unknown flag bits");
  if (!std::isfinite(p->eps) || !(p->eps > 0)) return fail("myo_batch_inverse_fd: eps must be finite and > 0");
  if (p->actuation != 0 && p->actuation != 1) return fail("myo_batch_inverse_fd: actuation must be 0 or 1");
  InvFdArgs a; memset(&a, 0, sizeof(a)); int nblk = 0;
  if (d->DfDq) a.blk[nblk++] = 0;
  if (d->DfDv) a.blk[nblk++] = 1;
  if (d->DfDa) a.blk[nblk++] = 2;
  const DevModel& dm = b->dm; const long long items = (long long)b->n_env*nblk*dm.nv;
  if (items > 0x7fffffffLL) return fail("myo_batch_inverse_fd: n_env * columns must fit in int32");
  CUDA_OK(cudaSetDevice(b->device)); cudaStream_t st = (cudaStream_t)stream;
  if (analysis_shape(b, (const void*)myo_inverse_fd_kernel, b->ifd_shape)) return -1;
  if (b->ifd_items != items) { cudaDeviceProp prop; CUDA_OK(cudaGetDeviceProperties(&prop, b->device));
    if (launch_shape((const void*)myo_inverse_fd_kernel, prop, dm.n_per_warp*8, b->const_bytes, (int)items, false, 0, b->ifd_item_shape)) return -1;
    b->ifd_items = items; }
  if (!b->dIfdNom) CUDA_OK(cudaMalloc(&b->dIfdNom, (size_t)b->n_env*imax(dm.nv, 1)*8));
  const myo_buffers& q = b->bufs;
  myo_buffers& c = a.b;      // the start state, read only
  c.qpos = d->qpos0 ? (double*)d->qpos0 : q.qpos; c.qvel = d->qvel0 ? (double*)d->qvel0 : q.qvel; c.act = d->act0 ? (double*)d->act0 : q.act;
  c.qacc_warmstart = q.qacc_warmstart; c.env_prm = q.env_prm;
  a.d = *d; a.nom = b->dIfdNom; a.eps = p->eps; a.rinv = 1.0/p->eps; a.n_env = b->n_env; a.ncol = nblk*dm.nv; a.flags = flags; a.actuation = p->actuation;
  const LaunchShape &s0 = b->ifd_shape.s, &s1 = b->ifd_item_shape;
  a.stage = 0;
  myo_inverse_fd_kernel<<<s0.grid, s0.warps*32, s0.smem, st>>>(b->dm, a);
  CUDA_OK(cudaGetLastError()); b->launches++;
  a.stage = 1;
  myo_inverse_fd_kernel<<<s1.grid, s1.warps*32, s1.smem, st>>>(b->dm, a);
  CUDA_OK(cudaGetLastError()); b->launches++; return 0;
}

// First rollout of a batch: the launch shape of the rollout kernel that matches the env step's instantiation (from its own attributes,
// with the env step's sizing rule and tuning override) and the carry state.  With the env step's shape the rollout also runs on its slot
// map (load-sorted when the batch regroups); with another shape, on the balanced map without regrouping.
static int roll_setup(myo_batch* b) {
  cudaDeviceProp prop; CUDA_OK(cudaGetDeviceProperties(&prop, b->device));
  const char* want_env = getenv("MYO_B200_WARPS_PER_CTA"); const int want = want_env ? atoi(want_env) : 0;
  LaunchShape& s = b->roll_shape.s;
  if (launch_shape(b->use_w14 ? (const void*)myo_roll_kernel_w14 : (const void*)myo_roll_kernel, prop, b->dm.n_per_warp*8, b->const_bytes, b->n_env, b->big, want, s)) return -1;
  const bool same = s.warps == b->prod.warps && s.grid == b->prod.grid && s.smem == b->prod.smem - b->cold_bytes;      // (less the hand kernel's cold tables)
  b->roll_regroup = same && b->regroup; b->roll_balanced = same ? b->balanced : 1;
  const DevModel& d = b->dm;
  CUDA_OK(cudaMalloc(&b->dCarry, (size_t)b->n_env*(d.nq + 2*d.nv + d.na + 1)*8));
  b->roll_shape.ready = true; return 0;
}

static int roll_run(myo_batch* b, const myo_rollout_buffers* r, int nstep, int substeps, void* stream);
// The StepArgs of a physics-only interval of `substeps` substeps (rollout and transition FD): the batch's model and solver with no task,
// fatigue, reafferentation or auto-reset; the caller sets the state buffers, the roll / fd blocks, the slot map and the slot count
static StepArgs physics_args(const myo_batch* b, int substeps) {
  StepArgs a; memset(&a, 0, sizeof(a)); a.mode = 0;
  a.cfg = b->cfg; a.cfg.task = MYO_TASK_NONE; a.cfg.muscle_condition = MYO_COND_NONE; a.cfg.reaf_dst = a.cfg.reaf_src = 0; a.cfg.auto_reset = 0; a.cfg.frame_skip = substeps;
  a.dt = b->dm.timestep*substeps; a.tol = b->tol; a.seed = b->seed; a.env_offset = b->env_offset;
  return a;
}
extern "C" int myo_batch_rollout(myo_batch* b, const myo_rollout_buffers* r, int nstep, int substeps, void* stream) {
  if (!b || !r) return fail("myo_batch_rollout: null");
  if (!r->ctrl) return fail("myo_batch_rollout: ctrl is required");
  if (const int rc = require_bound(b)) return rc;
  if (nstep < 1 || substeps < 1) return fail("myo_batch_rollout: nstep and substeps must be >= 1");
  CUDA_OK(cudaSetDevice(b->device));
  return roll_run(b, r, nstep, substeps, stream);
}

// The carry of a checked rollout, on the current device: the start state from the caller's rows (r's *0 fields) or the bound buffers, and
// r->overflow cleared; no launch
static int roll_carry(myo_batch* b, const myo_rollout_buffers* r, cudaStream_t st, myo_buffers& c) {
  if (!b->roll_shape.ready) { if (const int rc = roll_setup(b)) { cudaFree(b->dCarry); b->dCarry = nullptr; return rc; } }
  const DevModel& d = b->dm; const size_t n = b->n_env;
  memset(&c, 0, sizeof(c));
  c.qpos = b->dCarry; c.qvel = c.qpos + n*d.nq; c.act = c.qvel + n*d.nv; c.qacc_warmstart = c.act + n*d.na; c.time = c.qacc_warmstart + n*d.nv;
  const myo_buffers& q = b->bufs;
  const struct { double* dst; const double* src; int width; } init[5] = {{c.qpos, r->qpos0 ? r->qpos0 : q.qpos, d.nq}, {c.qvel, r->qvel0 ? r->qvel0 : q.qvel, d.nv},
    {c.act, r->act0 ? r->act0 : q.act, d.na}, {c.qacc_warmstart, r->qacc_warmstart0 ? r->qacc_warmstart0 : q.qacc_warmstart, d.nv}, {c.time, r->time0 ? r->time0 : q.time, 1}};
  for (const auto& f : init) {
    if (f.width == 0) continue;
    if (f.src) CUDA_OK(cudaMemcpyAsync(f.dst, f.src, n*f.width*8, cudaMemcpyDeviceToDevice, st));
    else CUDA_OK(cudaMemsetAsync(f.dst, 0, n*f.width*8, st)); }      // (an unbound time buffer: the rollout starts at 0)
  if (r->overflow) CUDA_OK(cudaMemsetAsync(r->overflow, 0, n*4, st));
  c.env_prm = q.env_prm; c.overflow = r->overflow;
  return 0;
}
// The StepArgs of the intervals of r (rows [n, nstep]) over the carry c, on the rollout's slot map
static StepArgs roll_args(const myo_batch* b, const myo_buffers& c, const myo_rollout_buffers* r, int nstep, int substeps) {
  StepArgs a = physics_args(b, substeps); a.b = c; a.roll = *r; a.roll_nstep = nstep; a.n_env = b->n_env; a.balanced = b->roll_balanced;
  if (b->roll_regroup) { a.load = b->dLoad; a.perm = b->dPerm; a.perm_rounds = b->perm_rounds; a.load_wn = LOAD_WN; a.load_wi = LOAD_WI; }
  return a;
}
// Interval a.roll_t: the regroup launch when the rollouts run on the load-sorted map, then the rollout kernel
static int roll_interval(myo_batch* b, const StepArgs& a, cudaStream_t st) {
  const LaunchShape& s = b->roll_shape.s;
  if (b->roll_regroup) { myo_regroup_kernel<<<1, 1024, 0, st>>>(b->dLoad, b->dPerm, b->n_env, s.grid, s.warps, b->perm_slots); b->launches++; }
  if (b->use_w14) myo_roll_kernel_w14<<<s.grid, s.warps*32, s.smem, st>>>(b->dm, a);
  else myo_roll_kernel<<<s.grid, s.warps*32, s.smem, st>>>(b->dm, a);
  CUDA_OK(cudaGetLastError()); b->launches++; return 0;
}
// The launches of a checked rollout, on the current device: the carry from the start state, then one launch per interval
static int roll_run(myo_batch* b, const myo_rollout_buffers* r, int nstep, int substeps, void* stream) {
  cudaStream_t st = (cudaStream_t)stream; myo_buffers c;
  if (const int rc = roll_carry(b, r, st, c)) return rc;
  StepArgs a = roll_args(b, c, r, nstep, substeps);
  for (int t = 0; t < nstep; t++) {
    a.roll_t = t;
    if (const int rc = roll_interval(b, a, st)) return rc; }
  return 0;
}

// Per-site kernel arguments of myo_batch_ik from the model blob: the site's program body, its ancestor dofs (the Jacobian's non-zero
// columns) and its position in that body, or, on a static body, its world position and the body's world rotation (MuJoCo's pose chain)
static int ik_sites(const myo_batch* b, const int32_t* sid, int ns, IkArgs& a) {
  const int32_t* I = b->model->I.data(); const double* D = b->model->D.data();
  const int nsite = MYO_DIM(I, MYO_DIM_nsite);
  const int32_t *parent = MYO_ISEC(I, MYO_SEC_body_parentid), *dofadr = MYO_ISEC(I, MYO_SEC_body_dofadr), *dofnum = MYO_ISEC(I, MYO_SEC_body_dofnum);
  const int32_t *sbody = MYO_ISEC(I, MYO_SEC_site_bodyid), *pbm = MYO_ISEC(I, MYO_SEC_PB_model_id);
  const double *spos = MYO_DSEC(I, D, MYO_SEC_site_pos), *bpos = MYO_DSEC(I, D, MYO_SEC_body_pos), *bquat = MYO_DSEC(I, D, MYO_SEC_body_quat);
  for (int s = 0; s < ns; s++) {
    if (sid[s] < 0 || sid[s] >= nsite) return fail("myo_batch_ik: site id " + std::to_string(sid[s]) + " outside [0, nsite)");
    const int body = sbody[sid[s]]; int k = -1;
    for (int q = 0; q < b->dm.nbd; q++) if (pbm[q] == body) k = q;
    unsigned long long mk = 0;
    for (int bb = body; bb > 0; bb = parent[bb]) for (int i = dofadr[bb]; i < dofadr[bb] + dofnum[bb]; i++) mk |= 1ull << i;
    double* f = a.site_frame[s]; const double* sp = spos + 3*sid[s];
    for (int c = 0; c < 12; c++) f[c] = 0;
    f[3] = f[7] = f[11] = 1;
    if (k >= 0) for (int c = 0; c < 3; c++) f[c] = sp[c];
    else {      // static body: xpos = xpos(parent) + xmat(parent) body_pos, xquat = xquat(parent) body_quat, from the world down
      std::vector<int> chain; for (int bb = body; bb > 0; bb = parent[bb]) chain.push_back(bb);
      double x[3] = {0, 0, 0}, q[4] = {1, 0, 0, 0}, R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
      for (int t = (int)chain.size() - 1; t >= 0; t--) { const int bb = chain[t]; const double* bp = bpos + 3*bb; const double* r = bquat + 4*bb;
        for (int c = 0; c < 3; c++) x[c] += R[3*c]*bp[0] + R[3*c+1]*bp[1] + R[3*c+2]*bp[2];
        const double n[4] = {q[0]*r[0]-q[1]*r[1]-q[2]*r[2]-q[3]*r[3], q[0]*r[1]+q[1]*r[0]+q[2]*r[3]-q[3]*r[2], q[0]*r[2]-q[1]*r[3]+q[2]*r[0]+q[3]*r[1], q[0]*r[3]+q[1]*r[2]-q[2]*r[1]+q[3]*r[0]};
        const double nn = sqrt(n[0]*n[0] + n[1]*n[1] + n[2]*n[2] + n[3]*n[3]); for (int c = 0; c < 4; c++) q[c] = n[c]/nn;
        const double w_ = q[0], x_ = q[1], y_ = q[2], z_ = q[3];
        const double M[9] = {w_*w_+x_*x_-y_*y_-z_*z_, 2*(x_*y_-w_*z_), 2*(x_*z_+w_*y_), 2*(x_*y_+w_*z_), w_*w_-x_*x_+y_*y_-z_*z_, 2*(y_*z_-w_*x_), 2*(x_*z_-w_*y_), 2*(y_*z_+w_*x_), w_*w_-x_*x_-y_*y_+z_*z_};
        for (int c = 0; c < 9; c++) R[c] = M[c]; }
      for (int c = 0; c < 3; c++) f[c] = x[c] + R[3*c]*sp[0] + R[3*c+1]*sp[1] + R[3*c+2]*sp[2];
      for (int c = 0; c < 9; c++) f[3+c] = R[c]; }
    a.site_body[s] = k; a.site_dofs[s] = mk; }
  return 0;
}

static_assert(sizeof(DevModel) + sizeof(IkArgs) <= 4096, "myo_ik_kernel's arguments fit the 4 KB kernel parameter space");

extern "C" int myo_batch_ik(myo_batch* b, const myo_ik_buffers* d, const myo_ik_params* p, void* stream) {
  if (!b || !d || !p) return fail("myo_batch_ik: null");
  if (!d->site_id || !d->site_quat || !d->target_pos || !d->qpos) return fail("myo_batch_ik: site_id, site_quat, target_pos and qpos are required");
  if (const int rc = require_bound(b)) return rc;
  const int ns = p->nsite;
  if (ns < 1 || ns > MYO_IK_MAXSITE) return fail("myo_batch_ik: nsite must be in [1, " + std::to_string(MYO_IK_MAXSITE) + "]");
  if (!std::isfinite(p->tol) || !std::isfinite(p->damping) || !std::isfinite(p->max_step) || !std::isfinite(p->posture_weight) || !std::isfinite(p->eq_weight))
    return fail("myo_batch_ik: non-finite parameter");
  if (p->damping <= 0 || p->max_step <= 0 || p->tol < 0 || p->max_iter < 0 || p->posture_weight < 0 || p->eq_weight < 0)
    return fail("myo_batch_ik: needs damping > 0, max_step > 0, tol >= 0, max_iter >= 0, posture_weight >= 0 and eq_weight >= 0");
  if (const int rc = require_64_dofs(b, "myo_batch_ik")) return rc;
  CUDA_OK(cudaSetDevice(b->device));
  int32_t sid[MYO_IK_MAXSITE]; cudaStream_t st = (cudaStream_t)stream;      // the site list decides the kernel arguments: read it back
  CUDA_OK(cudaMemcpyAsync(sid, d->site_id, (size_t)ns*4, cudaMemcpyDeviceToHost, st)); CUDA_OK(cudaStreamSynchronize(st));
  IkArgs a; memset(&a, 0, sizeof(a));
  if (const int rc = ik_sites(b, sid, ns, a)) return rc;
  if (analysis_shape(b, (const void*)myo_ik_kernel, b->ik_shape)) return -1;
  a.d = *d; a.p = *p; a.bound_qpos = b->bufs.qpos; a.n_env = b->n_env; const LaunchShape& s = b->ik_shape.s;
  myo_ik_kernel<<<s.grid, s.warps*32, s.smem, st>>>(b->dm, a);
  CUDA_OK(cudaGetLastError()); b->launches++; return 0;
}

// Transition FD: the nominal interval is a rollout into the carry (so it is that rollout, bit for bit); then myo_fd_kernel runs every
// (env, column) item from the env's start state (the caller's rows or the bound buffers, read only) and writes A and B in place.
extern "C" int myo_batch_transition_fd(myo_batch* b, const myo_fd_buffers* d, const myo_fd_params* p, void* stream) {
  if (!b || !d || !p) return fail("myo_batch_transition_fd: null");
  if (!d->ctrl) return fail("myo_batch_transition_fd: ctrl is required");
  if (!d->A && !d->B) return fail("myo_batch_transition_fd: at least one of A and B is required");
  if (const int rc = require_bound(b)) return rc;
  if (!std::isfinite(p->eps) || !(p->eps > 0)) return fail("myo_batch_transition_fd: eps must be finite and > 0");
  if (p->substeps < 1) return fail("myo_batch_transition_fd: substeps must be >= 1");
  if (p->centered != 0 && p->centered != 1) return fail("myo_batch_transition_fd: centered must be 0 or 1");
  const DevModel& dm = b->dm; const int nx = 2*dm.nv + dm.na, nxa = d->A ? nx : 0, ncol = nxa + (d->B ? dm.nu : 0);
  const long long items = (long long)b->n_env*ncol;
  if (items > 0x7fffffffLL) return fail("myo_batch_transition_fd: n_env * columns must fit in int32");
  CUDA_OK(cudaSetDevice(b->device)); cudaStream_t st = (cudaStream_t)stream;
  myo_rollout_buffers r; memset(&r, 0, sizeof(r));
  r.ctrl = d->ctrl; r.qfrc_applied = d->qfrc_applied; r.qpos0 = d->qpos0; r.qvel0 = d->qvel0; r.act0 = d->act0; r.qacc_warmstart0 = d->qacc_warmstart0; r.overflow = d->overflow;
  if (const int rc = roll_run(b, &r, 1, p->substeps, stream)) return rc;
  if (items == 0) return 0;
  if (b->fd_items != items) { cudaDeviceProp prop; CUDA_OK(cudaGetDeviceProperties(&prop, b->device));
    if (launch_shape((const void*)myo_fd_kernel, prop, dm.n_per_warp*8, b->const_bytes, (int)items, b->big, 0, b->fd_shape)) return -1;
    b->fd_items = items; }
  const LaunchShape& s = b->fd_shape;
  const size_t rows = (size_t)s.grid*s.warps*(dm.nu + dm.nq + dm.nv + dm.na)*8;
  if (rows > b->fd_rows_bytes) { cudaFree(b->dFdRows); b->dFdRows = nullptr; b->fd_rows_bytes = 0;
    CUDA_OK(cudaMalloc(&b->dFdRows, rows)); b->fd_rows_bytes = rows; }
  const myo_buffers& q = b->bufs;
  myo_buffers c; memset(&c, 0, sizeof(c));      // the start state, read only: no state is stored back in this kernel
  c.qpos = d->qpos0 ? (double*)d->qpos0 : q.qpos; c.qvel = d->qvel0 ? (double*)d->qvel0 : q.qvel; c.act = d->act0 ? (double*)d->act0 : q.act;
  c.qacc_warmstart = d->qacc_warmstart0 ? (double*)d->qacc_warmstart0 : q.qacc_warmstart; c.env_prm = q.env_prm; c.overflow = d->overflow;
  StepArgs a = physics_args(b, p->substeps); a.b = c; a.roll.ctrl = d->ctrl; a.roll.qfrc_applied = d->qfrc_applied; a.roll_nstep = 1; a.roll_t = 0;
  a.n_env = (int)items; a.balanced = 0;
  a.fd.A = d->A; a.fd.B = d->B; a.fd.nom = b->dCarry; a.fd.rows = b->dFdRows; a.fd.eps = p->eps; a.fd.rinv1 = 1.0/p->eps; a.fd.rinv2 = 1.0/(2.0*p->eps);
  a.fd.n_env = b->n_env; a.fd.ncol = ncol; a.fd.nxa = nxa; a.fd.npass = p->centered ? 2 : 1;
  myo_fd_kernel<<<s.grid, s.warps*32, s.smem, st>>>(b->dm, a);
  CUDA_OK(cudaGetLastError()); b->launches++; return 0;
}

// Placement of myo_static_opt_kernel's arrays (SoArgs order: H, x, l, cg, tf, s, gm, bm), first fit by decreasing size in the per-env
// scratch and the persistent dof axes and mass matrix (dead after the tendon pass).  gm and bm go first, outside the tendon moments, lengths
// and velocities (the gain pass reads those while it writes them); the rest outside mom, gm and bm.  Offsets from the warp base, in doubles.
static int so_plan(const DevModel& d, int* off) {
  const int np = d.nvp, size[8] = {al2(np*(np + 1)/2), al2(np), al2(d.nv), al2(d.nta), al2(d.nta), al2(d.nu), al2(d.nu), al2(d.nu)};
  int lo[16] = {d.s_mom, d.s_tlen, d.s_tvel}, hi[16] = {d.s_mom + al2(d.nnz), d.s_tlen + al2(d.nta), d.s_tvel + al2(d.nta)}, nused = 3;
  const int room[2][2] = {{d.o_scr, d.n_per_warp}, {d.o_dax, d.o_fsm}};      // (dax, dan, qM are consecutive)
  const int order[8] = {6, 7, 0, 1, 2, 3, 4, 5};
  bool done[8] = {};
  for (int r = 0; r < 8; r++) {
    int k = -1;
    if (r < 2) k = order[r];
    else { if (r == 2) { lo[1] = lo[2] = hi[1] = hi[2] = 0; }      // tlen and tvel are dead after the gain pass
      for (int q = 0; q < 6; q++) if (!done[q] && (k < 0 || size[q] > size[k])) k = q; }
    int at = -1;
    for (int g = 0; g < 2 && at < 0; g++) {
      int c = room[g][0];      // the lowest start in this room that overlaps no used interval
      for (bool moved = true; moved; ) { moved = false;
        for (int u = 0; u < nused; u++) if (c < hi[u] && lo[u] < c + size[k]) { c = hi[u]; moved = true; } }
      if (c + size[k] <= room[g][1]) at = c; }
    if (at < 0) return fail("myo_batch_static_opt: the model's per-env scratch has no room for the dual Newton's arrays");
    off[k] = at; lo[nused] = at; hi[nused] = at + size[k]; nused++; done[k] = true; }
  return 0;
}

static_assert(sizeof(DevModel) + sizeof(SoArgs) <= 4096, "myo_static_opt_kernel's arguments fit the 4 KB kernel parameter space");

// The checks of the static optimisation's flags and parameters, shared by the calls that launch it (`call` names the call in the message)
static int so_check(const myo_batch* b, const std::string& call, int flags, int max_iter, double tol) {
  if (flags & ~(MYO_INV_NOCONSTRAINT | MYO_INV_DISCRETE)) return fail(call + ": unknown flag bits");
  if (const int rc = require_bound(b)) return rc;
  if (!std::isfinite(tol)) return fail(call + ": non-finite parameter");
  if (tol < 0 || max_iter < 0) return fail(call + ": needs tol >= 0 and max_iter >= 0");
  return require_64_dofs(b, call);
}
// myo_static_opt_kernel's scratch placement and launch shape, set by the first call that launches it; on the current device
static int so_setup(myo_batch* b) {
  return !b->so_shape.ready && so_plan(b->dm, b->so_off) ? -1 : analysis_shape(b, (const void*)myo_static_opt_kernel, b->so_shape); }
// The SoArgs of a launch over the state buffers c, with every buffer of a.d null
static SoArgs so_args(const myo_batch* b, int max_iter, double tol, int flags, const myo_buffers& c) {
  SoArgs a; memset(&a, 0, sizeof(a));
  a.p.max_iter = max_iter; a.p.tol = tol; a.b = c; a.n_env = b->n_env; a.flags = flags;
  a.o_H = b->so_off[0]; a.o_x = b->so_off[1]; a.o_l = b->so_off[2]; a.o_cg = b->so_off[3]; a.o_tf = b->so_off[4]; a.o_s = b->so_off[5]; a.o_gm = b->so_off[6]; a.o_bm = b->so_off[7];
  return a;
}

extern "C" int myo_batch_static_opt(myo_batch* b, const myo_static_opt_buffers* d, const myo_static_opt_params* p, int flags, void* stream) {
  if (!b || !d || !p) return fail("myo_batch_static_opt: null");
  if (!d->qacc || !d->reserve || !d->act) return fail("myo_batch_static_opt: qacc, reserve and act are required");
  if (const int rc = so_check(b, "myo_batch_static_opt", flags, p->max_iter, p->tol)) return rc;
  CUDA_OK(cudaSetDevice(b->device));
  if (so_setup(b)) return -1;
  SoArgs a = so_args(b, p->max_iter, p->tol, flags, b->bufs); a.d = *d;
  const LaunchShape& s = b->so_shape.s;
  myo_static_opt_kernel<<<s.grid, s.warps*32, s.smem, (cudaStream_t)stream>>>(b->dm, a);
  CUDA_OK(cudaGetLastError()); b->launches++; return 0;
}

// ------------------------------------------------------------------ computed muscle control (myo_batch_cmc)
// Each frame is the unchanged myo_static_opt_kernel and rollout interval launches, with this kernel around them (include/myo_b200.h states
// the loop).  One env per warp on the balanced map.  Stage 0 of frame t (t = 0 .. nstep): row t - 1 of the caller's outputs, the frame's
// solve from the per-frame rows and the state after its interval from the rollout carry (which holds s_t); then, for t < nstep, qacc_des_t
// from the carry and the reference rows, into the per-frame row the static optimisation reads.  Stage 1 (substeps > 1): the excitation
// over the interval, from the carry's act and a*, in place of the static optimisation's one-step ctrl (which it then does not write).
// Per-frame rows, [n, width] each (cmc_rows): qacc_des, a*, ctrl, reserve force, lambda of even and of odd frames, residual, niter | converged.
struct CmcArgs { myo_cmc_buffers d; myo_buffers c; int n_env, nstep, t, stage, substeps;
  double *qdes, *act, *ctrl, *rf, *lam, *res; int32_t *niter, *conv; };      // lam: the rows frame t - 1 wrote

extern "C" __global__ void __launch_bounds__(320) myo_cmc_kernel(const __grid_constant__ DevModel m, const __grid_constant__ CmcArgs a) {
  WARP_KERNEL_PROLOGUE(m, true)
  const myo_cmc_buffers& d = a.d; const myo_buffers& c = a.c; const int nq = m.nq, nv = m.nv, nu = m.nu, na = m.na, lane = w.lane;
  FOR_EACH_WARP_ENV(env, a.n_env) {
    if (a.stage == 1) {
      const idx_t* acls = CI(PA_cls); const double* __restrict__ PAc = GD(PA_d);
      for (int i = lane; i < nu; i += 32) { const double* __restrict__ ag = PAc + acls[i]*PA_STRIDE; const double dyn[3] = {LDC(ag), LDC(ag + 1), LDC(ag + 2)};
        double lo, hi; excitation_range(m, ag, lo, hi);
        a.ctrl[(size_t)env*nu + i] = excitation(dyn, c.act[(size_t)env*na + i], a.act[(size_t)env*nu + i], m.timestep, a.substeps, lo, hi); }
      continue; }
    if (a.t > 0) { const size_t row = (size_t)env*a.nstep + a.t - 1;
      for (int i = lane; i < nu; i += 32) { const size_t o = (size_t)env*nu + i;
        if (d.ctrl) d.ctrl[row*nu + i] = a.ctrl[o];
        if (d.act_opt) d.act_opt[row*nu + i] = a.act[o]; }
      for (int i = lane; i < nv; i += 32) { const size_t o = (size_t)env*nv + i;
        if (d.reserve_force) d.reserve_force[row*nv + i] = a.rf[o];
        if (d.lambda) d.lambda[row*nv + i] = a.lam[o];
        if (d.qvel) d.qvel[row*nv + i] = c.qvel[o];
        if (d.qacc) d.qacc[row*nv + i] = c.qacc_warmstart[o]; }
      if (d.qpos) for (int i = lane; i < nq; i += 32) d.qpos[row*nq + i] = c.qpos[(size_t)env*nq + i];
      if (d.act) for (int i = lane; i < na; i += 32) d.act[row*na + i] = c.act[(size_t)env*na + i];
      if (lane == 0) { if (d.niter) d.niter[row] = a.niter[env]; if (d.converged) d.converged[row] = a.conv[env];
        if (d.residual) d.residual[row] = a.res[env]; if (d.time) d.time[row] = c.time[env]; } }
    if (a.t < a.nstep) { const size_t row = (size_t)env*a.nstep + a.t;
      differentiate_pos(m, w, S_g, c.qpos + (size_t)env*nq, d.ref_qpos + row*nq);
      __syncwarp();
      for (int i = lane; i < nv; i += 32) {
        const double v = d.ref_qacc[row*nv + i] + d.kv[i]*(d.ref_qvel[row*nv + i] - c.qvel[(size_t)env*nv + i]) + d.kp[i]*S_g[i];
        a.qdes[(size_t)env*nv + i] = v;
        if (d.qacc_des) d.qacc_des[row*nv + i] = v; } }
    __syncwarp();
  }
}
static_assert(sizeof(DevModel) + sizeof(CmcArgs) <= 4096, "myo_cmc_kernel's arguments fit the 4 KB kernel parameter space");

// The per-frame rows of myo_batch_cmc (CmcArgs), allocated by the first call
static int cmc_rows(myo_batch* b, CmcArgs& a, double* lam[2]) {
  const size_t n = b->n_env, nv = b->dm.nv, nu = b->dm.nu;
  if (!b->dCmc) CUDA_OK(cudaMalloc(&b->dCmc, n*(4*nv + 2*nu + 2)*8));
  a.qdes = b->dCmc; a.act = a.qdes + n*nv; a.ctrl = a.act + n*nu; a.rf = a.ctrl + n*nu; lam[0] = a.rf + n*nv; lam[1] = lam[0] + n*nv;
  a.res = lam[1] + n*nv; a.niter = (int32_t*)(a.res + n); a.conv = a.niter + n;
  return 0;
}

extern "C" int myo_batch_cmc(myo_batch* b, const myo_cmc_buffers* d, const myo_cmc_params* p, int nstep, int flags, void* stream) {
  if (!b || !d || !p) return fail("myo_batch_cmc: null");
  if (!d->ref_qpos || !d->ref_qvel || !d->ref_qacc || !d->kp || !d->kv || !d->reserve) return fail("myo_batch_cmc: ref_qpos, ref_qvel, ref_qacc, kp, kv and reserve are required");
  if (nstep < 1 || p->substeps < 1) return fail("myo_batch_cmc: nstep and substeps must be >= 1");
  if (const int rc = so_check(b, "myo_batch_cmc", flags, p->max_iter, p->tol)) return rc;
  CUDA_OK(cudaSetDevice(b->device)); cudaStream_t st = (cudaStream_t)stream;
  if (so_setup(b) || analysis_shape(b, (const void*)myo_cmc_kernel, b->cmc_shape)) return -1;
  CmcArgs ca; memset(&ca, 0, sizeof(ca)); double* lam[2];
  if (const int rc = cmc_rows(b, ca, lam)) return rc;
  // the rollout's carry from the start state; its intervals read the frame's ctrl and reserve force rows
  myo_rollout_buffers r; memset(&r, 0, sizeof(r));
  r.ctrl = ca.ctrl; r.qfrc_applied = ca.rf; r.qpos0 = d->qpos0; r.qvel0 = d->qvel0; r.act0 = d->act0; r.qacc_warmstart0 = d->qacc_warmstart0; r.time0 = d->time0;
  r.overflow = d->overflow;
  myo_buffers c;
  if (const int rc = roll_carry(b, &r, st, c)) return rc;
  const StepArgs ra = roll_args(b, c, &r, 1, p->substeps);
  SoArgs so = so_args(b, p->max_iter, p->tol, flags, c);
  so.d.qacc = ca.qdes; so.d.weight = d->weight; so.d.reserve = d->reserve; so.d.act = ca.act; so.d.reserve_force = ca.rf; so.d.ctrl = p->substeps == 1 ? ca.ctrl : nullptr;
  so.d.niter = ca.niter; so.d.converged = ca.conv; so.d.residual = ca.res;
  ca.d = *d; ca.c = c; ca.n_env = b->n_env; ca.nstep = nstep; ca.substeps = p->substeps;
  const LaunchShape &sc = b->cmc_shape.s, &ss = b->so_shape.s;
  for (int t = 0; ; t++) {
    ca.t = t; ca.stage = 0; ca.lam = lam[(t + 1) & 1];
    myo_cmc_kernel<<<sc.grid, sc.warps*32, sc.smem, st>>>(b->dm, ca);
    CUDA_OK(cudaGetLastError()); b->launches++;
    if (t == nstep) break;
    so.d.lambda0 = t == 0 ? d->lambda0 : lam[(t + 1) & 1]; so.d.lambda = lam[t & 1];
    myo_static_opt_kernel<<<ss.grid, ss.warps*32, ss.smem, st>>>(b->dm, so);
    CUDA_OK(cudaGetLastError()); b->launches++;
    if (p->substeps > 1) { ca.stage = 1;
      myo_cmc_kernel<<<sc.grid, sc.warps*32, sc.smem, st>>>(b->dm, ca);
      CUDA_OK(cudaGetLastError()); b->launches++; }
    if (const int rc = roll_interval(b, ra, st)) return rc;
  }
  return 0;
}

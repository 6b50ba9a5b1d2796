// myo_b200.cu -- kernels + C-ABI of libmyo_b200.so (see include/myo_b200.h for the boundary contract).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -shared -Xcompiler -fPIC
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>

#include "myo_solver.cuh"

// ------------------------------------------------------------------ kernel arguments
#ifndef MYO_BMASK
#define MYO_BMASK 0x40      /* phases of the product kernels that start with a CTA barrier (bit k = phase k).  0x40: only the solver entry, whose inner
                               barriers need aligned warps anyway; with load-sorted rounds the warps of a CTA stay close without the other phase barriers. */
#endif
struct StepArgs {
  myo_buffers b; myo_task_cfg cfg;
  int n_env, obs_dim, mode;     // mode 0: env step ; 1: debug forward (ctrl verbatim, optional substeps) ; 2: reset only
  int n_substeps;               // mode 1
  int balanced;                 // env -> CTA map: 1 = e % grid (equal env counts per CTA, big models), 0 = contiguous groups of warps (small models: neighbouring rows share cache lines)
  const double* dbg_ctrl;       // mode 1
  const uint8_t* reset_mask;    // mode 2 (nullable)
  int* load;                    // mode 0, product kernels (nullable): per-env load key written at the end of the step (mean contacts + Newton iterations per substep)
  const int* perm;              // mode 0, product kernels (nullable): slot -> env, built from last step's load keys by myo_regroup_kernel (-1 = idle slot)
  int perm_rounds;              // rounds of warps each CTA walks when perm is set
  int load_wn, load_wi;         // load key = (load_wn * contacts + load_wi * Newton iterations) averaged over the substeps
  unsigned long long seed; long long env_offset;
  double tol, dt;
};

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
__device__ __forceinline__ void philox_init(Philox& p, unsigned long long seed, unsigned long long env, unsigned long long episode, uint32_t lane) {
  p.k0 = (uint32_t)seed; p.k1 = (uint32_t)(seed >> 32); p.c0 = 0; p.c1 = lane; p.c2 = (uint32_t)env ^ (uint32_t)(episode << 20); p.c3 = (uint32_t)(env >> 32) ^ (uint32_t)(episode >> 12) ^ 0x4D594F42u; p.have = 0; }
__device__ __noinline__ double philox_uniform(Philox& p) {   // [0,1) with 53 random bits; consumes the outputs in pairs (0,1) then (2,3)
  if (p.have < 2) philox_gen(p);
  uint32_t a = p.have == 4 ? p.o0 : p.o2, b = p.have == 4 ? p.o1 : p.o3; p.have -= 2;
  return ((double)(((unsigned long long)(a >> 5) << 26) | (b >> 6))) * (1.0/9007199254740992.0); }

// ------------------------------------------------------------------ parity taps
__device__ void write_taps_solve(const DevModel& m, const Warp w, const StepArgs& a, int env) {   // after the Newton solve
  const myo_buffers& b = a.b;
  if (b.tap_qacc) for (int i = w.lane; i < m.nv; i += 32) b.tap_qacc[(size_t)env*m.nv+i] = S_a[i];
  if (b.tap_qfrc_smooth) for (int i = w.lane; i < m.nv; i += 32) b.tap_qfrc_smooth[(size_t)env*m.nv+i] = W_(fsm)[i];
  if (b.tap_qM) for (int i = w.lane; i < m.nM; i += 32) b.tap_qM[(size_t)env*m.nM+i] = W_(qM)[i];
  if (b.tap_ncon && w.lane == 0) { int* t = b.tap_ncon + 4*(size_t)env; t[0] = WI_(ncon); t[1] = WI_(nefc); t[2] = WI_(niter); t[3] = WI_(overflow); }
  __syncwarp();
}
__device__ void write_taps_contacts(const DevModel& m, const Warp w, const StepArgs& a, int env) {   // after constraint assembly (con is overwritten by the solve)
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
__device__ void env_reset(const DevModel& m, const Warp w, const StepArgs& a, int env) {
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

__device__ void write_obs_pose(const DevModel& m, const Warp w, const StepArgs& a, int env, double* dist_out, double* actmag_out) {
  const myo_buffers& b = a.b; float* o = b.obs ? b.obs + (size_t)env*a.obs_dim : nullptr; double d2 = 0, a2 = 0;
  for (int i = w.lane; i < m.nq; i += 32) { double tgt = b.target ? b.target[(size_t)env*m.nq+i] : 0.0, err = tgt - W_(qpos)[i]; d2 += err*err;
    if (o) { o[i] = (float)W_(qpos)[i]; o[m.nq+m.nv+i] = (float)err; } }
  if (o) for (int i = w.lane; i < m.nv; i += 32) o[m.nq+i] = (float)(W_(qvel)[i]*a.dt);
  for (int i = w.lane; i < m.na; i += 32) { a2 += W_(act)[i]*W_(act)[i]; if (o) o[2*m.nq+m.nv+i] = (float)W_(act)[i]; }
  *dist_out = sqrt(warp_sum(d2)); double am = sqrt(warp_sum(a2)); *actmag_out = m.na ? am/m.na : am;
}

// reward / done of the current state (pose_v0.py:113-140); lane 0 writes
__device__ void pose_reward_done(const DevModel& m, const Warp w, const StepArgs& a, int env, double* rw_out, bool* done_out) {
  double dist, am; write_obs_pose(m, w, a, env, &dist, &am);
  const double far_th = a.cfg.task_d[0] > 0 ? a.cfg.task_d[0] : 4*3.14159265358979323846/2; double thd = a.cfg.pose_thd;      // PoseEnvV0: 2 pi (pose_v0.py:117); TorsoEnvV0: pi (torso_v0.py:104), passed in task_d[0]
  *rw_out = a.cfg.weights[0]*(-dist) + a.cfg.weights[1]*((dist < thd ? 1.0 : 0.0)+(dist < 1.5*thd ? 1.0 : 0.0)) + a.cfg.weights[2]*(-am) + a.cfg.weights[3]*(dist > far_th ? -1.0 : 0.0);
  *done_out = dist > far_th; }

// spatial velocity [omega; v_origin] of dynamic body k from its dof chain
__device__ __forceinline__ void body_velocity(const DevModel& m, const Warp w, int k, double* v) {
  const idx_t* cadr = CI(PCH_adr); const idx_t* ch = CI(PCH);
  for (int c = 0; c < 6; c++) v[c] = 0;
  #pragma unroll 1
  for (int e = cadr[k]; e < cadr[k+1]; e++) { int d = ch[e] >> 1; double S[6], qd = W_(qvel)[d]; dof_motion(m, w, d, S); for (int c = 0; c < 6; c++) v[c] += S[c]*qd; } }

// WalkEnvV0 obs / reward / done (walk_v0.py:268-319,358-494) on the post-step state; needs kinematics + tendon + actuation of that
// state in scratch (the reference's extra mj_forward, robot.py:607).  `steps` = WalkEnvV0.steps BEFORE its increment (walk_v0.py:339-342).
__device__ void walk_observe(const DevModel& m, const Warp w, const StepArgs& a, int env, int steps, double* rw_out, bool* done_out) {
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
__device__ void hold_observe(const DevModel& m, const Warp w, const StepArgs& a, int env, double* rw_out, bool* done_out) {
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
__device__ __noinline__ double qvel_dt_norm(const DevModel& m, const Warp w, const StepArgs& a) {
  double v2 = 0; for (int i = w.lane; i < m.nv; i += 32) { const double v = W_(qvel)[i]*a.dt; v2 += v*v; }
  return sqrt(warp_sum(v2)); }

// ReachEnvV0 obs / reward / done (reach_v0.py:98-160): needs kinematics of the post-step state in scratch.  tnow = mjData.time of that state
__device__ void reach_observe(const DevModel& m, const Warp w, const StepArgs& a, int env, double tnow, double* rw_out, bool* done_out) {
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
__device__ __noinline__ RwDone task_observe(const DevModel& m, const Warp w, const StepArgs& a, int env, int steps, double tnow) {
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

// ------------------------------------------------------------------ the kernel
// DBG = false: the product step / reset / observe kernel (modes 0, 2, 3): no parity taps, no cycle counters, fixed barrier scheme.
// DBG = true: everything -- forward-debug mode (1), parity taps, per-phase cycle counters, the barrier / lockstep-group tuning knobs.
// MAXT: launch bound (threads per CTA) -> register budget of the instantiation.
template <bool DBG, int MAXT>
__device__ __forceinline__ void env_kernel_body(const DevModel& m, const StepArgs& a) {
  __shared__ __align__(8) unsigned long long mbar;
  const int wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  // ---- stage the model constants into shared memory: bulk async copies (TMA), completion on an mbarrier
  double* s_d = smem; idx_t* s_i = (idx_t*)(smem + m.nD);
  const unsigned mb = (unsigned)__cvta_generic_to_shared(&mbar);
  if (threadIdx.x == 0) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(mb)); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned bytes_d = (unsigned)m.nD*8u, bytes_i = (unsigned)m.nI16w*4u;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mb), "r"(bytes_d + bytes_i) : "memory");
    const unsigned CH = 32768u;   // chunked: every piece 16-byte aligned and a multiple of 16 bytes
    for (unsigned o = 0; o < bytes_d; o += CH) { unsigned n = bytes_d - o < CH ? bytes_d - o : CH;
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   :: "r"((unsigned)__cvta_generic_to_shared((char*)s_d + o)), "l"((const char*)m.gD + o), "r"(n), "r"(mb) : "memory"); }
    for (unsigned o = 0; o < bytes_i; o += CH) { unsigned n = bytes_i - o < CH ? bytes_i - o : CH;
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   :: "r"((unsigned)__cvta_generic_to_shared((char*)s_i + o)), "l"((const char*)m.gI16 + o), "r"(n), "r"(mb) : "memory"); }
  }
  { unsigned done = 0; while (!done) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(mb) : "memory"); }

  const Warp w = { m.nD + (m.nI16w + 1)/2 + wid*m.n_per_warp, (int)(threadIdx.x & 31) };
  if (w.lane < CNT_N) ((int*)(smem + w.base + m.o_cnt))[w.lane] = 0;
  __syncwarp();
  const myo_buffers& b = a.b;
  // All warps of a CTA walk the phases in lockstep (CTA barriers between phases) so that they share instruction fetches:
  // the step is a long, mostly straight-line program and the instruction cache, not the data path, is the scarce resource.
  const int nsub = a.mode == 0 ? a.cfg.frame_skip : ((DBG && a.mode == 1) ? (a.n_substeps > 0 ? a.n_substeps : 1) : 0);
  const bool integrate = a.mode == 0 || (DBG && a.mode == 1 && a.n_substeps > 0);
  const bool prof = DBG && b.tap_phase_cycles != nullptr;
  // env e belongs to CTA e % gridDim.x: every CTA gets floor or ceil of n_env / gridDim.x envs, so no CTA runs a full extra round
  // while the others idle (4096 envs on 132 SMs at 11 warps: rounds of 11, 11, 9 or 10 everywhere instead of 11, 11, 11 on four fifths of the SMs)
  // With a.perm (big models, env steps of the product kernels) the slot -> env map is the load-sorted one: the envs of a round carry
  // similar contact loads, so the lockstep barriers wait for a slowest env that is close to the average one.
  const bool regrouped = !DBG && a.perm != nullptr;
  const int per_cta = regrouped ? a.perm_rounds*nw : (a.balanced ? (a.n_env + (int)gridDim.x - 1)/(int)gridDim.x : ((a.n_env + nw - 1)/nw + (int)gridDim.x - 1)/(int)gridDim.x*nw);
  for (int j0 = 0; j0 < per_cta; j0 += nw) {
    const int env = regrouped ? a.perm[(int)blockIdx.x + (int)gridDim.x*(j0 + wid)] : (a.balanced ? (int)blockIdx.x + (int)gridDim.x*(j0 + wid) : ((int)blockIdx.x + (int)gridDim.x*(j0/nw))*nw + wid);
    const bool live = (j0 + wid) < per_cta && env >= 0 && env < a.n_env; const long long tstep_ = prof ? clock64() : 0; int load_acc = 0;
    if (live) {
      // ---- load state (coalesced: one env's row per warp)
      for (int i = w.lane; i < m.nq; i += 32) W_(qpos)[i] = b.qpos[(size_t)env*m.nq+i];
      for (int i = w.lane; i < m.nv; i += 32) { W_(qvel)[i] = b.qvel[(size_t)env*m.nv+i]; W_(qws)[i] = b.qacc_warmstart[(size_t)env*m.nv+i]; }
      for (int i = w.lane; i < m.na; i += 32) W_(act)[i] = b.act[(size_t)env*m.na+i];
      if (w.lane < m.neprm) W_(eprm)[w.lane] = b.env_prm ? b.env_prm[(size_t)env*8 + w.lane] : 0.0;     // per-env model overrides (hold task only)
      for (int i = w.lane; i < m.nwz; i += 32) W_(wz)[i] = -1.0;     // cold start of the inverse-wrap roots at the first substep
      __syncwarp();
      if (a.mode == 2) {
        if (!a.reset_mask || a.reset_mask[env]) { env_reset(m, w, a, env);
          task_observe(m, w, a, env, 0, 0.0);
          if (w.lane == 0) { if (b.done) b.done[env] = 0; if (b.truncated) b.truncated[env] = 0; if (b.reward) b.reward[env] = 0; if (b.overflow) b.overflow[env] = 0; } }
      } else if (a.mode == 3) {   // observe: obs/reward/done of the current state, nothing advanced (env.forward(), env_base.py:393-432)
        { const RwDone rd = task_observe(m, w, a, env, b.step_count ? b.step_count[env] : 0, b.time ? b.time[env] : 0.0);
          if (w.lane == 0) { if (b.reward) b.reward[env] = (float)rd.rw; if (b.done) b.done[env] = rd.done != 0; } }
      } else if (DBG && a.mode == 1) {
        for (int i = w.lane; i < m.nu; i += 32) m.g_ctrl[(size_t)env*m.nu+i] = a.dbg_ctrl[(size_t)env*m.nu+i];
      } else if (a.mode == 0) {
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
      PH(2, phase_actuation(m, w, integrate, m.g_ctrl + (size_t)env*m.nu, tap && b.tap_actuator_force ? b.tap_actuator_force + (size_t)env*m.nu : nullptr, tap && b.tap_ten_length ? b.tap_ten_length + (size_t)env*m.nu : nullptr));
      PH(3, phase_body_inertia(m, w); phase_crb(m, w); phase_bias(m, w));
      PH(4, phase_collision(m, w); overflow_seen |= WI_(overflow));
      PH(5, phase_constraints(m, w); if (tap) write_taps_contacts(m, w, a, env));
#ifdef MYO_SOLVE_NOSYNC
      const bool solver_aligned = DBG && ngroups == 1 && m.solve_sync;
#else
      const bool solver_aligned = ngroups == 1 && (!DBG || m.solve_sync);
#endif
      if (solver_aligned) {   // every warp enters the solver: its inner CTA barriers need the idle warps too (the unaligned variant is a debug-kernel experiment)
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
    if (live) {
      if (DBG && a.mode == 1) { if (integrate && w.lane == 0 && b.time) b.time[env] += nsub*m.timestep; }
      else if (a.mode == 0) {
        // ---- obs / reward / done / TimeLimit / auto-reset
        // mjData.time advances by one timestep per substep (the accumulated rounding is visible to ReachEnvV0's `time > 2 dt` test)
        double tnow = b.time ? b.time[env] : 0.0; for (int s_ = 0; s_ < a.cfg.frame_skip; s_++) tnow += m.timestep;
        if (overflow_seen && w.lane == 0 && b.overflow) b.overflow[env] |= 1;      // sticky until the next reset of this env
        if (!DBG && a.load && w.lane == 0) a.load[env] = load_acc/(nsub > 0 ? nsub : 1);
        if (a.cfg.task != MYO_TASK_NONE) { const RwDone rd = task_observe(m, w, a, env, b.step_count ? b.step_count[env] : 0, tnow); const double rw = rd.rw; const bool done = rd.done != 0;
          int sc = b.step_count ? b.step_count[env]+1 : 0; bool trunc = a.cfg.max_episode_steps > 0 && sc >= a.cfg.max_episode_steps;
          __syncwarp();
          // truncated follows gym's TimeLimit: set whenever the step budget is reached, also when the episode terminated on the same step
          if (w.lane == 0) { if (b.reward) b.reward[env] = (float)rw; if (b.done) b.done[env] = done; if (b.truncated) b.truncated[env] = trunc;
            if (b.step_count) b.step_count[env] = sc; if (b.time) b.time[env] = tnow;
            if (b.ep_return) { float R = b.ep_return[env] + (float)rw; b.ep_return[env] = R; if ((done || trunc) && b.last_return) b.last_return[env] = R; } }
          __syncwarp();
          if ((done || trunc) && a.cfg.auto_reset) { env_reset(m, w, a, env); task_observe(m, w, a, env, 0, 0.0); if (w.lane == 0 && b.overflow) b.overflow[env] = 0; }
        } else if (w.lane == 0 && b.time) b.time[env] = tnow;
      }
      __syncwarp();
      // ---- store state
      for (int i = w.lane; i < m.nq; i += 32) b.qpos[(size_t)env*m.nq+i] = W_(qpos)[i];
      for (int i = w.lane; i < m.nv; i += 32) { b.qvel[(size_t)env*m.nv+i] = W_(qvel)[i]; b.qacc_warmstart[(size_t)env*m.nv+i] = W_(qws)[i]; }
      for (int i = w.lane; i < m.na; i += 32) b.act[(size_t)env*m.na+i] = W_(act)[i];
      __syncwarp();
    }
  }
}
// product kernel: up to 10 env-warps per CTA (204 registers per thread)
// Register budget of the product kernel.  ptxas keeps ~36 registers back for the callees of a kernel that makes ABI calls: the entry function
// gets 168 under launch_bounds(320) (10 env-warps per CTA) and 128 under launch_bounds(448) (14).  __maxnreg__(200) spills a third as much
// but the kernel then launches with at most 8 warps per CTA (measured round 2: "too many resources requested" at 9).
#if defined(MYO_LB_MODE) && MYO_LB_MODE == 0
#define MYO_LB __maxnreg__(200)
#elif defined(MYO_LB_MODE) && MYO_LB_MODE == 3
#define MYO_LB __launch_bounds__(448)
#elif defined(MYO_LB_MODE) && MYO_LB_MODE == 4
#define MYO_LB __launch_bounds__(384)
#else
#define MYO_LB __launch_bounds__(320)
#endif
extern "C" __global__ void MYO_LB myo_env_kernel(const __grid_constant__ DevModel m, const __grid_constant__ StepArgs a) { env_kernel_body<false, 320>(m, a); }
// the same product body under launch_bounds(448): 128 registers for the entry function, up to 14 env-warps per CTA.  Chosen when the model's
// shared-memory footprint lets that many warps cut the number of rounds (hand, 4096 envs: 2 rounds of 14 instead of 3 of 10).
#ifndef MYO_EXPERIMENT_NO_W14
#ifndef MYO_W14_REGS
#define MYO_W14_REGS 144
#endif
extern "C" __global__ void __launch_bounds__(448) myo_env_kernel_w14(const __grid_constant__ DevModel m, const __grid_constant__ StepArgs a) { env_kernel_body<false, 448>(m, a); }
#else
#define myo_env_kernel_w14 myo_env_kernel
#endif
// parity taps / forward-debug / profiling counters / tuning knobs
#ifndef MYO_EXPERIMENT_NO_DBG     // (compile-time experiments build the product kernel only)
extern "C" __global__ void __launch_bounds__(320) myo_env_kernel_dbg(const __grid_constant__ DevModel m, const __grid_constant__ StepArgs a) { env_kernel_body<true, 320>(m, a); }
#else
#define myo_env_kernel_dbg myo_env_kernel
#endif

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

struct myo_batch { const myo_model* model; int device, n_env; myo_task_cfg cfg; myo_buffers bufs; bool bound; DevModel dm; int32_t* dI; double* dD; double* dCtrl; int const_bytes;
  int warps_per_cta, grid, smem_bytes, obs_dim; int dbg_warps, dbg_grid, dbg_smem; bool use_w14; bool force_dbg; bool regroup; int* dLoad; int* dPerm; int perm_rounds, perm_slots, load_wn, load_wi; bool perm_built; long long launches; unsigned long long seed; long long env_offset; };

extern "C" const char* myo_last_error(void) { return g_err.c_str(); }
extern "C" int myo_version(void) { return 1; }

extern "C" int myo_model_from_blob(const int32_t* I, int64_t nI, const double* D, int64_t nD, myo_model** out) {
  if (!I || !out || nI < MYO_BLOB_HDR + MYO_NDIM + 3*MYO_NSEC) return fail("myo_model_from_blob: bad arguments");
  if (I[0] != MYO_BLOB_MAGIC || I[1] != MYO_BLOB_VERSION || I[2] != MYO_NDIM || I[3] != MYO_NSEC) return fail("myo_model_from_blob: blob magic/version/layout mismatch");
  for (int s = 0; s < MYO_NSEC; s++) { long long off = MYO_SEC_OFF(I, s), len = MYO_SEC_LEN(I, s); int kind = I[MYO_BLOB_HDR+MYO_NDIM+3*s];
    if (off < 0 || len < 0 || off + len > (kind ? nD : nI)) return fail("myo_model_from_blob: section out of range"); }
  if (MYO_SEC_LEN(I, MYO_SEC_P_dims) < 30 || MYO_SEC_LEN(I, MYO_SEC_HOT_off) != MYO_NSEC + 1) return fail("myo_model_from_blob: blob carries no kernel program (pack with program=build_program(m))");
  myo_model* m = new myo_model(); m->I.assign(I, I+nI); m->D.assign(D, D+nD); *out = m; return 0;
}
extern "C" void myo_model_destroy(myo_model* m) { delete m; }

static int al2(int x) { return (x + 1) & ~1; }
static int imax(int a, int b) { return a > b ? a : b; }
static void fill_devmodel(const myo_model* mm, const myo_task_cfg* cfg, DevModel& d) {
  const int32_t* I = mm->I.data(); const double* D = mm->D.data(); memset(&d, 0, sizeof(d));
  const int32_t* hoff = MYO_ISEC(I, MYO_SEC_HOT_off);
  for (int s = 0; s < MYO_NSEC; s++) d.hoff[s] = hoff[s];
  d.nI16w = MYO_SEC_LEN(I, MYO_SEC_HOT_I16); d.nD = hoff[MYO_NSEC] >= 0 ? hoff[MYO_NSEC] : MYO_SEC_LEN(I, MYO_SEC_HOT_D);      // doubles staged to shared memory (the cold tables behind them stay in HBM)
  d.nq = MYO_DIM(I, MYO_DIM_nq); d.nv = MYO_DIM(I, MYO_DIM_nv); d.nu = MYO_DIM(I, MYO_DIM_nu); d.na = MYO_DIM(I, MYO_DIM_na); d.nM = MYO_DIM(I, MYO_DIM_nM); d.njnt = MYO_DIM(I, MYO_DIM_njnt);
  const int32_t* P = MYO_ISEC(I, MYO_SEC_P_dims);
  d.nbd = P[PD_NBD]; d.nlevel = P[PD_NLEVEL]; d.nsp = P[PD_NSP]; d.nwe = P[PD_NWE]; d.nta = P[PD_NTA]; d.nnz = P[PD_NNZ]; d.nlim = P[PD_NLIM]; d.neq = P[PD_NEQ];
  { const int sp_[3] = {0, P[PD_SPLIT_SP], d.nsp}, we_[3] = {0, P[PD_SPLIT_WE], d.nwe}, ta_[3] = {0, P[PD_SPLIT_TA], d.nta}, nz_[3] = {0, P[PD_SPLIT_NZ], d.nnz};
    for (int k = 0; k < 3; k++) { d.tg_sp[k] = sp_[k]; d.tg_we[k] = we_[k]; d.tg_ta[k] = ta_[k]; d.tg_nz[k] = nz_[k]; } }
  d.npair = P[PD_NPAIR]; d.npair_an = P[PD_NPAIR_ANALYTIC]; d.maxpath = P[PD_MAXPATH]; d.ndepth = P[PD_NDEPTH]; d.eq_tree = P[PD_EQ_TREE];
  const double* opt = MYO_DSEC(I, D, MYO_SEC_opt); d.timestep = opt[0]; d.gx = opt[1]; d.gy = opt[2]; d.gz = opt[3]; d.tolerance = opt[4]; d.meaninertia = opt[6];
  d.ovr_geom = (cfg && cfg->task == MYO_TASK_HOLD) ? cfg->task_i[1] : -1;
  { const char* e = getenv("MYO_B200_SOLVE_SYNC"); d.solve_sync = e ? atoi(e) : 1; }   // CTA barriers inside the Newton loop (0 = warps run the solver phase unaligned)
  int mc = cfg && cfg->maxcon > 0 ? cfg->maxcon : 32; if (mc > 64) mc = 64; if (mc > 2*d.npair) mc = 2*d.npair; /* (the contact-order merge handles up to 64) */ d.maxcon = mc; d.nlimrow = P[PD_NLIMROW] > 0 ? P[PD_NLIMROW] : 2*d.nlim; d.maxefc = d.neq + d.nlimrow + 4*mc;
  int o = 0;
  #define TAKE(field, n) d.field = o; o += al2(n)
  // persistent per-env arrays.  ctrl is NOT here: it is written once per control step to a library-owned global row and re-read by the actuation
  // phase of every substep (an L2 hit); the solver's warm start lives in the tail of the Hessian region when that tail is provably idle (below).
  TAKE(o_qpos, d.nq); TAKE(o_qvel, d.nv); TAKE(o_act, d.na); TAKE(o_dax, 3*d.nv); TAKE(o_dan, 3*d.nv); TAKE(o_qM, d.nM); TAKE(o_fsm, d.nv);
  d.neprm = (cfg && cfg->task == MYO_TASK_HOLD) ? 8 : 0; TAKE(o_eprm, d.neprm); d.nwz = P[PD_NWE_SPH_IN] + P[PD_NWE_CYL_IN]; TAKE(o_wz, d.nwz); TAKE(o_cnt, CNT_N/2);
  d.nvp = chol_pad(d.nv);
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
  d.s_xpos = head; d.s_xmat = head + al2(3*d.nbd); const int afterK = head + K;
  int c0, c1, ext;      // two cursors: inside [0, head) and after K
  #define PLACE(field, n) { const int n_ = al2(n); if (c0 + n_ <= head) { d.field = c0; c0 += n_; } else { d.field = c1; c1 += n_; } }
  c0 = 0; c1 = afterK;
  PLACE(s_mom, d.nnz); PLACE(s_tlen, d.nta); PLACE(s_tvel, d.nta); PLACE(s_tfrc, d.nta); { const int nsA = d.tg_sp[1], nsB = d.nsp - nsA, nwA = d.tg_we[1], nwB = d.nwe - nwA;      // one tendon group at a time lives in U / PL
    PLACE(s_PL, imax(nsA + nwA, nsB + nwB)); PLACE(s_U, 3*imax(nsA + 2*nwA, nsB + 2*nwB)); }
  ext = c1;
  c0 = 0; c1 = afterK;
  PLACE(s_cin, 10*d.nbd); PLACE(s_crb, 10*d.nbd); PLACE(s_bf, 6*d.nbd);
  ext = imax(ext, c1);
  d.kcand = d.npair - d.npair_an; d.ngc = P[PD_NGC];
  d.s_gpose = afterK; d.s_clist = afterK + al2(6*d.ngc); ext = imax(ext, d.s_clist + al2((d.kcand + 1)/2));
  const int extNonSolve = ext;
  int t = head;
  d.s_conJ = t; t += al2(imax((3*d.maxpath*mc*JAC_BYTES + 7)/8, (mc + 1)/2)); d.s_efD = t; t += al2(d.neq + d.nlimrow + mc); d.s_eqJ = t; t += al2(d.neq);      /* (the Jacobian region doubles as the int rank keys of the contact ordering) */
  d.s_va = t; t += al2(d.nvp); d.s_vg = t; d.s_vp = t; t += al2(d.nvp); d.s_vMa = t; t += al2(d.nvp); d.s_vMp = t; t += al2(d.nvp);
  const int hsize = imax(al2(d.nvp*(d.nvp+1)/2), 2*al2(d.nM) + al2(d.nv)); const bool arefInH = rows <= hsize;
  d.s_efA = t; if (!arefInH) t += rows;      /* aref (constraints -> start of the solve) lives in the Hessian region when it fits: H is first written after its last read */
  d.s_H = t; d.s_Hs = t; d.s_LD = t + al2(d.nM); d.s_Dinv = t + 2*al2(d.nM); if (arefInH) d.s_efA = t; t += hsize;
  // warm start in the last nv slots of the Hessian region: read once at the start of the solve (before any write to H), rewritten at the end
  // of the integrator (after the last read of H).  Requires that no other stage reaches that far and that aref (head of H) does not overlap it.
  int qws = t - al2(d.nv);
  const bool qwsInH = qws >= extNonSolve && (!arefInH || d.s_H + rows <= qws) && d.s_H + al2(d.nvp*(d.nvp+1)/2) <= t;
  ext = imax(ext, t);
  int scratch = ext;
  if (qwsInH) { d.o_scr = o; d.o_qws = o + qws; } else { d.o_qws = o_qws_persistent; o += al2(d.nv); d.o_scr = o; }
  #undef PLACE
  #undef TAKE
  // scratch offsets are used relative to the warp base
  { int32_t* f[] = {&d.s_xpos, &d.s_xmat, &d.s_U, &d.s_PL, &d.s_mom, &d.s_tlen, &d.s_tvel, &d.s_tfrc, &d.s_cin, &d.s_crb, &d.s_bf, &d.s_conJ, &d.s_efD, &d.s_efA, &d.s_eqJ,
                    &d.s_icon, &d.s_con, &d.s_clist, &d.s_gpose, &d.s_efR, &d.s_efV, &d.s_va, &d.s_vg, &d.s_vp, &d.s_vMa, &d.s_vMp, &d.s_H, &d.s_Hs, &d.s_LD, &d.s_Dinv};
    for (int32_t* q : f) *q += d.o_scr; }
  d.n_per_warp = d.o_scr + scratch;
}

extern "C" int myo_model_dims(const myo_model* m, const myo_task_cfg* cfg, myo_dims* out) {
  if (!m || !out) return fail("myo_model_dims: null"); DevModel d; fill_devmodel(m, cfg, d); const int32_t* I = m->I.data();
  memset(out, 0, sizeof(*out)); out->nq = d.nq; out->nv = d.nv; out->nu = d.nu; out->na = d.na; out->nbody = MYO_DIM(I, MYO_DIM_nbody); out->njnt = d.njnt; out->ntendon = MYO_DIM(I, MYO_DIM_ntendon);
  out->nM = d.nM; out->npair = d.npair; out->nta = d.nta; out->maxcon = d.maxcon; out->maxefc = d.maxefc; out->smem_bytes_per_env = d.n_per_warp*8; out->reserved[0] = d.nnz; out->reserved[1] = d.nD*8 + ((d.nI16w + 1)/2)*8; return 0;
}

extern "C" int myo_batch_create(const myo_model* m, int device, int n_env, const myo_task_cfg* cfg, myo_batch** out) {
  if (!m || !cfg || !out || n_env <= 0) return fail("myo_batch_create: bad arguments");
  int ndev = 0; cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) return fail("myo_batch_create: no CUDA device available (this library has no CPU fallback)");
  if (device < 0 || device >= ndev) return fail("myo_batch_create: bad device index");
  CUDA_OK(cudaSetDevice(device));
  myo_batch* b = new myo_batch(); memset(&b->bufs, 0, sizeof(b->bufs)); b->model = m; b->device = device; b->n_env = n_env; b->cfg = *cfg; b->bound = false; b->force_dbg = getenv("MYO_B200_DEBUG_KERNEL") && atoi(getenv("MYO_B200_DEBUG_KERNEL")); b->launches = 0; b->seed = 0; b->env_offset = 0;
  fill_devmodel(m, cfg, b->dm);
  if (b->cfg.frame_skip <= 0) b->cfg.frame_skip = 1;
  if (cfg->task == MYO_TASK_POSE && b->dm.nq != b->dm.nv) { delete b; return fail("pose task needs nq == nv"); }
  b->obs_dim = 0;
  if (cfg->task == MYO_TASK_POSE) b->obs_dim = 2*b->dm.nq + b->dm.nv + b->dm.na;
  else if (cfg->task == MYO_TASK_WALK) b->obs_dim = (b->dm.nq - 2) + b->dm.nv + 16 + 4*b->dm.nu;
  else if (cfg->task == MYO_TASK_HOLD) b->obs_dim = (b->dm.nq - 7) + (b->dm.nv - 6) + 6 + b->dm.na;
  else if (cfg->task == MYO_TASK_REACH) { if (cfg->task_i[0] < 1 || cfg->task_i[0] > 7 || 3*cfg->task_i[0] > b->dm.nq) { delete b; return fail("reach task: 1..7 tips and 3*ntip <= nq"); }
    b->obs_dim = b->dm.nq + b->dm.nv + 6*cfg->task_i[0] + b->dm.na; }
  { const int32_t* I = m->I.data(); const double* D = m->D.data();
    size_t nI = (size_t)b->dm.nI16w*4, nD = (size_t)MYO_SEC_LEN(I, MYO_SEC_HOT_D)*8;      /* ALL hot doubles go to HBM; the first dm.nD of them are staged per CTA */
    CUDA_OK(cudaMalloc(&b->dI, nI ? nI : 16)); CUDA_OK(cudaMalloc(&b->dD, nD ? nD : 16));
    CUDA_OK(cudaMemcpy(b->dI, MYO_ISEC(I, MYO_SEC_HOT_I16), nI, cudaMemcpyHostToDevice)); CUDA_OK(cudaMemcpy(b->dD, MYO_DSEC(I, D, MYO_SEC_HOT_D), nD, cudaMemcpyHostToDevice)); }
  CUDA_OK(cudaMalloc(&b->dCtrl, (size_t)n_env*imax(b->dm.nu, 1)*8)); CUDA_OK(cudaMemset(b->dCtrl, 0, (size_t)n_env*imax(b->dm.nu, 1)*8));
  b->dm.gI16 = b->dI; b->dm.gD = b->dD; b->dm.g_ctrl = b->dCtrl;
  cudaDeviceProp prop; CUDA_OK(cudaGetDeviceProperties(&prop, device));
  b->const_bytes = b->dm.nD*8 + ((b->dm.nI16w + 1)/2)*8;
  int per = b->dm.n_per_warp*8, maxs = (int)prop.sharedMemPerBlockOptin - b->const_bytes - 64;
  // Launch configurations.  Product: the launch_bounds(320) kernel (168 registers, <= 10 warps) unless more warps fit in shared memory AND cut the
  // number of rounds, then the launch_bounds(448) kernel (128 registers, <= 14 warps).  Debug kernel: its own configuration (<= 10 warps).
  cudaFuncAttributes fa_p, fa_w, fa_d; CUDA_OK(cudaFuncGetAttributes(&fa_p, myo_env_kernel)); CUDA_OK(cudaFuncGetAttributes(&fa_w, myo_env_kernel_w14)); CUDA_OK(cudaFuncGetAttributes(&fa_d, myo_env_kernel_dbg));
  const int sms = prop.multiProcessorCount, fit = maxs/per;
  if (fit < 1) { delete b; return fail("model working set exceeds shared memory of one CTA"); }
  if (b->dm.neq + b->dm.nlimrow + b->dm.maxcon > 255) { delete b; return fail("equality + limit rows + contact capacity exceed the 255 regulariser slots of the row map"); }
  const bool big = (size_t)per*(fit < 4 ? fit : 4) + b->const_bytes > 50*1024;      // a 4-warp CTA already takes > 50 KB: one CTA per SM, sized by the round count below (small models run several CTAs per SM instead)
  auto pick = [&](int maxw) { int wpc = fit < maxw ? fit : maxw; if (n_env < wpc) wpc = n_env;
    // wave quantisation: with one CTA per SM the batch takes ceil(n_env / (SMs * wpc)) rounds; among the warp counts that reach the
    // minimal number of rounds take the SMALLEST (same rounds, less issue contention and less lockstep imbalance per round)
    if (big) { int best = wpc, rounds = (n_env + sms*wpc - 1)/(sms*wpc); for (int q = wpc - 1; q >= 1; q--) if ((n_env + sms*q - 1)/(sms*q) == rounds) best = q;
      if ((size_t)b->dm.n_per_warp*8*best + b->const_bytes > 100*1024) wpc = best; }
    return wpc; };
  auto rounds_of = [&](int wpc) { return (n_env + sms*wpc - 1)/(sms*wpc); };
  int wp = pick(fa_p.maxThreadsPerBlock/32), ww = pick(fa_w.maxThreadsPerBlock/32), wd = pick(fa_d.maxThreadsPerBlock/32);
  b->use_w14 = ww > wp && rounds_of(ww) < rounds_of(wp);      // (small models too: the elbow runs 4096 envs in 2 rounds of 14 warps instead of 3 of 10 -- registers, not shared memory, keep it at one CTA per SM)
  if (const char* e = getenv("MYO_B200_W14")) b->use_w14 = atoi(e) != 0 && fa_w.maxThreadsPerBlock > fa_p.maxThreadsPerBlock;      // tuning override
  int wpc = b->use_w14 ? ww : wp;
  if (const char* e = getenv("MYO_B200_WARPS_PER_CTA")) { int q = atoi(e), cap = (b->use_w14 ? fa_w.maxThreadsPerBlock : fa_p.maxThreadsPerBlock)/32; if (cap > fit) cap = fit;
    if (q >= 1 && q <= cap) wpc = q; if (q >= 1 && q <= (fa_d.maxThreadsPerBlock/32 < fit ? fa_d.maxThreadsPerBlock/32 : fit)) wd = q; }     // tuning override (never above what fits)
  b->warps_per_cta = wpc; b->smem_bytes = b->const_bytes + wpc*per; b->dbg_warps = wd; b->dbg_smem = b->const_bytes + wd*per;
  CUDA_OK(cudaFuncSetAttribute(myo_env_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, b->smem_bytes));
  CUDA_OK(cudaFuncSetAttribute(myo_env_kernel_w14, cudaFuncAttributeMaxDynamicSharedMemorySize, b->smem_bytes));
  CUDA_OK(cudaFuncSetAttribute(myo_env_kernel_dbg, cudaFuncAttributeMaxDynamicSharedMemorySize, b->dbg_smem));
  { int c = 1; if (b->use_w14) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, myo_env_kernel_w14, wpc*32, b->smem_bytes); else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, myo_env_kernel, wpc*32, b->smem_bytes);
    if (c < 1) c = 1; int need = (n_env + wpc - 1)/wpc, cap = sms*c; b->grid = need < cap ? need : cap; }
  { int c = 1; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, myo_env_kernel_dbg, wd*32, b->dbg_smem); if (c < 1) c = 1; int need = (n_env + wd - 1)/wd, cap = sms*c; b->dbg_grid = need < cap ? need : cap; }
  // load-sorted env -> round map (one-CTA-per-SM models only; MYO_B200_REGROUP=0 switches it off)
  b->regroup = big; if (const char* e = getenv("MYO_B200_REGROUP")) b->regroup = big && atoi(e) != 0;
  b->dLoad = nullptr; b->dPerm = nullptr; b->perm_rounds = 0; b->perm_slots = 0; b->perm_built = false; b->load_wn = 2; b->load_wi = 3;
  if (const char* e = getenv("MYO_B200_LOADKEY")) sscanf(e, "%d,%d", &b->load_wn, &b->load_wi);      // tuning: weights of contacts and Newton iterations in the load key
  if (b->regroup) { const int per_cta = (n_env + b->grid - 1)/b->grid; b->perm_rounds = (per_cta + wpc - 1)/wpc; b->perm_slots = b->grid*wpc*b->perm_rounds;
    CUDA_OK(cudaMalloc(&b->dLoad, (size_t)n_env*4)); CUDA_OK(cudaMemset(b->dLoad, 0, (size_t)n_env*4)); CUDA_OK(cudaMalloc(&b->dPerm, (size_t)b->perm_slots*4)); }
  if (getenv("MYO_B200_VERBOSE")) fprintf(stderr, "[myo_b200] n_env %d: %s kernel, %d warps/CTA, grid %d, smem %d B (const %d + %d/env, %d fit); debug kernel %d warps, grid %d; max threads / regs: product %d / %d, w14 %d / %d, debug %d / %d\n",
    n_env, b->use_w14 ? "launch_bounds(448)" : "launch_bounds(320)", b->warps_per_cta, b->grid, b->smem_bytes, b->const_bytes, per, fit, b->dbg_warps, b->dbg_grid, fa_p.maxThreadsPerBlock, fa_p.numRegs, fa_w.maxThreadsPerBlock, fa_w.numRegs, fa_d.maxThreadsPerBlock, fa_d.numRegs);
  *out = b; return 0;
}
extern "C" void myo_batch_destroy(myo_batch* b) { if (!b) return; cudaSetDevice(b->device); cudaFree(b->dI); cudaFree(b->dD); cudaFree(b->dCtrl); if (b->dLoad) cudaFree(b->dLoad); if (b->dPerm) cudaFree(b->dPerm); delete b; }
extern "C" int myo_batch_obs_dim(const myo_batch* b) { return b ? b->obs_dim : -1; }
extern "C" int64_t myo_batch_launch_count(const myo_batch* b) { return b ? b->launches : -1; }
// Launch shape of the product kernels' env steps, as launch() and env_kernel_body compute it.  Fields (first min(n, 8) written):
// use_w14, warps_per_cta, grid, rounds per CTA, regroup, balanced, smem_bytes, perm_slots.
extern "C" int myo_batch_launch_info(const myo_batch* b, int32_t* out, int n) {
  if (!b || !out || n < 1) return fail("myo_batch_launch_info: bad arguments");
  const int nw = b->warps_per_cta, grid = b->grid, balanced = b->smem_bytes > 100*1024;
  // per_cta and the round loop of env_kernel_body (for j0 = 0; j0 < per_cta; j0 += nw)
  const int per_cta = b->regroup ? b->perm_rounds*nw : (balanced ? (b->n_env + grid - 1)/grid : ((b->n_env + nw - 1)/nw + grid - 1)/grid*nw);
  const int32_t v[8] = {b->use_w14 ? 1 : 0, nw, grid, (per_cta + nw - 1)/nw, b->regroup ? 1 : 0, balanced, b->smem_bytes, b->perm_slots};
  for (int i = 0; i < n && i < 8; i++) out[i] = v[i];
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

extern "C" int myo_batch_bind(myo_batch* b, const myo_buffers* bufs) {
  if (!b || !bufs) return fail("myo_batch_bind: null");
  if (!bufs->qpos || !bufs->qvel || !bufs->qacc_warmstart || (b->dm.na && !bufs->act)) return fail("myo_batch_bind: qpos/qvel/act/qacc_warmstart are required");
  if (b->cfg.muscle_condition == MYO_COND_FATIGUE && !bufs->fatigue) return fail("myo_batch_bind: fatigue buffer required for MYO_COND_FATIGUE");
  if (b->cfg.muscle_condition == MYO_COND_FATIGUE && b->cfg.fatigue_reset == 2 && !bufs->fatigue_reset_vec) return fail("myo_batch_bind: fatigue_reset_vec buffer required for fatigue_reset = 2");
  if (b->cfg.task == MYO_TASK_HOLD && !bufs->env_prm) return fail("myo_batch_bind: env_prm buffer required for MYO_TASK_HOLD");
  b->bufs = *bufs; b->bound = true; return 0;
}

static int launch(myo_batch* b, StepArgs& a, void* stream) {
  if (!b->bound) return fail("batch has no bound buffers (call myo_batch_bind)");
  CUDA_OK(cudaSetDevice(b->device));
  a.b = b->bufs; a.cfg = b->cfg; a.n_env = b->n_env; a.obs_dim = b->obs_dim; a.dt = b->dm.timestep*b->cfg.frame_skip;
  a.seed = b->seed; a.env_offset = b->env_offset;
  a.tol = b->cfg.solver_tolerance > 0 ? b->cfg.solver_tolerance : 1e-10;
  // the debug instantiation serves forward-debug calls, bound parity taps / cycle counters and the barrier / lockstep tuning knobs
  const myo_buffers& q = b->bufs;
  const bool dbg = a.mode == 1 || b->force_dbg || b->cfg.barrier_mode != 0 || b->cfg.reserved_i > 1 || q.tap_qacc || q.tap_actuator_force || q.tap_ten_length || q.tap_qfrc_smooth ||
                   q.tap_ncon || q.tap_contact_pair || q.tap_contact_dist || q.tap_moment || q.tap_qM || q.tap_phase_cycles;
  if (dbg) { a.balanced = b->dbg_smem > 100*1024; myo_env_kernel_dbg<<<b->dbg_grid, b->dbg_warps*32, b->dbg_smem, (cudaStream_t)stream>>>(b->dm, a); }
  else { a.balanced = b->smem_bytes > 100*1024;
    if (a.mode == 0 && b->regroup) {      // env steps: regroup by last step's load first (same stream), then step through the permutation
      myo_regroup_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(b->dLoad, b->dPerm, b->n_env, b->grid, b->warps_per_cta, b->perm_slots);
      a.load = b->dLoad; a.perm = b->dPerm; a.perm_rounds = b->perm_rounds; a.load_wn = b->load_wn; a.load_wi = b->load_wi; b->perm_built = true; b->launches++; }
    if (b->use_w14) myo_env_kernel_w14<<<b->grid, b->warps_per_cta*32, b->smem_bytes, (cudaStream_t)stream>>>(b->dm, a);
    else myo_env_kernel<<<b->grid, b->warps_per_cta*32, b->smem_bytes, (cudaStream_t)stream>>>(b->dm, a); }
  CUDA_OK(cudaGetLastError()); b->launches++; return 0;
}
extern "C" int myo_batch_step(myo_batch* b, void* stream) {
  if (!b) return fail("null batch"); if (!b->bufs.action) return fail("myo_batch_step: action buffer not bound");
  StepArgs a; memset(&a, 0, sizeof(a)); a.mode = 0; return launch(b, a, stream);
}
extern "C" int myo_batch_reset(myo_batch* b, const uint8_t* mask, uint64_t seed, int64_t env_offset, void* stream) {
  if (!b) return fail("null batch");
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

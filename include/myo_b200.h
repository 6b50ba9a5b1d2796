/* myo_b200.h -- C-ABI of the B200-native batched musculoskeletal simulator (libmyo_b200.so).
 *
 * Drop-in boundary for ONE hot path of MyoSuite: `env.step` of
 *   myosuite/envs/myo/base_v0.py:82-118  (BaseV0.step)
 * for thousands of parallel envs.  The reference has no FFI seam of its own on this path; what the
 * library semantically replaces is the MuJoCo C API the reference reaches through pybind11:
 *   mj_step      myosuite/robot/robot.py:861
 *   mj_forward   myosuite/robot/robot.py:607,1002 ; envs/env_base.py:91-92
 *   mj_resetData myosuite/robot/robot.py:999
 *   MjSpec.from_file().compile()  myosuite/envs/env_base.py:70-72,96-106
 * plus the per-step Python glue that must run on the device to keep envs resident in HBM:
 *   sigmoid action remap            base_v0.py:86-94
 *   3CC-r fatigue                   envs/myo/fatigue.py:38-76,82-99
 *   frame_skip substeps             robot/robot.py:901-905
 *   obs / reward / done (pose task) envs/myo/myobase/pose_v0.py:100-140
 *   random reset + target sampling  envs/myo/myobase/pose_v0.py:140-170,250-253
 *
 * Conventions: every function returns 0 on success, <0 on error (text via myo_last_error(), thread
 * local).  No exceptions cross the ABI, no torch types appear in it.  All per-env arrays are
 * CALLER-OWNED device buffers (e.g. torch CUDA tensors passed by data_ptr()), contiguous,
 * row-major [n_env, width], on the batch's device, and must outlive the batch.  Any number of
 * batches, on one device or several, are independent: calls on one batch never change another
 * batch's results or whether its launches succeed, in any order and from any stream or host
 * thread.  Each batch itself is single-stream and not re-entrant.  A model is immutable and
 * shareable.  `stream` arguments are `cudaStream_t` passed as void* (NULL = default).
 */
#ifndef MYO_B200_H
#define MYO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct myo_model myo_model;
typedef struct myo_batch myo_batch;

enum { MYO_TASK_NONE = 0, MYO_TASK_POSE = 1, MYO_TASK_WALK = 2, MYO_TASK_HOLD = 3, MYO_TASK_REACH = 4 };
enum { MYO_COND_NONE = 0, MYO_COND_FATIGUE = 2 };   /* sarcopenia / reafferentation are host-side model edits */

/* model dimensions (mirrors the mjModel sizes the reference reads: env.unwrapped.mj_model.{nq,nv,nu,na}) */
typedef struct {
  int32_t nq, nv, nu, na, nbody, njnt, ntendon, nM;
  int32_t npair;       /* collision candidate pairs evaluated on the device */
  int32_t nta;         /* actuated tendons */
  int32_t maxcon;      /* contact capacity per env */
  int32_t maxefc;      /* constraint-row capacity per env */
  int32_t smem_bytes_per_env;
  int32_t reserved[3];
} myo_dims;

/* task / stepping configuration (registry kwargs of the reference, envs/myo/myobase/__init__.py) */
typedef struct {
  int32_t task;              /* MYO_TASK_* */
  int32_t frame_skip;        /* physics substeps per env step (base_v0.py:27 default 10) */
  int32_t max_episode_steps; /* TimeLimit truncation (registry max_episode_steps) */
  int32_t normalize_act;     /* sigmoid remap of muscle actions (base_v0.py:86-94) */
  int32_t muscle_condition;  /* MYO_COND_* */
  int32_t auto_reset;        /* 1: envs that finish are reset inside the step kernel */
  int32_t reset_random;      /* reset_type="random": pose qpos ~ U(jnt_range); walk keyframe row 0/1 of init_qpos + N(0,0.02) (walk_v0.py:321-337); hold goal/size sampling. 0 = init_qpos */
  int32_t maxcon;            /* 0 = library default */
  int32_t reaf_dst, reaf_src;/* reafferentation (base_v0.py:104-108): ctrl[dst] = ctrl[src]; ctrl[src] = 0 ; dst == src = off */
  int32_t barrier_mode;      /* CTA phase barriers: 0 = before every phase (default), 1 = once per substep, 2 = none, >2 = bit mask of the 8 phases that start with a barrier (tuning knob) */
  int32_t reserved_i;        /* lockstep groups per CTA (tuning knob; 0/1 = the whole CTA is one group) */
  int32_t fatigue_reset;     /* fatigue state at reset (fatigue.py:82-99): 0 = MA 0, MR 1, MF 0 ; 1 = fatigue_reset_random (u1, u2 ~ U(0,1): MA = u1 u2, MR = u1 (1 - u2), MF = 1 - u1) ; 2 = fatigue_reset_vec (MF = vec, MR = 1 - vec, MA = 0) */
  double pose_thd;           /* pose_v0.py:43 */
  double weights[8];         /* reward weights in the task's own key order (pose_v0.py:18-23, walk_v0.py:205-211, obj_hold_v0.py:17-21; reach_v0.py:18-22 as reach, bonus, act_reg, penalty) */
  double solver_tolerance;   /* scaled-gradient stop of the Newton solver; 0 = library default (1e-10) */
  int32_t task_i[16];        /* task-specific indices, filled by the host mirror (vec_env.py): WALK body/joint ids, HOLD object ids, REACH [ntip, tip body x ntip] */
  double task_d[24];         /* task-specific constants: WALK targets / thresholds / torso quaternion offset, HOLD object site, REACH tip-site offsets [3 x ntip] then far_th */
  double reserved[2];        /* [0] != 0 with the phase-cycle tap bound: record the barrier wait before each phase instead of its work (profiling) */
  /* REACH reward shape: reach = c_off - d - c_vel |qvel dt| ; act_reg = -c_act |act|/na ; bonus thresholds near and 2 near with near = ntip near_per_tip.
   * {c_off, c_vel, c_act, near_per_tip}; all zero = reach_v0.py:120-160 (0, 0, 1, 0.0125).  The leg stand task (walk_v0.py:104-140) is (10, 10, 100, 0.05). */
  double reach_shape[4];
  /* REACH reset, when hi > lo: for every joint j, qpos[jnt_qposadr[j]] = clip(init_qpos[.] + U(lo, hi), jnt_range[j]) (walk_v0.py:142-186) */
  double joint_random[2];
} myo_task_cfg;

/* caller-owned device buffers; nullable ones are marked.  f64 state, f32 I/O like the reference
 * (obs cast to float32 in envs/obs_vec_dict.py:83, action space float32 in envs/env_base.py:155). */
typedef struct {
  const float* action;       /* [n, nu]  in  */
  double* qpos;              /* [n, nq]  in/out */
  double* qvel;              /* [n, nv]  in/out */
  double* act;               /* [n, na]  in/out */
  double* qacc_warmstart;    /* [n, nv]  in/out (mjData.qacc_warmstart) */
  double* time;              /* [n]      in/out */
  double* fatigue;           /* [n, 3, nu] MA,MR,MF (nullable unless MYO_COND_FATIGUE) */
  double* target;            /* [n, nq]  pose target_jnt_value, in/out */
  const double* target_range;/* [nq, 2]  per-qpos target sampling range (pose), model-level, in */
  const double* init_qpos;   /* [nq]     reset pose, in ([2,nq] for the walk task with reset_random: the two candidate keyframes) */
  const double* init_qvel;   /* [nv]     reset velocity (nullable = zeros), in ([2,nv] alongside a [2,nq] init_qpos) */
  double* env_prm;           /* [n, 8]   per-env model overrides (HOLD: goal site pos[3], object geom size[3]); nullable */
  int32_t* step_count;       /* [n] */
  int64_t* episode_count;    /* [n]  also keys the reset's Philox streams (myo_batch_reset) */
  float* obs;                /* [n, obs_dim] out */
  float* reward;             /* [n] out (rwd_dense) */
  uint8_t* done;             /* [n] out (terminated) */
  uint8_t* truncated;        /* [n] out (TimeLimit) */
  float* ep_return;          /* [n] running return of the current episode */
  float* last_return;        /* [n] return of the most recently finished episode */
  /* parity taps, all nullable: values of the LAST substep's forward pass (pre-integration state) */
  double* tap_qacc;          /* [n, nv] */
  double* tap_actuator_force;/* [n, nu] */
  double* tap_ten_length;    /* [n, nta] actuator_length order */
  double* tap_qfrc_smooth;   /* [n, nv] */
  int32_t* tap_ncon;         /* [n, 4]: ncon, nefc, newton iterations, overflow flag */
  int32_t* tap_contact_pair; /* [n, maxcon] program pair index of each contact, -1 padded */
  double* tap_contact_dist;  /* [n, maxcon] */
  double* tap_moment;        /* [n, nnz] structural non-zeros of the tendon moment */
  double* tap_qM;            /* [n, nM] */
  long long* tap_phase_cycles; /* [n, 20] SM-clock cycles per phase over the call (profiling aid; 8-11 solver parts, 12,13: max ncon / nefc, 14,15: Newton iterations / dense ones, 16: cooperative collision, 17: load..substeps) */
  const double* fatigue_reset_vec; /* [nu] nullable unless cfg.fatigue_reset == 2: the reference's fatigue_reset_vec (base_v0.py:29,48; fatigue.py:90-94) */
  int32_t* overflow;         /* [n] nullable: sticky flag, set when a substep of this env dropped contacts (more than maxcon, or more ellipsoid candidates than the list holds); cleared by the env's reset */
  /* Since version 2.  The observation of the state an episode ended in, written by myo_batch_step for the envs whose done or truncated
   * it sets, before the auto-reset (if on) overwrites their obs row; without auto-reset it equals obs.  The rows of the other envs are
   * not written, and reset / observe / forward-debug never write it.  A row is valid exactly where done | truncated of the same step is set. */
  float* final_obs;          /* [n, obs_dim] out, nullable (needs obs) */
} myo_buffers;

/* Caller-owned device buffers of a readout of mjData (myo_batch_data), all nullable: only the non-null fields are computed.  Every
 * value equals MuJoCo's mjData after mj_forward at the env's current (time, qpos, qvel, act) with the per-env overrides (env_prm,
 * targets) applied and ctrl = the last env step's ctrl (zeros before the first step).  MuJoCo ids and order, f64 unless noted. */
typedef struct {
  /* pose group: mj_kinematics (the quaternion chain: xquat carries MuJoCo's sign, xmat = quat2mat(xquat)) */
  double* xpos;              /* [n, nbody, 3] */
  double* xquat;             /* [n, nbody, 4] */
  double* xmat;              /* [n, nbody, 9] */
  double* site_xpos;         /* [n, nsite, 3] */
  /* [nsite, 2] in, nullable (every site at its model site_pos): where the local position of each site comes from, as (kind, index):
   * 0 model site_pos ; 1 target[env, index .. index+2] ; 2 env_prm[env, index .. index+2] ; 3 the world position of site `index` at the
   * forward kinematics of qpos := target[env] (the pose task's target markers).  Kinds 1-3 fall back to 0 when their buffer is unbound. */
  const int32_t* site_source;
  /* actuation group: transmission, velocities, muscle forces */
  double* actuator_length;   /* [n, nu] */
  double* actuator_velocity; /* [n, nu] */
  double* actuator_force;    /* [n, nu] */
  double* qfrc_actuator;     /* [n, nv] */
  /* dynamics group: collision and the constraint solve (no integration; the warm start is read, never written) */
  double* qacc;              /* [n, nv] */
  int32_t* ncon;             /* [n] */
  int32_t* contact_geom;     /* [n, maxcon, 2] geom1, geom2 in model pair order, -1 padded */
  double* contact_dist;      /* [n, maxcon]    0 padded */
  double* contact_pos;       /* [n, maxcon, 3] */
  double* contact_frame;     /* [n, maxcon, 9] rows normal, tangent1, tangent2 */
  double* contact_force;     /* [n, maxcon, 6] mj_contactForce: the pyramid forces decoded into the contact frame, normal first */
} myo_data_buffers;

/* Caller-owned device buffers of myo_batch_inverse (MuJoCo's mj_inverse): the generalized force that produces the acceleration qacc at
 * each env's current (qpos, qvel) with the per-env overrides (env_prm) applied,
 *   qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - qfrc_constraint
 * M with armature; qfrc_passive = -damping qvel; qfrc_constraint = J' efc_force with MuJoCo's soft-constraint inverse: jar = J qacc - aref,
 * efc_force = -D jar on equality rows and on limit and contact rows where jar < 0, else 0.  Contacts, rows and their order are those of
 * mj_forward at the same state (myo_batch_data's contact list).  act, ctrl and the warm start are not read.  Only the non-null outputs
 * are written. */
typedef struct {
  const double* qacc;        /* [n, nv] in, required */
  double* qfrc_inverse;      /* [n, nv] out, required */
  double* qfrc_constraint;   /* [n, nv] nullable */
  double* contact_force;     /* [n, maxcon, 6] nullable: mj_contactForce of the inverse's efc_force, in myo_data_buffers.contact_force's layout */
  double* actuator_moment;   /* [n, nu, nv] nullable, dense: gear x the tendon moment (mjData.actuator_moment through mju_sparse2dense) */
} myo_inverse_buffers;
#define MYO_INV_NOCONSTRAINT 1   /* mjDSBL_CONSTRAINT: no collision, no constraint rows, qfrc_constraint = 0 */
#define MYO_INV_DISCRETE 2       /* mjENBL_INVDISCRETE: qacc is (qvel' - qvel) / h of one Euler substep with implicit damping; it is converted to
                                    the continuous qacc_c = M^-1 (M + h B) qacc of the forward pass, which everything above then uses */

/* Caller-owned device buffers of myo_batch_rollout (MuJoCo's mj_step, nstep intervals of `substeps` mj_steps each).  ctrl is MuJoCo's
 * ctrl: clipped to ctrlrange inside the step, as mj_step does, with no action remap, fatigue or reafferentation.  qfrc_applied is
 * mjData.qfrc_applied: added to qfrc_smooth, so it enters the constraint solve and the implicit-damping Euler step.  The start state
 * fields are nullable: a null one is taken from the batch's bound buffer of the same name.  Every output is nullable; row t holds
 * mjData after the last mj_step of interval t. */
typedef struct {
  const double* ctrl;        /* [n, nstep, nu] in, required; row t is held for the substeps of interval t */
  const double* qfrc_applied;/* [n, nstep, nv] in, nullable (zero) */
  const double* qpos0;       /* [n, nq] start state, nullable (bound qpos) */
  const double* qvel0;       /* [n, nv] nullable (bound qvel) */
  const double* act0;        /* [n, na] nullable (bound act) */
  const double* qacc_warmstart0; /* [n, nv] nullable (bound qacc_warmstart) */
  const double* time0;       /* [n] nullable (bound time) */
  double* qpos;              /* [n, nstep, nq] out */
  double* qvel;              /* [n, nstep, nv] out */
  double* act;               /* [n, nstep, na] out */
  double* qacc;              /* [n, nstep, nv] out: mjData.qacc, which is also the next interval's warm start */
  double* time;              /* [n, nstep] out */
  int32_t* overflow;         /* [n] out: set when a substep of the rollout dropped contacts (myo_buffers.overflow's meaning), else 0 */
} myo_rollout_buffers;

/* Caller-owned device buffers of myo_batch_ik: damped least-squares inverse kinematics of ns sites (one list for the batch) to per-env
 * targets.  From q = q0 (qpos0, or the bound qpos) each iteration k = 0, 1, ... runs mj_kinematics at q; the site errors
 * e_s = target_pos_s - site_xpos_s and, with orientation targets, w_s = log(mat(target_quat_s) site_xmat_s') (world-frame rotation
 * vector, angle in [0, pi]); stops with converged = 1 when every |e_s| <= tol and every |w_s| <= tol, or with converged = 0 at
 * k = max_iter; else solves
 *   H = sum_s (wp_s jacp_s' jacp_s + wr_s jacr_s' jacr_s) + eq_weight sum_e J_e' J_e + posture_weight P + damping I
 *   g = sum_s (wp_s jacp_s' e_s + wr_s jacr_s' w_s) - eq_weight sum_e J_e' c_e + posture_weight P (qpos_ref - q)
 * for H dq = g (joint equalities e with residual c_e and row J_e as the constraint rows have them; P: 1 on hinge and slide dofs, 0 on
 * free-joint dofs; a dof outside dof_mask gets an identity row and column and g = 0), caps |dq| at max_step, and sets
 * q <- q (+) dq (mj_integratePos with dt = 1), then clamps every limited hinge or slide joint to its range.  Every output describes the
 * returned qpos; max_iter = 0 returns q0 with its Jacobians (mj_jacSite) and errors. */
#define MYO_IK_MAXSITE 16
typedef struct {
  const int32_t* site_id;    /* [ns] in, required: model site ids */
  const double* site_quat;   /* [ns, 4] in, required: each site's frame in its body, mjModel.site_quat (the model blob carries no site frames) */
  const double* site_weight; /* [ns, 2] nullable (1, 1): position and orientation weight of each site */
  const double* target_pos;  /* [n, ns, 3] in, required */
  const double* target_quat; /* [n, ns, 4] nullable (position targets only): w x y z, normalised here */
  const double* qpos0;       /* [n, nq] start, nullable (bound qpos) */
  const double* qpos_ref;    /* [n, nq] posture reference, nullable (the start) */
  const uint8_t* dof_mask;   /* [nv] nullable (every dof moves): 0 holds the dof */
  double* qpos;              /* [n, nq] out, required */
  int32_t* niter;            /* [n] nullable: updates applied */
  int32_t* converged;        /* [n] nullable */
  double* err;               /* [n, ns, 2] nullable: |e_s|, |w_s| (0 without orientation targets) */
  double* site_xpos;         /* [n, ns, 3] nullable */
  double* site_xmat;         /* [n, ns, 9] nullable */
  double* jacp;              /* [n, ns, 3, nv] nullable: mj_jacSite */
  double* jacr;              /* [n, ns, 3, nv] nullable */
} myo_ik_buffers;
typedef struct {
  int32_t nsite, max_iter;
  double tol, damping, max_step, posture_weight, eq_weight;
} myo_ik_params;

/* Caller-owned device buffers of myo_batch_transition_fd: MuJoCo's mjd_transitionFD (mjd_stepFD) with one mj_step replaced by one interval
 * of `substeps` mj_steps with ctrl held, x' ~ x'0 + A dx + B du.
 *   State: x = [dq (nv, the tangent space of mj_integratePos / mj_differentiatePos), qvel (nv), act (na)], nx = 2 nv + na; time is not
 *     part of it.
 *   Nominal: x'0 is one interval from the start state with ctrl and qfrc_applied, bit-identical to myo_batch_rollout with nstep = 1 and
 *     the same substeps from the same start.
 *   Warm start: every perturbed interval starts from the same start state with the start's qacc_warmstart (mjd_stepFD restores the warm
 *     start before each perturbation); its inverse-wrap roots start cold, as every rollout interval's do.
 *   Perturbations: qpos column j: mj_integratePos(qpos, e_j, +-eps); qvel column j: qvel[j] +- eps; act column j: act[j] +- eps
 *     (unclamped); ctrl column i: ctrl[i] +- eps, where with actuator_ctrllimited fwd = inRange(ctrl, ctrl + eps) and
 *     back = (centered || !fwd) && inRange(ctrl - eps, ctrl) (without the limit both are possible); state columns always go forward and
 *     go back when centered.
 *   Differences: both sides (x'+ (-) x'-) * (1 / (2 eps)); forward only (x'+ (-) x'0) * (1 / eps); back only (x'0 (-) x'-) * (1 / eps);
 *     neither 0.  (-) is mj_differentiatePos (dt = 1) on the qpos part and subtraction on the rest; 1 / eps and 1 / (2 eps) are the
 *     IEEE-rounded reciprocals, as mjd_stepFD's mju_scl(ds, ds, 1/h) has them. */
typedef struct {
  const double* ctrl;            /* [n, nu] in, required: MuJoCo ctrl, held for the substeps (clipped to ctrlrange inside the step, like rollout) */
  const double* qfrc_applied;    /* [n, nv] nullable (zero) */
  const double* qpos0;           /* [n, nq] start state, nullable field by field (bound buffers), as myo_rollout_buffers */
  const double* qvel0;           /* [n, nv] */
  const double* act0;            /* [n, na] */
  const double* qacc_warmstart0; /* [n, nv] */
  double* A;                     /* [n, nx, nx] out, nullable; nx = 2 nv + na, row-major, A[i][j] = d x'_i / d x_j */
  double* B;                     /* [n, nx, nu] out, nullable (at least one of A, B) */
  int32_t* overflow;             /* [n] out, nullable: set when any substep of any of the env's perturbed or nominal steps dropped contacts */
} myo_fd_buffers;
typedef struct { double eps; int32_t centered, substeps; } myo_fd_params;

/* Caller-owned device buffers of myo_batch_static_opt: muscle static optimisation with reserve actuators at each env's current (qpos, qvel,
 * act).  With tau = qfrc_inverse(qacc) (myo_batch_inverse with the same flags), AM [nu, nv] the actuator moments (gear x the tendon
 * moment), and g <= 0, b the muscle gain and bias at the current actuator length and velocity (actuator_force = g act + b), let
 * t = tau - AM' b and G = AM' diag(g) [nv, nu].  The solution of the strictly convex problem
 *   min_{a, r}  1/2 sum_m w_m a_m^2 + 1/2 sum_i (r_i / rho_i)^2   s.t.   G a + r = t,   0 <= a_m <= 1
 * (w: weight, rho: reserve; r is the reserve generalized force, exactly t on dofs no muscle crosses) comes from semismooth Newton on the
 * dual in nv space: a(l) = clip((G' l)_m / w_m, 0, 1), r(l) = rho^2 l, F(l) = G a(l) + rho^2 l - t; the step solves
 * (G_F W_F^-1 G_F' + diag rho^2) d = -F over the muscles F strictly inside the box and those at the kink (G'l)_m = 0 (the generalized
 * Jacobian's choice there; at l = 0 it is every muscle, which keeps the first step from overshooting), with Armijo backtracking (halving, slope 1e-4) on the
 * concave dual psi(l) = l't - 1/2 sum rho_i^2 l_i^2 - sum_m max_{a in [0, 1]} (a (G'l)_m - 1/2 w_m a^2).  From l = lambda0 (or 0) it stops
 * with converged = 1 at the first iterate where |F|_inf <= tol max(1, |t|_inf), else with converged = 0 after max_iter steps; every
 * output describes the returned l.  ctrl is the excitation that takes the current act to a in one mj_step of the muscle activation
 * dynamics (act' = act + h (clip(ctrl, 0, 1) - act) / tau(ctrl, act)): closed form with tausmooth = 0, bisection over the range to machine
 * precision otherwise; it is clipped to ctrlrange intersected with [0, 1] ([0, 1] without ctrllimited), where act moves toward a but does
 * not reach it.  Only the non-null outputs are written. */
typedef struct {
  const double* qacc;          /* [n, nv] in, required */
  const double* weight;        /* [nu] nullable (1): w > 0 */
  const double* reserve;       /* [nv] in, required: rho > 0 */
  const double* lambda0;       /* [n, nv] nullable (0): warm start of the dual */
  double* act;                 /* [n, nu] out, required: the optimal activations a */
  double* reserve_force;       /* [n, nv] nullable: r = rho^2 lambda */
  double* ctrl;                /* [n, nu] nullable: excitation reaching a in one mj_step */
  double* actuator_force;      /* [n, nu] nullable: g a + b */
  double* muscle_gain;         /* [n, nu] nullable: g */
  double* muscle_bias;         /* [n, nu] nullable: b */
  double* qfrc_inverse;        /* [n, nv] nullable: tau */
  double* lambda;              /* [n, nv] nullable: the dual solution */
  int32_t* niter;              /* [n] nullable: Newton steps taken */
  int32_t* converged;          /* [n] nullable */
  double* residual;            /* [n] nullable: |F|_inf at the returned lambda */
} myo_static_opt_buffers;
typedef struct { int32_t max_iter; double tol; } myo_static_opt_params;

/* Caller-owned device buffers of myo_batch_cmc: computed muscle control (OpenSim's CMC, MyoSuite tutorial 9) of every env along its own
 * reference motion, T = nstep frames.  From the start state s_0 (qpos0 ... time0, or the bound buffer of the same name, as
 * myo_rollout_buffers takes it) each frame t = 0 .. T-1 runs
 *   1. qacc_des_t = ref_qacc[t] + kv (ref_qvel[t] - qvel_t) + kp dq,  dq = mj_differentiatePos(qpos_t, ref_qpos[t]) (dt = 1: the tangent
 *      space, so free and ball joints are handled), products elementwise over the dofs;
 *   2. myo_batch_static_opt's problem at s_t for qacc_des_t with the call's flags, weight, reserve, max_iter and tol, warm-started from
 *      lambda_{t-1} (lambda_{-1} = lambda0, or 0): a*_t, r_t = reserve_force, lambda_t;
 *   3. the excitation u_t that, held for `substeps` mj_steps of the muscle activation dynamics from act_t, brings act to a*_t at the end of
 *      the interval, clipped to ctrlrange intersected with [0, 1] (myo_static_opt_buffers.ctrl at substeps = 1; bisection over the k-step
 *      map otherwise, on the monotonicity in ctrl that the one-step bisection assumes);
 *   4. one myo_batch_rollout interval of `substeps` mj_steps from s_t with ctrl u_t and qfrc_applied r_t, which gives s_{t+1}.
 * Steps 2 and 4 are myo_batch_static_opt and myo_batch_rollout themselves: row t of the outputs is bit-identical to those calls run from
 * row t-1's state (s_0 for t = 0).  Row t holds the frame's solve and the state after its interval (myo_rollout_buffers' meaning).
 * Every output is nullable; only the non-null ones are written. */
typedef struct {
  const double* ref_qpos;      /* [n, nstep, nq] in, required: reference positions */
  const double* ref_qvel;      /* [n, nstep, nv] in, required */
  const double* ref_qacc;      /* [n, nstep, nv] in, required */
  const double* kp;            /* [nv] in, required: position gains (>= 0; not checked on the device) */
  const double* kv;            /* [nv] in, required: velocity gains (>= 0) */
  const double* weight;        /* [nu] nullable (1): w > 0, as myo_static_opt_buffers.weight */
  const double* reserve;       /* [nv] in, required: rho > 0 */
  const double* lambda0;       /* [n, nv] nullable (0): warm start of frame 0's dual */
  const double* qpos0;         /* [n, nq] start state, nullable field by field (bound buffers), as myo_rollout_buffers */
  const double* qvel0;         /* [n, nv] */
  const double* act0;          /* [n, na] */
  const double* qacc_warmstart0; /* [n, nv] */
  const double* time0;         /* [n] */
  double* qacc_des;            /* [n, nstep, nv] out */
  double* ctrl;                /* [n, nstep, nu] out: u_t */
  double* act_opt;             /* [n, nstep, nu] out: a*_t */
  double* reserve_force;       /* [n, nstep, nv] out: r_t */
  double* lambda;              /* [n, nstep, nv] out: lambda_t */
  int32_t* niter;              /* [n, nstep] out */
  int32_t* converged;          /* [n, nstep] out */
  double* residual;            /* [n, nstep] out */
  double* qpos;                /* [n, nstep, nq] out: s_{t+1} */
  double* qvel;                /* [n, nstep, nv] out */
  double* act;                 /* [n, nstep, na] out */
  double* qacc;                /* [n, nstep, nv] out: mjData.qacc, the next interval's warm start */
  double* time;                /* [n, nstep] out */
  int32_t* overflow;           /* [n] out: myo_rollout_buffers.overflow's meaning over every interval */
} myo_cmc_buffers;
typedef struct { int32_t max_iter, substeps; double tol; } myo_cmc_params;

/* Caller-owned device buffers of myo_batch_inverse_fd: MuJoCo's mjd_inverseFD, finite-difference Jacobians of the inverse dynamics.  For
 * each env, at the start state (qpos, qvel, act) and the caller's qacc, let
 *   f(q, v, a) = qfrc_inverse(q, v, a)                     (actuation = 0)
 *   f(q, v, a) = qfrc_inverse(q, v, a) - qfrc_actuator(q, v, act)   (actuation = 1: flg_actuation, the residual the muscles do not supply,
 *                                                            myo_static_opt_buffers' t before the muscle bias is taken out)
 *   qfrc_inverse is myo_batch_inverse's, with the same MYO_INV_* flags and the per-env overrides (env_prm); qfrc_actuator is the readout's
 *   (myo_data_buffers.qfrc_actuator).  Every actuator on this path is a muscle, whose force reads act, not ctrl: ctrl is not an input.
 *   Differences are forward only, as in MuJoCo: row i of a block is (f(x + eps e_i) - f(x)) * (1 / eps), with 1 / eps the IEEE-rounded
 *   reciprocal (myo_fd_params' rule).  The qpos perturbation is mj_integratePos(qpos, e_i, eps) (free joints included); the qvel and qacc
 *   perturbations add eps to entry i.  Every pass, nominal and perturbed, starts from the start state with cold inverse-wrap roots.
 *   Layout is MuJoCo's, DfDq[env][i][j] = d f_j / d q_i (the same for DfDv and DfDa): transposed with respect to the control-theory
 *   convention and to myo_fd_buffers.A, whose A[i][j] = d x'_i / d x_j.  MuJoCo's API reference for mjd_inverseFD: "Finite differenced
 *   Jacobians of (force, sensors) = mj_inverse(state, acceleration) ... Output dimensions (transposed w.r.t Control Theory convention):
 *   DfDq: (nv x nv), DfDv: (nv x nv), DfDa: (nv x nv) ... flg_actuation specifies whether to subtract qfrc_actuator from qfrc_inverse".
 *   Precision: the inside-wrap root solve (wrap2d_inside) starts cold in every pass and stops on a tolerance, |residual| <= 1e-6 on the
 *   angle equation (at most 20 Newton steps from z = 1 - 1e-7), not at machine precision.  Where a perturbation changes the step at which
 *   it stops, the root moves by up to that tolerance over the equation's slope, so DfDq rows of dofs that move a tendon with an inside
 *   wrap carry noise of order that tolerance / eps, as MuJoCo's FD does.  The contact and the active constraint rows are those of each
 *   pass's own state: a perturbation that changes them gives that column a jump, as in MuJoCo.  The product build stores the contact
 *   Jacobian rows with 36 mantissa bits (p48), so with constraints the columns of a state with active contacts carry that rounding, of
 *   order 2^-36 |J' efc_force| / eps (measured: up to 3e-6 x the env's largest force term per unit of q, on the hold task at eps = 1e-4);
 *   the f64-rows build (MYO_F64_ROWS) does not.
 *   Not provided: the sensor blocks DsDq, DsDv, DsDa (there are no device sensors), DmDq, centred differences, xfrc_applied and analytic
 *   derivatives. */
typedef struct {
  const double* qacc;            /* [n, nv] in, required */
  const double* qpos0;           /* [n, nq] start state, nullable field by field (bound buffers), as myo_fd_buffers */
  const double* qvel0;           /* [n, nv] */
  const double* act0;            /* [n, na] */
  double* DfDq;                  /* [n, nv, nv] out, nullable (at least one of DfDq, DfDv, DfDa): DfDq[i][j] = d f_j / d q_i */
  double* DfDv;                  /* [n, nv, nv] out, nullable */
  double* DfDa;                  /* [n, nv, nv] out, nullable */
  double* qfrc_inverse;          /* [n, nv] out, nullable: the nominal f (minus qfrc_actuator with actuation) */
  int32_t* overflow;             /* [n] out, nullable: set when the nominal or any perturbed pass dropped contacts (myo_fd_buffers.overflow) */
} myo_inverse_fd_buffers;
typedef struct { double eps; int32_t actuation; } myo_inverse_fd_params;

const char* myo_last_error(void);
int myo_version(void);       /* 2: myo_buffers ends with final_obs.  Version 1 ended with overflow: a caller built against that header passes a
                                smaller struct, so callers check that this matches the version of the header they were compiled against */

/* Model from the packed blob produced by myosuite_b200.blob.pack (host arrays; copied).
 * Replaces: MjSpec.from_file(path).compile() + the model upload.  */
int myo_model_from_blob(const int32_t* I, int64_t nI, const double* D, int64_t nD, myo_model** out);
int myo_model_dims(const myo_model* m, const myo_task_cfg* cfg_or_null, myo_dims* out);
void myo_model_destroy(myo_model* m);

/* Shared-memory layout of one env's slice, as the step kernels of a batch created with this model and cfg use it (host only: needs no
 * device).  Writes the first min(cap, MYO_LAYOUT_N) of these int32 values; offsets and sizes are in doubles, offsets from the start of
 * the slice:
 *   [0, 12)   persistent offsets, in MYO_LAYOUT_PERSISTENT order (scr: start of the stage scratch; qws lies inside the scratch, in the
 *             tail of the Hessian region, when the qwsInH flag below is set)
 *   [12, 24)  their reserved sizes, same order (scr: size of the scratch)
 *   [24, 54)  scratch offsets, in MYO_LAYOUT_SCRATCH order
 *   [54, 84)  their reserved sizes, same order (aliases share storage: con / efR / efV, vg / vp, H / Hs, and efA / H when arefInH)
 *   84 head: end of the contact head (icon records, then contact records)     85 afterK: end of the body poses xpos / xmat behind it
 *   86 extNonSolve: end of the scratch the stages before the constraints use  87 end of the solve stage's regions (the Hessian region)
 *   88 arefInH: aref lives at the head of the Hessian region                  89 qwsInH: the warm start lives in its tail
 *   90 n_per_warp (doubles per env slice)    91 maxcon (cfg's, or 32 when 0, clamped to min(64, 2 npair))    92 maxefc */
#define MYO_LAYOUT_N 93
#define MYO_LAYOUT_PERSISTENT(X) X(qpos) X(qvel) X(act) X(qws) X(dax) X(dan) X(qM) X(fsm) X(eprm) X(wz) X(cnt) X(scr)
#define MYO_LAYOUT_SCRATCH(X) X(xpos) X(xmat) X(U) X(PL) X(mom) X(tlen) X(tvel) X(tfrc) X(cin) X(crb) X(bf) X(conJ) X(efD) X(efA) X(eqJ) \
  X(icon) X(con) X(clist) X(gpose) X(efR) X(efV) X(va) X(vg) X(vp) X(vMa) X(vMp) X(H) X(Hs) X(LD) X(Dinv)
int myo_model_layout(const myo_model* m, const myo_task_cfg* cfg_or_null, int32_t* out, int cap);

/* Batch of n_env envs of one model on one device. */
int myo_batch_create(const myo_model* m, int device, int n_env, const myo_task_cfg* cfg, myo_batch** out);
int myo_batch_bind(myo_batch* b, const myo_buffers* bufs);
void myo_batch_destroy(myo_batch* b);
int myo_batch_obs_dim(const myo_batch* b);

/* Reset envs whose mask byte is non-zero (mask == NULL: all).  Per-env Philox streams keyed
 * (seed, env_offset + env, episode_count).  Replaces env.reset() (pose_v0.py:174-257, robot.py:996-1002).
 * Each lane of an env's warp draws from its own Philox4x32-10 stream: key (k0, k1) = (seed lo, seed hi), counter
 *   c0 = draw block    c1 = lane | (u32)(env >> 20) << 5    c2 = (u32)env ^ (u32)(episode << 20)    c3 = (u32)(env >> 32) ^ (u32)(episode >> 12) ^ 0x4D594F42
 * with env the global index env_offset + i.  Distinct (seed, env, episode, lane) get distinct streams for env < 2^47 and episode < 2^44;
 * below 2^20 envs, c1 is the lane alone.  The call fails when env_offset < 0 or env_offset + n_env > MYO_RESET_ENV_LIMIT. */
#define MYO_RESET_ENV_LIMIT (1LL << 47)
int myo_batch_reset(myo_batch* b, const uint8_t* mask_dev_or_null, uint64_t seed, int64_t env_offset, void* stream);

/* One control step for every env: action->ctrl, [fatigue], frame_skip x (forward + Euler), obs,
 * reward, done, TimeLimit, optional auto-reset.  Asynchronous on `stream`.
 * Replaces BaseV0.step (base_v0.py:82-118) for the whole batch. */
int myo_batch_step(myo_batch* b, void* stream);

/* obs / reward / done of the CURRENT state without advancing it.
 * Replaces env.forward() (envs/env_base.py:393-432). */
int myo_batch_observe(myo_batch* b, void* stream);

/* Parity tap: ONE forward pass (mj_forward) on the bound qpos/qvel/act with ctrl := action taken
 * verbatim (no sigmoid), writing the tap_* buffers; state is not advanced.  If n_substeps > 0 the
 * state IS advanced by that many mj_step's with the same ctrl (taps hold the last forward). */
int myo_batch_forward_debug(myo_batch* b, const double* ctrl_dev /* [n, nu] */, int n_substeps, void* stream);

/* Readout of mjData for every env (the fields of myo_data_buffers that are non-null), one launch on `stream`; the state is not
 * advanced and no bound buffer is written.  The deepest requested group decides how much of the forward pass runs: the pose group
 * alone needs kinematics, the actuation group adds tendons and muscles, the dynamics group adds collision and the constraint solve.
 * Replaces reading env.unwrapped.mj_data after reset() / step() (envs/env_base.py:77-92, robot/robot.py:595-607). */
int myo_batch_data(myo_batch* b, const myo_data_buffers* d, void* stream);

/* Inverse dynamics of every env (myo_inverse_buffers), one launch on `stream`; flags: MYO_INV_* (0 = MuJoCo's defaults).  The state is
 * not advanced and no bound buffer is written.  Fails on a null batch, buffers, qacc or qfrc_inverse, an unbound batch or unknown flag bits.
 * Replaces mujoco.mj_inverse (MyoSuite tutorials 6_Inverse_Dynamics and 9_Computed_muscle_control). */
int myo_batch_inverse(myo_batch* b, const myo_inverse_buffers* d, int flags, void* stream);

/* Rollout of every env (myo_rollout_buffers): nstep intervals of `substeps` mj_steps each, from the given or the bound start state, with
 * the caller's ctrl and applied forces; one launch per interval on `stream`.  The per-env overrides (env_prm) apply; fatigue, the task
 * layer (obs, reward, done, counters) and auto-reset do not run.  No bound buffer is written, and results of later env steps and
 * readouts do not change (the load-sorted grouping of the next env step may).  Fails on a null batch, buffers or ctrl, an unbound
 * batch, nstep < 1 or substeps < 1.  Replaces mj_step loops over data.ctrl / data.qfrc_applied (MyoSuite tutorials
 * 6_Inverse_Dynamics and 9_Computed_muscle_control; sampling-based control, system identification, trajectory replay). */
int myo_batch_rollout(myo_batch* b, const myo_rollout_buffers* r, int nstep, int substeps, void* stream);

/* Inverse kinematics of every env (myo_ik_buffers, myo_ik_params), one launch on `stream`; each env iterates until its own stop test.
 * No bound buffer is written: adopting a solution is a separate state change.  Fails before any launch on a null batch, buffers,
 * site_id, site_quat, target_pos or qpos, an unbound batch, nsite outside [1, MYO_IK_MAXSITE], a site id outside [0, nsite), damping <= 0,
 * max_step <= 0, tol < 0, max_iter < 0 or a non-finite parameter.  Replaces mj_jacSite and the mink / dm_control IK loops over it
 * (MyoSuite tutorial 8_inverse_kinematics, marker and fingertip retargeting). */
int myo_batch_ik(myo_batch* b, const myo_ik_buffers* d, const myo_ik_params* p, void* stream);

/* Finite-difference transition Jacobians of every env (myo_fd_buffers, myo_fd_params): a nominal rollout interval, then one launch that
 * runs every (env, column) pair as its own warp, both on `stream`.  The per-env overrides (env_prm) apply; fatigue, the task layer and
 * auto-reset do not run.  No bound buffer is written: the call advances nothing.  With the iterative solver the columns carry solver noise
 * of order solver tolerance / eps, as in MuJoCo.  Fails before any launch on a null batch, buffers, params or ctrl, A and B both null, an
 * unbound batch, eps not finite or not > 0, substeps < 1 or centered not in {0, 1}.  Replaces mujoco.mjd_transitionFD (iLQR / DDP, LQR
 * about a reference pose, MPC warm starts, controllability and sensitivity studies). */
int myo_batch_transition_fd(myo_batch* b, const myo_fd_buffers* d, const myo_fd_params* p, void* stream);

/* Muscle static optimisation of every env (myo_static_opt_buffers, myo_static_opt_params), one launch on `stream`; flags: MYO_INV_* as
 * myo_batch_inverse's; each env iterates until its own stop test.  No bound buffer is written.  Fails before any launch on a null batch,
 * buffers, params, qacc, reserve or act, an unbound batch, unknown flag bits, tol < 0, max_iter < 0, a non-finite tol, a model with more
 * than 64 dofs, or a per-env slice without room for the iteration's arrays (the legs at maxcon 4); the device does not check the values of
 * weight and reserve.  Replaces the per-frame SLSQP / OSQP solves of MyoSuite
 * tutorials 6_Inverse_Dynamics (get_ctrl) and 9_Computed_muscle_control. */
int myo_batch_static_opt(myo_batch* b, const myo_static_opt_buffers* d, const myo_static_opt_params* p, int flags, void* stream);

/* Computed muscle control of every env over nstep frames (myo_cmc_buffers, myo_cmc_params), all on `stream` with no host synchronisation;
 * flags: MYO_INV_* as myo_batch_static_opt's.  Launches per call: nstep (3 + (substeps > 1) + R) + 1, where R = 1 when the batch's
 * rollouts run on the load-sorted map (a regroup launch before each interval) and 0 otherwise: per frame the qacc_des stage (which also
 * stores the previous frame's row), myo_static_opt_kernel, the k-step excitation when substeps > 1, and the rollout interval; then one
 * stage launch that stores the last row.  No bound buffer is written and the env's episode is left alone, as with myo_batch_rollout.  The
 * per-frame scratch is allocated by the first call.  Fails before any launch on a null batch, buffers or params, a null ref_qpos,
 * ref_qvel, ref_qacc, kp, kv or reserve, an unbound batch, unknown flag bits, nstep < 1, substeps < 1, tol < 0, max_iter < 0, a
 * non-finite tol, a model with more than 64 dofs, or a per-env slice without room for the dual Newton's arrays.  Replaces the per-frame
 * loop of MyoSuite tutorials 6_Inverse_Dynamics and 9_Computed_muscle_control. */
int myo_batch_cmc(myo_batch* b, const myo_cmc_buffers* d, const myo_cmc_params* p, int nstep, int flags, void* stream);

/* Finite-difference Jacobians of the inverse dynamics of every env (myo_inverse_fd_buffers, myo_inverse_fd_params); flags: MYO_INV_* as
 * myo_batch_inverse's.  Two launches on `stream`: the nominal f of every env, then one warp per (env, column) of the requested blocks.
 * No bound buffer is written and nothing is advanced; the nominal rows are allocated by the first call.  Fails before any launch on a null
 * batch, buffers, params or qacc, DfDq, DfDv and DfDa all null, an unbound batch, unknown flag bits, eps not finite or not > 0, actuation
 * not in {0, 1}, or n_env x columns beyond int32.  Replaces mujoco.mjd_inverseFD (inverse-dynamics trajectory optimisation: muscle-driven
 * direct collocation, MJPC's direct optimiser and batch estimator, static optimisation along a motion, system identification). */
int myo_batch_inverse_fd(myo_batch* b, const myo_inverse_fd_buffers* d, const myo_inverse_fd_params* p, int flags, void* stream);

/* number of kernel launches issued by this batch so far (bench.py's gpu_launches claim) */
int64_t myo_batch_launch_count(const myo_batch* b);

/* Read-only queries of how env steps are launched (for tests of the product kernels at their real launch shapes).
 * launch_info writes the first min(n, 9) of: use_w14 (1: the launch_bounds(448) kernel, 0: launch_bounds(320)), warps_per_cta,
 * grid, rounds of warps each CTA walks, regroup (1: load-sorted slot -> env map), balanced (1: env e on CTA e % grid when not
 * regrouped, 0: contiguous groups of warps), smem_bytes, perm_slots (entries of the slot -> env map, 0 without regroup), hand_shape
 * (1: the env steps run myo_env_kernel_w14_hand, the launch_bounds(352) kernel compiled for the hand's shape, in place of the launch_bounds(448) one;
 * smem_bytes then includes its cold-table region).
 * debug_perm copies the slot -> env map of the last env step to HOST memory (n >= perm_slots entries; slot
 * cta + grid*(round*warps_per_cta + warp), -1 = idle slot); it synchronises the device and fails when regroup is off or no step has run. */
int myo_batch_launch_info(const myo_batch* b, int32_t* out, int n);
int myo_batch_debug_perm(const myo_batch* b, int32_t* host_out, int n);

/* Unit-test hook for the dense solver the Newton and integrator phases use: solves H x = b for `count` independent SPD systems
 * (H_host: count x n(n+1)/2 packed lower triangles, row-major; x_host: count x n, rhs in / solution out; HOST pointers), one
 * warp per system (row-in-registers / column-through-shared-memory L D L' for n <= 32, bordered register Cholesky for 32 < n <= 36, shared-memory
 * fallback above).  `mode` is ignored (kept for ABI stability).  n <= 64. */
int myo_debug_chol_solve(int device, const double* H_host, double* x_host, int n, int count, int mode);

#ifdef __cplusplus
}
#endif
#endif

/* myo_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A scalar, f64, single-env restatement of what the reference's hot path computes per physics
 * substep: `mujoco.mj_step(model, data)` as called from
 *   myosuite/robot/robot.py:856-861 (Robot._advance)  and the
 * `mujoco.mj_forward` of myosuite/robot/robot.py:607 (Robot.sensor2sim).
 *
 * MuJoCo (pinned mujoco 3.5.0, uv.lock:1739-1740) is a third-party dependency that
 * is not part of the reference checkout nor of this project.  The algorithm below restates MuJoCo's
 * published pipeline (MuJoCo documentation, "Computation" chapter; SURVEY.md Appendix A) stage by
 * stage, in MuJoCo's own formulation (subtree-COM-centred spatial algebra, mj_crb/mj_rne/mj_tendon/
 * mju_wrap/mj_makeConstraint/Newton), deliberately different from the restructured formulation
 * used by the CUDA kernels so that agreement between the two is meaningful.
 *
 * PARITY UNPINNED for the physics: the reference holds no golden numeric vectors for this path
 * (SURVEY.md section 8c) and MuJoCo cannot be run here.  Only the Python-side logic (fatigue,
 * sigmoid remap, obs/reward) is pinned against outputs of the reference's own code
 * (tests/golden/, oracle/env_oracle.py).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline/reference legs may use this file.
 */
#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>

#include "../include/myo_blob_layout.h"

#define MINVAL 1e-15
#define MINIMP 0.0001
#define MAXIMP 0.9999
#define JNT_FREE 0
#define JNT_SLIDE 2
#define JNT_HINGE 3
#define GEOM_PLANE 0
#define GEOM_SPHERE 2
#define GEOM_CAPSULE 3
#define GEOM_ELLIPSOID 4
#define WRAP_SITE 3
#define WRAP_SPHERE 4
#define WRAP_CYLINDER 5

typedef struct {
  const int* I; const double* D;
  int nq, nv, nu, na, nbody, njnt, ngeom, nsite, ntendon, nwrap, nM, npair, neq;
  int maxcon, maxefc;
  /* state */
  double *qpos, *qvel, *act, *ctrl, *qacc_warmstart, time;
  /* position stage */
  double *xpos, *xquat, *xmat, *xipos, *ximat, *xanchor, *xaxis, *geom_xpos, *geom_xmat, *site_xpos;
  double *subtree_com, *cinert, *cdof, *crb;
  double *ten_length, *ten_J, *wrap_xpos; int *wrap_obj;
  double *qM, *qLD, *qLDiagInv;
  /* contacts */
  int ncon; int *con_geom1, *con_geom2, *con_pair; double *con_dist, *con_pos, *con_frame;
  /* constraints */
  int nefc, ne, nl; double *efc_J, *efc_pos, *efc_margin, *efc_diagApprox, *efc_R, *efc_D, *efc_KBIP, *efc_vel,
      *efc_aref, *efc_force; int *efc_type;
  /* velocity / actuation / acceleration */
  double *ten_velocity, *actuator_length, *actuator_velocity, *actuator_force, *act_dot, *cvel, *cdof_dot, *cacc, *cfrc;
  double *qfrc_bias, *qfrc_passive, *qfrc_actuator, *qfrc_smooth, *qacc_smooth, *qfrc_constraint, *qacc;
  int solver_niter;
  /* op counter (flops, coarse) */
  double flops;
} ora;

/* ---------------------------------------------------------------- small math */
static void cross3(double* r, const double* a, const double* b) {
  double x = a[1]*b[2]-a[2]*b[1], y = a[2]*b[0]-a[0]*b[2], z = a[0]*b[1]-a[1]*b[0]; r[0]=x; r[1]=y; r[2]=z; }
static double dot3(const double* a, const double* b) { return a[0]*b[0]+a[1]*b[1]+a[2]*b[2]; }
static double norm3(const double* a) { return sqrt(dot3(a,a)); }
static double normalize3(double* a) { double n = norm3(a); if (n < MINVAL) { a[0]=1; a[1]=0; a[2]=0; } else { a[0]/=n; a[1]/=n; a[2]/=n; } return n; }
static void quat_mul(double* r, const double* a, const double* b) {
  double w=a[0]*b[0]-a[1]*b[1]-a[2]*b[2]-a[3]*b[3], x=a[0]*b[1]+a[1]*b[0]+a[2]*b[3]-a[3]*b[2],
         y=a[0]*b[2]-a[1]*b[3]+a[2]*b[0]+a[3]*b[1], z=a[0]*b[3]+a[1]*b[2]-a[2]*b[1]+a[3]*b[0];
  r[0]=w; r[1]=x; r[2]=y; r[3]=z; }
static void quat_norm(double* q) { double n=sqrt(q[0]*q[0]+q[1]*q[1]+q[2]*q[2]+q[3]*q[3]); if (n<MINVAL){q[0]=1;q[1]=q[2]=q[3]=0;} else {q[0]/=n;q[1]/=n;q[2]/=n;q[3]/=n;} }
static void quat2mat(double* m, const double* q) {
  double w=q[0],x=q[1],y=q[2],z=q[3];
  m[0]=w*w+x*x-y*y-z*z; m[1]=2*(x*y-w*z); m[2]=2*(x*z+w*y);
  m[3]=2*(x*y+w*z); m[4]=w*w-x*x+y*y-z*z; m[5]=2*(y*z-w*x);
  m[6]=2*(x*z-w*y); m[7]=2*(y*z+w*x); m[8]=w*w-x*x-y*y+z*z; }
static void mat_vec(double* r, const double* m, const double* v) {
  double x=m[0]*v[0]+m[1]*v[1]+m[2]*v[2], y=m[3]*v[0]+m[4]*v[1]+m[5]*v[2], z=m[6]*v[0]+m[7]*v[1]+m[8]*v[2]; r[0]=x;r[1]=y;r[2]=z; }
static void matT_vec(double* r, const double* m, const double* v) {
  double x=m[0]*v[0]+m[3]*v[1]+m[6]*v[2], y=m[1]*v[0]+m[4]*v[1]+m[7]*v[2], z=m[2]*v[0]+m[5]*v[1]+m[8]*v[2]; r[0]=x;r[1]=y;r[2]=z; }
static void axisangle_quat(double* q, const double* axis, double ang) {
  double s = sin(0.5*ang); q[0]=cos(0.5*ang); q[1]=axis[0]*s; q[2]=axis[1]*s; q[3]=axis[2]*s; }
static double clip(double x, double lo, double hi) { return x < lo ? lo : (x > hi ? hi : x); }

#define ISEC(o, name) MYO_ISEC((o)->I, MYO_SEC_##name)
#define DSEC(o, name) MYO_DSEC((o)->I, (o)->D, MYO_SEC_##name)

/* ---------------------------------------------------------------- create / reset */
static double* dalloc(size_t n) { return (double*)calloc(n ? n : 1, sizeof(double)); }
static int* ialloc(size_t n) { return (int*)calloc(n ? n : 1, sizeof(int)); }

ora* oracle_create(const int* I, const double* D) {
  if (I[0] != MYO_BLOB_MAGIC || I[1] != MYO_BLOB_VERSION) return NULL;
  ora* o = (ora*)calloc(1, sizeof(ora));
  o->I = I; o->D = D;
  o->nq=MYO_DIM(I,MYO_DIM_nq); o->nv=MYO_DIM(I,MYO_DIM_nv); o->nu=MYO_DIM(I,MYO_DIM_nu); o->na=MYO_DIM(I,MYO_DIM_na);
  o->nbody=MYO_DIM(I,MYO_DIM_nbody); o->njnt=MYO_DIM(I,MYO_DIM_njnt); o->ngeom=MYO_DIM(I,MYO_DIM_ngeom);
  o->nsite=MYO_DIM(I,MYO_DIM_nsite); o->ntendon=MYO_DIM(I,MYO_DIM_ntendon); o->nwrap=MYO_DIM(I,MYO_DIM_nwrap);
  o->nM=MYO_DIM(I,MYO_DIM_nM); o->npair=MYO_DIM(I,MYO_DIM_npair); o->neq=MYO_DIM(I,MYO_DIM_neq);
  int nv=o->nv, nb=o->nbody;
  o->maxcon = 2*o->npair + 1; o->maxefc = o->neq + 2*o->njnt + 4*o->maxcon + 1;
  o->qpos=dalloc(o->nq); o->qvel=dalloc(nv); o->act=dalloc(o->na); o->ctrl=dalloc(o->nu); o->qacc_warmstart=dalloc(nv);
  o->xpos=dalloc(3*nb); o->xquat=dalloc(4*nb); o->xmat=dalloc(9*nb); o->xipos=dalloc(3*nb); o->ximat=dalloc(9*nb);
  o->xanchor=dalloc(3*o->njnt); o->xaxis=dalloc(3*o->njnt); o->geom_xpos=dalloc(3*o->ngeom); o->geom_xmat=dalloc(9*o->ngeom);
  o->site_xpos=dalloc(3*o->nsite); o->subtree_com=dalloc(3*nb); o->cinert=dalloc(10*nb); o->cdof=dalloc(6*nv); o->crb=dalloc(10*nb);
  o->ten_length=dalloc(o->ntendon); o->ten_J=dalloc((size_t)o->ntendon*nv); o->wrap_xpos=dalloc(6*o->nwrap); o->wrap_obj=ialloc(2*o->nwrap);
  o->qM=dalloc(o->nM); o->qLD=dalloc(o->nM); o->qLDiagInv=dalloc(nv);
  o->con_geom1=ialloc(o->maxcon); o->con_geom2=ialloc(o->maxcon); o->con_pair=ialloc(o->maxcon);
  o->con_dist=dalloc(o->maxcon); o->con_pos=dalloc(3*o->maxcon); o->con_frame=dalloc(9*o->maxcon);
  o->efc_J=dalloc((size_t)o->maxefc*nv); o->efc_pos=dalloc(o->maxefc); o->efc_margin=dalloc(o->maxefc);
  o->efc_diagApprox=dalloc(o->maxefc); o->efc_R=dalloc(o->maxefc); o->efc_D=dalloc(o->maxefc); o->efc_KBIP=dalloc(4*o->maxefc);
  o->efc_vel=dalloc(o->maxefc); o->efc_aref=dalloc(o->maxefc); o->efc_force=dalloc(o->maxefc); o->efc_type=ialloc(o->maxefc);
  o->ten_velocity=dalloc(o->ntendon); o->actuator_length=dalloc(o->nu); o->actuator_velocity=dalloc(o->nu);
  o->actuator_force=dalloc(o->nu); o->act_dot=dalloc(o->na); o->cvel=dalloc(6*nb); o->cdof_dot=dalloc(6*nv); o->cacc=dalloc(6*nb); o->cfrc=dalloc(6*nb);
  o->qfrc_bias=dalloc(nv); o->qfrc_passive=dalloc(nv); o->qfrc_actuator=dalloc(nv); o->qfrc_smooth=dalloc(nv);
  o->qacc_smooth=dalloc(nv); o->qfrc_constraint=dalloc(nv); o->qacc=dalloc(nv);
  memcpy(o->qpos, DSEC(o, qpos0), sizeof(double)*o->nq);
  return o;
}

void oracle_destroy(ora* o) { /* test-lifetime object: leak-free enough */
  if (!o) return;
  double** p[] = {&o->qpos,&o->qvel,&o->act,&o->ctrl,&o->qacc_warmstart,&o->xpos,&o->xquat,&o->xmat,&o->xipos,&o->ximat,&o->xanchor,
    &o->xaxis,&o->geom_xpos,&o->geom_xmat,&o->site_xpos,&o->subtree_com,&o->cinert,&o->cdof,&o->crb,&o->ten_length,&o->ten_J,&o->wrap_xpos,
    &o->qM,&o->qLD,&o->qLDiagInv,&o->con_dist,&o->con_pos,&o->con_frame,&o->efc_J,&o->efc_pos,&o->efc_margin,&o->efc_diagApprox,&o->efc_R,
    &o->efc_D,&o->efc_KBIP,&o->efc_vel,&o->efc_aref,&o->efc_force,&o->ten_velocity,&o->actuator_length,&o->actuator_velocity,&o->actuator_force,
    &o->act_dot,&o->cvel,&o->cdof_dot,&o->cacc,&o->cfrc,&o->qfrc_bias,&o->qfrc_passive,&o->qfrc_actuator,&o->qfrc_smooth,&o->qacc_smooth,
    &o->qfrc_constraint,&o->qacc};
  for (size_t i = 0; i < sizeof(p)/sizeof(p[0]); i++) free(*p[i]);
  free(o->wrap_obj); free(o->con_geom1); free(o->con_geom2); free(o->con_pair); free(o->efc_type); free(o);
}

/* mj_resetData semantics: qpos=qpos0, everything else zero (robot.py:999) */
void oracle_reset(ora* o) {
  memcpy(o->qpos, DSEC(o, qpos0), sizeof(double)*o->nq);
  memset(o->qvel, 0, sizeof(double)*o->nv); memset(o->act, 0, sizeof(double)*o->na); memset(o->ctrl, 0, sizeof(double)*o->nu);
  memset(o->qacc_warmstart, 0, sizeof(double)*o->nv); memset(o->qacc, 0, sizeof(double)*o->nv); o->time = 0;
}

/* ---------------------------------------------------------------- A.1 kinematics + comPos */
static void kinematics(ora* o) {
  const int *parent=ISEC(o,body_parentid), *jadr=ISEC(o,body_jntadr), *jnum=ISEC(o,body_jntnum), *jtype=ISEC(o,jnt_type), *jq=ISEC(o,jnt_qposadr);
  const double *bpos=DSEC(o,body_pos), *bquat=DSEC(o,body_quat), *jpos=DSEC(o,jnt_pos), *jaxis=DSEC(o,jnt_axis), *qpos0=DSEC(o,qpos0);
  const double *bipos=DSEC(o,body_ipos), *biquat=DSEC(o,body_iquat);
  o->xquat[0]=1; quat2mat(o->xmat, o->xquat); quat2mat(o->ximat, o->xquat);
  for (int b=1; b<o->nbody; b++) {
    int p=parent[b]; double pos[3], quat[4], v[3];
    if (jnum[b]==1 && jtype[jadr[b]]==JNT_FREE) {
      int a=jq[jadr[b]]; double* qp=o->qpos+a;
      memcpy(pos, qp, 24); memcpy(quat, qp+3, 32); quat_norm(quat);   /* normalised copy: mj_kinematics (MuJoCo >= 2.3) leaves qpos untouched */
      memcpy(o->xanchor+3*jadr[b], pos, 24); o->xaxis[3*jadr[b]]=0; o->xaxis[3*jadr[b]+1]=0; o->xaxis[3*jadr[b]+2]=1;
    } else {
      mat_vec(v, o->xmat+9*p, bpos+3*b); for (int k=0;k<3;k++) pos[k]=o->xpos[3*p+k]+v[k];
      quat_mul(quat, o->xquat+4*p, bquat+4*b);
      for (int j=jadr[b]; j<jadr[b]+jnum[b]; j++) {
        double m[9]; quat2mat(m, quat);
        double* anc=o->xanchor+3*j; double* ax=o->xaxis+3*j;
        mat_vec(ax, m, jaxis+3*j); mat_vec(v, m, jpos+3*j); for (int k=0;k<3;k++) anc[k]=pos[k]+v[k];
        double dq = o->qpos[jq[j]] - qpos0[jq[j]];
        if (jtype[j]==JNT_SLIDE) { for (int k=0;k<3;k++) pos[k]+=ax[k]*dq; }
        else if (jtype[j]==JNT_HINGE) {
          double ql[4], qn[4]; axisangle_quat(ql, jaxis+3*j, dq); quat_mul(qn, quat, ql); memcpy(quat, qn, 32);
          quat2mat(m, quat); mat_vec(v, m, jpos+3*j); for (int k=0;k<3;k++) pos[k]=anc[k]-v[k];
        }
      }
    }
    quat_norm(quat);
    memcpy(o->xpos+3*b, pos, 24); memcpy(o->xquat+4*b, quat, 32); quat2mat(o->xmat+9*b, quat);
    mat_vec(v, o->xmat+9*b, bipos+3*b); for (int k=0;k<3;k++) o->xipos[3*b+k]=pos[k]+v[k];
    double qi[4]; quat_mul(qi, quat, biquat+4*b); quat_norm(qi); quat2mat(o->ximat+9*b, qi);
  }
  const int* gb=ISEC(o,geom_bodyid); const double *gp=DSEC(o,geom_pos), *gq=DSEC(o,geom_quat);
  for (int g=0; g<o->ngeom; g++) { int b=gb[g]; double v[3], q[4];
    mat_vec(v, o->xmat+9*b, gp+3*g); for (int k=0;k<3;k++) o->geom_xpos[3*g+k]=o->xpos[3*b+k]+v[k];
    quat_mul(q, o->xquat+4*b, gq+4*g); quat_norm(q); quat2mat(o->geom_xmat+9*g, q); }
  const int* sb=ISEC(o,site_bodyid); const double* sp=DSEC(o,site_pos);
  for (int s=0; s<o->nsite; s++) { int b=sb[s]; double v[3];
    mat_vec(v, o->xmat+9*b, sp+3*s); for (int k=0;k<3;k++) o->site_xpos[3*s+k]=o->xpos[3*b+k]+v[k]; }
}

/* cinert[10] = (Ixx,Iyy,Izz,Ixy,Ixz,Iyz, m*dx,m*dy,m*dz, m) about the point `com - dif` (mju_inertCom) */
static void inert_com(double* r, const double* inert, const double* mat, const double* dif, double mass) {
  double t[9];
  for (int i=0;i<3;i++) for (int j=0;j<3;j++) t[3*i+j]=mat[3*i]*inert[0]*mat[3*j]+mat[3*i+1]*inert[1]*mat[3*j+1]+mat[3*i+2]*inert[2]*mat[3*j+2];
  r[0]=t[0]+mass*(dif[1]*dif[1]+dif[2]*dif[2]); r[1]=t[4]+mass*(dif[0]*dif[0]+dif[2]*dif[2]); r[2]=t[8]+mass*(dif[0]*dif[0]+dif[1]*dif[1]);
  r[3]=t[1]-mass*dif[0]*dif[1]; r[4]=t[2]-mass*dif[0]*dif[2]; r[5]=t[5]-mass*dif[1]*dif[2];
  r[6]=mass*dif[0]; r[7]=mass*dif[1]; r[8]=mass*dif[2]; r[9]=mass; }
/* f[6] = cinert * v[6]  (mju_mulInertVec); spatial vectors are [angular; linear] */
static void mul_inert_vec(double* r, const double* i, const double* v) {
  r[0]=i[0]*v[0]+i[3]*v[1]+i[4]*v[2]-i[8]*v[4]+i[7]*v[5];
  r[1]=i[3]*v[0]+i[1]*v[1]+i[5]*v[2]+i[8]*v[3]-i[6]*v[5];
  r[2]=i[4]*v[0]+i[5]*v[1]+i[2]*v[2]-i[7]*v[3]+i[6]*v[4];
  r[3]=i[8]*v[1]-i[7]*v[2]+i[9]*v[3]; r[4]=i[6]*v[2]-i[8]*v[0]+i[9]*v[4]; r[5]=i[7]*v[0]-i[6]*v[1]+i[9]*v[5]; }

static void com_pos(ora* o) {
  const int *parent=ISEC(o,body_parentid), *rootid=ISEC(o,body_rootid), *jtype=ISEC(o,jnt_type), *jb=ISEC(o,jnt_bodyid), *jd=ISEC(o,jnt_dofadr);
  const double *mass=DSEC(o,body_mass), *inertia=DSEC(o,body_inertia);
  int nb=o->nbody; double* sm=dalloc(nb);
  for (int b=0;b<nb;b++) { sm[b]=mass[b]; for (int k=0;k<3;k++) o->subtree_com[3*b+k]=mass[b]*o->xipos[3*b+k]; }
  for (int b=nb-1;b>0;b--) { int p=parent[b]; sm[p]+=sm[b]; for (int k=0;k<3;k++) o->subtree_com[3*p+k]+=o->subtree_com[3*b+k]; }
  for (int b=0;b<nb;b++) for (int k=0;k<3;k++) o->subtree_com[3*b+k] = sm[b]<MINVAL ? o->xipos[3*b+k] : o->subtree_com[3*b+k]/sm[b];
  free(sm);
  memset(o->cinert, 0, sizeof(double)*10);
  for (int b=1;b<nb;b++) { double dif[3]; for (int k=0;k<3;k++) dif[k]=o->xipos[3*b+k]-o->subtree_com[3*rootid[b]+k];
    inert_com(o->cinert+10*b, inertia+3*b, o->ximat+9*b, dif, mass[b]); }
  for (int j=0;j<o->njnt;j++) { int b=jb[j], d=jd[j]; double off[3];
    for (int k=0;k<3;k++) off[k]=o->subtree_com[3*rootid[b]+k]-o->xanchor[3*j+k];
    if (jtype[j]==JNT_FREE) {
      for (int k=0;k<3;k++) { double* c=o->cdof+6*(d+k); memset(c,0,48); c[3+k]=1; }
      for (int k=0;k<3;k++) { double* c=o->cdof+6*(d+3+k); double ax[3]={o->xmat[9*b+k],o->xmat[9*b+3+k],o->xmat[9*b+6+k]};
        memcpy(c, ax, 24); cross3(c+3, ax, off); }
    } else if (jtype[j]==JNT_SLIDE) { double* c=o->cdof+6*d; c[0]=c[1]=c[2]=0; memcpy(c+3, o->xaxis+3*j, 24); }
    else { double* c=o->cdof+6*d; memcpy(c, o->xaxis+3*j, 24); cross3(c+3, o->xaxis+3*j, off); }
  }
}

/* ---------------------------------------------------------------- Jacobian of a world point fixed to a body (mj_jac) */
static void jac_point(ora* o, double* jacp, double* jacr, const double* point, int body) {
  const int *rootid=ISEC(o,body_rootid), *dofadr=ISEC(o,body_dofadr), *dofnum=ISEC(o,body_dofnum), *parent=ISEC(o,body_parentid), *dpar=ISEC(o,dof_parentid);
  int nv=o->nv;
  if (jacp) memset(jacp, 0, sizeof(double)*3*nv);
  if (jacr) memset(jacr, 0, sizeof(double)*3*nv);
  while (body && dofnum[body]==0) body=parent[body];
  if (!body) return;
  double off[3]; for (int k=0;k<3;k++) off[k]=point[k]-o->subtree_com[3*rootid[body]+k];
  int d=dofadr[body]+dofnum[body]-1;
  while (d>=0) { const double* c=o->cdof+6*d;
    if (jacr) { jacr[d]=c[0]; jacr[nv+d]=c[1]; jacr[2*nv+d]=c[2]; }
    if (jacp) { double t[3]; cross3(t, c, off); jacp[d]=c[3]+t[0]; jacp[nv+d]=c[4]+t[1]; jacp[2*nv+d]=c[5]+t[2]; }
    d=dpar[d]; }
}

/* ---------------------------------------------------------------- A.2 tendon wrapping (mju_wrap and helpers) */
static int is_intersect(const double* p1, const double* p2, const double* p3, const double* p4) {
  double det=(p4[1]-p3[1])*(p2[0]-p1[0])-(p4[0]-p3[0])*(p2[1]-p1[1]);
  if (fabs(det)<MINVAL) return 0;
  double a=((p4[0]-p3[0])*(p1[1]-p3[1])-(p4[1]-p3[1])*(p1[0]-p3[0]))/det;
  double b=((p2[0]-p1[0])*(p1[1]-p3[1])-(p2[1]-p1[1])*(p1[0]-p3[0]))/det;
  return a>=0 && a<=1 && b>=0 && b<=1; }

static double wrap_circle(double* pnt, const double* d, const double* sd, double rad) {
  double sqlen0=d[0]*d[0]+d[1]*d[1], sqlen1=d[2]*d[2]+d[3]*d[3], sqrad=rad*rad;
  double dif[2]={d[2]-d[0], d[3]-d[1]}, dd=dif[0]*dif[0]+dif[1]*dif[1];
  if (sqlen0<sqrad || sqlen1<sqrad || rad<MINVAL) return -1;
  if (dd<MINVAL) return -1;
  double a=-(dif[0]*d[0]+dif[1]*d[1])/dd; a=clip(a,0,1);
  double tmp[2]={a*dif[0]+d[0], a*dif[1]+d[1]};
  if (tmp[0]*tmp[0]+tmp[1]*tmp[1]>sqrad && (!sd || tmp[0]*sd[0]+tmp[1]*sd[1]>=0)) return -1;
  double sqrt0=sqrt(sqlen0-sqrad), sqrt1=sqrt(sqlen1-sqrad), sol[2][4], good[2];
  for (int i=0;i<2;i++) { double sgn=i==0?1:-1;
    sol[i][0]=(d[0]*sqrad+sgn*rad*d[1]*sqrt0)/sqlen0; sol[i][1]=(d[1]*sqrad-sgn*rad*d[0]*sqrt0)/sqlen0;
    sol[i][2]=(d[2]*sqrad-sgn*rad*d[3]*sqrt1)/sqlen1; sol[i][3]=(d[3]*sqrad+sgn*rad*d[2]*sqrt1)/sqlen1;
    if (sd) { double t[2]={sol[i][0]+sol[i][2], sol[i][1]+sol[i][3]}; double n=sqrt(t[0]*t[0]+t[1]*t[1]);
      if (n<MINVAL) { t[0]=1; t[1]=0; } else { t[0]/=n; t[1]/=n; } good[i]=t[0]*sd[0]+t[1]*sd[1]; }
    else { double t[2]={sol[i][0]-sol[i][2], sol[i][1]-sol[i][3]}; good[i]=-(t[0]*t[0]+t[1]*t[1]); }
    if (is_intersect(d, sol[i], d+2, sol[i]+2)) good[i]=-10000; }
  int i = good[0]>good[1] ? 0 : 1;
  memcpy(pnt, sol[i], 32);
  if (is_intersect(d, pnt, d+2, pnt+2)) return -1;
  return rad*acos(clip((pnt[0]*pnt[2]+pnt[1]*pnt[3])/sqrad, -1, 1));
}

static double wrap_inside(double* pnt, const double* d, double rad) {
  const int maxiter=20; const double zinit=1-1e-7, tolerance=1e-6;
  double len0=sqrt(d[0]*d[0]+d[1]*d[1]), len1=sqrt(d[2]*d[2]+d[3]*d[3]);
  if (len0<=rad || len1<=rad || rad<MINVAL || len0<MINVAL || len1<MINVAL) return -1;
  double dif[2]={d[2]-d[0], d[3]-d[1]}, dd=dif[0]*dif[0]+dif[1]*dif[1];
  if (dd>MINVAL) { double a=-(dif[0]*d[0]+dif[1]*d[1])/dd;
    if (a>0 && a<1) { double t[2]={d[0]+a*dif[0], d[1]+a*dif[1]}; if (sqrt(t[0]*t[0]+t[1]*t[1])<=rad) return -1; } }
  { double t[2]={0.5*(d[0]+d[2]), 0.5*(d[1]+d[3])}; double n=sqrt(t[0]*t[0]+t[1]*t[1]);
    if (n<MINVAL) { t[0]=1; t[1]=0; n=1; } pnt[0]=pnt[2]=rad*t[0]/n; pnt[1]=pnt[3]=rad*t[1]/n; }
  double A=rad/len0, B=rad/len1, cosG=(len0*len0+len1*len1-dd)/(2*len0*len1);
  if (cosG<-1+MINVAL) return -1; else if (cosG>1-MINVAL) return 0;
  double G=acos(cosG), z=zinit, f=asin(A*z)+asin(B*z)-2*asin(z)+G;
  if (f>0) return 0;
  int iter;
  for (iter=0; iter<maxiter && fabs(f)>tolerance; iter++) {
    double df=A/fmax(MINVAL,sqrt(1-z*z*A*A))+B/fmax(MINVAL,sqrt(1-z*z*B*B))-2/fmax(MINVAL,sqrt(1-z*z));
    if (df>-MINVAL) return 0;
    double z1=z-f/df; if (z1>z) return 0;
    z=z1; f=asin(A*z)+asin(B*z)-2*asin(z)+G;
    if (f>tolerance) return 0; }
  if (iter>=maxiter) return 0;
  double vec[2], ang;
  if (d[0]*d[3]-d[1]*d[2]>0) { vec[0]=d[0]; vec[1]=d[1]; ang=asin(z)-asin(A*z); }
  else { vec[0]=d[2]; vec[1]=d[3]; ang=asin(z)-asin(B*z); }
  double n=sqrt(vec[0]*vec[0]+vec[1]*vec[1]); vec[0]/=n; vec[1]/=n;
  pnt[0]=rad*(cos(ang)*vec[0]-sin(ang)*vec[1]); pnt[1]=rad*(sin(ang)*vec[0]+cos(ang)*vec[1]); pnt[2]=pnt[0]; pnt[3]=pnt[1];
  return 0;
}

static double mju_wrap(double* wpnt, const double* x0, const double* x1, const double* xpos, const double* xmat,
                       double radius, int type, const double* side) {
  double p0[3], p1[3], s[3]={0,0,0}, d[4], sd[2]={0,0}, tmp[3], axis[2][3], pnt[4], res[6], normal[3], wlen;
  for (int k=0;k<3;k++) tmp[k]=x0[k]-xpos[k]; matT_vec(p0, xmat, tmp);
  for (int k=0;k<3;k++) tmp[k]=x1[k]-xpos[k]; matT_vec(p1, xmat, tmp);
  if (norm3(p0)<MINVAL || norm3(p1)<MINVAL) return -1;
  if (type==WRAP_SPHERE) {
    memcpy(axis[0], p0, 24); normalize3(axis[0]);
    cross3(normal, p0, p1); double nrm=norm3(normal);
    if (nrm<MINVAL) { int i=0; if (fabs(axis[0][1])>fabs(axis[0][i])) i=1; if (fabs(axis[0][2])>fabs(axis[0][i])) i=2;
      axis[1][0]=axis[1][1]=axis[1][2]=1; axis[1][i]=0; cross3(normal, axis[0], axis[1]); }
    normalize3(normal);
    cross3(axis[1], normal, axis[0]); normalize3(axis[1]);
  } else { axis[0][0]=1; axis[0][1]=0; axis[0][2]=0; axis[1][0]=0; axis[1][1]=1; axis[1][2]=0; }
  d[0]=dot3(p0,axis[0]); d[1]=dot3(p0,axis[1]); d[2]=dot3(p1,axis[0]); d[3]=dot3(p1,axis[1]);
  if (side) { for (int k=0;k<3;k++) tmp[k]=side[k]-xpos[k]; matT_vec(s, xmat, tmp);
    sd[0]=dot3(s,axis[0]); sd[1]=dot3(s,axis[1]); double n=sqrt(sd[0]*sd[0]+sd[1]*sd[1]);
    if (n<MINVAL) { sd[0]=radius; sd[1]=0; } else { sd[0]*=radius/n; sd[1]*=radius/n; } }
  if (side && norm3(s)<radius) wlen=wrap_inside(pnt, d, radius);
  else wlen=wrap_circle(pnt, d, side?sd:NULL, radius);
  if (wlen<0) return -1;
  for (int k=0;k<3;k++) { res[k]=axis[0][k]*pnt[0]+axis[1][k]*pnt[1]; res[3+k]=axis[0][k]*pnt[2]+axis[1][k]*pnt[3]; }
  if (type==WRAP_CYLINDER) {
    double L0=sqrt((p0[0]-pnt[0])*(p0[0]-pnt[0])+(p0[1]-pnt[1])*(p0[1]-pnt[1]));
    double L1=sqrt((p1[0]-pnt[2])*(p1[0]-pnt[2])+(p1[1]-pnt[3])*(p1[1]-pnt[3]));
    res[2]=p0[2]+(p1[2]-p0[2])*L0/(L0+wlen+L1); res[5]=p0[2]+(p1[2]-p0[2])*(L0+wlen)/(L0+wlen+L1);
    double h=fabs(res[5]-res[2]); wlen=sqrt(wlen*wlen+h*h); }
  mat_vec(wpnt, xmat, res); mat_vec(wpnt+3, xmat, res+3);
  for (int k=0;k<3;k++) { wpnt[k]+=xpos[k]; wpnt[3+k]+=xpos[k]; }
  return wlen;
}

static void tendon(ora* o) {
  const int *tadr=ISEC(o,tendon_adr), *tnum=ISEC(o,tendon_num), *wtype=ISEC(o,wrap_type), *wobj=ISEC(o,wrap_objid), *wside=ISEC(o,wrap_sidesite);
  const int *sbody=ISEC(o,site_bodyid), *gbody=ISEC(o,geom_bodyid); const double* gsize=DSEC(o,geom_size);
  int nv=o->nv; double *j0=dalloc(3*nv), *j1=dalloc(3*nv);
  memset(o->ten_J, 0, sizeof(double)*o->ntendon*nv);
  for (int t=0;t<o->ntendon;t++) {
    int adr=tadr[t], num=tnum[t], j=0; double len=0; double* J=o->ten_J+(size_t)t*nv;
    while (j<num-1) {
      int type1=wtype[adr+j+1];
      int id0=wobj[adr+j]; double wpnt[12]; int wbody[4]; double wlen=-1;
      memcpy(wpnt, o->site_xpos+3*id0, 24); wbody[0]=sbody[id0];
      int npnt, id1;
      if (type1==WRAP_SITE) { id1=wobj[adr+j+1]; memcpy(wpnt+3, o->site_xpos+3*id1, 24); wbody[1]=sbody[id1]; npnt=2; }
      else { int g=wobj[adr+j+1]; id1=wobj[adr+j+2]; int ss=wside[adr+j+1];
        wlen=mju_wrap(wpnt+3, o->site_xpos+3*id0, o->site_xpos+3*id1, o->geom_xpos+3*g, o->geom_xmat+9*g, gsize[3*g], type1,
                      ss>=0 ? o->site_xpos+3*ss : NULL);
        if (wlen<0) { memcpy(wpnt+3, o->site_xpos+3*id1, 24); wbody[1]=sbody[id1]; npnt=2; }
        else { wbody[1]=wbody[2]=gbody[g]; memcpy(wpnt+9, o->site_xpos+3*id1, 24); wbody[3]=sbody[id1]; npnt=4; } }
      if (npnt==4) len+=wlen;
      for (int k=0;k<npnt-1;k++) { if (npnt==4 && k==1) continue;
        double dif[3]; for (int c=0;c<3;c++) dif[c]=wpnt[3*k+3+c]-wpnt[3*k+c];
        double n=norm3(dif); len+=n; if (n<MINVAL) { dif[0]=1; dif[1]=dif[2]=0; } else { dif[0]/=n; dif[1]/=n; dif[2]/=n; }
        if (wbody[k]!=wbody[k+1]) { jac_point(o, j0, NULL, wpnt+3*k, wbody[k]); jac_point(o, j1, NULL, wpnt+3*k+3, wbody[k+1]);
          for (int dd=0;dd<nv;dd++) J[dd]+=dif[0]*(j1[dd]-j0[dd])+dif[1]*(j1[nv+dd]-j0[nv+dd])+dif[2]*(j1[2*nv+dd]-j0[2*nv+dd]); } }
      j += (type1==WRAP_SITE) ? 1 : 2;
    }
    o->ten_length[t]=len;
  }
  free(j0); free(j1);
}

/* ---------------------------------------------------------------- A.3 CRB, factorisation, solve */
static void crb(ora* o) {
  const int *parent=ISEC(o,body_parentid), *dbody=ISEC(o,dof_bodyid), *dpar=ISEC(o,dof_parentid), *madr=ISEC(o,dof_Madr);
  const double* arm=DSEC(o,dof_armature);
  memcpy(o->crb, o->cinert, sizeof(double)*10*o->nbody);
  for (int b=o->nbody-1;b>0;b--) if (parent[b]>0) for (int k=0;k<10;k++) o->crb[10*parent[b]+k]+=o->crb[10*b+k];
  for (int i=0;i<o->nv;i++) { double f[6]; mul_inert_vec(f, o->crb+10*dbody[i], o->cdof+6*i);
    int adr=madr[i];
    int j=i; while (j>=0) { const double* c=o->cdof+6*j; o->qM[adr++] = (j==i ? arm[i] : 0) + c[0]*f[0]+c[1]*f[1]+c[2]*f[2]+c[3]*f[3]+c[4]*f[4]+c[5]*f[5]; j=dpar[j]; } }
}
/* in-place L'DL over the tree sparsity (mj_factorI); qLD row i holds [D_ii, L_i,par(i), L_i,par(par(i)), ...] */
static void factor(const int* madr, const int* dpar, int nv, const double* M, int nM, double* LD, double* dinv) {
  memcpy(LD, M, sizeof(double)*nM);
  for (int k=nv-1;k>=0;k--) { int Madr_kk=madr[k]; int i=dpar[k], Madr_ki=Madr_kk+1;
    while (i>=0) { double tmp=LD[Madr_ki]/LD[Madr_kk]; int cnt=0, jj=i;   /* M(i,j) -= M(k,j)*M(k,i)/M(k,k) for j in ancestors(i) incl i */
      while (jj>=0) { LD[madr[i]+cnt] -= LD[Madr_ki+cnt]*tmp; cnt++; jj=dpar[jj]; }
      LD[Madr_ki]=tmp; i=dpar[i]; Madr_ki++; }
    dinv[k]=1.0/LD[Madr_kk]; }
}
static void solve_ld(const int* madr, const int* dpar, int nv, const double* LD, const double* dinv, double* x) {
  for (int i=nv-1;i>=0;i--) { int adr=madr[i]+1, j=dpar[i]; while (j>=0) { x[j]-=LD[adr++]*x[i]; j=dpar[j]; } }
  for (int i=0;i<nv;i++) x[i]*=dinv[i];
  for (int i=0;i<nv;i++) { int adr=madr[i]+1, j=dpar[i]; while (j>=0) { x[i]-=LD[adr++]*x[j]; j=dpar[j]; } }
}
static void mul_M(ora* o, double* r, const double* v) {
  const int *dpar=ISEC(o,dof_parentid), *madr=ISEC(o,dof_Madr);
  for (int i=0;i<o->nv;i++) r[i]=0;
  for (int i=0;i<o->nv;i++) { int adr=madr[i]; r[i]+=o->qM[adr]*v[i]; int j=dpar[i]; adr++;
    while (j>=0) { r[i]+=o->qM[adr]*v[j]; r[j]+=o->qM[adr]*v[i]; adr++; j=dpar[j]; } }
}

/* ---------------------------------------------------------------- A.4 collision (analytic primitives) */
static void make_frame(double* f) {   /* mju_makeFrame: complete [x | yhint | -] into an orthonormal frame (rows) */
  normalize3(f);
  if (norm3(f+3)<0.5) { f[3]=f[4]=f[5]=0; if (f[1]<0.5 && f[1]>-0.5) f[4]=1; else f[5]=1; }
  double d=dot3(f, f+3); for (int k=0;k<3;k++) f[3+k]-=d*f[k]; normalize3(f+3);
  cross3(f+6, f, f+3);
}
static int sphere_sphere(ora* o, int pair, int g1, int g2, double margin, const double* p1, double r1, const double* p2, double r2, const double* yhint) {
  double dif[3]={p2[0]-p1[0],p2[1]-p1[1],p2[2]-p1[2]}; double cd=norm3(dif), dist=cd-r1-r2;
  if (dist>margin) return 0;
  int c=o->ncon; if (c>=o->maxcon) return 0;
  double* f=o->con_frame+9*c; memset(f,0,72);
  if (cd<MINVAL) { f[0]=1; } else { f[0]=dif[0]/cd; f[1]=dif[1]/cd; f[2]=dif[2]/cd; }
  if (yhint) memcpy(f+3, yhint, 24);
  for (int k=0;k<3;k++) o->con_pos[3*c+k]=p1[k]+f[k]*(r1+0.5*dist);
  make_frame(f);
  o->con_dist[c]=dist; o->con_geom1[c]=g1; o->con_geom2[c]=g2; o->con_pair[c]=pair; o->ncon++; return 1;
}
static int plane_sphere(ora* o, int pair, int g1, int g2, double margin, const double* ppos, const double* pmat, const double* spos, double r, const double* yhint) {
  double n[3]={pmat[2],pmat[5],pmat[8]}, dif[3]={spos[0]-ppos[0],spos[1]-ppos[1],spos[2]-ppos[2]};
  double dist=dot3(dif,n)-r; if (dist>margin) return 0;
  int c=o->ncon; if (c>=o->maxcon) return 0;
  double* f=o->con_frame+9*c; memset(f,0,72); memcpy(f,n,24); if (yhint) memcpy(f+3,yhint,24);
  for (int k=0;k<3;k++) o->con_pos[3*c+k]=spos[k]-n[k]*(r+0.5*dist);
  make_frame(f);
  o->con_dist[c]=dist; o->con_geom1[c]=g1; o->con_geom2[c]=g2; o->con_pair[c]=pair; o->ncon++; return 1;
}
static int capsule_capsule(ora* o, int pair, int g1, int g2, double margin) {
  const double* gs=DSEC(o,geom_size); const double *pos1=o->geom_xpos+3*g1, *pos2=o->geom_xpos+3*g2, *m1=o->geom_xmat+9*g1, *m2=o->geom_xmat+9*g2;
  double r1=gs[3*g1], h1=gs[3*g1+1], r2=gs[3*g2], h2=gs[3*g2+1];
  double a1[3]={m1[2],m1[5],m1[8]}, a2[3]={m2[2],m2[5],m2[8]}, dif[3]={pos1[0]-pos2[0],pos1[1]-pos2[1],pos1[2]-pos2[2]};
  double ma=dot3(a1,a1), mb=-dot3(a1,a2), mc=dot3(a2,a2), u=-dot3(a1,dif), v=dot3(a2,dif), det=ma*mc-mb*mb;
  double v1[3], v2[3];
  if (fabs(det)>=MINVAL) {
    double x1=(mc*u-mb*v)/det, x2=(ma*v-mb*u)/det;
    if (x1>h1) { x1=h1; x2=(v-mb*h1)/mc; } else if (x1<-h1) { x1=-h1; x2=(v+mb*h1)/mc; }
    if (x2>h2) { x2=h2; x1=clip((u-mb*h2)/ma,-h1,h1); } else if (x2<-h2) { x2=-h2; x1=clip((u+mb*h2)/ma,-h1,h1); }
    for (int k=0;k<3;k++) { v1[k]=pos1[k]+a1[k]*x1; v2[k]=pos2[k]+a2[k]*x2; }
    return sphere_sphere(o,pair,g1,g2,margin,v1,r1,v2,r2,NULL);
  }
  int n=0; double x2, x1;
  for (int k=0;k<3;k++) v1[k]=pos1[k]+a1[k]*h1; x2=clip((v-mb*h1)/mc,-h2,h2); for (int k=0;k<3;k++) v2[k]=pos2[k]+a2[k]*x2;
  n+=sphere_sphere(o,pair,g1,g2,margin,v1,r1,v2,r2,NULL);
  for (int k=0;k<3;k++) v1[k]=pos1[k]-a1[k]*h1; x2=clip((v+mb*h1)/mc,-h2,h2); for (int k=0;k<3;k++) v2[k]=pos2[k]+a2[k]*x2;
  n+=sphere_sphere(o,pair,g1,g2,margin,v1,r1,v2,r2,NULL);
  if (n==2) return n;
  for (int k=0;k<3;k++) v2[k]=pos2[k]+a2[k]*h2; x1=clip((u-mb*h2)/ma,-h1,h1); for (int k=0;k<3;k++) v1[k]=pos1[k]+a1[k]*x1;
  n+=sphere_sphere(o,pair,g1,g2,margin,v1,r1,v2,r2,NULL);
  if (n==2) return n;
  for (int k=0;k<3;k++) v2[k]=pos2[k]-a2[k]*h2; x1=clip((u+mb*h2)/ma,-h1,h1); for (int k=0;k<3;k++) v1[k]=pos1[k]+a1[k]*x1;
  n+=sphere_sphere(o,pair,g1,g2,margin,v1,r1,v2,r2,NULL);
  return n;
}
/* ---- ellipsoid colliders.  MuJoCo sends ellipsoid-capsule / ellipsoid-ellipsoid pairs through its general convex
 * collider (signed distance / penetration depth along the minimum-translation direction, one contact at the midpoint of
 * the witness points).  Restated from that definition with ROBUST, SLOW numerics (bisection / golden section / pattern
 * search), deliberately unlike the Newton iterations of the CUDA kernels. */
/* signed distance from world point p to the ellipsoid (c, R, s); outward unit normal n (ellipsoid -> point); witness x on the surface */
static double point_ellipsoid(const double* p, const double* c, const double* R, const double* s, double* n, double* x) {
  double t[3] = {p[0]-c[0], p[1]-c[1], p[2]-c[2]}, q[3]; matT_vec(q, R, t);
  double inside = (q[0]/s[0])*(q[0]/s[0])+(q[1]/s[1])*(q[1]/s[1])+(q[2]/s[2])*(q[2]/s[2]);
  double xl[3], lo, hi;
  if (inside >= 1) { lo = 0; hi = norm3(q)*fmax(s[0],fmax(s[1],s[2])); }
  else { double mn = fmin(s[0],fmin(s[1],s[2])); lo = -mn*mn*(1-1e-12); hi = 0; }      /* closest surface point from inside */
  for (int it = 0; it < 200; it++) { double l = 0.5*(lo+hi), g = 0;
    for (int k = 0; k < 3; k++) { double v = s[k]*q[k]/(s[k]*s[k]+l); g += v*v; }
    if (g > 1) lo = l; else hi = l; }
  double l = 0.5*(lo+hi); for (int k = 0; k < 3; k++) xl[k] = s[k]*s[k]*q[k]/(s[k]*s[k]+l);
  double dl[3] = {q[0]-xl[0], q[1]-xl[1], q[2]-xl[2]}, dist = norm3(dl);
  /* outward surface normal at xl: gradient of the implicit function */
  double nl[3] = {xl[0]/(s[0]*s[0]), xl[1]/(s[1]*s[1]), xl[2]/(s[2]*s[2])}; normalize3(nl);
  mat_vec(n, R, nl); double xw[3]; mat_vec(xw, R, xl); for (int k = 0; k < 3; k++) x[k] = xw[k]+c[k];
  return inside >= 1 ? dist : -dist;
}
static long double ee_fl(long double th, long double ph, const double* dl, const double* R1, const double* s1, const double* R2, const double* s2) {
  long double d[3] = {sinl(th)*cosl(ph), sinl(th)*sinl(ph), cosl(th)}, f = d[0]*dl[0]+d[1]*dl[1]+d[2]*dl[2], q1 = 0, q2 = 0;
  for (int k = 0; k < 3; k++) { long double a = R1[k]*d[0]+R1[3+k]*d[1]+R1[6+k]*d[2], b = R2[k]*d[0]+R2[3+k]*d[1]+R2[6+k]*d[2]; q1 += (long double)s1[k]*s1[k]*a*a; q2 += (long double)s2[k]*s2[k]*b*b; }
  return f - sqrtl(q1) - sqrtl(q2); }
static void ang2dir(double th, double ph, double* d) { d[0] = sin(th)*cos(ph); d[1] = sin(th)*sin(ph); d[2] = cos(th); }
static int ellipsoid_ellipsoid(ora* o, int pair, int g1, int g2, double margin) {
  const double* gs = DSEC(o,geom_size); const double *c1=o->geom_xpos+3*g1, *c2=o->geom_xpos+3*g2, *R1=o->geom_xmat+9*g1, *R2=o->geom_xmat+9*g2, *s1=gs+3*g1, *s2=gs+3*g2;
  double dl[3] = {c2[0]-c1[0], c2[1]-c1[1], c2[2]-c1[2]};
  double rb1 = fmax(s1[0],fmax(s1[1],s1[2])), rb2 = fmax(s2[0],fmax(s2[1],s2[2]));
  if (norm3(dl)-rb1-rb2 > margin) return 0;
  { /* any direction gives a lower bound on the signed distance: try the centre line before the expensive search */
    double n = norm3(dl); if (n > MINVAL && ee_fl(acosl(dl[2]/n), atan2l(dl[1], dl[0]), dl, R1, s1, R2, s2) > margin) return 0; }
  /* signed distance = max over unit d of  d.(c2-c1) - h1(d) - h2(-d): coarse grid, then pattern search on the two angles */
  long double best = -1e30L, bt = 0, bp = 0; double d[3];
  for (int i = 1; i < 60; i++) for (int j = 0; j < 120; j++) { long double th = M_PI*i/60, ph = 2*M_PI*j/120, f = ee_fl(th, ph, dl, R1, s1, R2, s2); if (f > best) { best = f; bt = th; bp = ph; } }
  long double step = M_PI/60;
  while (step > 1e-13L) { int moved = 0;
    for (int k = 0; k < 4; k++) { long double th = bt + (k==0)*step - (k==1)*step, ph = bp + (k==2)*step - (k==3)*step, f = ee_fl(th, ph, dl, R1, s1, R2, s2); if (f > best) { best = f; bt = th; bp = ph; moved = 1; } }
    if (!moved) step *= 0.5L; }
  if ((double)best > margin) return 0;
  ang2dir((double)bt, (double)bp, d);
  int c = o->ncon; if (c >= o->maxcon) return 0;
  double a[3], b[3], u[3], pa[3], pb[3]; matT_vec(a, R1, d); for (int k = 0; k < 3; k++) u[k] = s1[k]*s1[k]*a[k]; double n1 = sqrt(dot3(a,u)); mat_vec(pa, R1, u);
  matT_vec(b, R2, d); for (int k = 0; k < 3; k++) u[k] = s2[k]*s2[k]*b[k]; double n2 = sqrt(dot3(b,u)); mat_vec(pb, R2, u);
  double* f = o->con_frame+9*c; memset(f, 0, 72); memcpy(f, d, 24);
  for (int k = 0; k < 3; k++) o->con_pos[3*c+k] = 0.5*((c1[k]+pa[k]/n1) + (c2[k]-pb[k]/n2));
  make_frame(f); o->con_dist[c] = (double)best; o->con_geom1[c] = g1; o->con_geom2[c] = g2; o->con_pair[c] = pair; o->ncon++; return 1;
}
static int capsule_ellipsoid(ora* o, int pair, int g1, int g2, double margin) {   /* g1 capsule, g2 ellipsoid */
  const double* gs = DSEC(o,geom_size); const double *cc=o->geom_xpos+3*g1, *mc=o->geom_xmat+9*g1, *ce=o->geom_xpos+3*g2, *Re=o->geom_xmat+9*g2, *se=gs+3*g2;
  double r = gs[3*g1], h = gs[3*g1+1], ax[3] = {mc[2], mc[5], mc[8]}, dl[3] = {ce[0]-cc[0], ce[1]-cc[1], ce[2]-cc[2]};
  if (norm3(dl)-(r+h)-fmax(se[0],fmax(se[1],se[2])) > margin) return 0;
  { /* lower bound from the direction (closest segment point -> ellipsoid centre) */
    double t0 = clip(dot3(dl, ax), -h, h), q[3] = {dl[0]-ax[0]*t0, dl[1]-ax[1]*t0, dl[2]-ax[2]*t0}, nq = norm3(q);
    if (nq > MINVAL) { double d0[3] = {q[0]/nq, q[1]/nq, q[2]/nq}, b[3]; matT_vec(b, Re, d0);
      if (nq - sqrt(se[0]*se[0]*b[0]*b[0]+se[1]*se[1]*b[1]*b[1]+se[2]*se[2]*b[2]*b[2]) - r > margin) return 0; } }
  /* min over the segment parameter of the (convex) point-ellipsoid distance: bisection on its derivative n.a */
  double lo = -h, hi = h, n[3], x[3], p[3];
  for (int k = 0; k < 3; k++) p[k] = cc[k]+ax[k]*lo; point_ellipsoid(p, ce, Re, se, n, x); double glo = dot3(n, ax);
  for (int k = 0; k < 3; k++) p[k] = cc[k]+ax[k]*hi; point_ellipsoid(p, ce, Re, se, n, x); double ghi = dot3(n, ax);
  if (glo >= 0) hi = lo; else if (ghi <= 0) lo = hi;
  else for (int it = 0; it < 200; it++) { double tm = 0.5*(lo+hi); for (int k = 0; k < 3; k++) p[k] = cc[k]+ax[k]*tm;
    point_ellipsoid(p, ce, Re, se, n, x); if (dot3(n, ax) > 0) hi = tm; else lo = tm; }
  double t = 0.5*(lo+hi); for (int k = 0; k < 3; k++) p[k] = cc[k]+ax[k]*t;
  double dist = point_ellipsoid(p, ce, Re, se, n, x) - r;
  if (dist > margin) return 0;
  int c = o->ncon; if (c >= o->maxcon) return 0;
  double* f = o->con_frame+9*c; memset(f, 0, 72); for (int k = 0; k < 3; k++) f[k] = -n[k];   /* normal from the capsule (geom1) to the ellipsoid (geom2) */
  for (int k = 0; k < 3; k++) o->con_pos[3*c+k] = 0.5*((p[k]-n[k]*r) + x[k]);
  make_frame(f); o->con_dist[c] = dist; o->con_geom1[c] = g1; o->con_geom2[c] = g2; o->con_pair[c] = pair; o->ncon++; return 1;
}
static int plane_ellipsoid(ora* o, int pair, int g1, int g2, double margin) {   /* mjc_PlaneEllipsoid: deepest point along -normal */
  const double* gs = DSEC(o,geom_size); const double *pp=o->geom_xpos+3*g1, *pm=o->geom_xmat+9*g1, *ce=o->geom_xpos+3*g2, *Re=o->geom_xmat+9*g2, *se=gs+3*g2;
  double n[3] = {pm[2], pm[5], pm[8]}, nl[3], u[3], pw[3]; matT_vec(nl, Re, n);
  for (int k = 0; k < 3; k++) u[k] = se[k]*se[k]*nl[k]; double nn = sqrt(dot3(nl,u)); mat_vec(pw, Re, u);
  double pos[3]; for (int k = 0; k < 3; k++) pos[k] = ce[k]-pw[k]/nn;
  double dv[3] = {pos[0]-pp[0], pos[1]-pp[1], pos[2]-pp[2]}, dist = dot3(dv, n);
  if (dist > margin) return 0;
  int c = o->ncon; if (c >= o->maxcon) return 0;
  double* f = o->con_frame+9*c; memset(f, 0, 72); memcpy(f, n, 24);
  for (int k = 0; k < 3; k++) o->con_pos[3*c+k] = pos[k]-n[k]*0.5*dist;
  make_frame(f); o->con_dist[c] = dist; o->con_geom1[c] = g1; o->con_geom2[c] = g2; o->con_pair[c] = pair; o->ncon++; return 1;
}
static void collision(ora* o) {
  const int *pg1=ISEC(o,pair_geom1), *pg2=ISEC(o,pair_geom2), *gt=ISEC(o,geom_type);
  const double *pm=DSEC(o,pair_margin), *gs=DSEC(o,geom_size);
  o->ncon=0;
  for (int p=0;p<o->npair;p++) { int g1=pg1[p], g2=pg2[p], t1=gt[g1], t2=gt[g2]; double margin=pm[p];
    const double *x1=o->geom_xpos+3*g1, *x2=o->geom_xpos+3*g2, *m1=o->geom_xmat+9*g1, *m2=o->geom_xmat+9*g2;
    if (t1==GEOM_CAPSULE && t2==GEOM_CAPSULE) capsule_capsule(o,p,g1,g2,margin);
    else if (t1==GEOM_SPHERE && t2==GEOM_SPHERE) sphere_sphere(o,p,g1,g2,margin,x1,gs[3*g1],x2,gs[3*g2],NULL);
    else if (t1==GEOM_SPHERE && t2==GEOM_CAPSULE) {   /* mjc_SphereCapsule: closest point on the segment */
      double ax[3]={m2[2],m2[5],m2[8]}, d[3]={x1[0]-x2[0],x1[1]-x2[1],x1[2]-x2[2]}, x=clip(dot3(ax,d),-gs[3*g2+1],gs[3*g2+1]), v[3];
      for (int k=0;k<3;k++) v[k]=x2[k]+ax[k]*x; sphere_sphere(o,p,g1,g2,margin,x1,gs[3*g1],v,gs[3*g2],NULL); }
    else if (t1==GEOM_PLANE && t2==GEOM_SPHERE) plane_sphere(o,p,g1,g2,margin,x1,m1,x2,gs[3*g2],NULL);
    else if (t1==GEOM_PLANE && t2==GEOM_CAPSULE) { double ax[3]={m2[2],m2[5],m2[8]}, e[3];
      for (int k=0;k<3;k++) e[k]=x2[k]+ax[k]*gs[3*g2+1]; plane_sphere(o,p,g1,g2,margin,x1,m1,e,gs[3*g2],ax);
      for (int k=0;k<3;k++) e[k]=x2[k]-ax[k]*gs[3*g2+1]; plane_sphere(o,p,g1,g2,margin,x1,m1,e,gs[3*g2],ax); }
    else if (t1==GEOM_PLANE && t2==GEOM_ELLIPSOID) plane_ellipsoid(o,p,g1,g2,margin);
    else if (t1==GEOM_CAPSULE && t2==GEOM_ELLIPSOID) capsule_ellipsoid(o,p,g1,g2,margin);
    else if (t1==GEOM_ELLIPSOID && t2==GEOM_ELLIPSOID) ellipsoid_ellipsoid(o,p,g1,g2,margin);
    /* mesh / hfield / cylinder pairs are dropped at model-compile time (proved unreachable) or listed in pair_unsupported */
  }
}

/* ---------------------------------------------------------------- A.5 constraint assembly */
static void get_solparam(const double* solref_in, const double* solimp_in, double* solref, double* solimp) {
  memcpy(solref, solref_in, 16); memcpy(solimp, solimp_in, 40);
  solimp[0]=clip(solimp[0],MINIMP,MAXIMP); solimp[1]=clip(solimp[1],MINIMP,MAXIMP); solimp[2]=fmax(0,solimp[2]);
  solimp[3]=clip(solimp[3],MINIMP,MAXIMP); solimp[4]=fmax(1,solimp[4]);
}
static double get_impedance(const double* solimp, double pos, double margin) {
  if (solimp[0]==solimp[1] || solimp[2]<=MINVAL) return 0.5*(solimp[0]+solimp[1]);
  double x=fabs((pos-margin)/solimp[2]);
  if (x>=1 || x<=0) return x>=1 ? solimp[1] : solimp[0];
  double y;
  if (solimp[4]==1) y=x;
  else if (x<=solimp[3]) y=pow(x,solimp[4])/pow(solimp[3],solimp[4]-1);
  else y=1-pow(1-x,solimp[4])/pow(1-solimp[3],solimp[4]-1);
  return solimp[0]+y*(solimp[1]-solimp[0]);
}
static int add_row(ora* o, int type, double pos, double margin, double diagApprox, const double* solref_in, const double* solimp_in) {
  int i=o->nefc; double solref[2], solimp[5]; get_solparam(solref_in, solimp_in, solref, solimp);
  double h=DSEC(o,opt)[0];
  o->efc_type[i]=type; o->efc_pos[i]=pos; o->efc_margin[i]=margin; o->efc_diagApprox[i]=diagApprox;
  double imp=get_impedance(solimp,pos,margin);
  o->efc_R[i]=fmax(MINVAL,(1-imp)*diagApprox/imp);
  double tc=fmax(solref[0],2*h), dr=solref[1], dmax=solimp[1];   /* refsafe */
  o->efc_KBIP[4*i]=1/fmax(MINVAL,dmax*dmax*tc*tc*dr*dr); o->efc_KBIP[4*i+1]=2/fmax(MINVAL,dmax*tc); o->efc_KBIP[4*i+2]=imp; o->efc_KBIP[4*i+3]=0;
  memset(o->efc_J+(size_t)i*o->nv, 0, sizeof(double)*o->nv);
  o->nefc++; return i;
}
static void make_constraint(ora* o) {
  const int *jtype=ISEC(o,jnt_type), *jq=ISEC(o,jnt_qposadr), *jd=ISEC(o,jnt_dofadr), *jlim=ISEC(o,jnt_limited), *gbody=ISEC(o,geom_bodyid);
  const double *jrange=DSEC(o,jnt_range), *jmargin=DSEC(o,jnt_margin), *jsolref=DSEC(o,jnt_solref), *jsolimp=DSEC(o,jnt_solimp);
  const double *dinv0=DSEC(o,dof_invweight0), *binv0=DSEC(o,body_invweight0), *qpos0=DSEC(o,qpos0);
  int nv=o->nv; o->nefc=0;
  /* equality: joint polynomial coupling */
  const int *e1=ISEC(o,eq_obj1id), *e2=ISEC(o,eq_obj2id), *eact=ISEC(o,eq_active0);
  const double *edata=DSEC(o,eq_data), *esolref=DSEC(o,eq_solref), *esolimp=DSEC(o,eq_solimp);
  for (int e=0;e<o->neq;e++) { if (!eact[e]) continue;
    int j0=e1[e], j1=e2[e]; const double* c=edata+5*e; double pos0=o->qpos[jq[j0]]-qpos0[jq[j0]], cpos, deriv=0, diag=dinv0[jd[j0]];
    if (j1>=0) { double dif=o->qpos[jq[j1]]-qpos0[jq[j1]];
      cpos=pos0-(c[0]+c[1]*dif+c[2]*dif*dif+c[3]*dif*dif*dif+c[4]*dif*dif*dif*dif);
      deriv=c[1]+2*c[2]*dif+3*c[3]*dif*dif+4*c[4]*dif*dif*dif; diag+=dinv0[jd[j1]]; }
    else cpos=pos0-c[0];
    int i=add_row(o,0,cpos,0,diag,esolref+2*e,esolimp+5*e);
    o->efc_J[(size_t)i*nv+jd[j0]]=1; if (j1>=0) o->efc_J[(size_t)i*nv+jd[j1]]=-deriv; }
  o->ne=o->nefc;
  /* joint limits */
  for (int j=0;j<o->njnt;j++) { if (!jlim[j] || (jtype[j]!=JNT_HINGE && jtype[j]!=JNT_SLIDE)) continue;
    double val=o->qpos[jq[j]];
    for (int side=-1;side<=1;side+=2) { double dist=side*(jrange[2*j+(side+1)/2]-val);
      if (dist<jmargin[j]) { int i=add_row(o,1,dist,jmargin[j],dinv0[jd[j]],jsolref+2*j,jsolimp+5*j); o->efc_J[(size_t)i*nv+jd[j]]=-side; } } }
  o->nl=o->nefc-o->ne;
  /* contacts (pyramidal cone / frictionless) */
  const int* pdim=ISEC(o,pair_dim); const double *pfr=DSEC(o,pair_friction), *psolref=DSEC(o,pair_solref), *psolimp=DSEC(o,pair_solimp),
      *pmargin=DSEC(o,pair_margin), *pgap=DSEC(o,pair_gap);
  double *jp1=dalloc(3*nv), *jp2=dalloc(3*nv), *jn=dalloc(nv), *jt=dalloc(nv);
  for (int c=0;c<o->ncon;c++) { int p=o->con_pair[c], dim=pdim[p]; double inc=pmargin[p]-pgap[p];
    if (o->con_dist[c]>=inc) continue;
    int b1=gbody[o->con_geom1[c]], b2=gbody[o->con_geom2[c]]; const double* f=o->con_frame+9*c;
    jac_point(o,jp1,NULL,o->con_pos+3*c,b1); jac_point(o,jp2,NULL,o->con_pos+3*c,b2);
    for (int d=0;d<nv;d++) jn[d]=f[0]*(jp2[d]-jp1[d])+f[1]*(jp2[nv+d]-jp1[nv+d])+f[2]*(jp2[2*nv+d]-jp1[2*nv+d]);
    double tran=binv0[2*b1]+binv0[2*b2];
    if (dim==1) { int i=add_row(o,2,o->con_dist[c],inc,tran,psolref+2*p,psolimp+5*p); memcpy(o->efc_J+(size_t)i*nv,jn,sizeof(double)*nv); }
    else { if (dim!=3) continue;   /* condim 4/6 are not used by the hot-path models */
      int first=o->nefc; double mu=pfr[5*p];
      for (int k=1;k<dim;k++) { double fri=pfr[5*p+k-1];
        for (int d=0;d<nv;d++) jt[d]=f[3*k]*(jp2[d]-jp1[d])+f[3*k+1]*(jp2[nv+d]-jp1[nv+d])+f[3*k+2]*(jp2[2*nv+d]-jp1[2*nv+d]);
        for (int s=0;s<2;s++) { int i=add_row(o,3,o->con_dist[c],inc,tran+fri*fri*tran,psolref+2*p,psolimp+5*p);
          for (int d=0;d<nv;d++) o->efc_J[(size_t)i*nv+d]=jn[d]+(s==0?fri:-fri)*jt[d]; } }
      /* pyramidal: one common regulariser for all edges, Rpy = 2 mu^2 R(first edge) */
      double Rpy=2*mu*mu*o->efc_R[first]; for (int i=first;i<o->nefc;i++) o->efc_R[i]=Rpy; } }
  free(jp1); free(jp2); free(jn); free(jt);
  for (int i=0;i<o->nefc;i++) o->efc_D[i]=1/o->efc_R[i];
}

/* ---------------------------------------------------------------- velocity stage */
static void cross_motion(double* r, const double* vel, const double* v) {
  double a[3], b[3]; cross3(r, vel, v); cross3(a, vel, v+3); cross3(b, vel+3, v); r[3]=a[0]+b[0]; r[4]=a[1]+b[1]; r[5]=a[2]+b[2]; }
static void cross_force(double* r, const double* vel, const double* f) {
  double a[3], b[3]; cross3(a, vel, f); cross3(b, vel+3, f+3); r[0]=a[0]+b[0]; r[1]=a[1]+b[1]; r[2]=a[2]+b[2]; cross3(r+3, vel, f+3); }
static void com_vel(ora* o) {
  const int *parent=ISEC(o,body_parentid), *dadr=ISEC(o,body_dofadr), *dnum=ISEC(o,body_dofnum), *djnt=ISEC(o,dof_jntid), *jtype=ISEC(o,jnt_type);
  memset(o->cvel,0,48);
  for (int b=1;b<o->nbody;b++) { double cv[6]; memcpy(cv,o->cvel+6*parent[b],48);
    int j=dadr[b], end=dadr[b]+dnum[b];
    while (j<end) {
      if (jtype[djnt[j]]==JNT_FREE) {
        memset(o->cdof_dot+6*j,0,sizeof(double)*18);
        for (int k=0;k<3;k++) for (int c=0;c<6;c++) cv[c]+=o->cdof[6*(j+k)+c]*o->qvel[j+k];
        j+=3;
        for (int k=0;k<3;k++) cross_motion(o->cdof_dot+6*(j+k), cv, o->cdof+6*(j+k));
        for (int k=0;k<3;k++) for (int c=0;c<6;c++) cv[c]+=o->cdof[6*(j+k)+c]*o->qvel[j+k];
        j+=3;
      } else { cross_motion(o->cdof_dot+6*j, cv, o->cdof+6*j); for (int c=0;c<6;c++) cv[c]+=o->cdof[6*j+c]*o->qvel[j]; j++; } }
    memcpy(o->cvel+6*b,cv,48); }
}
static void rne_bias(ora* o) {
  const int *parent=ISEC(o,body_parentid), *dadr=ISEC(o,body_dofadr), *dnum=ISEC(o,body_dofnum), *dbody=ISEC(o,dof_bodyid);
  const double* g=DSEC(o,opt)+1;
  o->cacc[0]=o->cacc[1]=o->cacc[2]=0; o->cacc[3]=-g[0]; o->cacc[4]=-g[1]; o->cacc[5]=-g[2]; memset(o->cfrc,0,48);
  for (int b=1;b<o->nbody;b++) { double* a=o->cacc+6*b; memcpy(a,o->cacc+6*parent[b],48);
    for (int j=dadr[b];j<dadr[b]+dnum[b];j++) for (int c=0;c<6;c++) a[c]+=o->cdof_dot[6*j+c]*o->qvel[j];
    double t[6], t2[6]; mul_inert_vec(o->cfrc+6*b, o->cinert+10*b, a); mul_inert_vec(t, o->cinert+10*b, o->cvel+6*b);
    cross_force(t2, o->cvel+6*b, t); for (int c=0;c<6;c++) o->cfrc[6*b+c]+=t2[c]; }
  for (int b=o->nbody-1;b>0;b--) if (parent[b]>0) for (int c=0;c<6;c++) o->cfrc[6*parent[b]+c]+=o->cfrc[6*b+c];
  for (int d=0;d<o->nv;d++) { const double *c=o->cdof+6*d, *f=o->cfrc+6*dbody[d]; o->qfrc_bias[d]=c[0]*f[0]+c[1]*f[1]+c[2]*f[2]+c[3]*f[3]+c[4]*f[4]+c[5]*f[5]; }
}

/* ---------------------------------------------------------------- A.6 muscle actuation */
static double muscle_dynamics(double ctrl, double act, const double* prm) {
  double c=clip(ctrl,0,1), a=clip(act,0,1), ta=prm[0]*(0.5+1.5*a), td=prm[1]/(0.5+1.5*a), dctrl=c-act, tau;
  if (prm[2]<MINVAL) tau = dctrl>0 ? ta : td;
  else { double x=clip(dctrl/prm[2]+0.5,0,1); double s=x*x*x*(3*x*(2*x-5)+10); tau=td+(ta-td)*s; }
  return dctrl/fmax(MINVAL,tau);
}
static double muscle_gain_length(double L, double lmin, double lmax) {
  if (lmin<=L && L<=lmax) { double a=0.5*(lmin+1), b=0.5*(1+lmax), x;
    if (L<=a) { x=(L-lmin)/fmax(MINVAL,a-lmin); return 0.5*x*x; }
    else if (L<=1) { x=(1-L)/fmax(MINVAL,1-a); return 1-0.5*x*x; }
    else if (L<=b) { x=(L-1)/fmax(MINVAL,b-1); return 1-0.5*x*x; }
    else { x=(lmax-L)/fmax(MINVAL,lmax-b); return 0.5*x*x; } }
  return 0;
}
static double muscle_gain(double len, double vel, const double* lr, double acc0, const double* prm) {
  double force=prm[2]; if (force<0) force=prm[3]/fmax(MINVAL,acc0);
  double L0=(lr[1]-lr[0])/fmax(MINVAL,prm[1]-prm[0]), L=prm[0]+(len-lr[0])/fmax(MINVAL,L0), V=vel/fmax(MINVAL,L0*prm[6]);
  double FL=muscle_gain_length(L,prm[4],prm[5]), y=prm[8]-1, FV;
  if (V<=-1) FV=0; else if (V<=0) FV=(V+1)*(V+1); else if (V<=y) FV=prm[8]-(y-V)*(y-V)/fmax(MINVAL,y); else FV=prm[8];
  return -force*FL*FV;
}
static double muscle_bias(double len, const double* lr, double acc0, const double* prm) {
  double force=prm[2]; if (force<0) force=prm[3]/fmax(MINVAL,acc0);
  double L0=(lr[1]-lr[0])/fmax(MINVAL,prm[1]-prm[0]), L=prm[0]+(len-lr[0])/fmax(MINVAL,L0), b=0.5*(1+prm[5]), x;
  if (L<=1) return 0;
  else if (L<=b) { x=(L-1)/fmax(MINVAL,b-1); return -force*prm[7]*0.5*x*x; }
  else { x=(L-b)/fmax(MINVAL,b-1); return -force*prm[7]*(0.5+x); }
}

/* ---------------------------------------------------------------- Newton solver (primal, exact line search) */
static double ls_deriv(int nefc, int ne, const double* D, const double* jar, const double* jv, double alpha,
                       double gauss_a, double gauss_b, double* hess) {
  /* d/dalpha [ gauss(alpha) + sum s_i(jar_i + alpha*jv_i) ];  gauss'(alpha) = gauss_a + gauss_b*alpha */
  double d=gauss_a+gauss_b*alpha, h=gauss_b;
  for (int i=0;i<nefc;i++) { double x=jar[i]+alpha*jv[i]; if (i<ne || x<0) { d+=D[i]*x*jv[i]; h+=D[i]*jv[i]*jv[i]; } }
  *hess=h; return d;
}
static void solve_constraint(ora* o) {
  int nv=o->nv, nefc=o->nefc; const int *dpar=ISEC(o,dof_parentid), *madr=ISEC(o,dof_Madr);
  memset(o->qfrc_constraint,0,sizeof(double)*nv); o->solver_niter=0;
  if (nefc==0) { memcpy(o->qacc,o->qacc_smooth,sizeof(double)*nv); return; }
  double *a=dalloc(nv), *Ma=dalloc(nv), *g=dalloc(nv), *p=dalloc(nv), *Mp=dalloc(nv), *jar=dalloc(nefc), *jv=dalloc(nefc), *H=dalloc((size_t)nv*nv), *t=dalloc(nv);
  const double *J=o->efc_J, *D=o->efc_D; int ne=o->ne;
  /* cost at a candidate */
  #define COST(acc, out) do { double cst=0; mul_M(o,t,acc); for (int d_=0;d_<nv;d_++) cst+=0.5*(t[d_]-o->qfrc_smooth[d_])*(acc[d_]-o->qacc_smooth[d_]); \
    for (int i_=0;i_<nefc;i_++) { double x_=-o->efc_aref[i_]; for (int d_=0;d_<nv;d_++) x_+=J[(size_t)i_*nv+d_]*acc[d_]; if (i_<ne||x_<0) cst+=0.5*D[i_]*x_*x_; } out=cst; } while (0)
  double c_warm, c_smooth; COST(o->qacc_warmstart,c_warm); COST(o->qacc_smooth,c_smooth);
  memcpy(a, c_warm<c_smooth ? o->qacc_warmstart : o->qacc_smooth, sizeof(double)*nv);
  double scale=1.0/(DSEC(o,opt)[6]*fmax(1,nv)), gn_prev=0;
  for (int iter=0; iter<200; iter++) {
    mul_M(o,Ma,a);
    for (int i=0;i<nefc;i++) { double x=-o->efc_aref[i]; for (int d=0;d<nv;d++) x+=J[(size_t)i*nv+d]*a[d]; jar[i]=x; }
    for (int d=0;d<nv;d++) g[d]=Ma[d]-o->qfrc_smooth[d];
    for (int i=0;i<nefc;i++) if (i<ne||jar[i]<0) for (int d=0;d<nv;d++) g[d]+=J[(size_t)i*nv+d]*D[i]*jar[i];
    double gn=0; for (int d=0;d<nv;d++) gn+=g[d]*g[d]; gn=sqrt(gn);
    if (getenv("ORACLE_DEBUG")) fprintf(stderr, "iter %d scaled grad %.3e\n", iter, scale*gn);
    if (scale*gn<1e-12 || (iter>0 && gn>=0.5*gn_prev && scale*gn<1e-9)) break;   /* converged to round-off */
    gn_prev=gn;
    /* H = M + J' D_active J (dense), Cholesky solve */
    memset(H,0,sizeof(double)*nv*nv);
    for (int i=0;i<nv;i++) { int adr=madr[i], j=i; while (j>=0) { H[i*nv+j]=H[j*nv+i]=o->qM[adr++]; j=dpar[j]; } }
    for (int r=0;r<nefc;r++) if (r<ne||jar[r]<0) for (int i=0;i<nv;i++) { double ji=J[(size_t)r*nv+i]*D[r]; if (ji!=0) for (int j=0;j<nv;j++) H[i*nv+j]+=ji*J[(size_t)r*nv+j]; }
    if (getenv("ORACLE_DEBUG")) { int nn=0; for (int i=0;i<nv*nv;i++) if (isnan(H[i])) nn++; int nj=0; for (int i=0;i<nefc*nv;i++) if (isnan(J[i])) nj++; int nd=0; for (int i=0;i<nefc;i++) if (isnan(D[i])||isnan(jar[i])) nd++; fprintf(stderr,"  H nan %d J nan %d D/jar nan %d\n",nn,nj,nd); }
    for (int i=0;i<nv;i++) { for (int j=0;j<=i;j++) { double s=H[i*nv+j]; for (int k=0;k<j;k++) s-=H[i*nv+k]*H[j*nv+k];
        if (i==j) { if (getenv("ORACLE_DEBUG") && !(s>1e-12)) fprintf(stderr,"   pivot %d = %.3e (H0 %.3e)\n", i, s, H[i*nv+i]); H[i*nv+i]=sqrt(fmax(s,MINVAL)); } else H[i*nv+j]=s/H[j*nv+j]; } }
    for (int i=0;i<nv;i++) { double s=-g[i]; for (int k=0;k<i;k++) s-=H[i*nv+k]*p[k]; p[i]=s/H[i*nv+i]; }
    for (int i=nv-1;i>=0;i--) { double s=p[i]; for (int k=i+1;k<nv;k++) s-=H[k*nv+i]*p[k]; p[i]=s/H[i*nv+i]; }
    /* exact line search: safeguarded Newton on the (piecewise linear, increasing) derivative */
    mul_M(o,Mp,p);
    for (int i=0;i<nefc;i++) { double x=0; for (int d=0;d<nv;d++) x+=J[(size_t)i*nv+d]*p[d]; jv[i]=x; }
    double ga=0, gb=0; for (int d=0;d<nv;d++) { ga+=p[d]*(Ma[d]-o->qfrc_smooth[d]); gb+=p[d]*Mp[d]; }
    double alpha=0, lo=0, hi=-1, h, dv=ls_deriv(nefc,ne,D,jar,jv,0,ga,gb,&h);
    if (dv>=0) break;   /* not a descent direction: converged to round-off */
    for (int it=0; it<100; it++) {
      double an=alpha-dv/h;
      if (an<=lo || (hi>0 && an>=hi)) an = hi>0 ? 0.5*(lo+hi) : 2*alpha+1;
      alpha=an; dv=ls_deriv(nefc,ne,D,jar,jv,alpha,ga,gb,&h);
      if (dv<0) lo=alpha; else hi=alpha;
      if (fabs(dv)<1e-15*fmax(1.0,fabs(ga))) break; }
    if (getenv("ORACLE_DEBUG")) { double pn=0; for (int d=0;d<nv;d++) pn+=p[d]*p[d]; fprintf(stderr, "  alpha %.6e dv %.3e h %.3e ga %.3e gb %.3e |p| %.3e\n", alpha, dv, h, ga, gb, sqrt(pn)); }
    for (int d=0;d<nv;d++) a[d]+=alpha*p[d];
    o->solver_niter=iter+1;
  }
  #undef COST
  memcpy(o->qacc,a,sizeof(double)*nv);
  for (int i=0;i<nefc;i++) { double x=-o->efc_aref[i]; for (int d=0;d<nv;d++) x+=J[(size_t)i*nv+d]*a[d];
    o->efc_force[i] = (i<ne||x<0) ? -D[i]*x : 0; for (int d=0;d<nv;d++) o->qfrc_constraint[d]+=J[(size_t)i*nv+d]*o->efc_force[i]; }
  free(a); free(Ma); free(g); free(p); free(Mp); free(jar); free(jv); free(H); free(t);
}

/* ---------------------------------------------------------------- A.0 mj_forward / mj_step */
void oracle_forward(ora* o) {
  int nv=o->nv, nu=o->nu; const int *dpar=ISEC(o,dof_parentid), *madr=ISEC(o,dof_Madr);
  /* fwdPosition */
  kinematics(o); com_pos(o); tendon(o); crb(o); factor(madr,dpar,nv,o->qM,o->nM,o->qLD,o->qLDiagInv); collision(o); make_constraint(o);
  /* transmission (tendon, gear) */
  const int* trnid=ISEC(o,actuator_trnid); const double* gear=DSEC(o,actuator_gear);
  for (int i=0;i<nu;i++) o->actuator_length[i]=gear[i]*o->ten_length[trnid[i]];
  /* fwdVelocity */
  for (int t=0;t<o->ntendon;t++) { double s=0; for (int d=0;d<nv;d++) s+=o->ten_J[(size_t)t*nv+d]*o->qvel[d]; o->ten_velocity[t]=s; }
  for (int i=0;i<nu;i++) o->actuator_velocity[i]=gear[i]*o->ten_velocity[trnid[i]];
  com_vel(o);
  { const int *djnt=ISEC(o,dof_jntid), *jtype=ISEC(o,jnt_type), *jq=ISEC(o,jnt_qposadr), *jd=ISEC(o,jnt_dofadr);
    const double *damp=DSEC(o,dof_damping), *stiff=DSEC(o,jnt_stiffness), *qs=DSEC(o,qpos_spring);
    for (int d=0;d<nv;d++) { int j=djnt[d]; o->qfrc_passive[d]=-damp[d]*o->qvel[d];
      if (jtype[j]!=JNT_FREE && stiff[j]!=0) o->qfrc_passive[d]-=stiff[j]*(o->qpos[jq[j]]-qs[jq[j]]); (void)jd; } }
  for (int i=0;i<o->nefc;i++) { double s=0; for (int d=0;d<nv;d++) s+=o->efc_J[(size_t)i*nv+d]*o->qvel[d]; o->efc_vel[i]=s;
    o->efc_aref[i]=-o->efc_KBIP[4*i+1]*s-o->efc_KBIP[4*i]*o->efc_KBIP[4*i+2]*(o->efc_pos[i]-o->efc_margin[i]); }
  rne_bias(o);
  /* fwdActuation */
  { const int *cl=ISEC(o,actuator_ctrllimited); const double *cr=DSEC(o,actuator_ctrlrange), *dyn=DSEC(o,actuator_dynprm), *gp=DSEC(o,actuator_gainprm),
        *bp=DSEC(o,actuator_biasprm), *lr=DSEC(o,actuator_lengthrange), *acc0=DSEC(o,actuator_acc0);
    memset(o->qfrc_actuator,0,sizeof(double)*nv);
    for (int i=0;i<nu;i++) { double c=o->ctrl[i]; if (cl[i]) c=clip(c,cr[2*i],cr[2*i+1]);
      o->act_dot[i]=muscle_dynamics(c,o->act[i],dyn+3*i);
      double gain=muscle_gain(o->actuator_length[i],o->actuator_velocity[i],lr+2*i,acc0[i],gp+9*i), bias=muscle_bias(o->actuator_length[i],lr+2*i,acc0[i],bp+9*i);
      o->actuator_force[i]=gain*o->act[i]+bias;
      for (int d=0;d<nv;d++) o->qfrc_actuator[d]+=gear[i]*o->ten_J[(size_t)trnid[i]*nv+d]*o->actuator_force[i]; } }
  /* fwdAcceleration */
  for (int d=0;d<nv;d++) { o->qfrc_smooth[d]=o->qfrc_passive[d]-o->qfrc_bias[d]+o->qfrc_actuator[d]; o->qacc_smooth[d]=o->qfrc_smooth[d]; }
  solve_ld(madr,dpar,nv,o->qLD,o->qLDiagInv,o->qacc_smooth);
  /* fwdConstraint */
  solve_constraint(o);
}

void oracle_step(ora* o) {
  int nv=o->nv; const int *dpar=ISEC(o,dof_parentid), *madr=ISEC(o,dof_Madr); double h=DSEC(o,opt)[0];
  oracle_forward(o);
  /* mj_Euler with implicit joint damping (eulerdamp) */
  const double* damp=DSEC(o,dof_damping); int any=0; for (int d=0;d<nv;d++) if (damp[d]>0) any=1;
  double* qacc=dalloc(nv);
  if (any) { double *MH=dalloc(o->nM), *LD=dalloc(o->nM), *di=dalloc(nv); memcpy(MH,o->qM,sizeof(double)*o->nM);
    for (int d=0;d<nv;d++) MH[madr[d]]+=h*damp[d];
    factor(madr,dpar,nv,MH,o->nM,LD,di);
    for (int d=0;d<nv;d++) qacc[d]=o->qfrc_smooth[d]+o->qfrc_constraint[d];
    solve_ld(madr,dpar,nv,LD,di,qacc); free(MH); free(LD); free(di); }
  else memcpy(qacc,o->qacc,sizeof(double)*nv);
  for (int i=0;i<o->na;i++) o->act[i]+=h*o->act_dot[i];
  for (int d=0;d<nv;d++) o->qvel[d]+=h*qacc[d];
  { const int *jtype=ISEC(o,jnt_type), *jq=ISEC(o,jnt_qposadr), *jd=ISEC(o,jnt_dofadr);
    for (int j=0;j<o->njnt;j++) { int qa=jq[j], da=jd[j];
      if (jtype[j]==JNT_FREE) { for (int k=0;k<3;k++) o->qpos[qa+k]+=h*o->qvel[da+k];
        double w[3]={o->qvel[da+3],o->qvel[da+4],o->qvel[da+5]}, ang=h*normalize3(w), ql[4], qn[4];
        axisangle_quat(ql,w,ang); quat_mul(qn,o->qpos+qa+3,ql); quat_norm(qn); memcpy(o->qpos+qa+3,qn,32); }
      else o->qpos[qa]+=h*o->qvel[da]; } }
  o->time+=h; memcpy(o->qacc_warmstart,o->qacc,sizeof(double)*nv); free(qacc);
}

void oracle_step_n(ora* o, int n) { for (int i = 0; i < n; i++) oracle_step(o); }

/* ---------------------------------------------------------------- field access for the Python test harness */
double* oracle_field(ora* o, const char* name, int* len) {
  #define F(n, ptr, l) if (!strcmp(name, n)) { *len=(l); return (ptr); }
  int nv=o->nv, nb=o->nbody;
  F("qpos",o->qpos,o->nq) F("qvel",o->qvel,nv) F("act",o->act,o->na) F("ctrl",o->ctrl,o->nu) F("qacc",o->qacc,nv)
  F("qacc_warmstart",o->qacc_warmstart,nv) F("xpos",o->xpos,3*nb) F("xquat",o->xquat,4*nb) F("xmat",o->xmat,9*nb) F("xipos",o->xipos,3*nb)
  F("geom_xpos",o->geom_xpos,3*o->ngeom) F("geom_xmat",o->geom_xmat,9*o->ngeom) F("site_xpos",o->site_xpos,3*o->nsite)
  F("subtree_com",o->subtree_com,3*nb) F("cvel",o->cvel,6*nb) F("ten_length",o->ten_length,o->ntendon) F("ten_J",o->ten_J,o->ntendon*nv)
  F("ten_velocity",o->ten_velocity,o->ntendon) F("actuator_length",o->actuator_length,o->nu) F("actuator_velocity",o->actuator_velocity,o->nu)
  F("actuator_force",o->actuator_force,o->nu) F("act_dot",o->act_dot,o->na) F("qM",o->qM,o->nM) F("qLD",o->qLD,o->nM)
  F("qfrc_bias",o->qfrc_bias,nv) F("qfrc_passive",o->qfrc_passive,nv) F("qfrc_actuator",o->qfrc_actuator,nv) F("qfrc_smooth",o->qfrc_smooth,nv)
  F("qacc_smooth",o->qacc_smooth,nv) F("qfrc_constraint",o->qfrc_constraint,nv) F("efc_J",o->efc_J,o->nefc*nv) F("efc_pos",o->efc_pos,o->nefc)
  F("efc_D",o->efc_D,o->nefc) F("efc_R",o->efc_R,o->nefc) F("efc_aref",o->efc_aref,o->nefc) F("efc_force",o->efc_force,o->nefc)
  F("efc_vel",o->efc_vel,o->nefc) F("con_dist",o->con_dist,o->ncon) F("con_pos",o->con_pos,3*o->ncon) F("con_frame",o->con_frame,9*o->ncon)
  F("time",&o->time,1)
  #undef F
  *len=0; return NULL;
}
int* oracle_ifield(ora* o, const char* name, int* len) {
  if (!strcmp(name,"con_geom1")) { *len=o->ncon; return o->con_geom1; }
  if (!strcmp(name,"con_geom2")) { *len=o->ncon; return o->con_geom2; }
  if (!strcmp(name,"con_pair")) { *len=o->ncon; return o->con_pair; }
  if (!strcmp(name,"efc_type")) { *len=o->nefc; return o->efc_type; }
  *len=0; return NULL;
}
int oracle_info(ora* o, int what) { switch (what) { case 0: return o->ncon; case 1: return o->nefc; case 2: return o->ne; case 3: return o->nl; case 4: return o->solver_niter; } return -1; }
void oracle_set_time(ora* o, double t) { o->time=t; }

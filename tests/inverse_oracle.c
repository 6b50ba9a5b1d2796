/* inverse_oracle.c -- mj_inverse on the CPU oracle (test infrastructure only; compiled by tests/inverse_oracle.py).
 *
 * The oracle's own source is included unchanged, so that the inverse runs on exactly its position and velocity stages.  What this file
 * adds follows MuJoCo's mj_inverse:
 *   M qacc + qfrc_bias     recursive Newton-Euler WITH the acceleration (mj_rne with flg_acc = 1), plus armature * qacc: the route MuJoCo
 *                          takes, not the oracle's mass matrix times qacc, so that a comparison with the device's CRB mass matrix sets two
 *                          formulations against each other
 *   qfrc_passive           as oracle_forward computes it
 *   qfrc_constraint        J' efc_force, efc_force = -D (J qacc - aref) on equality rows and on the other rows where that is negative
 *   INV_DISCRETE           (mjENBL_INVDISCRETE) qacc is first converted to M^-1 (M + h B) qacc with the oracle's factor / solve_ld
 *   INV_NOCONSTRAINT       (mjDSBL_CONSTRAINT) no collision and no constraint rows */
#include "../oracle/myo_oracle.c"

#define INV_NOCONSTRAINT 1
#define INV_DISCRETE 2

/* cfrc of every body for the accelerations cacc = cacc(parent) + cdof_dot qvel + cdof qacc, summed up the tree; out = cdof' cfrc */
static void rne_acc(ora* o, const double* qacc, double* out) {
  const int *parent=ISEC(o,body_parentid), *dadr=ISEC(o,body_dofadr), *dnum=ISEC(o,body_dofnum), *dbody=ISEC(o,dof_bodyid);
  const double* g=DSEC(o,opt)+1;
  o->cacc[0]=o->cacc[1]=o->cacc[2]=0; o->cacc[3]=-g[0]; o->cacc[4]=-g[1]; o->cacc[5]=-g[2]; memset(o->cfrc,0,48);
  for (int b=1;b<o->nbody;b++) { double* a=o->cacc+6*b; memcpy(a,o->cacc+6*parent[b],48);
    for (int j=dadr[b];j<dadr[b]+dnum[b];j++) for (int c=0;c<6;c++) a[c]+=o->cdof_dot[6*j+c]*o->qvel[j]+o->cdof[6*j+c]*qacc[j];
    double t[6], t2[6]; mul_inert_vec(o->cfrc+6*b, o->cinert+10*b, a); mul_inert_vec(t, o->cinert+10*b, o->cvel+6*b);
    cross_force(t2, o->cvel+6*b, t); for (int c=0;c<6;c++) o->cfrc[6*b+c]+=t2[c]; }
  for (int b=o->nbody-1;b>0;b--) if (parent[b]>0) for (int c=0;c<6;c++) o->cfrc[6*parent[b]+c]+=o->cfrc[6*b+c];
  for (int d=0;d<o->nv;d++) { const double *c=o->cdof+6*d, *f=o->cfrc+6*dbody[d]; out[d]=c[0]*f[0]+c[1]*f[1]+c[2]*f[2]+c[3]*f[3]+c[4]*f[4]+c[5]*f[5]; }
}

/* mj_inverse at the oracle's (qpos, qvel) for the caller-set qacc (left untouched).  Writes qfrc_inverse [nv] and the oracle's
 * qfrc_constraint and efc_force fields; the position and velocity fields are those of oracle_forward at the same state. */
void oracle_inverse(ora* o, int flags, double* qfrc_inverse) {
  int nv=o->nv; const int *dpar=ISEC(o,dof_parentid), *madr=ISEC(o,dof_Madr); const double h=DSEC(o,opt)[0];
  kinematics(o); com_pos(o); tendon(o); crb(o); factor(madr,dpar,nv,o->qM,o->nM,o->qLD,o->qLDiagInv);
  if (flags & INV_NOCONSTRAINT) { o->ncon=0; o->nefc=0; o->ne=0; o->nl=0; }
  else { collision(o); make_constraint(o); }
  com_vel(o);
  { const int *djnt=ISEC(o,dof_jntid), *jtype=ISEC(o,jnt_type), *jq=ISEC(o,jnt_qposadr);
    const double *damp=DSEC(o,dof_damping), *stiff=DSEC(o,jnt_stiffness), *qs=DSEC(o,qpos_spring);
    for (int d=0;d<nv;d++) { int j=djnt[d]; o->qfrc_passive[d]=-damp[d]*o->qvel[d];
      if (jtype[j]!=JNT_FREE && stiff[j]!=0) o->qfrc_passive[d]-=stiff[j]*(o->qpos[jq[j]]-qs[jq[j]]); } }
  for (int i=0;i<o->nefc;i++) { double s=0; for (int d=0;d<nv;d++) s+=o->efc_J[(size_t)i*nv+d]*o->qvel[d]; o->efc_vel[i]=s;
    o->efc_aref[i]=-o->efc_KBIP[4*i+1]*s-o->efc_KBIP[4*i]*o->efc_KBIP[4*i+2]*(o->efc_pos[i]-o->efc_margin[i]); }
  double* a=dalloc(nv); memcpy(a,o->qacc,sizeof(double)*nv);
  if (flags & INV_DISCRETE) { const double* damp=DSEC(o,dof_damping); double* t=dalloc(nv);
    mul_M(o,t,a); for (int d=0;d<nv;d++) t[d]+=h*damp[d]*a[d];
    solve_ld(madr,dpar,nv,o->qLD,o->qLDiagInv,t); memcpy(a,t,sizeof(double)*nv); free(t); }
  rne_acc(o,a,qfrc_inverse);
  const double* arm=DSEC(o,dof_armature);
  memset(o->qfrc_constraint,0,sizeof(double)*nv);
  for (int i=0;i<o->nefc;i++) { double x=-o->efc_aref[i]; for (int d=0;d<nv;d++) x+=o->efc_J[(size_t)i*nv+d]*a[d];
    o->efc_force[i] = (i<o->ne || x<0) ? -o->efc_D[i]*x : 0; for (int d=0;d<nv;d++) o->qfrc_constraint[d]+=o->efc_J[(size_t)i*nv+d]*o->efc_force[i]; }
  for (int d=0;d<nv;d++) qfrc_inverse[d]+=arm[d]*a[d]-o->qfrc_passive[d]-o->qfrc_constraint[d];
  free(a);
}

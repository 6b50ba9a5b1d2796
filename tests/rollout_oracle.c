/* rollout_oracle.c -- mjData.qfrc_applied on the CPU oracle (test infrastructure only; compiled by tests/rollout_oracle.py).
 *
 * The oracle's own source is included unchanged.  MuJoCo adds qfrc_applied to qfrc_smooth in fwdAcceleration; nothing before that line
 * of oracle_forward reads qfrc_smooth, and solve_constraint reads qfrc_smooth, qacc_smooth, the warm start and the constraint rows but
 * none of its own outputs.  So the forward pass with an applied force is oracle_forward followed by that line and the two solves again:
 *   qfrc_smooth += f        qacc_smooth = M^-1 qfrc_smooth        solve_constraint
 * The step is that forward pass followed by mj_Euler with implicit joint damping, restated from oracle_step.  With f = 0 both agree with
 * oracle_forward / oracle_step bit for bit (tests/test_rollout.py checks it), which also pins the restated integrator to the oracle's. */
#include "../oracle/myo_oracle.c"

void oracle_forward_applied(ora* o, const double* f) {
  int nv=o->nv; const int *dpar=ISEC(o,dof_parentid), *madr=ISEC(o,dof_Madr);
  oracle_forward(o);
  for (int d=0;d<nv;d++) { o->qfrc_smooth[d]+=f[d]; o->qacc_smooth[d]=o->qfrc_smooth[d]; }
  solve_ld(madr,dpar,nv,o->qLD,o->qLDiagInv,o->qacc_smooth);
  solve_constraint(o);
}

void oracle_step_applied(ora* o, const double* f) {
  int nv=o->nv; const int *dpar=ISEC(o,dof_parentid), *madr=ISEC(o,dof_Madr); double h=DSEC(o,opt)[0];
  oracle_forward_applied(o, f);
  /* mj_Euler with implicit joint damping (eulerdamp), as oracle_step */
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

// objective_common.cuh -- host checks of a compiled objective (bb_objective), shared by bb_objective_score
// (objective.cu) and bb_objective_grad (objgrad.cu).  `fn` prefixes every message.
#pragma once

#include <math.h>

#include "common.cuh"

namespace bb {

// Dry run of one program on the host: opcodes, op count and stack depth (BB_OBJ_MAX_STACK).
static inline int check_program(const char* fn, const bb_objective* obj, int m) {
  const int n = obj->n_ops[m];
  BB_CHECK_SUPPORTED(n >= 0 && n <= BB_OBJ_MAX_OPS, "%s: target %d has %d ops outside [0,%d]", fn, m, n,
                     BB_OBJ_MAX_OPS);
  int depth = 1;
  for (int i = 0; i < n; ++i) {
    const bb_obj_instr& in = obj->prog[m][i];
    BB_CHECK_ARG(in.op >= BB_OBJ_AFFINE && in.op <= BB_OBJ_MUL, "%s: target %d op %d: unknown opcode %d", fn, m, i,
                 in.op);
    if (in.op == BB_OBJ_DUP_INPUT) ++depth;
    if (in.op == BB_OBJ_ADD || in.op == BB_OBJ_MUL) {
      BB_CHECK_ARG(depth >= 2, "%s: target %d op %d pops an empty stack", fn, m, i);
      --depth;
    }
    BB_CHECK_SUPPORTED(depth <= BB_OBJ_MAX_STACK, "%s: target %d op %d: stack depth %d above %d", fn, m, i, depth,
                       BB_OBJ_MAX_STACK);
    if (in.op == BB_OBJ_POW_INT)
      BB_CHECK_SUPPORTED(in.arg[0] == rintf(in.arg[0]), "%s: target %d op %d: non-integer power %g", fn, m, i,
                         (double)in.arg[0]);
  }
  BB_CHECK_ARG(depth == 1, "%s: target %d leaves %d stack entries (need 1)", fn, m, depth);
  return BB_OK;
}

// The acquisition kind and its temperatures, the target count, the scalariser, every program and weight, and the
// analytic kinds' envelope (MEAN over affine targets: the scalarised posterior must stay Gaussian).  a, obj non-null.
static inline int check_objective(const char* fn, const bb_acq_spec* a, const bb_objective* obj) {
  BB_CHECK_ARG(a->kind >= BB_ACQ_QLOGEI && a->kind <= BB_ACQ_PSTD,
               "%s: kind %d is not a single-objective acquisition function", fn, a->kind);
  const bool analytic = a->kind >= BB_ACQ_UCB;
  BB_CHECK_ARG(!(a->kind == BB_ACQ_QLOGEI) || (a->tau_relu > 0.f && a->tau_max > 0.f),
               "%s: qLogEI needs tau_relu > 0 and tau_max > 0", fn);
  BB_CHECK_ARG(!(a->kind == BB_ACQ_QPI) || a->tau_pi > 0.f, "%s: qPI needs tau_pi > 0", fn);
  const int M = obj->n_targets;
  BB_CHECK_SUPPORTED(M >= 1 && M <= BB_OBJ_MAX_TARGETS, "%s: n_targets=%d outside [1,%d]", fn, M, BB_OBJ_MAX_TARGETS);
  BB_CHECK_ARG(obj->scalarizer >= BB_OBJ_SCALAR_NONE && obj->scalarizer <= BB_OBJ_SCALAR_GEOM_MEAN,
               "%s: unknown scalarizer %d", fn, obj->scalarizer);
  BB_CHECK_ARG((obj->scalarizer == BB_OBJ_SCALAR_NONE) == (M == 1),
               "%s: scalarizer NONE is for exactly one target (got %d targets)", fn, M);
  for (int m = 0; m < M; ++m) {
    const int rc = check_program(fn, obj, m);
    if (rc != BB_OK) return rc;
    BB_CHECK_ARG(isfinite(obj->weight[m]), "%s: weight %d is not finite", fn, m);
  }
  if (analytic) {
    BB_CHECK_SUPPORTED(obj->scalarizer == BB_OBJ_SCALAR_MEAN,
                       "%s: analytic kinds need MEAN scalarisation (the posterior must stay Gaussian)", fn);
    for (int m = 0; m < M; ++m)
      BB_CHECK_SUPPORTED(obj->n_ops[m] == 0 || (obj->n_ops[m] == 1 && obj->prog[m][0].op == BB_OBJ_AFFINE),
                         "%s: analytic kinds need affine targets (target %d is not)", fn, m);
  }
  return BB_OK;
}

}  // namespace bb

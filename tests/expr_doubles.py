"""Double of er_expr_eval (ExprFeature columns) for the host tests (TEST INFRASTRUCTURE): the programs of a kernels.ExprPlan
run in numpy on the host, float64 ops and one rounding to float32 as the kernel does.  `install` lets the plan be built
on a host device and puts the double in place of kernels.expr_eval; install it after host_doubles.install_all."""
import numpy as np
import torch

from easyrec_b200 import expr as X, kernels as K

_NUMPY = {X.EXPR_ADD: np.add, X.EXPR_SUB: np.subtract, X.EXPR_MUL: np.multiply, X.EXPR_DIV: np.divide,
          X.EXPR_GT: np.greater, X.EXPR_GE: np.greater_equal, X.EXPR_LT: np.less, X.EXPR_LE: np.less_equal,
          X.EXPR_EQ: np.equal, X.EXPR_AND: lambda a, b: (a != 0) & (b != 0),
          X.EXPR_OR: lambda a, b: (a != 0) | (b != 0)}


def evaluate(ops, inputs):
  """one program's ops [(opcode, input, constant)] on inputs float64 [B, n] -> float32 [B]"""
  st = []
  with np.errstate(all='ignore'):
    for op, arg, value in ops:
      if op == X.EXPR_LOAD:
        st.append(np.asarray(inputs[:, arg], np.float64))
      elif op == X.EXPR_CONST:
        st.append(np.full(inputs.shape[0], value, np.float64))
      elif op == X.EXPR_NEG:
        st.append(-st.pop())
      else:
        b, a = st.pop(), st.pop()
        st.append(np.asarray(_NUMPY[op](a, b), np.float64))
    return st[0].astype(np.float32)


def install(patch=setattr):
  def expr_plan(programs, out_cols, n_inputs, device):
    plan = K.ExprPlan(programs, out_cols, n_inputs, device)
    plan.programs, plan.out_cols = list(programs), list(out_cols)
    return plan

  def expr_eval(plan, inputs, dense):
    x = inputs.numpy()
    assert x.dtype == np.float64 and x.shape == (dense.shape[0], plan.n_inputs)
    for p, col in zip(plan.programs, plan.out_cols):
      dense[:, col] = torch.from_numpy(evaluate(p.ops, x))
    return dense
  patch(K, 'expr_plan', expr_plan)
  patch(K, 'expr_eval', expr_eval)

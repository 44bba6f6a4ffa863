// ExprFeature columns (input/input.py:507-535): every expression of the model is a postfix program over float64 inputs,
// compiled once on the host (easyrec_b200/expr.py).  One thread evaluates one (expression, sample) pair; consecutive
// threads take consecutive samples of one expression, so a warp runs one program in lock step.  The operand stack is
// ER_EXPR_MAX_STACK registers: a push shifts every slot down one place and an operator shifts them up, at indices known
// at compile time, so the stack never goes to local memory.  Arithmetic is float64 with the rounded intrinsics (never
// contracted into an FMA, as TF's separate ops are not); a comparison pushes 1.0 / 0.0, and the result is rounded to
// float32 (tf.cast of the bool or float64 value, compat/feature_column/feature_column.py:2710-2718).
#include "common.cuh"

namespace er {

constexpr int kExprThreads = 256;

template <typename F>
__device__ __forceinline__ void stack_shift_up(double (&s)[ER_EXPR_MAX_STACK], F top) {
  const double r = top(s[1], s[0]);
#pragma unroll
  for (int k = 1; k < ER_EXPR_MAX_STACK - 1; ++k) s[k] = s[k + 1];
  s[0] = r;
}

__global__ void __launch_bounds__(kExprThreads)
    expr_eval_kernel(const double* __restrict__ inputs, int64_t batch, int32_t n_inputs,
                     const er_expr_t* __restrict__ exprs, int32_t n_expr, const er_expr_op_t* __restrict__ ops,
                     int32_t n_ops, float* __restrict__ dense, int64_t dense_pitch) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= batch * n_expr) return;
  const int64_t e = t / batch, b = t - e * batch;
  const er_expr_t x = exprs[e];
  const double* in = inputs + b * n_inputs;
  double s[ER_EXPR_MAX_STACK];
#pragma unroll
  for (int k = 0; k < ER_EXPR_MAX_STACK; ++k) s[k] = 0.0;
  // (a descriptor reaching past the ops array stops there: the kernel reads nothing outside the arrays it is given)
  const int end = (unsigned)x.begin <= (unsigned)n_ops && x.n_ops <= n_ops - x.begin ? x.begin + x.n_ops : 0;
  for (int i = x.begin; i < end; ++i) {
    const er_expr_op_t op = ops[i];
    switch (op.op) {
      case ER_EXPR_LOAD:
      case ER_EXPR_CONST: {
        // an input index outside [0, n_inputs) reads NaN: no program can make this kernel read outside its inputs
        const double v = op.op == ER_EXPR_CONST ? op.value
                         : ((unsigned)op.arg < (unsigned)n_inputs ? in[op.arg] : __longlong_as_double(0x7ff8000000000000ll));
#pragma unroll
        for (int k = ER_EXPR_MAX_STACK - 1; k > 0; --k) s[k] = s[k - 1];
        s[0] = v;
        break;
      }
      case ER_EXPR_NEG: s[0] = -s[0]; break;
      case ER_EXPR_ADD: stack_shift_up(s, [](double a, double c) { return __dadd_rn(a, c); }); break;
      case ER_EXPR_SUB: stack_shift_up(s, [](double a, double c) { return __dsub_rn(a, c); }); break;
      case ER_EXPR_MUL: stack_shift_up(s, [](double a, double c) { return __dmul_rn(a, c); }); break;
      case ER_EXPR_DIV: stack_shift_up(s, [](double a, double c) { return __ddiv_rn(a, c); }); break;
      case ER_EXPR_GT: stack_shift_up(s, [](double a, double c) { return a > c ? 1.0 : 0.0; }); break;
      case ER_EXPR_GE: stack_shift_up(s, [](double a, double c) { return a >= c ? 1.0 : 0.0; }); break;
      case ER_EXPR_LT: stack_shift_up(s, [](double a, double c) { return a < c ? 1.0 : 0.0; }); break;
      case ER_EXPR_LE: stack_shift_up(s, [](double a, double c) { return a <= c ? 1.0 : 0.0; }); break;
      case ER_EXPR_EQ: stack_shift_up(s, [](double a, double c) { return a == c ? 1.0 : 0.0; }); break;
      case ER_EXPR_AND: stack_shift_up(s, [](double a, double c) { return (a != 0.0 && c != 0.0) ? 1.0 : 0.0; }); break;
      case ER_EXPR_OR: stack_shift_up(s, [](double a, double c) { return (a != 0.0 || c != 0.0) ? 1.0 : 0.0; }); break;
      default: break;
    }
  }
  if ((uint64_t)x.out_col < (uint64_t)dense_pitch) dense[b * dense_pitch + x.out_col] = __double2float_rn(s[0]);
}

}  // namespace er

extern "C" int er_expr_eval(const double* inputs, int64_t batch, int32_t n_inputs, const er_expr_t* exprs,
                            int32_t n_expr, const er_expr_op_t* ops, int32_t n_ops, int32_t max_depth, float* dense,
                            int64_t dense_pitch, er_stream_t stream) {
  using namespace er;
  ER_REQUIRE(batch >= 0 && n_inputs >= 0 && n_expr >= 0, "batch, n_inputs and n_expr must be >= 0");
  ER_REQUIRE(n_ops >= 0 && n_ops <= ER_EXPR_MAX_OPS, "n_ops must be in [0, ER_EXPR_MAX_OPS]");
  ER_REQUIRE(max_depth >= 0 && max_depth <= ER_EXPR_MAX_STACK, "max_depth must be in [0, ER_EXPR_MAX_STACK]");
  ER_REQUIRE(dense_pitch >= 1, "dense_pitch must be >= 1");
  if (batch == 0 || n_expr == 0) return ER_OK;
  ER_REQUIRE(n_ops >= n_expr && max_depth >= 1, "every program has at least one op and a stack of one");
  ER_REQUIRE(exprs && ops && dense, "null exprs, ops or dense array");
  ER_REQUIRE(n_inputs == 0 || inputs, "null inputs array");
  const int64_t grid = ceil_div(batch * n_expr, (int64_t)kExprThreads);
  ER_REQUIRE(grid <= 0x7fffffff, "batch * n_expr too large");
  expr_eval_kernel<<<(unsigned)grid, kExprThreads, 0, as_stream(stream)>>>(inputs, batch, n_inputs, exprs, n_expr, ops,
                                                                          n_ops, dense, dense_pitch);
  count_launches(1);
  ER_CUDA_LAUNCH_CHECK();
  return ER_OK;
}

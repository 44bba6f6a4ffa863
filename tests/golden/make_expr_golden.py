"""Golden vectors for ExprFeature, produced by EXECUTING THE REFERENCE'S OWN GRAMMAR.

utils/expr_util.py imports no TensorFlow: it is loaded from an EasyRec checkout as it is and its get_expression turns
every expression below into the Python text input/input.py:507-535 evals.  That text is evaluated here on float64
numpy arrays with `tf.greater / greater_equal / less / less_equal / equal` bound to numpy's comparisons, and the result
is cast to float32 (the numeric column's tf.cast).  numpy accepts a few forms TF rejects when it builds the graph (a
bare number left of a comparison, a bool compared with a number); tests/test_expr_feature_host.py refuses those by name.

  python tests/golden/make_expr_golden.py <EasyRec checkout>  -> tests/golden/reference_expr.json

Values travel as bit patterns (hex of the float64 inputs and float32 outputs), so NaN and -0.0 survive."""
import importlib.util
import json
import os
import sys
import types

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'reference_expr.json')

# input k of an expression = column k of a row
ROWS = [
    [0.0, 0.0, 0.0], [1.0, 1.0, 2.0], [2.0, 1.0, 1.0], [-1.0, 1.0, -2.0], [-0.0, 0.0, 1.0], [3.0, 5.0, 7.0],
    [5.0, 3.0, 8.0], [7.0, 2.0, 5.0], [2.5, -2.5, 0.1], [0.1, 0.2, 0.3], [16777216.0, 16777217.0, 16777218.0],
    [16777217.0, 16777216.0, 3.0], [9007199254740992.0, 9007199254740994.0, 1.0], [2.0 ** 60, -2.0 ** 60, 2.0 ** -60],
    [1e300, 1e300, 1e-300], [5e-324, -5e-324, 0.0], [float('nan'), 1.0, 2.0], [1.0, float('nan'), float('nan')],
    [float('inf'), float('-inf'), 0.0], [float('inf'), float('inf'), float('nan')], [4.0, 0.0, -0.0],
    [-7.0, -7.0, -7.0], [6.0, 1.0, 5.0], [0.3, 0.1, 0.2], [1.0 / 3.0, 3.0, 1.0], [3.4e38, 3.4e38, 10.0],
]

XYZ = ['x', 'y', 'z']
AGE = ['age_level', 'item_age_level']
EXPRESSIONS = [
    # multi_tower_on_taobao_for_expr.config
    ('age_level>=1', AGE), ('age_level<(item_age_level+5)', AGE), ('age_level==item_age_level', AGE),
    ('(age_level>=item_age_level) & (age_level<=(item_age_level+5))', AGE),
    ('(age_level>=item_age_level) | (age_level>5)', AGE),
    # comparisons, arithmetic, Python's precedence inside an operand, number arithmetic folded by Python
    ('x>y', XYZ), ('x>=y', XYZ), ('x<y', XYZ), ('x<=y', XYZ), ('x==y', XYZ), ('x + y', XYZ), ('x-y', XYZ),
    ('x*y', XYZ), ('x/y', XYZ), ('y/x', XYZ), ('x/0', XYZ), ('0/x', XYZ), ('x-y*z', XYZ), ('x*y+z', XYZ),
    ('x*y-z*x', XYZ), ('-x', XYZ), ('-x+y', XYZ), ('x - -y', XYZ), ('x+1e-3', XYZ), ('x + 9007199254740993', XYZ),
    ('x*3+0.1', XYZ), ('0.1+0.2+x', XYZ), ('x+0.1+0.2', XYZ), ('1/3+x', XYZ), ('2*3*x', XYZ), ('x*2**3', XYZ),
    ('x>=-1', XYZ), ('x >= y + z', XYZ), ('(x+1)>y', XYZ), ('x>(y+1)', XYZ), (' x== y ', XYZ),
    # & / |: folded left to right, then Python's precedence between the unparenthesised & and |
    ('(x>y) & (y>z)', XYZ), ('(x>y) | (y>z) & (z>x)', XYZ), ('(x>y)&(y>z)|(z>x)', XYZ), ('(x>=1)&(x<=5)|(y==2)', XYZ),
    ('(x>1)&((y>1)&((z>1)&(x<5)))', XYZ), ('((x>y))', XYZ), ('(x>y)==(y>z)', XYZ), ('x>y & y>z', XYZ),
    ('x>y | y', XYZ), ('(x>y)==((y>z)==((x>z)|(z>1)&(x>y-z*x)))', XYZ),
    # odd cases: an operand before "(" is dropped, an unclosed "(", "-" before "(", "=" alone, chains, spaces
    ('x*(y+z)', XYZ), ('(x>y', XYZ), ('-(x>y)', XYZ), ('x=y', XYZ), ('x>y>z', XYZ), ('x==y==z', XYZ),
    ('x>y)', XYZ), ('x y>1', XYZ), ('x>>y', XYZ), ('x<>y', XYZ), ('', XYZ),
    # a ")" that pops an operand where a sign was saved: the reference's _solve asserts
    ('+=><==&&)2)z', XYZ), ('2====0.5x<====y)x', XYZ),
    # forms TF rejects (or the reference cannot evaluate)
    ('w>1', XYZ), ('x>True', XYZ), ('x&y', XYZ), ('x+1&y>1', XYZ), ('5<x', XYZ), ('x**2>1', XYZ), ('x//2>1', XYZ),
    ('+x', XYZ), ('2>1', XYZ), ('1/0+x', XYZ), ('(x>y)>(y>z)', XYZ), ('(x>y)==1', XYZ), ('x%2', XYZ), ('x>1 & 1', XYZ),
]


def load_expr_util(checkout):
  path = os.path.join(checkout, 'easy_rec', 'python', 'utils', 'expr_util.py')
  spec = importlib.util.spec_from_file_location('expr_util', path)
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def main(checkout):
  expr_util = load_expr_util(checkout)
  rows = np.array(ROWS, np.float64)
  tf = types.SimpleNamespace(greater=np.greater, greater_equal=np.greater_equal, less=np.less,
                             less_equal=np.less_equal, equal=np.equal)
  cases = []
  for text, names in EXPRESSIONS:
    case = dict(expression=text, input_names=names)
    try:
      case['reference'] = expr_util.get_expression(text, names, prefix='expr_')
    except Exception as e:   # noqa: BLE001 - recorded: the reference fails on it
      case['error'] = 'get_expression: %s' % type(e).__name__
      cases.append(case)
      continue
    parsed = {'expr_' + n: rows[:, k].copy() for k, n in enumerate(names)}
    try:
      with np.errstate(all='ignore'):
        v = eval(case['reference'], {'tf': tf, 'parsed_dict': parsed})   # noqa: S307 - the reference's own step
      v = np.asarray(v)
      if v.shape != (rows.shape[0],) or v.dtype.kind not in 'bf':
        raise TypeError('not a per-sample bool / float tensor: %s %s' % (v.dtype, v.shape))
      case['out'] = [format(int(b), '08x') for b in v.astype(np.float32).view(np.uint32)]
    except Exception as e:   # noqa: BLE001 - recorded: the reference's eval fails on it
      case['error'] = 'eval: %s' % type(e).__name__
    cases.append(case)
  with open(OUT, 'w') as f:
    json.dump(dict(rows=[[format(int(b), '016x') for b in r.view(np.uint64)] for r in rows], cases=cases), f, indent=1)
    f.write('\n')
  print('wrote %s: %d expressions, %d evaluated' % (OUT, len(cases), sum('out' in c for c in cases)))


if __name__ == '__main__':
  main(sys.argv[1])

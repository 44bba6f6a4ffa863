"""ExprFeature: the reference's expression grammar (utils/expr_util.py, evaluated by input/input.py:507-535) compiled
once on the host into a postfix program that er_expr_eval runs per sample on the device.

The reference rewrites the expression into a Python string of tf.greater / greater_equal / less / less_equal / equal
calls joined by `&` / `|`, and `eval`s it on float64 tensors.  Its rules, followed here step for step:

  * every character of `+ - * / ( ) > < = & |` is an operator character, everything else (spaces included) operand
    text; a run of operand text is stripped and, when it is one of the feature's input_names, becomes that input;
  * a run of operator characters splits greedily into `>=`, `<=`, `==` and single characters;
  * `+ - * /` and a lone `=` are glued to the operand text around them, so an operand is Python arithmetic over
    inputs and numbers, evaluated with Python's precedence (a lone `=` makes it a syntax error);
  * `( ) > >= < <= == & |` are folded strictly left to right with one stack, with no precedence; only parentheses
    nest.  An operand followed by `(` is dropped (`a*(b+c)` is `b+c`), `a>b>c` compares the bool `a>b` with `c`, a
    `(` that is never closed is accepted, a `)` without its `(` is an error;
  * the comparisons become calls, `&` / `|` are written between their operands WITHOUT parentheses, so the string
    Python finally parses gives `&` precedence over `|`: `x | y & z` is `x | (y & z)`.

The compiler builds the same string, with `_in(k)` for input k and `_gt(a, b)`-style calls, parses it with Python's
own parser, and turns the tree into the program.  Anything the reference would not evaluate, or that TF would reject
when it builds the graph, is refused naming the feature: an unknown identifier (True / False included), `&` / `|` on
a non-bool, a comparison of a bool with a number or an ordering of two bools, a comparison whose left side is a bare
number (TF converts it to int32 / float32 first and then rejects the float64 right side), unary `+` on an input
(tf.Tensor defines no `__pos__`), an expression that reads no input, division by a literal zero in pure-number
arithmetic, and an empty or malformed expression.  `**` / `//` / `%` on an input are refused as not supported: TF
would evaluate them, but the program has no power, floor-division or modulo op (numbers alone are Python's: `x*2**3`
is `x*8`).  Sub-expressions without an input are evaluated by
Python as the reference's `eval` does (exact integers, then one conversion to float64).
"""
import ast
import collections
import operator

EXPR_LOAD, EXPR_CONST, EXPR_ADD, EXPR_SUB, EXPR_MUL, EXPR_DIV, EXPR_NEG = 0, 1, 2, 3, 4, 5, 6
EXPR_GT, EXPR_GE, EXPR_LT, EXPR_LE, EXPR_EQ, EXPR_AND, EXPR_OR = 7, 8, 9, 10, 11, 12, 13
MAX_STACK = 8       # ER_EXPR_MAX_STACK: er_expr_eval's register stack
MAX_OPS = 4096      # ER_EXPR_MAX_OPS: the ops of all programs of one call

# a compiled expression: ops [(opcode, input index, float64 constant)], 'bool' | 'float', the deepest stack it needs
Program = collections.namedtuple('Program', ['ops', 'result', 'depth'])

_OP_CHARS = set('+-*/()><=&|')
_TWO_CHAR = ('>=', '<=', '==')
_FOLD = ('(', ')', '>=', '<=', '==', '>', '<', '&', '|')
_CMP = {'>': '_gt', '>=': '_ge', '<': '_lt', '<=': '_le', '==': '_eq'}
_CMP_OP = {'_gt': EXPR_GT, '_ge': EXPR_GE, '_lt': EXPR_LT, '_le': EXPR_LE, '_eq': EXPR_EQ}
_ARITH = {ast.Add: EXPR_ADD, ast.Sub: EXPR_SUB, ast.Mult: EXPR_MUL, ast.Div: EXPR_DIV}
_PY_ARITH = {ast.Add: operator.add, ast.Sub: operator.sub, ast.Mult: operator.mul, ast.Div: operator.truediv,
             ast.Pow: operator.pow, ast.FloorDiv: operator.floordiv, ast.Mod: operator.mod}


class ExprError(ValueError):
  pass


def _tokens(expression, input_names):
  """operand strings and fold operators, in order (expr_util._get_expression_list)"""
  pieces, word, ops = [], '', ''

  def operand(w):
    w = w.strip()
    return '_in(%d)' % input_names.index(w) if w in input_names else w

  def split(run):
    i = 0
    while i < len(run):
      n = 2 if run[i:i + 2] in _TWO_CHAR else 1
      pieces.append(run[i:i + n])
      i += n
  for ch in expression:
    if ch in _OP_CHARS:
      if word:
        pieces.append(operand(word))
        word = ''
      ops += ch
    else:
      word += ch
      if ops:
        split(ops)
        ops = ''
  if word:
    pieces.append(operand(word))
  if ops:
    split(ops)
  out = ['']
  for p in pieces:
    if p in _FOLD or out[-1] in _FOLD:
      out.append(p)
    else:
      out[-1] += p
  return [p for p in out if p]


def source(expression, input_names):
  """the Python text the reference evaluates, with `_in(k)` for input k and `_gt(a, b)`... for tf.greater..."""
  stack, sign, operand = [], '', ''

  def reduce(rhs, sign):
    if not stack or rhs == '' or sign == '':
      return rhs
    lhs = stack.pop()
    if sign not in _CMP and sign not in ('&', '|'):
      # a ")" popped an operand where its "(" saved a sign: the reference's _solve asserts on it
      raise ExprError('%r stands where an operator belongs' % sign)
    if sign in _CMP:
      return '%s(%s, %s)' % (_CMP[sign], lhs, rhs)
    return '%s %s %s' % (lhs, sign, rhs)
  for t in _tokens(expression, list(input_names)):
    if t not in _FOLD:
      operand = t
    elif t == '(':
      stack.append(sign)
      sign = ''
    else:
      r = reduce(operand, sign)
      operand = ''
      if t == ')':
        if not stack:
          raise ExprError('a ")" without its "("')
        sign = stack.pop()
        operand = reduce(r, sign)
        sign = ''
      else:
        sign = t
        stack.append(r)
  return reduce(operand, sign)


class _Node(object):
  """a typed sub-expression: ops of the program that compute it, or a Python number when it reads no input"""

  def __init__(self, kind, ops=(), value=None, depth=0):
    self.kind, self.ops, self.value, self.depth = kind, list(ops), value, depth


def _num(v):
  try:
    return float(v)
  except OverflowError:
    raise ExprError('the number %r does not fit a float64' % (v,))


def _load(node):
  """the ops that push a node's value (a number becomes a float64 constant)"""
  if node.kind == 'const':
    return [(EXPR_CONST, 0, _num(node.value))], 1
  return node.ops, node.depth


def _binary(code, a, b, kind):
  oa, da = _load(a)
  ob, db = _load(b)
  return _Node(kind, oa + ob + [(code, 0, 0.0)], depth=max(da, db + 1))


def _walk(n, input_names):
  if isinstance(n, ast.Constant):
    if type(n.value) not in (int, float):
      raise ExprError('%r is not a number' % (n.value,))
    return _Node('const', value=n.value)
  if isinstance(n, ast.Name):
    raise ExprError('%r is not one of input_names %s' % (n.id, list(input_names)))
  if isinstance(n, ast.Call) and isinstance(n.func, ast.Name) and n.func.id == '_in':
    return _Node('float', [(EXPR_LOAD, n.args[0].value, 0.0)], depth=1)
  if isinstance(n, ast.Call) and isinstance(n.func, ast.Name) and n.func.id in _CMP_OP:
    a, b = (_walk(x, input_names) for x in n.args)
    name = {v: k for k, v in _CMP.items()}[n.func.id]
    if a.kind == 'const' and b.kind == 'const':
      raise ExprError('the comparison %s of two numbers reads no input' % name)
    if a.kind == 'const':
      raise ExprError('a bare number on the left of %s (TF converts it to int32 / float32 and then rejects the float64 '
                      'right side)' % name)
    if (a.kind == 'bool') != (b.kind == 'bool'):
      raise ExprError('%s compares a bool with a number' % name)
    if a.kind == 'bool' and n.func.id != '_eq':
      raise ExprError('%s orders two bools' % name)
    return _binary(_CMP_OP[n.func.id], a, b, 'bool')
  if isinstance(n, ast.UnaryOp) and isinstance(n.op, (ast.USub, ast.UAdd)):
    a = _walk(n.operand, input_names)
    if a.kind == 'const':
      return _Node('const', value=-a.value if isinstance(n.op, ast.USub) else +a.value)
    if a.kind == 'bool' or isinstance(n.op, ast.UAdd):
      raise ExprError('unary %s on %s' % ('-' if isinstance(n.op, ast.USub) else '+',
                                          'a bool' if a.kind == 'bool' else 'an input (tf.Tensor has no __pos__)'))
    return _Node('float', a.ops + [(EXPR_NEG, 0, 0.0)], depth=a.depth)
  if isinstance(n, ast.BinOp) and type(n.op) in _PY_ARITH:
    a, b = _walk(n.left, input_names), _walk(n.right, input_names)
    if 'bool' in (a.kind, b.kind):
      raise ExprError('arithmetic on a bool')
    if a.kind == 'const' and b.kind == 'const':
      # numbers only: Python computes it, exact integers included, before any tensor sees it
      if isinstance(n.op, ast.Pow) and abs(b.value) > 1100:
        raise ExprError('the power %r ** %r' % (a.value, b.value))
      try:
        return _Node('const', value=_PY_ARITH[type(n.op)](a.value, b.value))
      except (ZeroDivisionError, OverflowError) as e:
        raise ExprError('the number arithmetic fails in Python: %s' % e)
    if type(n.op) not in _ARITH:
      raise ExprError('the operator %s on an input is not one of + - * /' % type(n.op).__name__)
    return _binary(_ARITH[type(n.op)], a, b, 'float')
  if isinstance(n, ast.BinOp) and isinstance(n.op, (ast.BitAnd, ast.BitOr)):
    a, b = _walk(n.left, input_names), _walk(n.right, input_names)
    sym = '&' if isinstance(n.op, ast.BitAnd) else '|'
    if a.kind != 'bool' or b.kind != 'bool':
      raise ExprError('%s on a non-bool operand' % sym)
    return _binary(EXPR_AND if sym == '&' else EXPR_OR, a, b, 'bool')
  if isinstance(n, ast.BinOp):
    raise ExprError('the operator %s is not one of + - * /' % type(n.op).__name__)
  raise ExprError('%s is not an arithmetic expression' % type(n).__name__)


def compile_expression(name, expression, input_names):
  """ExprFeature `name` -> Program over its input_names (input k = column k of its inputs).  Raises ExprError (a
  ValueError) naming the feature for anything the reference would not evaluate or TF would reject."""
  try:
    text = source(expression, input_names)
    if not text.strip():
      raise ExprError('the expression is empty')
    try:
      tree = ast.parse(text.strip(), mode='eval')
    except SyntaxError:
      raise ExprError('%r is not valid once rewritten: %r' % (expression, text))
    node = _walk(tree.body, input_names)
    if node.kind == 'const':
      raise ExprError('the expression reads no input')
    if node.depth > MAX_STACK:
      raise ExprError('it needs a stack of %d values; er_expr_eval holds %d' % (node.depth, MAX_STACK))
  except ExprError as e:
    raise ExprError('ExprFeature %s: expression %r: %s' % (name, expression, e))
  return Program(tuple(node.ops), node.kind, node.depth)


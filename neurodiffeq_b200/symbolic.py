"""Symbolic tracing of the user's problem definition into a per-point residual program.

The reference evaluates ``conditions.parameterize`` (conditions.py:41-57) and the user's ``diff_eqs`` (solvers.py:380)
eagerly on torch tensors and differentiates them with ``torch.autograd.grad(create_graph=True)``
(neurodiffeq.py:6-34).  Here the SAME Python callables are run ONCE on :class:`Sym` placeholders.  A ``Sym`` is a
node of a hash-consed expression DAG over per-point scalars:

* ``coord(i)``                -- the i-th sampled coordinate,
* ``net(n, o, alpha)``        -- the derivative jet of raw output ``o`` of network ``n``; ``alpha`` is a sorted tuple of
  coordinate indices (``()`` value, ``(0,)`` d/dx0, ``(0, 0)`` d2/dx0^2, ...).  These are what the forward kernel
  propagates through the FCNN in Taylor mode (SURVEY.md Appendix A),
* arithmetic / elementary functions of those.

``diff(u, t, order)`` on Syms is exact symbolic differentiation w.r.t. a coordinate leaf; differentiating something
that does not depend on ``t`` gives the constant 0, matching the reference's ``allow_unused`` -> zeros behaviour
(neurodiffeq.py:22-31).  The traced residuals are then (optionally) reverse-differentiated symbolically w.r.t. every
``net`` leaf to obtain the per-point seeds  dL/d(jet)  that the reverse kernel needs, and everything is lowered to a
compact register-allocated bytecode (``lower``) that the CUDA kernels interpret in their epilogue.
"""
import math
import numbers

import numpy as np
import torch

# --- bytecode opcodes (must match csrc/pinnjet_program.cuh) -----------------------------------------------------------
OP_CONST, OP_COORD, OP_NET, OP_RBAR, OP_PARAM = 0, 1, 2, 3, 4
OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_NEG = 5, 6, 7, 8, 9
OP_SIN, OP_COS, OP_EXP, OP_LOG, OP_TANH, OP_SQRT, OP_ABS, OP_SIGN, OP_POWC, OP_RCP = 10, 11, 12, 13, 14, 15, 16, 17, 18, 19
OP_ST_U, OP_ST_R, OP_ST_SEED = 20, 21, 22
OP_TAN, OP_SINH, OP_COSH, OP_ATAN, OP_ERF = 23, 24, 25, 26, 27
OP_ST_W = 28   # store a per-point weight of the combined second-order channel
OP_POW = 29    # slot ** slot: double programs only (an exponent float32 cannot hold, Program.to_f64)
OP_ST_COT = 30  # add a per-point cotangent dL/d(coefficient k) to the forward kernel's batch sum of coefficient k
OP_FIELD = 31   # load row `a` of the problem's coordinate-only field table (thin-plate-spline maps) at the point
MAX_FIELD_ROWS = 64   # field rows per problem (PJ_MAX_FIELD_ROWS of include/pinnjet.h)

_UNARY = {"neg": OP_NEG, "sin": OP_SIN, "cos": OP_COS, "exp": OP_EXP, "log": OP_LOG, "tanh": OP_TANH,
          "sqrt": OP_SQRT, "abs": OP_ABS, "sign": OP_SIGN, "rcp": OP_RCP, "tan": OP_TAN, "sinh": OP_SINH,
          "cosh": OP_COSH, "atan": OP_ATAN, "erf": OP_ERF}
_BINARY = {"add": OP_ADD, "sub": OP_SUB, "mul": OP_MUL, "div": OP_DIV}
_PY_UNARY = {"neg": lambda a: -a, "sin": math.sin, "cos": math.cos, "exp": math.exp, "log": math.log,
             "tanh": math.tanh, "sqrt": math.sqrt, "abs": abs, "sign": lambda a: (a > 0) - (a < 0),
             "rcp": lambda a: 1.0 / a, "tan": math.tan, "sinh": math.sinh, "cosh": math.cosh, "atan": math.atan,
             "erf": math.erf}

PARAM_LOSS_SCALE = 0  # OP_PARAM index: 2 / (N_global * n_eq)


class Graph:
    """Hash-consing context (one per traced problem)."""

    def __init__(self):
        self.table = {}
        self.nodes = []
        self.nets = []  # list of (module, in_coord tuple)
        self._net_ids = {}
        self.n_sampled = None   # number of sampled coordinates (set by the tracer); constant coordinates follow them
        self.const_coords = []  # values of the constant ("virtual") coordinates n_sampled, n_sampled + 1, ...
        self.coef_tensors = []  # trainable tensors whose elements are coefficients of the trace, in order of first use
        self.tps_groups = []    # thin-plate-spline centre sets: dict(centres [M, 2] float64, stiffness, coords (i, j))
        self.tps_maps = []      # (group, coefficients [M + 3] float64) of every distinct TPS map
        self._tps_keys = {}

    def _mk(self, op, args=(), imm=None):
        key = (op, tuple(a.idx for a in args), imm)
        node = self.table.get(key)
        if node is None:
            node = Sym(self, op, tuple(args), imm, len(self.nodes))
            self.table[key] = node
            self.nodes.append(node)
        return node

    # leaves
    def const(self, v):
        return self._mk("const", (), float(v))

    def coord(self, i):
        return self._mk("coord", (), int(i))

    def const_coord(self, value):
        """A coordinate leaf that has the same value at every sample point: what the reference builds with
        ``x1 = x_max * torch.ones_like(x, requires_grad=True)`` (conditions.py:585, 823) to evaluate -- and differentiate --
        the network AT a boundary.  It is a genuine extra coordinate of the traced problem: ``diff(net(x1, t), x1)`` is
        the derivative w.r.t. that network input, and nothing else depends on it."""
        if self.n_sampled is None:
            raise RuntimeError("constant coordinates can only be created while a problem is being traced")
        value = float(value)
        if value not in self.const_coords:
            self.const_coords.append(value)
        return self.coord(self.n_sampled + self.const_coords.index(value))

    def net(self, n, o, alpha=()):
        return self._mk("net", (), (int(n), int(o), tuple(sorted(alpha))))

    def ych(self, n, o, c):
        """channel-resolved jet leaf: output ``o`` of net ``n``, kernel channel ``c`` (after ChannelScheme)."""
        return self._mk("ych", (), (int(n), int(o), int(c)))

    def rbar(self, e):
        return self._mk("rbar", (), int(e))

    def theta(self, key):
        """A trainable scalar that enters the residual program directly (not through a network jet): the entries of a
        Resnet's bias-free shortcut matrix, and the user's equation coefficients (:meth:`coefficient`).  Constant w.r.t. the
        coordinates; lowered as an OP_CONST whose immediate the engine re-writes whenever the parameters change
        (``Program.patch``)."""
        return self._mk("theta", (), key)

    def coefficient(self, x):
        """The ``theta`` leaf of a trainable coefficient: a one-element tensor that requires grad and is either a leaf
        (``nn.Parameter(torch.tensor(0.5))``) or a one-element view of one (``c[0]`` of ``c = nn.Parameter(torch.zeros(3))``).
        Key ``("coef", id(leaf), flat index)``; the leaf tensors are kept in ``coef_tensors``.  Anything else that requires
        grad (a tensor computed from a trainable one, a multi-element view) raises ``NotImplementedError``."""
        leaf = x if x.is_leaf else x._base
        if x.numel() != 1 or leaf is None or not leaf.is_leaf or not leaf.requires_grad:
            raise NotImplementedError(f"{describe_tensor(x)} requires grad but is not a trainable coefficient: the fused "
                                      f"kernels train 1-element leaf tensors and 1-element views of leaf tensors only")
        if leaf is x:
            index = 0
        else:
            if x.dtype != leaf.dtype or not leaf.is_contiguous():
                raise NotImplementedError(f"{describe_tensor(x)}: a coefficient must be an element of a contiguous tensor "
                                          f"of the same dtype")
            index = x.storage_offset() - leaf.storage_offset()
            if not 0 <= index < leaf.numel():
                raise NotImplementedError(f"{describe_tensor(x)}: not an element of its base tensor")
        if not any(t is leaf for t in self.coef_tensors):
            self.coef_tensors.append(leaf)
        return self.theta(("coef", id(leaf), int(index)))

    def param(self, k):
        return self._mk("param", (), int(k))

    def tps_group(self, centres, stiffness, coords):
        """Index of the thin-plate-spline group with these centres [M, 2], stiffness and sampled coordinate indices (i, j),
        shared by every map over the same centres."""
        centres = np.ascontiguousarray(centres, dtype=np.float64).reshape(-1, 2)
        key = ("group", centres.tobytes(), float(stiffness), tuple(int(c) for c in coords))
        if key not in self._tps_keys:
            self._tps_keys[key] = len(self.tps_groups)
            self.tps_groups.append(dict(centres=centres, stiffness=float(stiffness), coords=key[3]))
        return self._tps_keys[key]

    def tps_map(self, group, coefs):
        """Index of the TPS map of ``group`` with coefficients [c_1..c_M, c_0, c_x, c_y] (de-duplicated by value)."""
        coefs = np.ascontiguousarray(coefs, dtype=np.float64).reshape(-1)
        if coefs.size != self.tps_groups[group]["centres"].shape[0] + 3:
            raise ValueError("a TPS map needs M + 3 coefficients")
        key = ("map", int(group), coefs.tobytes())
        if key not in self._tps_keys:
            self._tps_keys[key] = len(self.tps_maps)
            self.tps_maps.append((int(group), coefs))
        return self._tps_keys[key]

    def tps(self, group, map_idx, alpha=()):
        """Derivative ``alpha`` (sorted coordinate indices, order <= 2) of TPS map ``map_idx``: a coordinate-only leaf that
        the kernels read from a field row (OP_FIELD)."""
        return self._mk("tps", (), (int(group), int(map_idx), tuple(sorted(alpha))))

    def register_net(self, module, in_coord):
        key = (id(module), tuple(in_coord))
        if key not in self._net_ids:   # the same module at another coordinate list is another instance sharing its weights
            self._net_ids[key] = len(self.nets)
            self.nets.append((module, tuple(in_coord)))
        return self._net_ids[key]

    def lift(self, x):
        if isinstance(x, Sym):
            if x.g is not self:
                raise ValueError("mixing symbols of two traces")
            return x
        if isinstance(x, numbers.Number):
            return self.const(x)
        if isinstance(x, np.ndarray) and x.size == 1:
            return self.const(float(x.reshape(-1)[0]))
        if isinstance(x, torch.Tensor) and x.requires_grad:
            return self.coefficient(x)
        if isinstance(x, torch.Tensor) and x.numel() == 1:
            return self.const(float(x.detach().reshape(-1)[0]))
        raise TypeError(f"cannot use {type(x).__name__} inside a traced (fused) expression; "
                        f"only python numbers, 1-element tensors and symbols are allowed")

    # ---- constructors with local simplification ----------------------------------------------------------------------
    def add(self, a, b):
        a, b = self.lift(a), self.lift(b)
        if a.op == "const" and b.op == "const":
            return self.const(a.imm + b.imm)
        if a.is_zero():
            return b
        if b.is_zero():
            return a
        if b.op == "neg":
            return self.sub(a, b.args[0])
        if a.op == "neg":
            return self.sub(b, a.args[0])
        if a.idx > b.idx:
            a, b = b, a
        return self._mk("add", (a, b))

    def sub(self, a, b):
        a, b = self.lift(a), self.lift(b)
        if a.op == "const" and b.op == "const":
            return self.const(a.imm - b.imm)
        if b.is_zero():
            return a
        if a.is_zero():
            return self.neg(b)
        if a is b:
            return self.const(0.0)
        if b.op == "neg":
            return self.add(a, b.args[0])
        return self._mk("sub", (a, b))

    def mul(self, a, b):
        a, b = self.lift(a), self.lift(b)
        if a.op == "const" and b.op == "const":
            return self.const(a.imm * b.imm)
        if a.is_zero() or b.is_zero():
            return self.const(0.0)
        if a.is_const(1.0):
            return b
        if b.is_const(1.0):
            return a
        if a.is_const(-1.0):
            return self.neg(b)
        if b.is_const(-1.0):
            return self.neg(a)
        if a.op == "neg" and b.op == "neg":
            return self.mul(a.args[0], b.args[0])
        if a.op == "neg":
            return self.neg(self.mul(a.args[0], b))
        if b.op == "neg":
            return self.neg(self.mul(a, b.args[0]))
        # c1 * (c2 * x) -> (c1*c2) * x
        if a.op == "const" and b.op == "mul" and b.args[0].op == "const":
            return self.mul(self.const(a.imm * b.args[0].imm), b.args[1])
        if b.op == "const" and a.op == "mul" and a.args[0].op == "const":
            return self.mul(self.const(b.imm * a.args[0].imm), a.args[1])
        if a.idx > b.idx:
            a, b = b, a
        if b.op == "const":  # constants first
            a, b = b, a
        return self._mk("mul", (a, b))

    def div(self, a, b):
        a, b = self.lift(a), self.lift(b)
        if b.op == "const":
            if b.imm == 0.0:
                raise ZeroDivisionError("division by the constant 0 in a traced expression")
            return self.mul(a, self.const(1.0 / b.imm)) if not (a.op == "const") else self.const(a.imm / b.imm)
        if a.is_zero():
            return a
        if a.is_const(1.0):
            return self.unary("rcp", b)
        return self._mk("div", (a, b))

    def neg(self, a):
        a = self.lift(a)
        if a.op == "const":
            return self.const(-a.imm)
        if a.op == "neg":
            return a.args[0]
        if a.op == "sub":
            return self.sub(a.args[1], a.args[0])
        return self._mk("neg", (a,))

    def unary(self, name, a):
        a = self.lift(a)
        if name == "neg":
            return self.neg(a)
        if a.op == "const":
            return self.const(_PY_UNARY[name](a.imm))
        if name == "abs" and a.op == "abs":
            return a
        return self._mk(name, (a,))

    def powc(self, a, p):
        """a ** p for a python-number exponent."""
        a = self.lift(a)
        p = float(p)
        if a.op == "const":
            return self.const(a.imm ** p)
        if p == 0.0:
            return self.const(1.0)
        if p == 1.0:
            return a
        if p == 2.0:
            return self.mul(a, a)
        if p == 3.0:
            return self.mul(self.mul(a, a), a)
        if p == 4.0:
            s = self.mul(a, a)
            return self.mul(s, s)
        if p == -1.0:
            return self.unary("rcp", a)
        if p == -2.0:
            return self.unary("rcp", self.mul(a, a))
        if p == 0.5:
            return self.unary("sqrt", a)
        return self._mk("powc", (a,), p)

    def pow(self, a, b):
        if isinstance(b, numbers.Number):
            return self.powc(a, b)
        b = self.lift(b)
        if b.op == "const":
            return self.powc(a, b.imm)
        a = self.lift(a)
        return self.unary("exp", self.mul(b, self.unary("log", a)))  # a > 0 assumed, as torch.pow's real branch


class Sym:
    """A per-point scalar expression; quacks like the ``(N, 1)`` tensors the reference passes around."""
    __slots__ = ("g", "op", "args", "imm", "idx")
    __array_priority__ = 1000

    def __init__(self, g, op, args, imm, idx):
        self.g, self.op, self.args, self.imm, self.idx = g, op, args, imm, idx

    # -- predicates
    def is_zero(self):
        return self.op == "const" and self.imm == 0.0

    def is_const(self, v):
        return self.op == "const" and self.imm == v

    # -- tensor-like surface -------------------------------------------------------------------------------------------
    @property
    def shape(self):
        return _SymShape()

    def dim(self):
        return 2

    def size(self, d=None):
        return self.shape if d is None else self.shape[d]

    def view(self, *shape):
        return self

    reshape = view

    def requires_grad_(self, *a, **k):
        return self

    def detach(self):
        return self

    def clone(self):
        return self

    def to(self, *a, **k):
        return self

    def double(self):
        return self

    float = double

    def __getitem__(self, item):  # u[:, 0] style indexing of an (N,1) symbol
        return self

    def __hash__(self):
        return id(self)

    def __bool__(self):
        raise TypeError("the truth value of a traced (fused) expression is undefined; data-dependent Python control "
                        "flow cannot be fused into the residual kernel")

    # -- arithmetic (an (N, k) operand -- a traced block or k per-column constants -- makes the result a block)
    def __add__(self, o):
        return _columns_binary("add", self, o) if _is_block(o) else self.g.add(self, o)

    def __radd__(self, o):
        return _columns_binary("add", o, self) if _is_block(o) else self.g.add(o, self)

    def __sub__(self, o):
        return _columns_binary("sub", self, o) if _is_block(o) else self.g.sub(self, o)

    def __rsub__(self, o):
        return _columns_binary("sub", o, self) if _is_block(o) else self.g.sub(o, self)

    def __mul__(self, o):
        return _columns_binary("mul", self, o) if _is_block(o) else self.g.mul(self, o)

    def __rmul__(self, o):
        return _columns_binary("mul", o, self) if _is_block(o) else self.g.mul(o, self)

    def __truediv__(self, o):
        return _columns_binary("div", self, o) if _is_block(o) else self.g.div(self, o)

    def __rtruediv__(self, o):
        return _columns_binary("div", o, self) if _is_block(o) else self.g.div(o, self)

    def __neg__(self):
        return self.g.neg(self)

    def __pos__(self):
        return self

    def __abs__(self):
        return self.g.unary("abs", self)

    def __pow__(self, p):
        return self.g.pow(self, p)

    def __rpow__(self, base):
        if isinstance(base, numbers.Number):
            if base <= 0:
                raise ValueError("non-positive constant base in traced power")
            return self.g.unary("exp", self.g.mul(math.log(base), self))
        return self.g.pow(base, self)

    # methods torch tensors have and user lambdas use
    def sin(self):
        return self.g.unary("sin", self)

    def cos(self):
        return self.g.unary("cos", self)

    def tan(self):
        return self.g.unary("tan", self)

    def exp(self):
        return self.g.unary("exp", self)

    def log(self):
        return self.g.unary("log", self)

    def tanh(self):
        return self.g.unary("tanh", self)

    def sinh(self):
        return self.g.unary("sinh", self)

    def cosh(self):
        return self.g.unary("cosh", self)

    def atan(self):
        return self.g.unary("atan", self)

    arctan = atan

    def erf(self):
        return self.g.unary("erf", self)

    def sqrt(self):
        return self.g.unary("sqrt", self)

    def abs(self):
        return self.g.unary("abs", self)

    def sign(self):
        return self.g.unary("sign", self)

    def square(self):
        return self.g.mul(self, self)

    def pow(self, p):
        return self.g.pow(self, p)

    def reciprocal(self):
        return self.g.unary("rcp", self)

    # -- numpy / torch protocol hooks ----------------------------------------------------------------------------------
    def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
        name = ufunc.__name__
        if method != "__call__":
            return NotImplemented
        return _dispatch_function(name, inputs, kwargs)

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        name = getattr(func, "__name__", str(func))
        return _dispatch_function(name, args, kwargs or {})

    def __repr__(self):
        return f"Sym#{self.idx}<{self.op}{'' if self.imm is None else ':' + str(self.imm)}>"


class SymColumns:
    """An (N, k) block of traced columns -- what ``EnsembleCondition.enforce`` returns for a k-output network
    (reference conditions.py:197-202 concatenates the re-parameterised columns) and what the function-basis code builds
    (reference function_basis.py).  Supports what user code does with such a tensor: ``u[:, i]``, ``u[:, i:i+1]`` (a
    column = a :class:`Sym`), ``u[:, i:j]`` (a narrower block), ``u.shape``; element-wise ``+ - * / **`` with numbers,
    (N, 1) columns, blocks of the same width and 1-D or (1, k) tensors / arrays (one constant per column); column-wise
    unary functions; ``torch.cat(..., dim=1)``; ``x.sum(dim=1)`` (a column); ``x.split(1, dim=1)``."""
    __array_priority__ = 1000

    def __init__(self, cols):
        self.cols = tuple(cols)
        if not self.cols or not all(isinstance(c, Sym) for c in self.cols):
            raise TypeError("SymColumns needs at least one traced column")

    @property
    def g(self):
        return self.cols[0].g

    @property
    def shape(self):
        return (-1, len(self.cols))

    def dim(self):
        return 2

    def size(self, d=None):
        return self.shape if d is None else self.shape[d]

    def __len__(self):
        raise TypeError("the number of sample points of a traced block is not known at trace time")

    def __getitem__(self, item):
        if not (isinstance(item, tuple) and len(item) == 2 and item[0] == slice(None)):
            raise NotImplementedError("traced (N, k) blocks support column indexing only: u[:, i] or u[:, i:j]")
        sel = item[1]
        if isinstance(sel, int):
            return self.cols[sel]
        if isinstance(sel, slice):
            picked = self.cols[sel]
        elif isinstance(sel, (list, tuple)):
            picked = tuple(self.cols[i] for i in sel)
        else:
            raise NotImplementedError(f"column selector {sel!r} on a traced block")
        if len(picked) == 0:
            raise IndexError("empty column selection")
        return picked[0] if len(picked) == 1 else SymColumns(picked)

    def __repr__(self):
        return f"SymColumns({len(self.cols)})"

    def __hash__(self):
        return id(self)

    def __bool__(self):
        raise TypeError("the truth value of a traced (fused) expression is undefined")

    def __add__(self, o):
        return _columns_binary("add", self, o)

    def __radd__(self, o):
        return _columns_binary("add", o, self)

    def __sub__(self, o):
        return _columns_binary("sub", self, o)

    def __rsub__(self, o):
        return _columns_binary("sub", o, self)

    def __mul__(self, o):
        return _columns_binary("mul", self, o)

    def __rmul__(self, o):
        return _columns_binary("mul", o, self)

    def __truediv__(self, o):
        return _columns_binary("div", self, o)

    def __rtruediv__(self, o):
        return _columns_binary("div", o, self)

    def __pow__(self, p):
        return _columns_binary("pow", self, p)

    def __neg__(self):
        return SymColumns([-c for c in self.cols])

    def __pos__(self):
        return self

    def __abs__(self):
        return _columns_unary("abs", (self,), {})

    def sum(self, dim=None, keepdim=False):
        return _columns_sum(self, dim)

    def split(self, split_size, dim=0):
        return _columns_split(self, split_size, dim)

    def __getattr__(self, name):   # tensor methods that are column-wise unary functions: x.sin(), x.exp(), ...
        if name in _COLUMNWISE_METHODS:
            return lambda *a, **k: _columns_unary(name, (self,) + a, k)
        raise AttributeError(name)

    def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
        if method != "__call__":
            return NotImplemented
        return _dispatch_function(ufunc.__name__, inputs, kwargs)

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        return _dispatch_function(getattr(func, "__name__", str(func)), args, kwargs or {})


class _SymShape(tuple):
    """Shape of a traced (N,1) column: compares equal to any other traced shape; index 1 is 1."""

    def __new__(cls):
        return super().__new__(cls, (-1, 1))

    def __eq__(self, other):
        return isinstance(other, _SymShape) or (isinstance(other, tuple) and len(other) == 2 and other[1] == 1)

    def __ne__(self, other):
        return not self.__eq__(other)

    def __hash__(self):
        return hash((-1, 1))


_NAME_ALIASES = {"multiply": "mul", "true_divide": "div", "divide": "div", "subtract": "sub", "negative": "neg",
                 "power": "pow", "absolute": "abs", "arctan": "atan", "float_power": "pow", "fabs": "abs"}


def _first_graph(args):
    for a in args:
        if isinstance(a, (Sym, SymColumns)):
            return a.g
        if isinstance(a, (list, tuple)):
            g = _first_graph(a)
            if g is not None:
                return g
    return None


_COLUMNWISE_METHODS = set(_UNARY) | {"square", "reciprocal", "rsqrt", "exp2", "sigmoid", "pow", "arctan", "absolute"}
_DUNDER = {"__add__": ("add", False), "__radd__": ("add", True), "__sub__": ("sub", False), "__rsub__": ("sub", True),
           "__mul__": ("mul", False), "__rmul__": ("mul", True), "__truediv__": ("div", False),
           "__rtruediv__": ("div", True), "__div__": ("div", False), "__rdiv__": ("div", True), "__pow__": ("pow", False)}


def describe_tensor(x):
    """How a refusal names a tensor: shape, dtype and the operation that computed it."""
    origin = "leaf" if x.grad_fn is None else type(x.grad_fn).__name__
    return f"tensor(shape={tuple(x.shape)}, dtype={x.dtype}, {origin})"


def _is_block(x):
    """An (N, k) operand: a traced block, or a tensor / array of k > 1 per-column constants."""
    return isinstance(x, SymColumns) or (isinstance(x, (torch.Tensor, np.ndarray)) and _numel(x) > 1)


def _numel(x):
    return x.numel() if isinstance(x, torch.Tensor) else x.size


def _column_values(x, width):
    """``x`` as a list of ``width`` per-column operands (numbers, Syms)."""
    if isinstance(x, SymColumns):
        if len(x.cols) == width:
            return list(x.cols)
        if len(x.cols) == 1:
            return list(x.cols) * width
        raise ValueError(f"traced blocks of widths {len(x.cols)} and {width} do not broadcast")
    if isinstance(x, torch.Tensor) and x.requires_grad:
        if x.numel() == 1:
            return [x] * width      # a trainable coefficient: Graph.lift makes it a theta leaf
        raise NotImplementedError(f"{describe_tensor(x)} requires grad: a trainable tensor of several elements cannot "
                                  f"enter a traced expression (use its elements, c[0], c[1], ..., as coefficients)")
    if isinstance(x, (torch.Tensor, np.ndarray)):
        a = x.detach().cpu().double().numpy() if isinstance(x, torch.Tensor) else np.asarray(x, dtype=np.float64)
        if a.size == 1:
            return [float(a.reshape(-1)[0])] * width
        if a.ndim == 1 or (a.ndim == 2 and a.shape[0] == 1):
            a = a.reshape(-1)
            if a.size == width:
                return [float(v) for v in a]
        raise NotImplementedError(f"a constant of shape {tuple(a.shape)} with a traced (N, {width}) block: only 1-D or "
                                  f"(1, {width}) per-column constants are supported")
    return [x] * width


def _block_width(args):
    widths = set()
    for a in args:
        if isinstance(a, SymColumns):
            widths.add(len(a.cols))
        elif isinstance(a, (torch.Tensor, np.ndarray)) and _numel(a) > 1:
            widths.add(_numel(a))
    widths.discard(1)
    if len(widths) > 1:
        raise ValueError(f"operands of widths {sorted(widths)} do not broadcast")
    return widths.pop() if widths else 1


def _columns_binary(name, a, b):
    width = _block_width((a, b))
    if not any(isinstance(x, (Sym, SymColumns)) for x in (a, b)):
        raise TypeError("no traced operand")
    g = _first_graph((a, b))
    out = []
    for x, y in zip(_column_values(a, width), _column_values(b, width)):
        out.append(g.pow(x, y) if name == "pow" else getattr(g, name)(x, y))
    return SymColumns(out)


def _columns_unary(name, args, kwargs):
    x = args[0]
    return SymColumns([_dispatch_function(name, (c,) + tuple(args[1:]), kwargs) for c in x.cols])


def _columns_sum(x, dim):
    if dim not in (1, -1):
        raise NotImplementedError("a traced (N, k) block can only be summed over its columns: sum(dim=1)")
    out = x.cols[0]
    for c in x.cols[1:]:
        out = out + c
    return out


def _columns_split(x, split_size, dim):
    if dim not in (1, -1):
        raise NotImplementedError("a traced (N, k) block can only be split into columns: split(size, dim=1)")
    if not isinstance(split_size, int) or split_size < 1:
        raise NotImplementedError("split of a traced block: an integer chunk size only")
    chunks = [x.cols[i:i + split_size] for i in range(0, len(x.cols), split_size)]
    return tuple(c[0] if len(c) == 1 else SymColumns(c) for c in chunks)


def _concat_columns(args, kwargs):
    seq = args[0]
    dim = kwargs.get("dim", kwargs.get("axis", args[1] if len(args) > 1 else 0))
    if dim not in (1, -1):
        raise NotImplementedError("torch.cat of traced columns: only along dim=1 (a block of columns); the network "
                                  "inputs are concatenated by `condition.enforce(net, *coords)`")
    cols = []
    for x in seq:
        if isinstance(x, SymColumns):
            cols += list(x.cols)
        elif isinstance(x, Sym):
            cols.append(x)
        else:
            raise NotImplementedError(f"torch.cat of a traced column with {type(x).__name__}")
    return SymColumns(cols)


def _dispatch_function(name, args, kwargs):
    """torch.<name>(...) / numpy.<name>(...) with at least one Sym / SymColumns argument."""
    g = _first_graph(args)
    name = _NAME_ALIASES.get(name, name)
    if name in _DUNDER:
        op, swap = _DUNDER[name]
        a, b = (args[1], args[0]) if swap else (args[0], args[1])
        if _is_block(a) or _is_block(b):
            return _columns_binary(op, a, b)
        return g.pow(a, b) if op == "pow" else getattr(g, op)(a, b)
    if name in ("cat", "concatenate", "concat"):
        return _concat_columns(args, kwargs)
    if name == "sum" and isinstance(args[0], SymColumns):
        return _columns_sum(args[0], kwargs.get("dim", args[1] if len(args) > 1 else None))
    if name == "split" and isinstance(args[0], SymColumns):
        return _columns_split(args[0], args[1] if len(args) > 1 else kwargs.get("split_size_or_sections"),
                              kwargs.get("dim", args[2] if len(args) > 2 else 0))
    if name in ("add", "sub", "mul", "div", "pow", "atan2") and (_is_block(args[0]) or _is_block(args[1])):
        if name in ("add", "sub") and kwargs.get("alpha", 1) != 1:
            raise NotImplementedError("alpha= in traced add/sub")
        if name == "atan2":
            width = _block_width(args[:2])
            return SymColumns([_dispatch_function("atan2", (y, x), {}) for y, x in
                               zip(_column_values(args[0], width), _column_values(args[1], width))])
        return _columns_binary(name, args[0], args[1])
    if isinstance(args[0], SymColumns):
        if name in _COLUMNWISE_METHODS:
            return _columns_unary(name, args, kwargs)
        if name in ("clone", "detach", "contiguous"):
            return args[0]
        raise NotImplementedError(f"`{name}` is not supported on a traced (N, k) block")
    if name in _UNARY:
        return g.unary(name, args[0])
    if name in ("add", "sub", "mul", "div"):
        out = getattr(g, name)(args[0], args[1])
        if name in ("add", "sub") and kwargs.get("alpha", 1) != 1:
            raise NotImplementedError("alpha= in traced add/sub")
        return out
    if name == "pow":
        return g.pow(args[0], args[1])
    if name == "square":
        a = g.lift(args[0])
        return g.mul(a, a)
    if name == "reciprocal":
        return g.unary("rcp", args[0])
    if name == "rsqrt":
        return g.unary("rcp", g.unary("sqrt", args[0]))
    if name in ("zeros_like", "ones_like", "full_like"):
        return g.const(0.0 if name == "zeros_like" else 1.0 if name == "ones_like" else args[1])
    if name in ("clone", "detach", "squeeze", "unsqueeze", "reshape", "view", "flatten", "contiguous"):
        return args[0]
    if name == "exp2":
        return g.unary("exp", g.mul(math.log(2.0), args[0]))
    if name == "sigmoid":
        return g.unary("rcp", g.add(1.0, g.unary("exp", g.neg(args[0]))))
    if name in ("atan2", "arctan2"):
        # half-angle form  atan2(y, x) = 2 atan(y / (sqrt(x^2 + y^2) + x)):  exact away from the non-positive x axis
        # (where the reference's own coordinate conversions are singular for the angles too)
        y, x = g.lift(args[0]), g.lift(args[1])
        r = g.unary("sqrt", g.add(g.mul(x, x), g.mul(y, y)))
        return g.mul(2.0, g.unary("atan", g.div(y, g.add(r, x))))
    if name == "stack":
        raise NotImplementedError("torch.stack of traced columns")
    raise NotImplementedError(f"`{name}` is not supported inside a fused residual / condition expression")


def is_symbolic(*xs):
    return any(isinstance(x, (Sym, SymColumns)) for x in xs)


# ----------------------------------------------------------------------------------------------------------------------
# differentiation
# ----------------------------------------------------------------------------------------------------------------------
def derivative(node, i, memo=None):
    """d node / d coord_i  as a new Sym (forward symbolic differentiation, memoised per (node, i))."""
    g = node.g
    if memo is None:
        memo = {}
    stack_guard = {}

    def d(n):
        key = n.idx
        if key in memo:
            return memo[key]
        op = n.op
        if op in ("const", "rbar", "param", "theta"):
            r = g.const(0.0)
        elif op == "ych":
            raise ValueError("cannot differentiate a channel-resolved expression")
        elif op == "coord":
            r = g.const(1.0 if n.imm == i else 0.0)
        elif op == "tps":
            group, map_idx, alpha = n.imm
            if i not in g.tps_groups[group]["coords"]:
                r = g.const(0.0)
            elif len(alpha) >= 2:
                raise NotImplementedError("derivative of order 3 of a thin-plate-spline interpolant: the field kernel "
                                          "evaluates them up to order 2")
            else:
                r = g.tps(group, map_idx, alpha + (i,))
        elif op == "net":
            net_idx, o, alpha = n.imm
            r = g.net(net_idx, o, alpha + (i,)) if i in g.nets[net_idx][1] else g.const(0.0)
        elif op == "add":
            r = g.add(d(n.args[0]), d(n.args[1]))
        elif op == "sub":
            r = g.sub(d(n.args[0]), d(n.args[1]))
        elif op == "mul":
            a, b = n.args
            r = g.add(g.mul(d(a), b), g.mul(a, d(b)))
        elif op == "div":
            a, b = n.args
            da, db = d(a), d(b)
            r = g.div(g.sub(da, g.mul(n, db)), b) if not db.is_zero() else g.div(da, b)
        elif op == "neg":
            r = g.neg(d(n.args[0]))
        else:
            a = n.args[0]
            da = d(a)
            if da.is_zero():
                r = da
            elif op == "sin":
                r = g.mul(g.unary("cos", a), da)
            elif op == "cos":
                r = g.neg(g.mul(g.unary("sin", a), da))
            elif op == "tan":
                r = g.mul(g.add(1.0, g.mul(n, n)), da)
            elif op == "exp":
                r = g.mul(n, da)
            elif op == "log":
                r = g.div(da, a)
            elif op == "tanh":
                r = g.mul(g.sub(1.0, g.mul(n, n)), da)
            elif op == "sinh":
                r = g.mul(g.unary("cosh", a), da)
            elif op == "cosh":
                r = g.mul(g.unary("sinh", a), da)
            elif op == "atan":
                r = g.div(da, g.add(1.0, g.mul(a, a)))
            elif op == "erf":
                r = g.mul(g.mul(2.0 / math.sqrt(math.pi), g.unary("exp", g.neg(g.mul(a, a)))), da)
            elif op == "sqrt":
                r = g.div(da, g.mul(2.0, n))
            elif op == "abs":
                r = g.mul(g.unary("sign", a), da)
            elif op == "sign":
                r = g.const(0.0)
            elif op == "rcp":
                r = g.neg(g.mul(g.mul(n, n), da))
            elif op == "powc":
                p = n.imm
                r = g.mul(g.mul(p, g.powc(a, p - 1.0)), da)
            else:
                raise NotImplementedError(op)
        memo[key] = r
        return r

    del stack_guard
    return d(node)


def sym_diff(u, t, order=1):
    """``diff`` on symbols (reference neurodiffeq.py:63-82 semantics for per-point-independent samples)."""
    g = _first_graph((u, t))
    u = g.lift(u)
    if not isinstance(t, Sym) or t.op != "coord":
        raise NotImplementedError("fused diff(u, t): `t` must be one of the sampled coordinates")
    out = u
    memo_by_level = {}
    for _ in range(order):
        out = derivative(out, t.imm, memo_by_level.setdefault(t.imm, {}))
    return out


def reverse_gradients(roots_and_cotangents, wrt_filter=lambda n: n.op in ("net", "ych")):
    """Symbolic reverse mode: returns {leaf Sym: adjoint Sym} for sum_k <cotangent_k, root_k>."""
    if not roots_and_cotangents:
        return {}
    g = roots_and_cotangents[0][0].g
    adj = {}
    order = topo_order([r for r, _ in roots_and_cotangents])
    for r, c in roots_and_cotangents:
        adj[r.idx] = g.add(adj[r.idx], c) if r.idx in adj else g.lift(c)
    out = {}

    def acc(n, v):
        if v.is_zero():
            return
        adj[n.idx] = g.add(adj[n.idx], v) if n.idx in adj else v

    for n in reversed(order):
        a_bar = adj.get(n.idx)
        if a_bar is None or a_bar.is_zero():
            continue
        op = n.op
        if wrt_filter(n):
            out[n] = a_bar
            continue
        if op in ("const", "coord", "rbar", "param", "theta", "net", "ych", "sign", "tps"):
            continue
        if op == "add":
            acc(n.args[0], a_bar)
            acc(n.args[1], a_bar)
        elif op == "sub":
            acc(n.args[0], a_bar)
            acc(n.args[1], g.neg(a_bar))
        elif op == "mul":
            a, b = n.args
            acc(a, g.mul(a_bar, b))
            acc(b, g.mul(a_bar, a))
        elif op == "div":
            a, b = n.args
            q = g.div(a_bar, b)
            acc(a, q)
            acc(b, g.neg(g.mul(q, n)))
        elif op == "neg":
            acc(n.args[0], g.neg(a_bar))
        else:
            a = n.args[0]
            if op == "sin":
                acc(a, g.mul(a_bar, g.unary("cos", a)))
            elif op == "cos":
                acc(a, g.neg(g.mul(a_bar, g.unary("sin", a))))
            elif op == "tan":
                acc(a, g.mul(a_bar, g.add(1.0, g.mul(n, n))))
            elif op == "exp":
                acc(a, g.mul(a_bar, n))
            elif op == "log":
                acc(a, g.div(a_bar, a))
            elif op == "tanh":
                acc(a, g.mul(a_bar, g.sub(1.0, g.mul(n, n))))
            elif op == "sinh":
                acc(a, g.mul(a_bar, g.unary("cosh", a)))
            elif op == "cosh":
                acc(a, g.mul(a_bar, g.unary("sinh", a)))
            elif op == "atan":
                acc(a, g.div(a_bar, g.add(1.0, g.mul(a, a))))
            elif op == "erf":
                acc(a, g.mul(a_bar, g.mul(2.0 / math.sqrt(math.pi), g.unary("exp", g.neg(g.mul(a, a))))))
            elif op == "sqrt":
                acc(a, g.div(a_bar, g.mul(2.0, n)))
            elif op == "abs":
                acc(a, g.mul(a_bar, g.unary("sign", a)))
            elif op == "rcp":
                acc(a, g.neg(g.mul(a_bar, g.mul(n, n))))
            elif op == "powc":
                acc(a, g.mul(a_bar, g.mul(n.imm, g.powc(a, n.imm - 1.0))))
            else:
                raise NotImplementedError(op)
    return out


def topo_order(roots):
    seen, order = set(), []
    for root in roots:
        if root.idx in seen:
            continue
        stack = [(root, 0)]
        while stack:
            node, k = stack.pop()
            if k == 0:
                if node.idx in seen:
                    continue
                seen.add(node.idx)
            if k < len(node.args):
                stack.append((node, k + 1))
                child = node.args[k]
                if child.idx not in seen:
                    stack.append((child, 0))
            else:
                order.append(node)
    return order


def substitute(roots, mapping):
    """Rebuild ``roots`` with leaf nodes replaced according to ``mapping`` {Sym: Sym}."""
    if not roots:
        return []
    g = roots[0].g
    memo = {k.idx: v for k, v in mapping.items()}
    for n in topo_order(roots):
        if n.idx in memo:
            continue
        if not n.args:
            memo[n.idx] = n
            continue
        new_args = [memo[a.idx] for a in n.args]
        if all(x is y for x, y in zip(new_args, n.args)):
            memo[n.idx] = n
        elif n.op in _BINARY:
            memo[n.idx] = getattr(g, n.op)(*new_args)
        elif n.op == "powc":
            memo[n.idx] = g.powc(new_args[0], n.imm)
        else:
            memo[n.idx] = g.unary(n.op, new_args[0])
    return [memo[r.idx] for r in roots]


# ----------------------------------------------------------------------------------------------------------------------
# jet channel scheme + lowering to bytecode
# ----------------------------------------------------------------------------------------------------------------------
class ChannelScheme:
    """Which derivative channels the kernels carry: value, n1 first-order directional derivatives D_v, the pure
    second derivatives D_v D_v of the FIRST n2 directions and, with ``max_order=3``, the pure third derivatives D_v^3 of the
    first n3 directions.  Mixed second partials are obtained by polarisation:
    d2/dxi dxj = ( D_{ei+ej}^2 - D_ei^2 - D_ej^2 ) / 2, so pure directional seconds suffice for every order-2 jet.  Of order
    3 only the pure partials d3/dxi3 exist (mixed ones would need third-order channels along polarisation directions)."""

    def __init__(self, n_coords, multi_indices, merged=None, max_order=2):
        """``merged``: optional list of coordinate groups that may share ONE direction because no network instance takes
        two members of a group as inputs (constant coordinates of different boundary instances): the direction is the sum
        of the group's axes, and restricted to any instance's inputs it is the axis of the one member that instance sees.
        ``max_order``: 2, or 3 to accept pure third-order multi-indices ``(i, i, i)``."""
        self.n_coords = n_coords
        self._group = {}
        for grp in (merged or []):
            for i in grp:
                self._group[i] = tuple(sorted(grp))
        firsts, seconds, thirds = set(), set(), set()
        self.mixed = set()
        for alpha in multi_indices:
            if len(alpha) == 0:
                continue
            if len(alpha) == 1:
                firsts.add(self.axis(alpha[0]))
            elif len(alpha) == 2:
                i, j = alpha
                if i == j:
                    seconds.add(self.axis(i))
                else:
                    if self.axis(i) == self.axis(j):
                        raise NotImplementedError("mixed derivative w.r.t. two coordinates that share a jet direction")
                    self.mixed.add((i, j))
                    seconds.add(self.axis(i))
                    seconds.add(self.axis(j))
                    seconds.add(self.mixed_dir(i, j))
            elif len(alpha) == 3 and max_order >= 3:
                if len(set(alpha)) != 1:
                    raise NotImplementedError(
                        f"mixed third-order derivative {tuple(alpha)} of a network output: the fused kernels carry pure "
                        f"third-order jets only (d3/dx3 along one coordinate)")
                thirds.add(self.axis(alpha[0]))
            else:
                raise NotImplementedError(
                    f"derivative of order {len(alpha)} of a network output: the fused kernels carry jets up to "
                    f"order {min(max_order, 3)} (SURVEY.md Appendix C caveat); higher orders are not implemented yet")
        seconds |= thirds
        firsts |= seconds
        # directions with a third-order channel first, then those with a second-order channel, then first-only ones;
        # axis-aligned ones in coordinate order within each group
        key = lambda v: (sum(abs(x) for x in v) != 1.0, [-x for x in v])  # noqa: E731
        third_sorted = sorted(thirds, key=key)
        sec_sorted = third_sorted + sorted(seconds - thirds, key=key)
        first_only = sorted(firsts - seconds, key=key)
        self.dirs = sec_sorted + first_only
        self.n1, self.n2, self.n3 = len(self.dirs), len(sec_sorted), len(third_sorted)

    def axis(self, i):
        """direction vector that differentiates w.r.t. coordinate i (its whole group when directions are shared)"""
        v = [0.0] * self.n_coords
        for k in self._group.get(i, (i,)):
            v[k] = 1.0
        return tuple(v)

    def mixed_dir(self, i, j):
        """polarisation direction for d2/dxi dxj"""
        return tuple(a + b for a, b in zip(self.axis(i), self.axis(j)))

    def pad_to(self, n1, n2, n3=0):
        """Add inert channels (zero direction vectors / unused second- and third-order slots) up to a compiled
        (n1, n2, n3)."""
        if n1 < self.n1 or n2 < self.n2 or n3 < self.n3 or n2 > n1 or n3 > n2:
            raise ValueError("cannot shrink a channel scheme")
        self.dirs = list(self.dirs) + [tuple([0.0] * self.n_coords)] * (n1 - self.n1)
        self.n1, self.n2, self.n3 = n1, n2, n3

    @property
    def n_channels(self):
        return 1 + self.n1 + self.n2 + self.n3

    def channel_of(self, alpha):
        """channel index of a (non-mixed) multi-index."""
        if len(alpha) == 0:
            return 0
        d = self.dirs.index(self.axis(alpha[0]))
        if len(alpha) == 1:
            return 1 + d
        if len(alpha) == 2:
            assert alpha[0] == alpha[1] and d < self.n2
            return 1 + self.n1 + d
        assert len(alpha) == 3 and len(set(alpha)) == 1 and d < self.n3
        return 1 + self.n1 + self.n2 + d

    def second_channel_of_dir(self, v):
        d = self.dirs.index(tuple(v))
        assert d < self.n2
        return 1 + self.n1 + d


class Program:
    """Lowered bytecode: int32 array [len, 4]  (op, dst, a, b)  -- see csrc/pinnjet_program.cuh."""

    def __init__(self, code, n_slots, exact_imm=None, patch=None, f64=False):
        self.code = np.asarray(code, dtype=np.int32).reshape(-1, 4)
        self.n_slots = n_slots
        self.exact_imm = exact_imm or {}  # instruction index -> float64 immediate (host-side checks only)
        self.patch = patch or {}          # instruction index -> key of the trainable scalar its immediate must hold
        self.f64 = f64                    # lowering for the double kernels (see to_f64)

    def __len__(self):
        return self.code.shape[0]

    def to_f64(self):
        """The program for the double kernels, with every immediate the exact double the host traced: OP_CONST holds the
        double's low word in ``a`` and its high word in ``b`` (patched constants: both words); an OP_POWC exponent
        float32 cannot hold exactly becomes OP_CONST into a fresh slot + OP_POW (two slots, double programs only).
        The float program is left as it is."""
        if self.f64:
            return self
        code, exact, patch, extra = [], {}, {}, self.n_slots
        for pc, (op, dst, a, b) in enumerate(self.code.tolist()):
            if op == OP_CONST:
                if pc in self.patch:
                    patch[len(code)] = self.patch[pc]
                    lo = hi = 0
                else:
                    v = self.exact_imm.get(pc, float(np.int32(a).view(np.float32)))
                    exact[len(code)] = v
                    lo, hi = _f64_words(v)
                code.append((OP_CONST, dst, lo, hi))
            elif op == OP_POWC and pc in self.exact_imm and float(np.float32(self.exact_imm[pc])) != self.exact_imm[pc]:
                exact[len(code)] = self.exact_imm[pc]
                code.append((OP_CONST, extra, *_f64_words(self.exact_imm[pc])))
                code.append((OP_POW, dst, a, extra))
            else:
                if op == OP_POWC and pc in self.exact_imm:
                    exact[len(code)] = self.exact_imm[pc]
                code.append((op, dst, a, b))
        n_slots = extra + 1 if any(c[0] == OP_POW for c in code) else self.n_slots
        return Program(code, n_slots, exact, patch, f64=True)


def _f32_bits(v):
    return int(np.array([v], dtype=np.float32).view(np.int32)[0])


def _f64_words(v):
    lo, hi = np.array([v], dtype=np.float64).view(np.int32).tolist()   # little endian: low word first
    return lo, hi


def _f64_of_words(lo, hi):
    return float(np.array([lo, hi], dtype=np.int32).view(np.float64)[0])


def lower(outputs, yrow_of, field_row_of=None):
    """``outputs``: list of (store_op, index, Sym).  ``yrow_of(net, out, channel_alpha) -> row`` in the y table,
    ``field_row_of(tps leaf imm) -> row`` in the field table.

    Emits instructions in topological order with liveness-based slot reuse (so that the interpreter's per-thread
    value file is small enough for shared memory)."""
    roots = [s for _, _, s in outputs]
    order = topo_order(roots)
    pos = {n.idx: k for k, n in enumerate(order)}
    last_use = {}
    for n in order:
        for a in n.args:
            last_use[a.idx] = max(last_use.get(a.idx, -1), pos[n.idx])
    store_at = {}
    for op, index, s in outputs:
        store_at.setdefault(s.idx, []).append((op, index))
        last_use[s.idx] = max(last_use.get(s.idx, -1), pos[s.idx])  # store happens right after definition
    free, slot_of, code, n_slots, exact, patch = [], {}, [], 0, {}, {}
    for k, n in enumerate(order):
        # allocate destination (operands may be released first only if this is their last use -> allows dst==src)
        srcs = [slot_of[a.idx] for a in n.args]
        for a in set(n.args):
            if last_use[a.idx] == k:
                free.append(slot_of[a.idx])
        if free:
            dst = free.pop()
        else:
            dst = n_slots
            n_slots += 1
        slot_of[n.idx] = dst
        op = n.op
        if op == "const":
            exact[len(code)] = n.imm
            code.append((OP_CONST, dst, _f32_bits(n.imm), 0))
        elif op == "theta":
            patch[len(code)] = n.imm
            code.append((OP_CONST, dst, 0, 0))
        elif op == "coord":
            code.append((OP_COORD, dst, n.imm, 0))
        elif op == "tps":
            code.append((OP_FIELD, dst, field_row_of(n.imm), 0))
        elif op == "ych":
            code.append((OP_NET, dst, yrow_of(*n.imm), 0))
        elif op == "net":
            raise ValueError("unresolved jet leaf: run ChannelScheme resolution before lowering")
        elif op == "rbar":
            code.append((OP_RBAR, dst, n.imm, 0))
        elif op == "param":
            code.append((OP_PARAM, dst, n.imm, 0))
        elif op in _BINARY:
            code.append((_BINARY[op], dst, srcs[0], srcs[1]))
        elif op == "powc":
            exact[len(code)] = n.imm
            code.append((OP_POWC, dst, srcs[0], _f32_bits(n.imm)))
        else:
            code.append((_UNARY[op], dst, srcs[0], 0))
        for st_op, index in store_at.get(n.idx, ()):
            code.append((st_op, index, dst, 0))
        if last_use.get(n.idx, -1) <= k:  # dead right away (store-only value)
            free.append(dst)
    return Program(code, max(n_slots, 1), exact, patch)


def depends_on_jets(expr):
    """True if the expression reads any network-output jet (i.e. is not a function of the coordinates alone)."""
    return any(n.op in ("net", "ych") for n in topo_order([expr]))


def evaluate_program(program, coords, y, rbar=None, params=None, n_u=0, n_r=0, n_seed=0, n_w=0, theta=None, n_cot=0,
                     fields=None):
    """Pure-numpy interpreter of the bytecode (host-side check of the lowering; float64).  ``theta``: values of the
    trainable scalars the program's patched constants stand for (``Program.patch`` keys -> float).  Float programs take
    their immediates from ``exact_imm``; double programs (``Program.to_f64``) are decoded from the code alone.
    ``n_cot > 0``: also return the per-point coefficient cotangents [n_cot, N] (OP_ST_COT) as a fourth result.
    ``fields``: the field rows [n_rows, N] that OP_FIELD reads."""
    n = coords.shape[1]
    val = np.zeros((program.n_slots, n))
    u, r, seed = np.zeros((n_u, n)), np.zeros((n_r, n)), np.zeros((n_seed, n))
    cot = np.zeros((n_cot, n))
    wout = np.zeros((n_w, n))
    bits = lambda b: float(np.array([b], dtype=np.int32).view(np.float32)[0])  # noqa: E731
    un = {OP_NEG: np.negative, OP_SIN: np.sin, OP_COS: np.cos, OP_EXP: np.exp, OP_LOG: np.log, OP_TANH: np.tanh,
          OP_SQRT: np.sqrt, OP_ABS: np.abs, OP_SIGN: np.sign, OP_RCP: lambda a: 1.0 / a, OP_TAN: np.tan,
          OP_SINH: np.sinh, OP_COSH: np.cosh, OP_ATAN: np.arctan}
    for pc, (op, dst, a, b) in enumerate(program.code.tolist()):
        if op == OP_CONST:
            if pc in program.patch:
                val[dst] = theta[program.patch[pc]]
            else:
                val[dst] = _f64_of_words(a, b) if program.f64 else program.exact_imm.get(pc, bits(a))
        elif op == OP_COORD:
            val[dst] = coords[a]
        elif op == OP_NET:
            val[dst] = y[a]
        elif op == OP_FIELD:
            val[dst] = fields[a]
        elif op == OP_RBAR:
            val[dst] = rbar[a]
        elif op == OP_PARAM:
            val[dst] = params[a]
        elif op == OP_ADD:
            val[dst] = val[a] + val[b]
        elif op == OP_SUB:
            val[dst] = val[a] - val[b]
        elif op == OP_MUL:
            val[dst] = val[a] * val[b]
        elif op == OP_DIV:
            val[dst] = val[a] / val[b]
        elif op == OP_POWC:
            val[dst] = val[a] ** (bits(b) if program.f64 else program.exact_imm.get(pc, bits(b)))
        elif op == OP_POW:
            val[dst] = val[a] ** val[b]
        elif op == OP_ERF:
            from scipy.special import erf
            val[dst] = erf(val[a])
        elif op == OP_ST_U:
            u[dst] = val[a]
        elif op == OP_ST_R:
            r[dst] = val[a]
        elif op == OP_ST_SEED:
            seed[dst] = val[a]
        elif op == OP_ST_W:
            wout[dst] = val[a]
        elif op == OP_ST_COT:
            cot[dst] += val[a]
        else:
            val[dst] = un[op](val[a])
    if n_w:
        return wout
    return (u, r, seed, cot) if n_cot else (u, r, seed)

"""Trace (conditions, diff_eqs) once -> the static description the CUDA engine needs.

This replaces, for the fused path, everything the reference does per batch in Python between ``_generate_batch`` and
``loss.backward()`` (solvers.py:369-395): the closed forms are extracted ONCE at solver construction:

* which networks are evaluated, fed by which coordinates (``BaseCondition.enforce``, conditions.py:41-57),
* which derivative jets of every raw network output the residuals need (-> :class:`ChannelScheme`),
* an *eval* program   coords, jets -> u_k (re-parameterised functions), r_e (residuals),
* a *train* program   coords, jets -> r_e and the seeds  dL/d(jet)  for  L = mean(r^2)  (solvers.py:218) or for an
  externally supplied  dL/dr  (custom ``loss_fn``), obtained by symbolic reverse differentiation.
"""
import numpy as np
import torch.nn as nn

from . import symbolic as S
from .networks import SinActv

ACT_TANH, ACT_SIN, ACT_SIGMOID, ACT_SILU, ACT_ELU = 0, 1, 2, 3, 4   # PJ_ACT_* of include/pinnjet.h
# torch modules with a jet rule in the kernels, matched by exact type: a subclass may compute something else (the
# product's own Swish(beta=1) equals SiLU but stays on the autograd path with its trainable-scalar variants)
_TORCH_ACTS = {nn.Sigmoid: ACT_SIGMOID, nn.SiLU: ACT_SILU, nn.ELU: ACT_ELU}


def check_jet_order(jet_order):
    """``None`` / ``2`` (the default: jets up to order 2) or ``3`` (also pure third derivatives); else ``ValueError``."""
    if jet_order is None or (isinstance(jet_order, int) and jet_order == 2):
        return 2
    if isinstance(jet_order, int) and jet_order == 3:
        return 3
    raise ValueError(f"jet_order must be 2 or 3, not {jet_order!r}")


class NetDescription:
    """Static view of one distinct network: widths, activation, the nn.Linear modules, input coordinates."""

    def __init__(self, module, in_coord):
        self.module = module
        self.in_coord = tuple(in_coord)
        self.skip = None
        if hasattr(module, "residual") and hasattr(module, "skip_connection"):   # Resnet (reference networks.py:73-106)
            self.skip = module.skip_connection
            if not isinstance(self.skip, nn.Linear) or self.skip.bias is not None:
                raise NotImplementedError("a Resnet shortcut must be a bias-free nn.Linear")
            module = module.residual
        seq = getattr(module, "NN", module)
        if not isinstance(seq, nn.Sequential):
            raise NotImplementedError(
                f"fused path supports FCNN-style networks (nn.Sequential of Linear/activation); got "
                f"{type(module).__name__}.  (Resnet / MonomialNN / custom modules: not implemented)")
        mods = list(seq)
        self.linears, acts = [], []
        for k, m in enumerate(mods):
            if k % 2 == 0:
                if not isinstance(m, nn.Linear):
                    raise NotImplementedError(f"expected nn.Linear at position {k} of the network, got {type(m).__name__}")
                if m.bias is None:
                    raise NotImplementedError("Linear layers without bias are not supported by the fused kernels")
                self.linears.append(m)
            else:
                acts.append(m)
        if len(mods) % 2 == 0 or len(self.linears) < 2:
            raise NotImplementedError("network must be Linear, actv, ..., Linear with at least one hidden layer")
        kinds = set()
        for a in acts:
            if isinstance(a, nn.Tanh):
                kinds.add(ACT_TANH)
            elif isinstance(a, SinActv) or type(a).__name__ == "SinActv":
                kinds.add(ACT_SIN)
            elif type(a) in _TORCH_ACTS:
                if type(a) is nn.ELU and a.alpha != 1.0:
                    raise NotImplementedError(f"nn.ELU(alpha={a.alpha}) has no jet rule in the fused kernels (alpha = 1 only)")
                kinds.add(_TORCH_ACTS[type(a)])
            else:
                raise NotImplementedError(f"activation {type(a).__name__} has no jet rule in the fused kernels "
                                          f"(implemented: nn.Tanh, SinActv, nn.Sigmoid, nn.SiLU, nn.ELU with alpha=1)")
        if len(kinds) != 1:
            raise NotImplementedError("all hidden activations of one network must be the same")
        self.act = kinds.pop()
        self.widths = [self.linears[0].in_features] + [m.out_features for m in self.linears]
        for a, b in zip(self.linears[:-1], self.linears[1:]):
            if a.out_features != b.in_features:
                raise ValueError("inconsistent layer widths")
        if self.skip is not None and (self.skip.in_features, self.skip.out_features) != (self.widths[0], self.widths[-1]):
            raise ValueError("Resnet shortcut and body disagree on the input / output widths")
        if self.widths[0] != len(self.in_coord):
            raise ValueError(f"network expects {self.widths[0]} inputs but the condition passes "
                             f"{len(self.in_coord)} coordinates")

    @property
    def n_out(self):
        return self.widths[-1]

    def parameters(self):
        out = []
        for m in self.linears:
            out += [m.weight, m.bias]
        if self.skip is not None:
            out.append(self.skip.weight)
        return out


class TracedProblem:
    def __init__(self, nets, conditions, diff_eqs, n_coords, coords_for_condition=None, pad_scheme=None,
                 combine_seconds=None, aux_outputs=None, enforce=None, jet_order=2):
        """``nets[k]`` / ``conditions[k]`` as in the reference solver; ``diff_eqs(*funcs, *coords)``.
        ``coords_for_condition(k, cond, coords) -> tuple`` lets SolverSpherical trim coordinates
        (reference solvers.py:894-916).  ``jet_order=3`` also accepts pure third derivatives of a network output
        (``pad_scheme`` is then called with a third argument, n3, when the problem has any)."""
        max_order = check_jet_order(jet_order)
        g = S.Graph()
        self.graph = g
        g.n_sampled = n_coords
        self.n_sampled = n_coords
        coords = [g.coord(i) for i in range(n_coords)]
        func_args, funcs, self.func_rows = [], [], []     # func_rows[k]: rows of u that make up function k (1 unless ensemble)
        for k, (net, cond) in enumerate(zip(nets, conditions)):
            cc = coords if coords_for_condition is None else coords_for_condition(k, cond, coords)
            # `enforce(net, cond, *coords)`: the solver's `compute_func_val` hook (reference solvers.py:267-279), which users
            # may override; default: the condition's own enforce
            f = cond.enforce(net, *cc) if enforce is None else enforce(net, cond, *cc)
            if isinstance(f, S.SymColumns):          # EnsembleCondition: one function = an (N, k) block of columns
                func_args.append(f)
                self.func_rows.append(list(range(len(funcs), len(funcs) + len(f.cols))))
                funcs += list(f.cols)
            else:
                f = g.lift(f)
                func_args.append(f)
                self.func_rows.append([len(funcs)])
                funcs.append(f)
        res = diff_eqs(*func_args, *coords) if diff_eqs is not None else []   # None: solution-only problem (u, no residual)
        # auxiliary per-point outputs (same arguments as diff_eqs): extra rows of `u` behind the functions, evaluated by
        # the forward kernel but not part of any loss (the 'h1 semi' loss keeps the user's residuals available this way)
        self.aux_rows = []
        if aux_outputs is not None:
            aux = aux_outputs(*func_args, *coords)
            aux = list(aux) if isinstance(aux, (list, tuple)) else [aux]
            self.aux_rows = list(range(len(funcs), len(funcs) + len(aux)))
            funcs += [g.lift(a) for a in aux]
        if isinstance(res, S.Sym) or not hasattr(res, "__len__"):
            res = [res]
        if any(isinstance(r, S.SymColumns) for r in res):
            raise NotImplementedError("a residual must be one (N, 1) column per equation; got a traced (N, k) block")
        residuals = [g.lift(r) for r in res]
        # constant coordinates created by the conditions (network evaluated at a boundary) follow the sampled ones; for the
        # kernels they are ordinary coordinate arrays (filled with the constant by the engine)
        self.const_coords = tuple(g.const_coords)
        n_coords = self.n_sampled + len(self.const_coords)
        self.n_coords = n_coords
        self.n_funcs, self.n_eq = len(funcs), len(residuals)
        self.nets = [NetDescription(m, ic) for m, ic in g.nets]
        if not self.nets:
            raise ValueError("no network is evaluated by the conditions")

        # --- which jets are needed -> channel scheme ------------------------------------------------------------------
        leaves = [n for n in S.topo_order(funcs + residuals) if n.op == "net"]
        for n in leaves:
            net_idx, o, _ = n.imm
            if o >= self.nets[net_idx].n_out:
                raise ValueError(f"condition selects output unit {o} of a network with "
                                 f"{self.nets[net_idx].n_out} outputs")
        self.scheme = S.ChannelScheme(n_coords, [n.imm[2] for n in leaves], merged=self._mergeable_constant_coords(),
                                      max_order=max_order)
        if pad_scheme is not None:  # round the scheme up to one the engine has a compiled kernel for
            sch = self.scheme
            self.scheme.pad_to(*(pad_scheme(sch.n1, sch.n2, sch.n3) if sch.n3 else pad_scheme(sch.n1, sch.n2)))
        C = self.scheme.n_channels
        self.yrow0 = []
        row = 0
        for nd in self.nets:
            self.yrow0.append(row)
            row += nd.n_out * C
        self.n_yrows = row

        mapping = {}
        for n in leaves:
            net_idx, o, alpha = n.imm
            if len(alpha) == 2 and alpha[0] != alpha[1]:
                i, j = alpha
                cd = self.scheme.second_channel_of_dir(self.scheme.mixed_dir(i, j))
                mapping[n] = g.mul(0.5, g.sub(g.sub(g.ych(net_idx, o, cd),
                                                    g.ych(net_idx, o, self.scheme.channel_of((i, i)))),
                                              g.ych(net_idx, o, self.scheme.channel_of((j, j)))))
            else:
                mapping[n] = g.ych(net_idx, o, self.scheme.channel_of(alpha))
        resolved = S.substitute(funcs + residuals, mapping)
        self.funcs, self.residuals = resolved[:self.n_funcs], resolved[self.n_funcs:]

        # --- combined second-order channel ("forward Laplacian" with per-point weights) ---------------------------------
        # If a residual is AFFINE in the pure second derivatives of a network output with coefficients that depend on the
        # coordinates only (Laplacians, spherical/cylindrical Laplacians, diffusion terms, ...), the kernels can carry ONE
        # channel  L = sum_d w_d(x) D_d^2  instead of n2 separate ones: linear layers commute with the weighted sum and the
        # activation rule becomes  a_L = s'' * sum_d w_d z_d^2 + s' z_L.  C drops from 1+n1+n2 to 2+n1 (C2: 5 -> 4 channels,
        # C4: 7 -> 5); the executed FLOPs shrink accordingly, the result is the same function of theta.
        self.wl = 0
        self.weight_exprs = []
        # (not with third-order channels: their rule needs the pure seconds of their directions)
        if combine_seconds is not None and not self.scheme.n3 and combine_seconds(self.scheme.n1, self.scheme.n2):
            self._try_combine_seconds()
            C = self.n_channels
            self.yrow0, row = [], 0
            for nd in self.nets:
                self.yrow0.append(row)
                row += nd.n_out * C
            self.n_yrows = row

        yrow = lambda net_idx, o, c: self.yrow0[net_idx] + o * C + c  # noqa: E731
        self._yrow = yrow
        # trainable coefficients (Graph.coefficient): their tensors follow the network parameters in the flat theta, element
        # by element; coef_index[key] is the position of a coefficient in that tail
        self.coef_tensors = list(g.coef_tensors)
        self.coef_index, off = {}, 0
        for t in self.coef_tensors:
            for i in range(t.numel()):
                self.coef_index[("coef", id(t), i)] = off + i
            off += t.numel()
        self.n_coef = off
        self._build_field_table()
        self.prog_w = (S.lower([(S.OP_ST_W, row, e) for row, e in self.weight_exprs], yrow, self._field_row)
                       if self.wl else None)
        # --- programs ---------------------------------------------------------------------------------------------------
        self.prog_eval = S.lower([(S.OP_ST_U, k, f) for k, f in enumerate(self.funcs)]
                                 + [(S.OP_ST_R, e, r) for e, r in enumerate(self.residuals)], yrow, self._field_row)
        self.prog_train = self._train_program(external_rbar=False)
        self._prog_train_ext = None

    def _build_field_table(self):
        """Thin-plate-spline leaves (pde.CustomBoundaryCondition) -> the field table the field kernel fills before the
        forward kernel runs: ``tps_groups`` (centres, stiffness, coordinate indices), ``tps_maps`` (group, coefficients)
        and ``field_rows``, one (group, map, alpha) per distinct leaf, which OP_FIELD reads by index."""
        g = self.graph
        exprs = self.funcs + self.residuals + [e for _, e in self.weight_exprs]
        leaves = sorted({n.imm for n in S.topo_order(exprs) if n.op == "tps"})
        if len(leaves) > S.MAX_FIELD_ROWS:
            raise NotImplementedError(f"{len(leaves)} thin-plate-spline field rows (the field kernel and the engine take "
                                      f"at most {S.MAX_FIELD_ROWS})")
        self.tps_groups, self.tps_maps = list(g.tps_groups), list(g.tps_maps)
        self.field_rows = leaves
        self._field_index = {imm: k for k, imm in enumerate(leaves)}

    def _field_row(self, imm):
        return self._field_index[imm]

    def _mergeable_constant_coords(self):
        """Constant coordinates (boundary abscissae) that never feed the same network instance can share one jet
        direction: e.g. IBVP1D with Neumann data on both ends evaluates the net at (x0, t) and at (x1, t) -- the
        derivative directions of x0 and x1 merge, and 4 directions (x, t, boundary, t + boundary) serve both instances."""
        consts = list(range(self.n_sampled, self.n_coords))
        groups = []
        for c in consts:
            for grp in groups:
                if all(not (c in nd.in_coord and m in nd.in_coord) for m in grp for nd in self.nets):
                    grp.append(c)
                    break
            else:
                groups.append([c])
        return [g for g in groups if len(g) > 1]

    @property
    def n_channels(self):
        return 2 + self.scheme.n1 if self.wl else self.scheme.n_channels

    def _try_combine_seconds(self):
        g = self.graph
        n1, n2 = self.scheme.n1, self.scheme.n2
        first_sec = 1 + n1
        is_sec = lambda leaf: leaf.op == "ych" and leaf.imm[2] >= first_sec  # noqa: E731
        for f in self.funcs:
            if any(is_sec(n) for n in S.topo_order([f])):
                return
        zero = g.const(0.0)
        owner, weights = {}, {}
        for e, r in enumerate(self.residuals):
            for leaf, coef in S.reverse_gradients([(r, g.const(1.0))]).items():
                if not is_sec(leaf):
                    continue
                if S.depends_on_jets(coef) or any(n.op == "theta" and n.imm[0] == "coef" for n in S.topo_order([coef])):
                    return                       # not affine in the second derivatives / jet-dependent coefficient / a
                    #                              trainable coefficient (the train program could not see its cotangent)
                net_idx, o, c = leaf.imm
                if owner.setdefault(net_idx, (e, o)) != (e, o):
                    return                       # two equations / outputs need different combinations of one net's jets
                weights.setdefault(net_idx, [zero] * n2)[c - first_sec] = coef
        if not owner:
            return
        new_res = list(self.residuals)
        for net_idx, (e, o) in owner.items():
            zero_map = {}
            for node in S.topo_order([new_res[e]]):
                if is_sec(node) and node.imm[0] == net_idx:
                    zero_map[node] = zero
            rest = S.substitute([new_res[e]], zero_map)[0]
            new_res[e] = g.add(rest, g.ych(net_idx, o, first_sec))
        self.residuals = new_res
        self.wl = n2
        self.weight_exprs = [(n * n2 + d, weights.get(n, [zero] * n2)[d]) for n in range(len(self.nets))
                             for d in range(n2)]

    def _train_program(self, external_rbar, with_func_adjoint=False):
        g = self.graph
        if external_rbar:
            cots = [(r, g.rbar(e)) for e, r in enumerate(self.residuals)]
            if with_func_adjoint:   # rows n_eq .. n_eq + n_funcs - 1 of the external buffer carry dL/du
                cots += [(f, g.rbar(self.n_eq + k)) for k, f in enumerate(self.funcs)]
        else:  # L = scale/2 * sum r^2 with scale = 2/(N n_eq)  ->  dL/dr = scale * r
            cots = [(r, g.mul(g.param(S.PARAM_LOSS_SCALE), r)) for r in self.residuals]
        is_coef = lambda n: n.op == "theta" and n.imm[0] == "coef"  # noqa: E731
        adj = S.reverse_gradients(cots, wrt_filter=lambda n: n.op in ("net", "ych") or is_coef(n))
        by_row = {self._yrow(*leaf.imm): expr for leaf, expr in adj.items() if not is_coef(leaf)}
        outs = [(S.OP_ST_R, e, r) for e, r in enumerate(self.residuals)]
        zero = g.const(0.0)
        for row in range(self.n_yrows):
            outs.append((S.OP_ST_SEED, row, by_row.get(row, zero)))
        # per-point cotangents of the coefficients; the forward kernel sums them over the batch
        outs += sorted(((S.OP_ST_COT, self.coef_index[leaf.imm], expr) for leaf, expr in adj.items() if is_coef(leaf)),
                       key=lambda o: o[1])
        return S.lower(outs, self._yrow, self._field_row)

    @property
    def prog_train_ext(self):
        if self._prog_train_ext is None:
            self._prog_train_ext = self._train_program(external_rbar=True)
        return self._prog_train_ext

    def extend_coords(self, coords):
        """[n_sampled, N] sampled coordinates -> [n_coords, N] with the constant coordinate rows appended."""
        coords = np.asarray(coords)
        if coords.shape[0] == self.n_coords or not self.const_coords:
            return coords
        extra = np.repeat(np.asarray(self.const_coords, dtype=coords.dtype)[:, None], coords.shape[1], axis=1)
        return np.concatenate([coords, extra], axis=0)

    @property
    def prog_train_ext_u(self):
        """Train program for a loss that depends on the residuals AND on the functions: the external cotangent buffer
        has n_eq + n_funcs rows, [dL/dr | dL/du]."""
        if getattr(self, "_prog_train_ext_u", None) is None:
            self._prog_train_ext_u = self._train_program(external_rbar=True, with_func_adjoint=True)
        return self._prog_train_ext_u

    def direction_matrix(self):
        """[n1, n_coords] float32: direction vectors of the first-order channels."""
        return np.asarray(self.scheme.dirs, dtype=np.float32).reshape(self.scheme.n1, self.n_coords)

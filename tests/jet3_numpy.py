"""TEST INFRASTRUCTURE ONLY (CPU, numpy float64): the numpy mirror of the kernels' algorithm (oracle/jet_numpy.py) for
channel schemes with pure third-order channels (``jet_order=3``).

Channels: 0 value | 1..n1 first order | n1+1..n1+n2 pure second order of the first n2 directions | n1+n2+1..n1+n2+n3
pure third order of the first n3 directions.  Along one direction, with s_k = sigma^(k)(z0):

    a3 = s3 z1^3 + 3 s2 z1 z2 + s1 z3
    z3_bar = s1 a3_bar,  z2_bar += 3 s2 z1 a3_bar,  z1_bar += (3 s3 z1^2 + 3 s2 z2) a3_bar,
    z0_bar += (s4 z1^3 + 3 s3 z1 z2 + s2 z3) a3_bar

Schemes without third-order channels are oracle/jet_numpy.py's business.  Never imported by the product.
"""
import numpy as np


def act_derivs4(act, z0):
    """value and first four derivatives of the activation at z0 (tanh: in terms of a = tanh(z0), as the kernels)."""
    if act == 0:
        a = np.tanh(z0)
        s1 = 1.0 - a * a
        s2 = -2.0 * a * s1
        s3 = -2.0 * s1 * s1 - 2.0 * a * s2
        s4 = -6.0 * s1 * s2 - 2.0 * a * s3
        return a, s1, s2, s3, s4
    a, c = np.sin(z0), np.cos(z0)
    return a, c, -a, -c, a


def _input_jet(x_in, dirs_in, C):
    a = np.zeros((C, x_in.shape[0], x_in.shape[1]))
    a[0] = x_in
    for f in range(dirs_in.shape[0]):
        a[1 + f] = dirs_in[f][:, None]
    return a        # second- and third-order channels of the inputs: 0


def a_from_z(act, z, n1, n2, n3):
    a0, s1, s2, s3, _ = act_derivs4(act, z[0])
    a = np.empty_like(z)
    a[0] = a0
    for f in range(n1):
        a[1 + f] = s1 * z[1 + f]
    for s in range(n2):
        a[1 + n1 + s] = s2 * z[1 + s] ** 2 + s1 * z[1 + n1 + s]
    for t in range(n3):
        z1, z2, z3 = z[1 + t], z[1 + n1 + t], z[1 + n1 + n2 + t]
        a[1 + n1 + n2 + t] = s3 * z1 ** 3 + 3.0 * s2 * z1 * z2 + s1 * z3
    return a


def forward_jets(weights, biases, act, x_in, dirs_in, n2, n3):
    """weights[l]: [out, in] (torch layout); x_in: [n_in, N]; dirs_in: [n1, n_in].  Returns (z-jets per hidden layer
    [C, h, N], raw output jets [C, n_out, N])."""
    n1 = dirs_in.shape[0]
    a = _input_jet(x_in, dirs_in, 1 + n1 + n2 + n3)
    z_store = []
    for l, (W, b) in enumerate(zip(weights, biases)):
        z = np.einsum("oi,cin->con", W, a)
        z[0] += b[:, None]
        if l == len(weights) - 1:
            return z_store, z
        z_store.append(z)
        a = a_from_z(act, z, n1, n2, n3)


def backward(weights, act, x_in, dirs_in, n2, n3, z_store, ybar):
    """ybar: [C, n_out, N] seeds dL/dy.  Returns (grad_W list [out, in], grad_b list)."""
    n1 = dirs_in.shape[0]
    C = 1 + n1 + n2 + n3
    L = len(weights)
    gW, gb = [None] * L, [None] * L
    zbar = ybar
    for l in range(L - 1, -1, -1):
        a_prev = a_from_z(act, z_store[l - 1], n1, n2, n3) if l > 0 else _input_jet(x_in, dirs_in, C)
        gW[l] = np.einsum("con,cin->oi", zbar, a_prev)
        gb[l] = zbar[0].sum(axis=1)
        if l == 0:
            break
        ab = np.einsum("oi,con->cin", weights[l], zbar)
        z = z_store[l - 1]
        _, s1, s2, s3, s4 = act_derivs4(act, z[0])
        zb = np.empty_like(z)
        zb[0] = s1 * ab[0]
        for f in range(n1):
            zb[1 + f] = s1 * ab[1 + f]
            zb[0] += s2 * z[1 + f] * ab[1 + f]
        for s in range(n2):
            zb[1 + n1 + s] = s1 * ab[1 + n1 + s]
            zb[1 + s] += 2.0 * s2 * z[1 + s] * ab[1 + n1 + s]
            zb[0] += (s3 * z[1 + s] ** 2 + s2 * z[1 + n1 + s]) * ab[1 + n1 + s]
        for t in range(n3):
            z1, z2, z3, a3 = z[1 + t], z[1 + n1 + t], z[1 + n1 + n2 + t], ab[1 + n1 + n2 + t]
            zb[1 + n1 + n2 + t] = s1 * a3
            zb[1 + n1 + t] += 3.0 * s2 * z1 * a3
            zb[1 + t] += (3.0 * s3 * z1 ** 2 + 3.0 * s2 * z2) * a3
            zb[0] += (s4 * z1 ** 3 + 3.0 * s3 * z1 * z2 + s2 * z3) * a3
        zbar = zb
    return gW, gb


def run_traced(tp, params_per_net, coords, n_global=None, want_grad=True, rbar=None, ubar=None):
    """oracle.jet_numpy.run_traced for a TracedProblem of any scheme, including third-order channels (no combined
    second-order channel, no Resnet shortcut: neither exists with n3 > 0 in the tests)."""
    from neurodiffeq_b200 import symbolic as S
    from oracle import jet_numpy
    if tp.scheme.n3 == 0:
        return jet_numpy.run_traced(tp, params_per_net, coords, n_global=n_global, want_grad=want_grad, rbar=rbar, ubar=ubar)
    assert not tp.wl and all(getattr(nd, "skip", None) is None for nd in tp.nets)
    coords = tp.extend_coords(np.asarray(coords, dtype=np.float64))
    N = coords.shape[1]
    dirs = np.asarray(tp.scheme.dirs, dtype=np.float64).reshape(tp.scheme.n1, tp.n_coords)
    n1, n2, n3 = tp.scheme.n1, tp.scheme.n2, tp.scheme.n3
    C = tp.n_channels
    y_rows = np.zeros((tp.n_yrows, N))
    stores = []
    for k, nd in enumerate(tp.nets):
        Ws = [np.asarray(p, dtype=np.float64) for p in params_per_net[k][0::2]]
        bs = [np.asarray(p, dtype=np.float64) for p in params_per_net[k][1::2]]
        x_in, d_in = coords[list(nd.in_coord)], dirs[:, list(nd.in_coord)]
        z_store, y = forward_jets(Ws, bs, nd.act, x_in, d_in, n2, n3)
        stores.append((Ws, x_in, d_in, z_store))
        for o in range(nd.n_out):
            for c in range(C):
                y_rows[tp.yrow0[k] + o * C + c] = y[c, o]
    u, r, _ = S.evaluate_program(tp.prog_eval, coords, y_rows, n_u=tp.n_funcs, n_r=tp.n_eq)
    out = dict(u=u, residual=r, loss=float((r ** 2).mean()) if r.size else 0.0, y=y_rows)
    if not want_grad:
        return out
    scale = 2.0 / ((N if n_global is None else n_global) * tp.n_eq)
    if rbar is None:
        _, r2, seeds = S.evaluate_program(tp.prog_train, coords, y_rows, params=[scale], n_r=tp.n_eq, n_seed=tp.n_yrows)
    elif ubar is None:
        _, r2, seeds = S.evaluate_program(tp.prog_train_ext, coords, y_rows, rbar=np.asarray(rbar, dtype=np.float64),
                                          params=[scale], n_r=tp.n_eq, n_seed=tp.n_yrows)
    else:
        ext = np.concatenate([np.asarray(rbar, dtype=np.float64), np.asarray(ubar, dtype=np.float64)], axis=0)
        _, r2, seeds = S.evaluate_program(tp.prog_train_ext_u, coords, y_rows, rbar=ext, params=[scale], n_r=tp.n_eq,
                                          n_seed=tp.n_yrows)
    assert np.allclose(r2, r)
    by_module = {}
    for k, nd in enumerate(tp.nets):
        Ws, x_in, d_in, z_store = stores[k]
        ybar = np.zeros((C, nd.n_out, N))
        for o in range(nd.n_out):
            for c in range(C):
                ybar[c, o] = seeds[tp.yrow0[k] + o * C + c]
        gW, gb = backward(Ws, nd.act, x_in, d_in, n2, n3, z_store, ybar)
        mine = [g for pair in zip(gW, gb) for g in pair]
        acc = by_module.setdefault(id(nd.module), mine)
        if acc is not mine:
            for a, m in zip(acc, mine):
                a += m
    out.update(grads=[g for gs in by_module.values() for g in gs], seeds=seeds, z_store=[s[3] for s in stores])
    return out

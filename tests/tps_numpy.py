"""TEST INFRASTRUCTURE: float64 numpy mirror of the field kernel (csrc/pinnjet_tps.cu) -- thin-plate-spline maps with their
first and second derivatives in closed form -- and of a traced irregular-domain problem: the network jets and parameter
gradients of oracle/jet_numpy.py with the residual programs interpreted on those field rows."""
import numpy as np

from neurodiffeq_b200 import symbolic as S
from oracle import jet_numpy


def tps_derivatives(centres, coefs, stiffness, x, y):
    """[6, N]: value, d/dx, d/dy, d2/dx2, d2/dxdy, d2/dy2 of the TPS map with coefficients [c_1..c_M, c_0, c_x, c_y]."""
    m = centres.shape[0]
    dx, dy = x[None, :] - centres[:, :1], y[None, :] - centres[:, 1:]
    q = dx ** 2 + dy ** 2 + stiffness ** 2
    lq = np.log(q)
    l1 = lq + 1.0
    phi = np.stack([q * lq, 2 * dx * l1, 2 * dy * l1, 2 * l1 + 4 * dx ** 2 / q, 4 * dx * dy / q, 2 * l1 + 4 * dy ** 2 / q])
    out = np.einsum("i,dik->dk", coefs[:m], phi)
    out[0] += coefs[m] + coefs[m + 1] * x + coefs[m + 2] * y
    out[1] += coefs[m + 1]
    out[2] += coefs[m + 2]
    return out


def field_rows(tp, coords):
    """The field rows [n_rows, N] of a traced problem at coords [n_coords, N]."""
    from neurodiffeq_b200.engine import field_derivative_code
    out = np.zeros((len(tp.field_rows), coords.shape[1]))
    for r, (gi, m, alpha) in enumerate(tp.field_rows):
        grp = tp.tps_groups[gi]
        cx, cy = grp["coords"]
        d = tps_derivatives(grp["centres"], tp.tps_maps[m][1], grp["stiffness"], coords[cx], coords[cy])
        out[r] = d[field_derivative_code(alpha, grp["coords"])]
    return out


def run_irregular(tp, params_per_net, coords, n_global=None, rbar=None, ubar=None, want_grad=True):
    """dict(u, residual, loss, grads) of a traced problem with field rows, as jet_numpy.run_traced returns them."""
    coords = tp.extend_coords(np.asarray(coords, dtype=np.float64))
    N = coords.shape[1]
    fields = field_rows(tp, coords)
    C, n2 = tp.n_channels, tp.scheme.n2
    dirs = np.asarray(tp.scheme.dirs, dtype=np.float64).reshape(tp.scheme.n1, tp.n_coords)
    wl_all = (S.evaluate_program(tp.prog_w, coords, np.zeros((1, N)), n_w=len(tp.nets) * tp.wl, fields=fields)
              if tp.wl else None)
    y_rows, stores = np.zeros((tp.n_yrows, N)), []
    for k, nd in enumerate(tp.nets):
        wl = wl_all[k * tp.wl:(k + 1) * tp.wl] if wl_all is not None else None
        Ws = [np.asarray(p, dtype=np.float64) for p in params_per_net[k][0::2]]
        bs = [np.asarray(p, dtype=np.float64) for p in params_per_net[k][1::2]]
        x_in, d_in = coords[list(nd.in_coord)], dirs[:, list(nd.in_coord)]
        z_store, y = jet_numpy.forward_jets(Ws, bs, nd.act, x_in, d_in, n2, wl)
        stores.append((Ws, x_in, d_in, z_store, wl))
        for o in range(nd.n_out):
            for c in range(C):
                y_rows[tp.yrow0[k] + o * C + c] = y[c, o]
    u, r, _ = S.evaluate_program(tp.prog_eval, coords, y_rows, n_u=tp.n_funcs, n_r=tp.n_eq, fields=fields)
    if not want_grad:
        return dict(u=u, residual=r)
    scale = 2.0 / ((N if n_global is None else n_global) * tp.n_eq)
    if rbar is None:
        prog, ext = tp.prog_train, None
    elif ubar is None:
        prog, ext = tp.prog_train_ext, np.asarray(rbar, np.float64)
    else:
        prog, ext = tp.prog_train_ext_u, np.concatenate([np.asarray(rbar, np.float64), np.asarray(ubar, np.float64)])
    _, _, seeds = S.evaluate_program(prog, coords, y_rows, rbar=ext, params=[scale], n_r=tp.n_eq, n_seed=tp.n_yrows,
                                     fields=fields)
    by_module = {}
    for k, nd in enumerate(tp.nets):
        Ws, x_in, d_in, z_store, wl = stores[k]
        ybar = np.zeros((C, nd.n_out, N))
        for o in range(nd.n_out):
            for c in range(C):
                ybar[c, o] = seeds[tp.yrow0[k] + o * C + c]
        gW, gb = jet_numpy.backward(Ws, nd.act, x_in, d_in, n2, z_store, ybar, wl)
        mine = [g for pair in zip(gW, gb) for g in pair]
        acc = by_module.setdefault(id(nd.module), mine)
        if acc is not mine:
            for a, m in zip(acc, mine):
                a += m
    return dict(u=u, residual=r, loss=float((r ** 2).mean()), grads=[g for gs in by_module.values() for g in gs])

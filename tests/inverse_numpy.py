"""TEST INFRASTRUCTURE: the numpy mirror (oracle/jet_numpy.py, float64) of a traced problem with trainable equation
coefficients: the network jets and parameter gradients of ``jet_numpy``, the residual programs interpreted with the
coefficients' values, and the coefficient gradients as the batch sums of the train program's OP_ST_COT cotangents."""
import numpy as np

from neurodiffeq_b200 import symbolic as S
from oracle import jet_numpy


def coefficient_values(tp):
    """Program.patch key -> current value of every coefficient of ``tp``."""
    flat = np.concatenate([t.detach().cpu().double().reshape(-1).numpy() for t in tp.coef_tensors])
    return {key: float(flat[k]) for key, k in tp.coef_index.items()}


def run_inverse(tp, params_per_net, coords, n_global=None, rbar=None, ubar=None):
    """dict(u, residual, loss, grads (per distinct module, as jet_numpy.run_traced), coef_grad [n_coef]).  ``rbar`` /
    ``ubar``: external cotangents dL/dr [n_eq, N] and dL/du [n_funcs, N] of a custom loss, as in run_traced."""
    coords = tp.extend_coords(np.asarray(coords, dtype=np.float64))
    N = coords.shape[1]
    theta = coefficient_values(tp)
    dirs = np.asarray(tp.scheme.dirs, dtype=np.float64).reshape(tp.scheme.n1, tp.n_coords)
    C, n2 = tp.n_channels, tp.scheme.n2
    wl_all = S.evaluate_program(tp.prog_w, coords, np.zeros((1, N)), n_w=len(tp.nets) * tp.wl, theta=theta) if tp.wl else None
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
    u, r, _ = S.evaluate_program(tp.prog_eval, coords, y_rows, n_u=tp.n_funcs, n_r=tp.n_eq, theta=theta)
    scale = 2.0 / ((N if n_global is None else n_global) * tp.n_eq)
    if rbar is None:
        prog, ext = tp.prog_train, None
    elif ubar is None:
        prog, ext = tp.prog_train_ext, np.asarray(rbar, np.float64)
    else:
        prog, ext = tp.prog_train_ext_u, np.concatenate([np.asarray(rbar, np.float64), np.asarray(ubar, np.float64)])
    _, _, seeds, cot = S.evaluate_program(prog, coords, y_rows, rbar=ext, params=[scale], n_r=tp.n_eq, n_seed=tp.n_yrows,
                                          theta=theta, n_cot=tp.n_coef)
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
    return dict(u=u, residual=r, loss=float((r ** 2).mean()), grads=[g for gs in by_module.values() for g in gs],
                coef_grad=cot.sum(axis=1))

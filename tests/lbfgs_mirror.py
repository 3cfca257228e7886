"""TEST INFRASTRUCTURE: torch mirrors of ``pj_lbfgs_step`` (csrc/pinnjet_lbfgs.cu).

``two_loop`` is the direction computation of ``torch.optim.LBFGS.step`` (torch/optim/lbfgs.py) as torch writes it, over
Python lists.  ``mirror_kernel`` has the signature of ``optim._lbfgs_kernel`` and does what one launch does, with torch
operations on the same buffers; the CPU tests swap it in so that ``FlatLBFGS``'s host logic runs without a GPU."""
import torch

from neurodiffeq_b200 import optim as O


def two_loop(g, old_dirs, old_stps, ro, H_diag):
    """d = -H g of torch's LBFGS.step for the pairs (oldest first); ``ro`` and ``H_diag`` as 0-dim tensors or numbers."""
    num_old = len(old_dirs)
    al = [None] * num_old
    q = g.neg()
    for i in range(num_old - 1, -1, -1):
        al[i] = old_stps[i].dot(q) * ro[i]
        q.add_(old_dirs[i], alpha=-al[i])
    d = r = torch.mul(q, H_diag)
    for i in range(num_old):
        be_i = old_dirs[i].dot(r) * ro[i]
        r.add_(old_stps[i], alpha=al[i] - be_i)
    return d


def ring_order(status, history):
    """Physical slots of the ring's pairs, oldest first."""
    head, num_old = int(status[O.HEAD]), int(status[O.NUM_OLD])
    return [(head + k) % history for k in range(num_old)]


def mirror_kernel(theta, grad, d, g_prev, old_dirs, old_stps, rho, status, loss, loss_host, lr, tolerance_grad,
                  tolerance_change, t_ls, flags, n_evals):
    st = status
    H = old_dirs.shape[0]
    n_iter0, prev_loss = float(st[O.N_ITER]), float(st[O.PREV_LOSS])
    line_search = bool(flags & O.LINE_SEARCH)
    take_ls_step = line_search and not flags & O.ENTRY
    t = t_ls if take_ls_step else float(st[O.T])
    loss = float(loss) if loss is not None else loss_host
    if take_ls_step:
        theta.add_(d, alpha=t)
    gmax, g1 = grad.abs().max(), grad.abs().sum()
    tdmax = d.mul(t).abs().max()
    y, s = grad.sub(g_prev), d.mul(t)
    ys, yy = y.dot(s), y.dot(y)
    opt = bool(gmax <= tolerance_grad)
    may_continue = bool(flags & O.MAY_CONTINUE)
    stop = O.RUNNING
    if flags & O.ENTRY:
        if opt:
            stop = O.STOP_GRAD
        elif not may_continue:
            stop = O.STOP_LIMIT
    elif not may_continue:
        stop = O.STOP_LIMIT
    elif opt:
        stop = O.STOP_GRAD
    elif bool(tdmax <= tolerance_change):
        stop = O.STOP_STEP
    elif abs(loss - prev_loss) < tolerance_change:
        stop = O.STOP_LOSS
    st[O.FUNC_EVALS] += n_evals
    st[O.LOSS], st[O.T], st[O.STOP] = loss, t, stop
    st[O.GMAX], st[O.G1], st[O.TDMAX] = float(gmax), float(g1), float(tdmax)
    if stop != O.RUNNING:
        return

    first = n_iter0 == 0
    if first:
        st[O.NUM_OLD], st[O.HEAD] = 0, 0
        d.copy_(grad.neg())
        H_diag = 1.0
    else:
        H_diag = st[O.H_DIAG].to(theta.dtype)
        if ys > 1e-10:
            num_old, head = int(st[O.NUM_OLD]), int(st[O.HEAD])
            if num_old == H:
                slot, head = head, (head + 1) % H
            else:
                slot, num_old = (head + num_old) % H, num_old + 1
            old_dirs[slot].copy_(y)
            old_stps[slot].copy_(s)
            rho[slot] = 1.0 / ys
            H_diag = ys / yy
            st[O.NUM_OLD], st[O.HEAD] = num_old, head
        order = ring_order(st, H)
        d.copy_(two_loop(grad, [old_dirs[k] for k in order], [old_stps[k] for k in order], [rho[k] for k in order], H_diag))
    g_prev.copy_(grad)
    t_new = min(1.0, 1.0 / g1) * lr if first else lr
    gtd = grad.dot(d)
    st[O.N_ITER] = n_iter0 + 1
    st[O.H_DIAG], st[O.T], st[O.GTD] = float(H_diag), float(t_new), float(gtd)
    st[O.PREV_LOSS], st[O.YS] = loss, float(ys)
    st[O.STOP] = O.STOP_DESCENT if gtd > -tolerance_change else O.RUNNING
    if not gtd > -tolerance_change and not line_search:
        theta.add_(d, alpha=t_new)

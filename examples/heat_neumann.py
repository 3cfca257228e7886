"""Heat equation u_t = 0.3 u_xx on [0, 1] with u(0, t) given and an insulated right end, u_x(1, t) = 0: the Neumann datum
makes ``IBVP1D`` evaluate the network AT x = 1 (reference conditions.py:585-596, 670-676); the fused engine runs that as a
second instance of the same network sharing its weights.  Trained with the 'h1'-free default loss and optim.FlatAdam.
python examples/heat_neumann.py   (needs an H100 and the built library)"""
import numpy as np
import torch

from neurodiffeq_b200 import diff
from neurodiffeq_b200.conditions import IBVP1D
from neurodiffeq_b200.generators import Generator2D
from neurodiffeq_b200.networks import FCNN
from neurodiffeq_b200.optim import FlatAdam
from neurodiffeq_b200.solvers import Solver2D


def main(epochs=3000):
    heat = lambda u, x, t: [diff(u, t) - 0.3 * diff(u, x, order=2)]                # noqa: E731
    rod = IBVP1D(x_min=0.0, x_max=1.0, t_min=0.0, t_min_val=lambda x: torch.sin(0.5 * np.pi * x),
                 x_min_val=lambda t: 0.0 * t, x_max_prime=lambda t: 0.0 * t)
    solver = Solver2D(heat, [rod], xy_min=(0, 0), xy_max=(1, 1), nets=[FCNN(2, 1, hidden_units=(64, 64))],
                      train_generator=Generator2D((128, 128), (0, 0), (1, 1), "equally-spaced-noisy"),
                      valid_generator=Generator2D((32, 32), (0, 0), (1, 1), "equally-spaced"))
    solver.optimizer = FlatAdam.for_solver(solver, lr=1e-3)
    solver.fit(max_epochs=epochs)
    xs, ts = np.meshgrid(np.linspace(0, 1, 51), np.linspace(0, 1, 51), indexing="ij")
    u = solver.get_solution()(xs, ts, to_numpy=True)
    exact = np.sin(0.5 * np.pi * xs) * np.exp(-0.3 * (0.5 * np.pi) ** 2 * ts)      # separable solution of this problem
    print(f"train loss {solver.metrics_history['train_loss'][-1]:.3e}   max |u - exact| = {np.abs(u - exact).max():.3e}")


if __name__ == "__main__":
    main()

"""Laplace's equation on the unit square -- the reference's README example (README.md:108-130 of NeuroDiffGym/neurodiffeq)
with the import root changed to ``neurodiffeq_b200``.  Needs an H100 (sm_90a) and the built library
(``python neurodiffeq_b200/csrc/build.py``).   python examples/laplace_2d.py"""
import numpy as np
import torch

from neurodiffeq_b200 import diff
from neurodiffeq_b200.conditions import DirichletBVP2D
from neurodiffeq_b200.generators import Generator2D
from neurodiffeq_b200.networks import FCNN
from neurodiffeq_b200.solvers import Solver2D


def main(epochs=2000):
    laplace = lambda u, x, y: [diff(u, x, order=2) + diff(u, y, order=2)]          # noqa: E731
    walls = DirichletBVP2D(x_min=0, x_min_val=lambda y: torch.sin(np.pi * y), x_max=1, x_max_val=lambda y: 0,
                           y_min=0, y_min_val=lambda x: 0, y_max=1, y_max_val=lambda x: 0)
    solver = Solver2D(laplace, [walls], xy_min=(0, 0), xy_max=(1, 1), nets=[FCNN(2, 1, hidden_units=(64, 64, 64))],
                      train_generator=Generator2D((128, 128), (0, 0), (1, 1), "equally-spaced-noisy"),
                      valid_generator=Generator2D((64, 64), (0, 0), (1, 1), "equally-spaced"))
    solver.fit(max_epochs=epochs)
    xs, ys = np.meshgrid(np.linspace(0, 1, 101), np.linspace(0, 1, 101), indexing="ij")
    u = solver.get_solution()(xs, ys, to_numpy=True)
    exact = np.sin(np.pi * ys) * np.sinh(np.pi * (1 - xs)) / np.sinh(np.pi)
    print(f"train loss {solver.metrics_history['train_loss'][-1]:.3e}   max |u - exact| = {np.abs(u - exact).max():.3e}")


if __name__ == "__main__":
    main()

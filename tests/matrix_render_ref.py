"""numpy restatement of the matrix-game frame (DESIGN.md §4.8 geometry, §4.9 board), the oracle of matrix_render_kernel.

Written from the specification: an N x A board of 40-px white cells behind 1-px black grid lines, row i for player i, column k for action k,
the cell of each player's previous action filled (46, 104, 190).  Integer arithmetic only, so frames compare bit for bit.
"""
from __future__ import annotations

import numpy as np

CELL = 40
CHOSEN = (46, 104, 190)


def frame_shape(n_agents, n_actions):
    return 1 + n_agents * (CELL + 1), 1 + n_actions * (CELL + 1), 3


def matrix_frame(last_action, n_actions):
    """last_action: int [N], each player's previous action (-1: none)."""
    last_action = np.asarray(last_action).astype(np.int64)
    H, W, _ = frame_shape(len(last_action), n_actions)
    f = np.zeros((H, W, 3), np.uint8)
    for i, a in enumerate(last_action):
        for k in range(n_actions):
            y, x = 1 + i * (CELL + 1), 1 + k * (CELL + 1)
            f[y:y + CELL, x:x + CELL] = CHOSEN if a == k else (255, 255, 255)
    return f

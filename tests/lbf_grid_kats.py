"""Hand-computed known-answer boards for the LBF grid observation (DESIGN.md Appendix A).

Each board: the field size, sight, food cells, players (row, col, level), the actions of one step (all NONE unless the board is about a
transition) and, per agent, the expected (3, W, W) window after that step, written out by hand as layer rows.  Window cell (y, x) of an agent
at (r, c) is field cell (r - k + y, c - k + x); off the field every layer is 0.  Layers: agents (levels), foods (levels), access (1 = an
empty field cell).
"""
import numpy as np

Z3 = ["000", "000", "000"]

KATS = [
    dict(name="corner_and_far_edge_k1", rows=5, cols=5, sight=1, foods={(1, 1): 3}, players=[(0, 0, 2), (4, 4, 1)], actions=[0, 0],
         want=[  # agent 0 at the top-left corner: the window's first row and column are padding
             (["000", "020", "000"], ["000", "000", "003"], ["000", "001", "010"]),
             # agent 1 at the bottom-right corner
             (["000", "010", "000"], Z3, ["110", "100", "000"])]),
    dict(name="top_edge_next_to_food_two_agents_k2", rows=6, cols=6, sight=2, foods={(1, 2): 2, (3, 3): 1}, players=[(0, 2, 1), (1, 3, 2)],
         actions=[0, 0],
         want=[  # agent 0 on the top edge, the food directly south, agent 1 diagonally south-east
             (["00000", "00000", "00100", "00020", "00000"], ["00000", "00000", "00000", "00200", "00000"],
              ["00000", "00000", "11011", "11001", "11111"]),
             # agent 1 at (1, 3): window rows -1..3, cols 1..5
             (["00000", "01000", "00200", "00000", "00000"], ["00000", "00000", "02000", "00000", "00100"],
              ["00000", "10111", "10011", "11111", "11011"])]),
    dict(name="food_removed_by_a_load_k1", rows=5, cols=5, sight=1, foods={(2, 2): 1, (4, 0): 1}, players=[(2, 1, 2), (0, 4, 1)], actions=[5, 0],
         want=[  # agent 0 loads the food east of it: the cell is empty and accessible afterwards
             (["000", "020", "000"], Z3, ["111", "101", "111"]),
             (["000", "010", "000"], Z3, ["000", "100", "110"])]),
    dict(name="two_players_on_one_cell_k1", rows=5, cols=5, sight=1, foods={(4, 4): 1}, players=[(2, 0, 1), (2, 1, 2), (2, 3, 3)],
         actions=[4, 4, 3],
         want=[  # players 1 and 2 both propose (2, 2) and stay; player 0 alone proposes (2, 1) and enters it, onto player 1: the later index's
                 # level is the one on the agents layer
             (["000", "020", "000"], Z3, ["111", "101", "111"]),
             (["000", "020", "000"], Z3, ["111", "101", "111"]),
             (["000", "030", "000"], Z3, ["111", "101", "111"])]),
    dict(name="k3_full_sight_3x3", rows=3, cols=3, sight=3, foods={(1, 1): 3}, players=[(0, 0, 1), (2, 2, 2)], actions=[0, 0],
         want=[  # agent 0 at (0, 0): the field occupies window rows / cols 3..5
             (["0000000", "0000000", "0000000", "0001000", "0000000", "0000020", "0000000"],
              ["0000000", "0000000", "0000000", "0000000", "0000300", "0000000", "0000000"],
              ["0000000", "0000000", "0000000", "0000110", "0001010", "0001100", "0000000"]),
             # agent 1 at (2, 2): the field occupies window rows / cols 1..3
             (["0000000", "0100000", "0000000", "0002000", "0000000", "0000000", "0000000"],
              ["0000000", "0000000", "0030000", "0000000", "0000000", "0000000", "0000000"],
              ["0000000", "0011000", "0101000", "0110000", "0000000", "0000000", "0000000"])]),
]


def materialise(kat):
    """(cfg kwargs, field int8 [R*C], players int8 [N][4], step, actions int32 [N])"""
    R, Cc, N = kat["rows"], kat["cols"], len(kat["players"])
    field = np.zeros((R, Cc), np.int8)
    for (r, c), lvl in kat["foods"].items():
        field[r, c] = lvl
    players = np.zeros((N, 4), np.int8)
    for i, (r, c, lvl) in enumerate(kat["players"]):
        players[i, :3] = (r, c, lvl)
    cfgkw = dict(rows=R, cols=Cc, n_agents=N, max_num_food=max(1, len(kat["foods"])), sight=kat["sight"], grid_observation=1)
    return cfgkw, field.reshape(-1), players, 0, np.array(kat["actions"], np.int32)


def expected(kat):
    """[N][D] float32: the hand-written windows, flattened in C order (layer, row, col)."""
    return np.stack([np.array([[[int(ch) for ch in row] for row in layer] for layer in agent], np.float32).reshape(-1) for agent in kat["want"]])

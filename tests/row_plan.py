"""The training pass's row split (csrc/learner.cuh: make_plan, episode_plan, cta_rows) restated in Python, and the branch class of a CTA; the
forward kernels' dense split (dense_plan, dense_classes, find_envs) after it; the recurrent kernels' sequence split (gru_plan, seq_class,
find_units) further down.

Which branches of the DQN tensor-core training pass run (csrc/tc_train.cu) depends on how many rows a CTA gets:
  - tc_dh1_kernel walks 128-row tiles; warpgroup 1 stages its two 32-row chunks of a tile at the top of the next tile, or after the loop when the
    last tile holds more than 64 rows; a chunk with no rows skips its MMAs;
  - tc_dw_kernel streams 32-row chunks in a do-while loop (one trip for a CTA of at most 32 rows), rebuilds H1 every second chunk into one of two
    buffers and zero-stages the rows past row_end of a partial chunk;
  - the fused FP32 train_kernel walks its tiles from the top down (its partial tile is the one at row_begin) and carries the next row's outputs
    across tile boundaries.
A CTA's class is (tiles: 1, 2 or 3+; 32-row chunks of its last tile that hold rows: 1-4; whether the last chunk is full), 24 classes in all.  Two
more cases concern a whole network: fewer than 64 rows in total, and a single CTA for the network.  find_batch picks a batch that reaches a class
on a given SM count, so that a device with another SM count still tests every class.

A CTA ends on an episode boundary, so its last rows are the final rows of its last episode, and row T of an episode has no TD error.  A tail
made of row T alone carries no gradient and tests nothing.  A CTA therefore counts for its class only when its last chunk is full or holds at
least TAIL_MIN rows, and the tests give the last episode of every CTA (last_episodes) its full length T: the tail -- the last chunk, and the rows warpgroup 1
stages after the loop -- then holds rows t < T that carry TD errors (tail_td_rows).

The actor-critic training pass (learner_kernels.cu: train_kernel<KP, kHeadA2cCritic> and <KP, kHeadA2cActor>, launched by a2c.cu's a2c_gradients
over episode_plan of the critic's and of the actor's networks) walks the same 128-row tiles from the top down, and row T of an episode carries
no loss there either (the heads run for t < T only): the same classes, find_batch, last_episodes and tail_td_rows apply to each of its passes.

The forward kernels serve the act step (model.act, get_value) over make_plan(ns, E, 1, n_sm, 32) (dense_plan: one row per environment and
agent, at most one CTA per 32 rows of a net), and the target-critic / PPO old-log-prob passes over episode_plan.  Each CTA walks its rows from
row_begin:
  - mlp_forward_kernel (FP32) in 128-row tiles, the last one partial unless the CTA's rows are a multiple of 128;
  - tc_forward_kernel (wgmma) with two warpgroups on alternating 64-row tiles: in the last 128 rows, c1 and c2 leave warpgroup 1 idle (c2-full
    is exactly 64 rows for warpgroup 0), c3 and c4 give it a partial or full tile.
So the 24 CLASSES name the forward's branches too; a forward has no loss rows, so every CTA counts (dense_classes)."""
from __future__ import annotations

import functools

TILE, CHUNK = 128, 32
TAIL_MIN = 8                   # rows of a partial last chunk for its CTA to count (TAIL_MIN - 1 of them carry TD errors)
CLASSES = tuple(f"t{t}{'+' if t == 3 else ''}-c{c}-{'full' if full else 'part'}" for t in (1, 2, 3) for c in (1, 2, 3, 4) for full in (True, False))
SMALL_NET = "net-rows<64"      # a network whose rows are fewer than the 64 a CTA is meant to get
ONE_CTA = "one-cta-net"        # a network trained by a single CTA
ALL_CLASSES = CLASSES + (SMALL_NET, ONE_CTA)


def nets_of(N, sharing):
    """agent -> network (codebase_b200.learner.sharing_to_nets): False one net per agent, True one shared net, a tuple of group labels"""
    if sharing is True:
        return [0] * N
    if sharing is False or sharing is None:
        return list(range(N))
    order = list(dict.fromkeys(sharing))
    return [order.index(i) for i in sharing]


def make_plan(agent_net, units_per_agent, unit_rows, n_cta_max, min_units):
    """make_plan: (cta_begin, slot_begin, slot_agent); CTAs [cta_begin[k], cta_begin[k + 1]) work on net k"""
    n_nets, N = max(agent_net) + 1, len(agent_net)
    slot_agent, slot_begin = [], []
    for k in range(n_nets):
        slot_begin.append(len(slot_agent))
        slot_agent += [a for a in range(N) if agent_net[a] == k]
    slot_begin.append(len(slot_agent))
    total = N * units_per_agent
    cta_begin, c = [], 0
    for k in range(n_nets):
        units = (slot_begin[k + 1] - slot_begin[k]) * units_per_agent
        want = n_cta_max * units // (total if total > 0 else 1)
        want = max(1, min(want, (units + min_units - 1) // min_units))
        cta_begin.append(c)
        c += want
    cta_begin.append(c)
    return dict(cta_begin=cta_begin, slot_begin=slot_begin, slot_agent=slot_agent, unit_rows=unit_rows, units_per_agent=units_per_agent)


def episode_plan(agent_net, episodes, T, n_cta_max):
    """a training pass over sampled episodes: one unit per episode (T + 1 rows), at least 64 rows per CTA"""
    return make_plan(agent_net, episodes, T + 1, n_cta_max, max(1, (64 + T) // (T + 1)))


def cta_rows(p, cta):
    """cta_rows: (net, row_begin, row_end) of CTA `cta`"""
    cb, sb = p["cta_begin"], p["slot_begin"]
    net = 0
    while net + 1 < len(cb) - 1 and cta >= cb[net + 1]:
        net += 1
    ncta, c = cb[net + 1] - cb[net], cta - cb[net]
    units = (sb[net + 1] - sb[net]) * p["units_per_agent"]
    return net, units * c // ncta * p["unit_rows"], units * (c + 1) // ncta * p["unit_rows"]


def all_cta_rows(p):
    return [cta_rows(p, c) for c in range(p["cta_begin"][-1])]


def classes(rows):
    """the branch class of a CTA of `rows` > 0 rows"""
    tiles = (rows + TILE - 1) // TILE
    last = rows - TILE * (tiles - 1)
    return f"t{min(tiles, 3)}{'+' if tiles >= 3 else ''}-c{(last + CHUNK - 1) // CHUNK}-{'full' if last % CHUNK == 0 else 'part'}"


def tail_counts(rows):
    """a CTA of `rows` rows counts for its class: its last chunk is full or holds at least TAIL_MIN rows"""
    return rows % CHUNK == 0 or rows % CHUNK >= TAIL_MIN


@functools.lru_cache(maxsize=None)
def plan_classes(agent_net, B, T, n_sm):
    """every class a training pass of B episodes of T steps reaches on n_sm SMs (agent_net: a tuple), the small-net cases included"""
    p = episode_plan(list(agent_net), B, T, n_sm)
    out = set()
    for net, r0, r1 in all_cta_rows(p):
        if r1 > r0 and tail_counts(r1 - r0):
            out.add(classes(r1 - r0))
    for k in range(len(p["cta_begin"]) - 1):
        if (p["slot_begin"][k + 1] - p["slot_begin"][k]) * B * (T + 1) < 64:
            out.add(SMALL_NET)
        if p["cta_begin"][k + 1] - p["cta_begin"][k] == 1:
            out.add(ONE_CTA)
    return frozenset(out)


def find_batch(N, sharing, T_choices, n_sm, cls, max_rows=20_000):
    """the smallest (B, T) -- fewest rows N B (T + 1), then smallest T -- with T in T_choices whose plan on n_sm SMs holds class `cls`; None when
    none does within max_rows rows"""
    nets = tuple(nets_of(N, sharing))
    cands = sorted((N * B * (T + 1), T, B) for T in T_choices for B in range(1, max_rows // (N * (T + 1)) + 1))
    for _, T, B in cands:
        if cls in plan_classes(nets, B, T, n_sm):
            return B, T
    return None


def last_episodes(agent_net, B, T, n_sm):
    """the episodes (batch indices b) that end a CTA: units are agent-major, unit u of a net is episode u % B of its (u // B)-th agent"""
    p = episode_plan(list(agent_net), B, T, n_sm)
    return sorted({(r1 // (T + 1) - 1) % B for _, r0, r1 in all_cta_rows(p) if r1 > r0})


# ---- the forward kernels' dense split -----------------------------------------------------------------------------------------------------------
def dense_plan(agent_net, E, n_sm):
    """the act step's plan (a2c_dense_forward, the DQN act forward): make_plan(ns, E, 1, n_sm, 32); unit = environment, one row each"""
    return make_plan(list(agent_net), E, 1, n_sm, 32)


@functools.lru_cache(maxsize=None)
def dense_classes(agent_net, E, n_sm):
    """every class a forward over E environments reaches on n_sm SMs (agent_net: a tuple).  cta_rows splits a net's `units` rows over `ncta`
    CTAs by floor division, so each CTA gets units // ncta rows or one more: two sizes per net instead of a walk over every CTA."""
    p = dense_plan(agent_net, E, n_sm)
    cb, sb = p["cta_begin"], p["slot_begin"]
    out = set()
    for k in range(len(cb) - 1):
        q, rem = divmod((sb[k + 1] - sb[k]) * E, cb[k + 1] - cb[k])
        out |= {classes(r) for r in ({q, q + 1} if rem else {q}) if r > 0}
    return frozenset(out)


def find_envs(N, sharing, n_sm, cls, max_envs):
    """the smallest E <= max_envs whose dense plan on n_sm SMs holds class `cls`; None when none does"""
    nets = tuple(nets_of(N, sharing))
    return next((E for E in range(1, max_envs + 1) if cls in dense_classes(nets, E, n_sm)), None)


# ---- the recurrent (GRU) split ------------------------------------------------------------------------------------------------------------------
# gru_backward_kernel (csrc/gru_kernels.cu) gets make_plan(ns, B, 1, n_sm, kGruSeqs): one unit per sequence (agent, b), a contiguous run
# [v_begin, v_end) of one net's sequences per CTA.  It walks the run in 16-sequence tiles, each split into two 8-sequence halves (one per 128-thread
# half of the block), resets the carried dL/dh per tile and adds each tile's sums into the CTA's scratch row.  A CTA's class is its tiles (1, 2,
# 3+) and its last tile: lower (1-7 sequences: the second half is all padding), half (8), upper (9-15), full (16).  Three more cases: a net of
# fewer than 16 sequences, a net trained by one CTA, and a tile of a multi-tile CTA that holds sequences of two agents (gru_seq crosses a slot).
# gru_forward_kernel tiles every net's sequences from 0 and launches ceil(max / 16) CTAs per net: its shapes are each net's nseq % 16 and whether
# a smaller net leaves CTAs idle.
SEQS = 16                      # kGruSeqs
SEQ_CLASSES = tuple(f"t{t}{'+' if t == 3 else ''}-{last}" for t in (1, 2, 3) for last in ("lower", "half", "upper", "full"))
GRU_SMALL_NET = "gru-small-net"
GRU_ONE_CTA = "gru-one-cta"
GRU_STRADDLE = "gru-straddle"
GRU_CLASSES = SEQ_CLASSES + (GRU_SMALL_NET, GRU_ONE_CTA, GRU_STRADDLE)
FWD_REMAINDERS = ("lower", "half", "upper", "full")


def _last_tile(n):
    last = n - SEQS * ((n - 1) // SEQS)
    return "lower" if last < 8 else "half" if last == 8 else "upper" if last < SEQS else "full"


def gru_plan(agent_net, B, n_sm):
    """the backward's plan: make_plan(ns, B, 1, n_sm, kGruSeqs); rows of cta_rows are sequences"""
    return make_plan(list(agent_net), B, 1, n_sm, SEQS)


def seq_class(n):
    """the class of a CTA of n > 0 sequences"""
    tiles = (n + SEQS - 1) // SEQS
    return f"t{min(tiles, 3)}{'+' if tiles >= 3 else ''}-{_last_tile(n)}"


def seq_of(p, net, v):
    """sequence v of net -> (agent, b), as gru_seq"""
    slot = v // p["units_per_agent"]
    return p["slot_agent"][p["slot_begin"][net] + slot], v - slot * p["units_per_agent"]


def tiles_of(v0, v1):
    """the tiles [vt, vt_end) of a CTA's run [v0, v1)"""
    return [(vt, min(vt + SEQS, v1)) for vt in range(v0, v1, SEQS)]


def straddles(B, v0, v1):
    """a tile of the multi-tile run [v0, v1) holds sequences of two agents (B sequences per agent)"""
    return v1 - v0 > SEQS and any((vt // B + 1) * B < ve for vt, ve in tiles_of(v0, v1))


@functools.lru_cache(maxsize=None)
def gru_classes(agent_net, B, n_sm):
    """every class the backward of B sequences per agent reaches on n_sm SMs (agent_net: a tuple)"""
    p = gru_plan(agent_net, B, n_sm)
    out = set()
    for _, v0, v1 in all_cta_rows(p):
        if v1 > v0:
            out.add(seq_class(v1 - v0))
            if straddles(B, v0, v1):
                out.add(GRU_STRADDLE)
    for k in range(len(p["cta_begin"]) - 1):
        if (p["slot_begin"][k + 1] - p["slot_begin"][k]) * B < SEQS:
            out.add(GRU_SMALL_NET)
        if p["cta_begin"][k + 1] - p["cta_begin"][k] == 1:
            out.add(GRU_ONE_CTA)
    return frozenset(out)


def find_units(N, sharing, n_sm, cls, max_seqs=7_000):
    """the smallest B (sequences per agent) whose backward plan on n_sm SMs holds class `cls`, with N B <= max_seqs; None when none does"""
    nets = tuple(nets_of(N, sharing))
    for B in range(1, max_seqs // N + 1):
        if cls in gru_classes(nets, B, n_sm):
            return B
    return None


def cta_edge_sequences(p):
    """(agent, b) of the first and the last sequence of every CTA and of every tile of the plan"""
    out = set()
    for net, v0, v1 in all_cta_rows(p):
        for vt, ve in tiles_of(v0, v1):
            out |= {seq_of(p, net, vt), seq_of(p, net, ve - 1)}
    return sorted(out)


def forward_shapes(agent_net, B):
    """the forward's launch: (each net's nseq % 16 class, whether some CTAs of the ceil(max / 16) x n_nets grid are idle)"""
    nseq = [agent_net.count(k) * B for k in range(max(agent_net) + 1)]
    tiles = [(n + SEQS - 1) // SEQS for n in nseq]
    return {_last_tile(n) for n in nseq}, min(tiles) < max(tiles)


def tail_td_rows(agent_net, B, T, n_sm, cls):
    """for every CTA of class `cls`: (rows of its last chunk, rows of warpgroup 1's after-loop phase -- chunks 2 and 3 of the last tile -- that
    carry a loss, t < T, in the CTA's last episode: a TD error in the DQN pass, a value or policy loss in the actor-critic passes); the after-loop
    count is None where the last tile holds 64 rows or fewer (no such phase)"""
    p = episode_plan(list(agent_net), B, T, n_sm)
    out = []
    for _, r0, r1 in all_cta_rows(p):
        if r1 <= r0 or not tail_counts(r1 - r0) or classes(r1 - r0) != cls:
            continue
        last_ep = r1 - (T + 1)
        td = lambda lo: sum(1 for vr in range(max(lo, last_ep), r1) if vr % (T + 1) < T)   # noqa: E731
        last_tile = r0 + (r1 - 1 - r0) // TILE * TILE
        out.append((td(r0 + (r1 - 1 - r0) // CHUNK * CHUNK), td(last_tile + 2 * CHUNK) if r1 - last_tile > 2 * CHUNK else None))
    return out

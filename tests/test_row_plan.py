"""No GPU: tests/row_plan.py against the library's own planner, the class search on both H100 SM counts, and the edges of
tests/test_tc_train_edges_gpu.py's, tests/test_ac_train_edges_gpu.py's and tests/test_gru_edges_gpu.py's shape tables.

The planner check compiles a host-only driver that includes csrc/gru.cuh and csrc/learner.cuh (nvcc with the library's flags, no device code
runs) and prints episode_plan's, the GRU backward's make_plan(ns, B, 1, n_sm, kGruSeqs) and the act step's make_plan(ns, E, 1, n_sm, 32)
cta_begin and every CTA's [row_begin, row_end).
cta_rows itself is device code: the driver restates its split in C++ integer arithmetic."""
import subprocess

import numpy as np
import pytest

from codebase_b200.csrc import build as native_build
from tests import row_plan as rp
from tests import test_ac_train_edges_gpu as ae
from tests import test_gru_edges_gpu as ge
from tests import test_tc_train_edges_gpu as g

DRIVER = r"""
#include "gru.cuh"
#include <stdio.h>
using namespace marl;
// stdin: lines "N B T n_sm agent_net[0..N)"; stdout per line, for episode_plan(ns, B, T, n_sm) and then for the GRU backward's
// make_plan(ns, B, 1, n_sm, kGruSeqs): "n_cta cta_begin[0..n_nets] | net row_begin row_end ..." (one triple per CTA), the two joined by " || ";
// then the GRU plan's slots, and the act step's dense plan make_plan(ns, E = B, 1, n_sm, 32) in the same form
static void print_plan(const RowPlan& p) {
  const int n_cta = p.cta_begin[p.n_nets];
  printf("%d", n_cta);
  for (int k = 0; k <= p.n_nets; ++k) printf(" %d", p.cta_begin[k]);
  printf(" |");
  for (int c = 0; c < n_cta; ++c) {   // cta_rows with blockIdx.x = c
    int net = 0;
    while (net + 1 < p.n_nets && c >= p.cta_begin[net + 1]) ++net;
    const int ncta = p.cta_begin[net + 1] - p.cta_begin[net], k = c - p.cta_begin[net];
    const long long units = (long long)(p.slot_begin[net + 1] - p.slot_begin[net]) * p.units_per_agent;
    printf(" %d %d %d", net, (int)(units * k / ncta) * p.unit_rows, (int)(units * (k + 1) / ncta) * p.unit_rows);
  }
}
int main() {
  int N, B, T, n_sm;
  while (scanf("%d %d %d %d", &N, &B, &T, &n_sm) == 4) {
    NetSet ns; ns.n_agents = N; ns.n_nets = 0;
    for (int a = 0; a < N; ++a) { scanf("%d", &ns.agent_net[a]); if (ns.agent_net[a] + 1 > ns.n_nets) ns.n_nets = ns.agent_net[a] + 1; }
    print_plan(episode_plan(ns, B, T, n_sm));
    printf(" || ");
    const RowPlan q = make_plan(ns, B, 1, n_sm, kGruSeqs);
    print_plan(q);
    printf(" || %d", q.n_nets);
    for (int k = 0; k <= q.n_nets; ++k) printf(" %d", q.slot_begin[k]);
    for (int a = 0; a < N; ++a) printf(" %d", q.slot_agent[a]);
    printf(" || ");
    print_plan(make_plan(ns, B, 1, n_sm, 32));
    printf("\n");
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("plan_driver")
    src, exe = d / "plan_driver.cu", d / "plan_driver"
    src.write_text(DRIVER)
    flags = [f for f in native_build.NVCC_FLAGS if f != "-shared"]
    subprocess.check_call([native_build.nvcc_path()] + flags + ["-I", native_build.HERE, str(src), "-o", str(exe)])
    return str(exe)


def _configs():
    """seeded configs: N 1-32; independent, shared and uneven sharing groups; B 1-2048; T 1-200; 114, 132 and 144 SMs"""
    rng = np.random.default_rng(0x9A7)
    out = []
    for i in range(300):
        N = int(rng.integers(1, 33))
        kind = i % 3
        nets = list(range(N)) if kind == 0 else [0] * N if kind == 1 else rp.nets_of(N, tuple(int(x) for x in rng.integers(0, max(1, N // 3) + 1, N)))
        B = int(rng.choice([rng.integers(1, 17), rng.integers(1, 257), rng.integers(1, 2049)]))
        T = int(rng.choice([rng.integers(1, 11), rng.integers(1, 201)]))
        out.append((N, B, T, int(rng.choice([114, 132, 144])), nets))
    return out


def test_mirror_matches_the_library_planner(driver):
    cfgs = _configs()
    stdin = "".join(f"{N} {B} {T} {n_sm} {' '.join(map(str, nets))}\n" for N, B, T, n_sm, nets in cfgs)
    lines = subprocess.run([driver], input=stdin, capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(lines) == len(cfgs)
    seen, seen_gru = set(), set()
    for (N, B, T, n_sm, nets), line in zip(cfgs, lines):
        episodes, seqs, slots, dense = line.split(" || ")
        for p, part in ((rp.episode_plan(nets, B, T, n_sm), episodes), (rp.gru_plan(nets, B, n_sm), seqs), (rp.dense_plan(nets, B, n_sm), dense)):
            head, rows = part.split("|")
            head, rows = [int(x) for x in head.split()], [int(x) for x in rows.split()]
            assert head[0] == p["cta_begin"][-1] and head[1:] == p["cta_begin"], (N, B, T, n_sm, nets)
            want = [x for r in rp.all_cta_rows(p) for x in r]
            assert rows == want, (N, B, T, n_sm, nets)
        slots = [int(x) for x in slots.split()]
        n_nets = slots[0]
        q = rp.gru_plan(nets, B, n_sm)
        assert slots[1:n_nets + 2] == q["slot_begin"] and slots[n_nets + 2:] == q["slot_agent"], (N, nets)   # what seq_of reads
        seen |= rp.plan_classes(tuple(nets), B, T, n_sm)
        seen_gru |= rp.gru_classes(tuple(nets), B, n_sm)
        # dense_classes reads two CTA sizes per net instead of walking every CTA
        d = rp.dense_plan(nets, B, n_sm)
        assert rp.dense_classes(tuple(nets), B, n_sm) == {rp.classes(r1 - r0) for _, r0, r1 in rp.all_cta_rows(d) if r1 > r0}, (N, B, n_sm, nets)
    assert len(seen) >= 12, sorted(seen)   # the random configs are not the coverage: find_batch / find_units are
    assert len(seen_gru) >= 6, sorted(seen_gru)


def test_classes_of_rows():
    assert rp.classes(1) == rp.classes(31) == "t1-c1-part" and rp.classes(32) == "t1-c1-full" and rp.classes(96) == "t1-c3-full"
    assert rp.classes(128) == "t1-c4-full" and rp.classes(129) == "t2-c1-part" and rp.classes(159) == "t2-c1-part" and rp.classes(160) == "t2-c1-full"
    assert rp.classes(257) == "t3+-c1-part" and rp.classes(383) == "t3+-c4-part" and rp.classes(384 + 96) == "t3+-c3-full"
    assert len(set(rp.CLASSES)) == 24 and {rp.classes(r) for r in range(1, 1025)} == set(rp.CLASSES)


@pytest.mark.parametrize("n_sm", [114, 132])
def test_every_class_is_found_within_the_row_budget(n_sm):
    """an H100 PCIe (114 SMs) and SXM (132 SMs) split the same batch differently: each case of the class sweep finds its class on both"""
    for cls, c in g.CLASS_CASES.items():
        found = rp.find_batch(c.N, c.sharing, c.T_choices, n_sm, cls, g.MAX_ROWS)
        assert found is not None, (n_sm, cls, c)
        B, T = found
        assert cls in rp.plan_classes(tuple(rp.nets_of(c.N, c.sharing)), B, T, n_sm) and c.N * B * (T + 1) <= g.MAX_ROWS
    assert set(g.CLASS_CASES) == set(rp.ALL_CLASSES)


@pytest.mark.parametrize("n_sm", [114, 132])
def test_the_tail_rows_of_every_case_carry_td_errors(n_sm):
    """With the last episode of every CTA at full length, every CTA of a case's class has TD rows (t < T) in its last chunk, and in the rows of
    warpgroup 1's after-loop phase exactly where the last tile holds more than 64 rows (chunks 3 and 4): a fault in either tail moves the gradient"""
    for name, c in {**g.CLASS_CASES, **g.WIDTH_CASES}.items():
        cls = c.cls or name
        if cls not in rp.CLASSES:
            continue
        B, T = rp.find_batch(c.N, c.sharing, c.T_choices, n_sm, cls, g.MAX_ROWS)
        tails = rp.tail_td_rows(rp.nets_of(c.N, c.sharing), B, T, n_sm, cls)
        assert tails, (n_sm, name)
        for last_chunk, after_loop in tails:
            assert last_chunk >= rp.TAIL_MIN - 1, (n_sm, name, B, T, last_chunk)
            assert (after_loop is not None) == (cls.split("-")[1] in ("c3", "c4")), (n_sm, name)
            assert after_loop is None or after_loop >= rp.TAIL_MIN - 1, (n_sm, name, B, T, after_loop)
    # two multi-tile classes hold several episodes per CTA: tile boundaries inside an episode, CTAs of one net split by cta_rows' rounding
    for cls in ("t2-c2-part", "t2-c3-part"):
        c = g.CLASS_CASES[cls]
        B, T = rp.find_batch(c.N, c.sharing, c.T_choices, n_sm, cls, g.MAX_ROWS)
        p = rp.episode_plan(rp.nets_of(c.N, c.sharing), B, T, n_sm)
        assert min(r1 - r0 for _, r0, r1 in rp.all_cta_rows(p)) >= 2 * (T + 1) and (T + 1) % rp.TILE != 0, (cls, B, T)


def test_tail_rows_of_a_small_plan():
    """tail_td_rows and last_episodes on a plan worked by hand: one net, 3 episodes of T = 63 (64 rows) in one CTA of 192 rows (t2-c2-full);
    the last episode is b = 2, its rows 128..191; the last chunk is rows 160..191, of which t < 63 are 160..190"""
    assert rp.episode_plan([0], 3, 63, 1)["cta_begin"] == [0, 1]
    assert rp.last_episodes([0], 3, 63, 1) == [2]
    assert rp.tail_td_rows([0], 3, 63, 1, "t2-c2-full") == [(31, None)]
    # 2 agents sharing the net, B = 2, T = 99: 4 units of 100 rows on 2 CTAs -> 200 rows each (t2-c3-part, after-loop rows 192..199)
    assert rp.last_episodes([0, 0], 2, 99, 2) == [1]
    assert rp.tail_td_rows([0, 0], 2, 99, 2, "t2-c3-part") == [(7, 7), (7, 7)]


def test_cases_sit_on_the_edges_they_claim():
    C, W = g.CLASS_CASES, g.WIDTH_CASES
    # the TD-head sources: the in-kernel head, td_ext with stride 0 (VDN), per agent (standardise_returns), the QMIX mixer
    kinds = [(c.kind, c.standardise) for c in C.values()]
    assert ("idqn", False) in kinds and ("vdn", False) in kinds and ("idqn", True) in kinds and 2 <= kinds.count(("qmix", False)) <= 3
    # independent, shared and uneven-group networks
    assert any(c.sharing is False and c.N > 1 for c in C.values()) and any(c.sharing is True and c.N > 1 for c in C.values())
    assert any(isinstance(c.sharing, tuple) and len(set(c.sharing)) > 1 for c in C.values())
    # double-Q only where a CTA holds few rows (near-ties grow with the rows) -- the single-action cases have no argmax to tie
    for cls, c in {**C, **W}.items():
        if c.double_q and c.A > 1:
            for n_sm in (114, 132):
                B, T = rp.find_batch(c.N, c.sharing, c.T_choices, n_sm, c.cls or cls, g.MAX_ROWS)
                assert B * T <= 160, (cls, n_sm, B, T)
    # the width sweep: the k1steps edges of layer1_tile (D = 8 k - 1, 8 k, 8 k + 1) and the widest input with a bias column
    assert sorted(c.D for c in W.values()) == [1, 2, 7, 8, 9, 16, 17, 24, 25, 31]
    for c in W.values():
        k1 = (c.D + 7) // 8
        assert c.D in (1, 2, 31) or c.D % 8 in (0, 1, 7), c
        assert (8 * k1 == c.D) == (c.D in (8, 16, 24))   # the gathered-row pitch equals D: the ones line of [X | 1] opens a new 8-line group
        assert c.D < g.MAX_OBS_TC
    # every action count 1, 2, 3, 5 and 8 at least twice (A = 1: no argmax, db3[0] only; 2 and 5: partial head columns; 8: kOutPad)
    counts = {a: sum(c.A == a for c in W.values()) for a in (1, 2, 3, 5, 8)}
    assert all(v >= 2 for v in counts.values()) and sum(counts.values()) == len(W), counts
    # each width case runs a multi-tile CTA whose last chunk is partial
    for c in W.values():
        assert c.cls.startswith(("t2", "t3")) and c.cls.endswith("part"), c
    # the forward: E = 1 and a ragged multi-tile split of E rows per network
    assert g.FWD_E[0] == 1 and g.FWD_E[1] % 32 != 0
    # handle reuse: a smaller batch and a shorter T than the handle was created for
    for name, (big, small) in g.REUSE_SHAPES.items():
        assert small[0] < big[0] and small[1] < big[1], name


# ---- the GRU split (tests/test_gru_edges_gpu.py) -------------------------------------------------------------------------------------------------
def test_seq_classes():
    assert [rp.seq_class(n) for n in (1, 7, 8, 9, 15, 16)] == ["t1-lower", "t1-lower", "t1-half", "t1-upper", "t1-upper", "t1-full"]
    assert [rp.seq_class(n) for n in (17, 24, 25, 32, 33, 48, 49, 1000)] == ["t2-lower", "t2-half", "t2-upper", "t2-full", "t3+-lower", "t3+-full",
                                                                             "t3+-lower", "t3+-half"]
    assert len(set(rp.SEQ_CLASSES)) == 12 and {rp.seq_class(n) for n in range(1, 200)} == set(rp.SEQ_CLASSES)


def test_edge_sequences_of_a_small_plan():
    """2 agents sharing a net, B = 21, 2 SMs: 42 sequences on 2 CTAs of 21 (t2-lower); CTA 0 holds agent 0's 0..20 (tiles 0..15, 16..20), CTA 1
    agent 1's, no tile straddles.  3 agents, B = 17, 2 SMs: 51 sequences on CTAs of 25 and 26; CTA 0's second tile 16..24 is agent 0's b = 16
    and agent 1's 0..7, CTA 1 (25..50) holds agent 1's 8..16 and agent 2's 0..16, its first tile 25..40 straddles too"""
    p = rp.gru_plan([0, 0], 21, 2)
    assert rp.all_cta_rows(p) == [(0, 0, 21), (0, 21, 42)] and rp.seq_class(21) == "t2-lower"
    assert rp.cta_edge_sequences(p) == [(0, 0), (0, 15), (0, 16), (0, 20), (1, 0), (1, 15), (1, 16), (1, 20)]
    assert not rp.straddles(21, 0, 21) and not rp.straddles(21, 21, 42)
    q = rp.gru_plan([0, 0, 0], 17, 2)
    assert rp.all_cta_rows(q) == [(0, 0, 25), (0, 25, 51)] and rp.straddles(17, 0, 25) and rp.straddles(17, 25, 51)
    assert rp.cta_edge_sequences(q) == [(0, 0), (0, 15), (0, 16), (1, 7), (1, 8), (2, 6), (2, 7), (2, 16)]
    assert rp.GRU_STRADDLE in rp.gru_classes((0, 0, 0), 17, 2) and rp.GRU_STRADDLE not in rp.gru_classes((0, 0), 21, 2)
    assert rp.forward_shapes([0, 1, 0, 0], 5) == ({"upper", "lower"}, False) and rp.forward_shapes([0, 1, 0, 0], 6) == ({"lower"}, True)   # 18 and 6 sequences: 2 tiles and 1


@pytest.mark.parametrize("n_sm", [114, 132])
def test_every_gru_case_finds_its_class(n_sm):
    """each case of tests/test_gru_edges_gpu.py finds its class on an H100 PCIe (114 SMs) and SXM (132 SMs) within the sequence budget; the class
    sweep covers all 15; its edge episodes are the first and last of every CTA and tile; the training forwards cover every nseq % 16 class and a
    launch with idle CTAs"""
    covered, fwd, idle = set(), set(), False
    for name, c in ge.all_train_cases():
        B = ge.units(c, n_sm)
        nets = rp.nets_of(c.N, c.sharing)
        assert c.cls in rp.gru_classes(tuple(nets), B, n_sm) and c.N * B <= ge.MAX_SEQS, (n_sm, name, B)
        if name in ge.CLASS_CASES:
            covered |= rp.gru_classes(tuple(nets), B, n_sm)
        p = rp.gru_plan(nets, B, n_sm)
        edges = rp.cta_edge_sequences(p)
        for net, v0, v1 in rp.all_cta_rows(p):
            assert rp.seq_of(p, net, v0) in edges and rp.seq_of(p, net, v1 - 1) in edges
        r, i = rp.forward_shapes(nets, B)
        fwd |= r; idle |= i
    assert covered == set(rp.GRU_CLASSES) and set(ge.CLASS_CASES) == set(rp.GRU_CLASSES), sorted(set(rp.GRU_CLASSES) - covered)
    assert fwd == set(rp.FWD_REMAINDERS) and idle, (fwd, idle)


def test_gru_cases_sit_on_the_edges_they_claim():
    C = ge.CLASS_CASES
    kinds = {c.kind for c in C.values()}
    assert kinds == {"idqn", "vdn", "qmix", "ia2c", "ippo", "maa2c", "mappo"}, kinds
    assert any(c.sharing is False and c.N > 1 for c in C.values()) and any(c.sharing is True for c in C.values())
    assert any(c.sharing == ge.SEPS for c in C.values()) and any(c.sharing == ge.GROUPS4 for c in C.values())
    # one recurrent actor with an MLP critic, one MLP actor with a recurrent centralised critic
    assert any(c.arnn and not c.crnn for c in C.values()) and any(not c.arnn and c.crnn and c.kind in ge.CENTRAL for c in C.values())
    for cls, c in C.items():   # short episodes at the multi-tile classes keep the oracle cheap
        assert not cls.startswith(("t2", "t3")) or 2 <= c.T <= 8, cls
    W = ge.WIDTH_CASES
    assert {1, 2, 37, 100, 127} <= {c.H for c in W.values()} | {c.critic_H for c in W.values() if not c.dqn}
    assert all(c.dqn or c.H != c.critic_H for c in W.values())
    assert {c.D for c in W.values() if c.dqn} == {1, 31, 32} and {33, 64, 128} <= {c.D for c in W.values() if not c.dqn}
    assert any(c.kind in ge.CENTRAL and c.N * c.D == 128 for c in W.values())
    assert {c.A for c in W.values()} == {1, 2, 3, 5, 8} and all(c.dqn for c in W.values() if c.A == 1)
    assert all(c.cls in ("t2-upper", "t3+-lower") for c in W.values())
    L = ge.LENGTH_CASES
    assert {c.T for c in L.values()} == {1, 2, 100} and {c.kind for c in L.values() if c.T == 100} == {"idqn", "vdn", "ippo"}
    assert all(c.cls.startswith("t1") for c in L.values() if c.T == 100)
    assert ge.ACT_E == (1, 17, 9001) and {c.H for c in ge.ACT_CASES.values()} == {37, 128}
    assert all(c.cls.startswith(("t2", "t3")) for c in ge.REUSE_CASES.values())
    rows = [c.N * P * c.T for c, P in ge.HEAD_CASES.values()]
    assert any(r % 256 == 0 for r in rows) and any(r % 256 == 1 and r > 256 for r in rows) and any(r < 256 for r in rows)


# ---- the actor-critic training pass and the forward kernels (tests/test_ac_train_edges_gpu.py) -----------------------------------------------------
def _kp(width):
    """the input tile of the FP32 kernels at an input width (learner_kernels_init / launch_train)"""
    return 16 if width <= 16 else 32 if width <= 32 else 64 if width <= 64 else 128


@pytest.mark.parametrize("n_sm", [114, 132])
def test_every_ac_case_finds_its_class_in_both_passes(n_sm):
    """On an H100 PCIe (114 SMs) and SXM (132 SMs), each training case finds its class within the row budget, in the actor pass and, over the
    critic's own networks, in the critic pass; with the edge episodes at full length, every CTA of that class has rows with a loss (t < T) in its
    last chunk in both passes: at least TAIL_MIN - 1 in its last episode, or all T of them where T is shorter.  Over the class sweep, the actor
    passes and the critic passes each cover all 26 classes."""
    actor, critic = set(), set()
    for name, c in ae.all_train_cases():
        found = rp.find_batch(c.N, c.sharing, c.T_choices, n_sm, c.cls, ae.MAX_ROWS)
        assert found is not None, (n_sm, name)
        P, T = found
        assert c.N * P * (T + 1) <= ae.MAX_ROWS
        for part, sharing in (("actor", c.sharing), ("critic", c.csharing)):
            nets = rp.nets_of(c.N, sharing)
            assert c.cls in rp.plan_classes(tuple(nets), P, T, n_sm), (n_sm, name, part, P, T)
            assert set(rp.last_episodes(nets, P, T, n_sm)) <= set(ae.edge_episodes(c, P, T, n_sm))
            if c.cls in rp.CLASSES:
                tails = rp.tail_td_rows(nets, P, T, n_sm, c.cls)
                assert tails and all(last >= min(rp.TAIL_MIN - 1, T) for last, _ in tails), (n_sm, name, part, P, T, tails)
        if name in ae.CLASS_CASES:
            actor |= rp.plan_classes(tuple(rp.nets_of(c.N, c.sharing)), P, T, n_sm)
            critic |= rp.plan_classes(tuple(rp.nets_of(c.N, c.csharing)), P, T, n_sm)
    assert set(ae.CLASS_CASES) == set(rp.ALL_CLASSES)
    assert actor == critic == set(rp.ALL_CLASSES), (sorted(set(rp.ALL_CLASSES) - actor), sorted(set(rp.ALL_CLASSES) - critic))


@pytest.mark.parametrize("n_sm", [114, 132])
def test_every_forward_case_finds_its_class(n_sm):
    """find_envs reaches each of the 24 classes for one agent, two independent agents and three in groups (0, 1, 0) within the environment
    budget, and returns the smallest such E; so do the FP32-only and joint-row cases"""
    for cls in rp.CLASSES:
        for N, sharing in ae.FWD_N:
            E = rp.find_envs(N, sharing, n_sm, cls, ae.FWD_MAX_ROWS // N)
            nets = tuple(rp.nets_of(N, sharing))
            assert E is not None and cls in rp.dense_classes(nets, E, n_sm), (n_sm, cls, N)
            assert E == 1 or cls not in rp.dense_classes(nets, E - 1, n_sm), (n_sm, cls, N, E)
    for name, (c, cls) in ae.FWD_EXTRA.items():
        E = rp.find_envs(c.N, c.sharing, n_sm, cls, ae.FWD_MAX_ROWS // c.N)
        assert E is not None and cls in rp.dense_classes(tuple(rp.nets_of(c.N, c.sharing)), E, n_sm), (n_sm, name)


def test_dense_plan_of_a_small_launch():
    """one agent, 2 SMs: E = 100 environments on 2 CTAs of 50 rows (t1-c2-part); E = 32 stays on one CTA, E = 40 takes two of 20 (at most
    ceil(E / 32) CTAs); the first CTA of 33 rows is at E = 65 (32 + 33).  Two agents in one group, 132 SMs, E = 4225: 8450 rows on 132 CTAs of 64
    or 65 (t1-c2-full and t1-c3-part)"""
    assert rp.all_cta_rows(rp.dense_plan([0], 100, 2)) == [(0, 0, 50), (0, 50, 100)] and rp.dense_classes((0,), 100, 2) == {"t1-c2-part"}
    assert rp.all_cta_rows(rp.dense_plan([0], 32, 2)) == [(0, 0, 32)] and rp.all_cta_rows(rp.dense_plan([0], 40, 2)) == [(0, 0, 20), (0, 20, 40)]
    assert rp.dense_classes((0, 0), 4225, 132) == {"t1-c2-full", "t1-c3-part"}
    assert rp.find_envs(1, False, 2, "t1-c2-part", 1000) == 65 and rp.find_envs(1, False, 2, "t3+-c1-part", 100) is None


def test_ac_cases_sit_on_the_edges_they_claim():
    C, W, L = ae.CLASS_CASES, ae.WIDTH_CASES, ae.LENGTH_CASES
    assert {c.kind for c in C.values()} == {"ia2c", "ippo", "maa2c", "mappo"}
    # independent, shared, uneven-group and SEPS actors; a few critics shared differently from their actor, so that cplan != aplan
    assert any(c.sharing is False and c.N > 1 for c in C.values()) and any(c.sharing is True and c.N > 1 for c in C.values())
    assert any(c.sharing == ae.SEPS for c in C.values()) and any(c.sharing in (ae.GROUPS3, ae.GROUPS4) for c in C.values())
    differ = [(k, c) for k, c in C.items() if c.csharing != c.sharing]
    assert len(differ) >= 3
    for n_sm in (114, 132):
        for cls, c in differ:
            P, T = rp.find_batch(c.N, c.sharing, c.T_choices, n_sm, cls, ae.MAX_ROWS)
            a, k = rp.episode_plan(rp.nets_of(c.N, c.sharing), P, T, n_sm), rp.episode_plan(rp.nets_of(c.N, c.csharing), P, T, n_sm)
            assert a["cta_begin"] != k["cta_begin"], (n_sm, cls)
    # KP 16, 32, 64 and 128 for the actor and for the critic; every actor KP at a t2 and at a t3+ class with a partial last tile
    assert {_kp(c.D) for c in C.values()} == {_kp(c.joint) for c in C.values()} == {16, 32, 64, 128}
    for kp in (16, 32, 64, 128):
        for t in ("t2", "t3+"):
            assert any(_kp(c.D) == kp and cls.startswith(t + "-") and cls.endswith("part") for cls, c in C.items()), (kp, t)
    assert any(c.standardise for c in C.values())
    # the tensor-core target and old-log-prob passes: cases of both kinds, PPO at 2, 3 and 4 epochs
    assert any(c.tc_forward and c.kind not in ae.PPO for c in C.values()) and any(c.tc_forward and c.joint > ae.MAX_OBS_TC for c in C.values())
    assert {c.epochs for c in C.values() if c.kind in ae.PPO and c.tc_forward} == {2, 3, 4}
    # the width sweep: every KP edge, hidden widths below 128 with actor and critic apart, every action count, joint inputs on both sides of 32 and 64
    assert {1, 16, 17, 32, 33, 64, 65, 127, 128} <= {c.D for c in W.values()}
    assert {1, 2, 37, 100, 127} <= {c.H for c in W.values()} | {c.critic_H for c in W.values()} and all(c.H != c.critic_H for c in W.values())
    assert {c.A for c in W.values()} == {1, 2, 3, 5, 8}
    assert {32, 33, 64, 65, 128} <= {c.joint for c in W.values() if c.kind in ae.CENTRAL}
    for c in list(W.values()) + list(L.values()):
        assert c.cls.startswith(("t2", "t3")), c
    assert all(c.cls.endswith("part") for c in W.values())
    # lengths: T = 1 and 2, and one environment whose single episode walks three tiles
    for n_sm in (114, 132):
        Ts = {}
        for name, c in L.items():
            P, T = rp.find_batch(c.N, c.sharing, c.T_choices, n_sm, c.cls, ae.MAX_ROWS)
            Ts.setdefault(T, []).append(P)
        assert set(Ts) == {1, 2, 383} and Ts[383] == [1] * len(Ts[383]), Ts
    # handle reuse at a t2 and a t3+ class
    assert {c.cls[:2] for c in ae.REUSE_CASES.values()} == {"t2", "t3"}
    # the forward's extra cases: an input of 100, a hidden width of 37, joint rows at 16 (tensor cores), 33 and 128
    X = {name: c for name, (c, _) in ae.FWD_EXTRA.items()}
    assert {c.joint for c in X.values() if c.kind in ae.CENTRAL} == {16, 33, 128} and any(c.D == 100 for c in X.values()) and any(c.H == 37 for c in X.values())

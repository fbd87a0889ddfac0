"""No GPU: the edges of tests/test_env_agent_range_gpu.py's case table, the shared-memory arithmetic of the env-step kernels, and the
observation-width limit of lbf_reset_kernel.

LBF's step kernel gives each env G = next_pow2(N) lanes and a CTA EPC = 4 * 32 / G envs; RWARE's one warp per env and 4 envs per CTA.  The
mirrors below restate step_smem_bytes (lbf_env.cu) and rware_warp_smem (rware_env.cu); the refusal test on the GPU checks the first against
the library's own message (REFUSED_LBF_SMEM)."""
import ctypes as C

import pytest

from codebase_b200 import _native as nat
from codebase_b200.lbf import LbfConfig
from codebase_b200.rware import RwareConfig
from oracle import rware_ref as rw
from tests import test_env_agent_range_gpu as g

H100_SMEM_OPTIN = 232_448   # cudaDevAttrMaxSharedMemoryPerBlockOptin on an H100
MAX_FOOD, MAX_AGENTS = 32, 32
MAX_VEC_OBS = 3 * MAX_FOOD + 4 * MAX_AGENTS   # kMaxVecObs: lbf_reset_kernel's observation buffer
OLD_RESET_BUF = 3 * (MAX_FOOD + MAX_AGENTS)   # the buffer's size before it was derived from the validator's limit


def lbf_G(cfg):
    G = 1
    while G < cfg.n_agents:
        G *= 2
    return G


def lbf_epc(cfg):
    return 4 * (32 // lbf_G(cfg))


def lbf_smem(cfg):
    """step_smem_bytes: field tile (pitch + 4), players, [foods], meta, [the observation tile]"""
    epc, G, pitch = lbf_epc(cfg), lbf_G(cfg), (cfg.rows * cfg.cols + 15) & ~15
    if cfg.grid_observation:
        return epc * (2 * (pitch + 4) + G * 4 + 16)
    return epc * (pitch + 4) + epc * G * 4 + epc * cfg.max_num_food * 4 + epc * 16 + epc * cfg.n_agents * cfg.obs_dim * 4


def rware_smem(cfg):
    """4 x rware_warp_smem: observations (16 B aligned), shelf grid, agents, requests, chain lengths, meta"""
    pitch = (cfg.rows * cfg.cols + 15) & ~15
    return 4 * (((cfg.n_agents * cfg.obs_dim * 4 + 15) & ~15) + pitch + 32 * 4 + 8 * 4 + 32 * 4 + 16)


def test_lbf_cases_sit_on_their_edges():
    L = g.LBF
    for name, (cfg, E) in L.items():
        assert E % lbf_epc(cfg) != 0, f"{name}: the last CTA must be ragged"
        assert lbf_smem(cfg) <= H100_SMEM_OPTIN, name
        assert 2 <= cfg.time_limit <= g.RESET_AT, f"{name}: every frozen env ends before the masked reset"
    assert [n for n, (c, _) in L.items() if c.grid_observation] == ["lbf_grid_n32_std_coop"]
    c = L["lbf_n9_g16"][0]
    assert (c.n_agents, lbf_G(c), lbf_epc(c)) == (9, 16, 8)
    c = L["lbf_n16_crowded"][0]
    assert (c.n_agents, lbf_G(c), c.force_coop, c.penalty) == (16, 16, 1, 0.1) and c.rows * c.cols == 64
    c = L["lbf_n17_std_coop"][0]
    assert (c.n_agents, lbf_G(c), c.standardise_rewards, c.cooperative_reward) == (17, 32, 1, 1)
    c = L["lbf_n24_upstream"][0]
    assert (c.n_agents, c.upstream_reset) == (24, 1)
    c = L["lbf_20x20_32p_10f"][0]
    assert (c.rows, c.cols, c.n_agents, c.max_num_food, c.grid_observation, lbf_G(c), lbf_epc(c)) == (20, 20, 32, 10, 0, 32, 4)
    c = L["lbf_grid_n32_std_coop"][0]
    assert (c.n_agents, lbf_G(c), c.sight, c.standardise_rewards, c.cooperative_reward) == (32, 32, 2, 1, 1)
    # the reset case: the widest vector observation there is, over the buffer lbf_reset_kernel had before
    c = L["lbf_n32_obsid_32f"][0]
    assert c.obs_dim == MAX_VEC_OBS == 224 > OLD_RESET_BUF == 192 and not c.grid_observation


def test_rware_cases_sit_on_their_edges():
    R = g.RWARE
    for name, (cfg, E) in R.items():
        assert E % 4 != 0, f"{name}: the last CTA must be ragged"
        assert rware_smem(cfg) <= H100_SMEM_OPTIN, name
        assert 2 <= cfg.time_limit <= g.RESET_AT, name
    assert R["rware_tiny_n31"][0].n_agents == R["rware_large_n31_s3"][0].n_agents == 31   # lane 31 is the sink
    c = R["rware_tiny_n31"][0]
    assert (c.rows, c.cols, c.shelf_rows, c.shelf_columns) == (11, 10, 1, 3)
    c = R["rware_large_n31_s3"][0]
    assert c.obs_dim == 8 + 7 * 49 + 31 == 382 and c.sensor_range == 3 and c.standardise_rewards and c.cooperative_reward
    assert rware_smem(c) == 192_576
    c = R["rware_medium_n24_hard"][0]
    assert (c.shelf_rows, c.shelf_columns, c.n_agents, c.request_queue_size) == (2, 5, 24, 12)
    # _queue_at_goals: 16 agents on highway cells of the two goal columns, the others side by side on a highway row
    for name in g.QUEUED:
        c = R[name][0]
        (gx, gy), (gx1, gy1) = rw.goals(c)
        assert gx1 == gx + 1 and gy1 == gy and 16 < c.n_agents <= 16 + c.cols, name
        assert all(rw.is_highway(c, gx + i % 2, gy - i // 2) for i in range(16)), name
        assert all(rw.is_highway(c, x, c.column_height + 1) for x in range(c.n_agents - 16)), name


def test_refused_vector_tile_is_over_the_limit():
    c = g.REFUSED_LBF
    assert not c.grid_observation and lbf_epc(c) == 64 and lbf_smem(c) == g.REFUSED_LBF_SMEM == 272_384 > H100_SMEM_OPTIN
    assert lbf_smem(LbfConfig(rows=60, cols=60, n_agents=2, sight=2, grid_observation=1)) > H100_SMEM_OPTIN   # the grid refusal's case


CASES = {**{n: c for n, (c, _) in {**g.LBF, **g.RWARE}.items()}, "refused_lbf_64x64": g.REFUSED_LBF}


@pytest.mark.parametrize("name", list(CASES))
def test_obs_dim_matches_the_library(name):
    cfg = CASES[name]
    ncfg = cfg.to_native()
    fn = nat.lib().marl_rware_obs_dim if isinstance(cfg, RwareConfig) else nat.lib().marl_lbf_obs_dim
    assert fn(C.byref(ncfg)) == cfg.obs_dim


def test_validators_admit_every_case_and_refuse_a_32nd_rware_agent():
    """marl_*_frame_shape runs the create validators on the host: D = 224 and 31 RWARE agents pass, 32 RWARE agents do not."""
    lib, h, w = nat.lib(), C.c_int32(), C.c_int32()
    for name, cfg in CASES.items():
        ncfg = cfg.to_native()
        fs = lib.marl_rware_frame_shape if isinstance(cfg, RwareConfig) else lib.marl_lbf_frame_shape
        nat.check(fs(C.byref(ncfg), C.byref(h), C.byref(w)), name)
    too_many = RwareConfig(n_agents=32, request_queue_size=16).to_native()
    with pytest.raises(nat.NativeError, match=r"n_agents 32 out of range \(1\.\.31\)"):
        nat.check(lib.marl_rware_frame_shape(C.byref(too_many), C.byref(h), C.byref(w)), "frame_shape")

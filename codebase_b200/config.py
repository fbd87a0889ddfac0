"""A small Hydra-compatible config composer (hydra / omegaconf are not dependencies of the GPU path).

Implements the subset of Hydra the reference's command lines use (README.md:80-120, marlbase/run.py:14-47):
  python -m codebase_b200.run +algorithm=idqn env.name="lbforaging:Foraging-8x8-2p-3f-v3" env.time_limit=25 seed=0
  * `configs/default.yaml` is the primary config, its `defaults:` list pulls `logger/<name>.yaml` under the `logger` key;
  * `+group=name` merges `configs/<group>/<name>.yaml`; files marked `# @package _global_` merge at the root and may
    inherit through their own `defaults:` list (vdn.yaml:3-4 -> idqn);
  * `a.b.c=value` / `+a.b.c=value` dotted overrides with YAML-typed values;
  * `_target_` strings are resolved against this package first (`dqn.train.main` -> `codebase_b200.dqn.train.main`),
    so the reference's own target names keep working.
"""
from __future__ import annotations

import importlib
import os

import yaml

CONFIG_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "configs")


class Config(dict):
    """dict with attribute access, nested (what the reference gets from OmegaConf's DictConfig)."""

    def __init__(self, d=None):
        super().__init__()
        for k, v in (d or {}).items():
            self[k] = v

    @staticmethod
    def _wrap(v):
        if isinstance(v, dict) and not isinstance(v, Config):
            return Config(v)
        if isinstance(v, list):
            return [Config._wrap(x) for x in v]
        return v

    def __setitem__(self, k, v):
        super().__setitem__(k, Config._wrap(v))

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v

    def __delattr__(self, k):
        del self[k]

    def to_dict(self):
        def un(v):
            if isinstance(v, dict):
                return {k: un(x) for k, x in v.items()}
            if isinstance(v, list):
                return [un(x) for x in v]
            return v
        return un(self)


def _merge(dst: dict, src: dict):
    for k, v in src.items():
        if isinstance(v, dict) and isinstance(dst.get(k), dict):
            _merge(dst[k], v)
        else:
            dst[k] = v
    return dst


def _load_group(group: str, name: str) -> tuple[dict, bool]:
    path = os.path.join(CONFIG_DIR, group, f"{name}.yaml")
    if not os.path.exists(path):
        raise FileNotFoundError(f"no config {group}/{name}.yaml under {CONFIG_DIR}")
    with open(path) as f:
        text = f.read()
    is_global = "@package _global_" in text.split("\n", 1)[0]
    data = yaml.safe_load(text) or {}
    out: dict = {}
    for d in data.pop("defaults", []) or []:
        if isinstance(d, str) and d != "_self_":
            base, _ = _load_group(group, d)
            _merge(out, base)
    _merge(out, data)
    return out, is_global


def _set_dotted(cfg: dict, key: str, value):
    parts = key.split(".")
    node = cfg
    for p in parts[:-1]:
        if not isinstance(node.get(p), dict):
            node[p] = {}
        node = node[p]
    node[parts[-1]] = value


def compose(overrides: list[str]) -> Config:
    with open(os.path.join(CONFIG_DIR, "default.yaml")) as f:
        root = yaml.safe_load(f)
    defaults = root.pop("defaults", [])
    root.pop("hydra", None)
    cfg: dict = {}
    _merge(cfg, root)
    for d in defaults:
        if isinstance(d, dict):
            for g, n in d.items():
                if g.startswith("override "):
                    continue
                data, is_global = _load_group(g, n)
                _merge(cfg, data) if is_global else _merge(cfg.setdefault(g, {}), data)
    groups, dotted = [], []
    for ov in overrides:
        key, _, val = ov.partition("=")
        plus = key.startswith("+")
        key = key.lstrip("+")
        if "." not in key and os.path.isdir(os.path.join(CONFIG_DIR, key)) and plus:
            groups.append((key, val))
        elif "." not in key and os.path.isdir(os.path.join(CONFIG_DIR, key)) and os.path.exists(os.path.join(CONFIG_DIR, key, f"{val}.yaml")):
            groups.append((key, val))
        else:
            dotted.append((key, yaml.safe_load(val) if val != "" else None))
    for g, n in groups:
        data, is_global = _load_group(g, n)
        _merge(cfg, data) if is_global else _merge(cfg.setdefault(g, {}), data)
    for k, v in dotted:
        _set_dotted(cfg, k, v)
    _check_missing(cfg)
    return Config(cfg)


def _check_missing(node, path=""):
    if isinstance(node, dict):
        for k, v in node.items():
            _check_missing(v, f"{path}.{k}" if path else k)
    elif node == "???":
        raise ValueError(f"missing mandatory config value: {path} (pass {path}=...)")


def resolve_target(target: str):
    mod, _, attr = target.rpartition(".")
    last = None
    for prefix in ("codebase_b200.", ""):
        try:
            return getattr(importlib.import_module(prefix + mod), attr)
        except (ImportError, AttributeError) as e:
            last = e
    raise ImportError(f"cannot resolve _target_ {target!r}: {last}")


def call(node, *args, **kwargs):
    """hydra.utils.call / instantiate with `_recursive_=False` semantics: nested configs are passed through as Config."""
    kw = {k: v for k, v in node.items() if k != "_target_"}
    kw.update(kwargs)
    return resolve_target(node["_target_"])(*args, **kw)


instantiate = call

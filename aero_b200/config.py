"""Hydra-less reader for ``conf/experiment/*.yaml``.

The reference builds its generator with ``Aero(**args.experiment.aero)`` from an OmegaConf
tree (reference ``src/models/modelFactory.py:6-8``, ``conf/experiment/aero_4-16_512_64.yaml:17-59``).
Hydra/OmegaConf are not installed in this image, so tests and ``bench.py`` use this loader; it
resolves ``${experiment.key}`` interpolations and coerces YAML-1.1 "1e-3"-style strings to float
the way OmegaConf does.
"""
from __future__ import annotations

import os
import re

import yaml

_CONF_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "conf")
_FLOAT = re.compile(r"^[+-]?(\d+\.?\d*|\.\d+)([eE][+-]?\d+)?$")
_INTERP = re.compile(r"^\$\{experiment\.([A-Za-z0-9_]+)\}$")


def _coerce(v):
    if isinstance(v, str) and _FLOAT.match(v):
        return float(v)
    if isinstance(v, dict):
        return {k: _coerce(x) for k, x in v.items()}
    if isinstance(v, list):
        return [_coerce(x) for x in v]
    return v


def _resolve(node, root):
    if isinstance(node, dict):
        return {k: _resolve(v, root) for k, v in node.items()}
    if isinstance(node, list):
        return [_resolve(v, root) for v in node]
    if isinstance(node, str):
        m = _INTERP.match(node)
        if m:
            return _resolve(root[m.group(1)], root)
        return re.sub(r"\$\{experiment\.([A-Za-z0-9_]+)\}", lambda mm: str(root[mm.group(1)]), node)
    return node


def load_experiment(name, conf_dir=None, **overrides):
    """Return the ``experiment`` dict for ``conf/experiment/<name>.yaml``."""
    path = name if os.path.isfile(name) else os.path.join(conf_dir or _CONF_DIR, "experiment", name + ".yaml")
    with open(path) as fh:
        raw = _coerce(yaml.safe_load(fh))
    raw.update(overrides)
    return _resolve(raw, raw)


def aero_kwargs(name, conf_dir=None, **overrides):
    """kwargs for ``Aero(**...)`` from an experiment file."""
    exp = load_experiment(name, conf_dir, **overrides)
    return dict(exp["aero"])


def seanet_kwargs(name, conf_dir=None, **overrides):
    """kwargs for ``Seanet(**...)`` from an experiment file."""
    exp = load_experiment(name, conf_dir, **overrides)
    return dict(exp["seanet"])

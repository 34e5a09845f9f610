"""The AERO forward of ``oracle/aero_oracle.py`` for any DConv activation (reference ``modules.py:194-199``: ``act_func``
'snake', 'gelu', any other name ReLU).  ``spec_upsample=False`` needs nothing here: it only changes the geometry, which
``aero_oracle.aero_forward`` already takes from ``geom``.

The restatement of the network stays in ``aero_oracle``.  Without Snake the DConv activation is pointwise, so it is run in
the place of ``aero_oracle.snake`` (whose layout permutes then do not matter) and the missing ``.act.a`` parameters read as
``None``.
"""
import torch

from . import aero_oracle as O

__all__ = ["aero_forward", "activation"]


def activation(act_func):
    """The pointwise DConv activation of a non-Snake ``act_func``."""
    return O.gelu if act_func == "gelu" else torch.relu


class _NoSnakeParams(dict):
    def __missing__(self, key):
        if key.endswith(".act.a"):
            return None
        raise KeyError(key)


def aero_forward(sd, geom, mix, return_spec=False, return_lr_spec=False, explicit=False, taps=None):
    """``aero_oracle.aero_forward`` with the DConv activation of ``geom.kw['act_func']``."""
    act_func = geom.kw["act_func"]
    if act_func == "snake":
        return O.aero_forward(sd, geom, mix, return_spec, return_lr_spec, explicit, taps)
    act = activation(act_func)
    saved = O.snake
    O.snake = lambda x, a: act(x)
    try:
        return O.aero_forward(_NoSnakeParams(sd), geom, mix, return_spec, return_lr_spec, explicit, taps)
    finally:
        O.snake = saved

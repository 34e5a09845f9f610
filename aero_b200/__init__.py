"""aero_b200: H100-native (sm_90a) implementation of the AERO generator forward path.

Public surface (mirrors the reference's ``src.models`` names):
  * ``Aero``                 -- drop-in for ``src.models.aero.Aero``
  * ``Seanet``               -- drop-in for ``src.models.seanet.Seanet``
  * ``spectro`` / ``ispectro`` -- drop-ins for ``src.models.spec``
  * ``load_experiment``      -- Hydra-less reader of ``conf/experiment/*.yaml``
  * ``resample``             -- ``torchaudio.functional.resample`` (default filter) on the GPU
"""
from .model import Aero, AeroGeometry  # noqa: F401
from .config import load_experiment, aero_kwargs, seanet_kwargs  # noqa: F401
from .seanet import Seanet  # noqa: F401
from .resampler import resample  # noqa: F401


def spectro(x, n_fft=512, hop_length=None, pad=0, win_length=None):
    from .spec import spectro as _s
    return _s(x, n_fft, hop_length, pad, win_length)


def ispectro(z, hop_length=None, length=None, pad=0, win_length=None):
    from .spec import ispectro as _i
    return _i(z, hop_length, length, pad, win_length)

"""Import-path shim: ``from src.models.seanet import Seanet`` (reference src/models/modelFactory.py:2) resolves to aero_b200.seanet."""
from aero_b200.seanet import Seanet  # noqa: F401

"""Generator factory with the reference's call shape (reference src/models/modelFactory.py:6-10).
The AERO and SEANet generators are provided by this repo; discriminators are outside the hot path."""
from aero_b200.model import Aero
from aero_b200.seanet import Seanet


def get_model(args):
    exp = args.experiment if hasattr(args, "experiment") else args["experiment"]
    model = exp.model if hasattr(exp, "model") else exp["model"]
    if model not in ("aero", "seanet"):
        raise NotImplementedError(f"aero_b200 provides the 'aero' and 'seanet' generators, got {model!r}")
    kw = getattr(exp, model) if hasattr(exp, model) else exp[model]
    return {"generator": Aero(**kw) if model == "aero" else Seanet(**kw)}

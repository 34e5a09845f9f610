"""Golden vectors for tests/test_oracle.py::test_oracle_blocks_match_reference_golden: one BLSTM block, one LocalState block
and a whole forward of the UNMODIFIED reference on seeded inputs (the comparison that test used to make against the live
reference package).  Block outputs are committed as a 16384-position sample, the waveform in full.

    python tests/golden/make_golden_blocks.py [reference checkout, default $AERO_REFERENCE]
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from util import ROOT, SEED, import_reference, sample_indices, trained_like_, weights_digest, white_noise  # noqa: E402

from aero_b200 import aero_kwargs  # noqa: E402

EXP = "aero_4-16_512_128"


def main():
    ref = import_reference(sys.argv[1] if len(sys.argv) > 1 else None)
    assert ref is not None, "needs a checkout of the reference (argument or $AERO_REFERENCE)"
    aero, kw = ref["aero"], aero_kwargs(EXP)
    torch.manual_seed(SEED)
    rmodel = aero.Aero(**kw).eval()
    rmodel.load_state_dict(trained_like_(rmodel.state_dict()))
    h = white_noise((6, 96, 251), seed=5)
    out = {"exp": EXP, "digest": weights_digest(rmodel.state_dict())}
    with torch.no_grad():
        layer = rmodel.encoder[3].dconv.layers[0]
        for tag in ("lstm", "time_attn"):
            y = layer[tag](h)
            idx = sample_indices(y.numel(), n=16384)
            out[tag + "_shape"] = np.array(y.shape)
            out[tag + "_idx"] = idx.numpy().astype(np.int32)
            out[tag + "_val"] = y.reshape(-1)[idx].numpy()
        out["out"] = rmodel(white_noise((1, 1, 5000))).numpy()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "blocks_4-16_hop128.npz"), **out)


if __name__ == "__main__":
    main()

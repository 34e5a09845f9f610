"""Functional torch restatement of the reference HiFi-GAN multi-period discriminator (reference
``src/models/discriminators.py:89-147``), in any dtype and on any device.

Used by the tests, ``smoke()`` and ``bench_mpd.py`` as the comparison point of ``aero_b200.mpd``.  It reads a ``state_dict`` with the
reference's keys (``discriminators.i.convs.j.{bias, weight_g, weight_v}``, ``discriminators.i.conv_post.*``) and returns what
``MultiPeriodDiscriminator.forward`` returns.  On CUDA its convolutions run on cuDNN, which is how the reference trains.
"""
import torch
import torch.nn.functional as F

SLOPE = 0.1           # discriminators.py:82 (LRELU_SLOPE)


def _w(sd, key):
    # torch.nn.utils.weight_norm with dim=0: w = g * v / ||v|| per output channel
    return torch._weight_norm(sd[key + ".weight_v"], sd[key + ".weight_g"], 0)


def period_forward(sd, prefix, period, x):
    """One DiscriminatorP (discriminators.py:104-121): x [B, 1, T] -> (logits [B, H*period], feature maps [B, C, H, period])."""
    T = x.shape[-1]
    if T % period:                                          # right reflection pad to a multiple of the period (:109-112)
        x = F.pad(x, (0, period - T % period), mode="reflect")
    h = x.reshape(x.shape[0], x.shape[1], -1, period)
    fmap = []
    for j in range(5):                                      # kernel (5, 1), padding (2, 0), stride (3, 1) but the last (:95-100)
        key = f"{prefix}convs.{j}"
        h = F.leaky_relu(F.conv2d(h, _w(sd, key), sd[key + ".bias"], stride=(3, 1) if j < 4 else 1, padding=(2, 0)), SLOPE)
        fmap.append(h)
    h = F.conv2d(h, _w(sd, prefix + "conv_post"), sd[prefix + "conv_post.bias"], padding=(1, 0))      # (:101)
    fmap.append(h)
    return torch.flatten(h, 1, -1), fmap


def mpd_forward(sd, periods, y, y_hat):
    """MultiPeriodDiscriminator.forward (discriminators.py:133-147): (y_d_rs, y_d_gs, fmap_rs, fmap_gs)."""
    out = ([], [], [], [])
    for i, p in enumerate(periods):
        r, fr = period_forward(sd, f"discriminators.{i}.", p, y)
        g, fg = period_forward(sd, f"discriminators.{i}.", p, y_hat)
        for lst, v in zip(out, (r, g, fr, fg)):
            lst.append(v)
    return out

"""H100-native forward pass of the Interactive Deep Colorization Local Hints Network.

Public surface (drop-in for /root/reference/data/colorize_image.py and
/root/reference/models/pytorch/model.py):

    colorize_image.ColorizeImageB200 / ColorizeImageB200Dist   wrapper classes
    model.SIGGRAPHGeneratorB200                                 network class
    engine.LhnContext                                           batched / device-tensor API
    parallel.ShardedColorizer                                   one process per GPU, image sharding

Everything numerical runs in lib/libidc_b200.so (hand-written sm_90a CUDA, csrc/); importing
the package does not load it, the first network call does -- and raises if it is missing.
"""
__version__ = "0.1.0"

from .colorize_image import (ColorizeImageBase, ColorizeImageB200, ColorizeImageB200Dist,  # noqa: F401
                             ColorizeImageB200GlobDist,
                             put_point, lab2rgb_transpose, rgb2lab_transpose)

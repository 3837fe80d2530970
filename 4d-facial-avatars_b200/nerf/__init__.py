"""Drop-in `nerf` package for the NeRFace render path on H100.

Exposes the names the reference's scripts import from `nerf` (train_transformed_rays.py:17-21,
eval_transformed_rays.py:30-39).  The render driver (`run_one_iter_of_nerf`, `predict_and_render_radiance`) and the
model class keep the reference's signatures; everything between ray batch and the seven output maps runs in one
hand-written sm_90a kernel behind the C ABI of include/nfb.h.  There is no PyTorch/CPU fallback for that path."""
from . import models
from .cfgnode import CfgNode
from .nerf_helpers import (get_embedding_function, get_minibatches, get_ray_bundle, img2mse, meshgrid_xy, mse2psnr,
                           positional_encoding, dump_rays)
from .train_utils import GaussianSmoothing, predict_and_render_radiance, render_frames, run_one_iter_of_nerf
from .load_flame import load_flame_data
from .load_llff import load_llff_data
from ._engine import get_precision, set_precision
from .fused_fit import FusedFitter

__all__ = ["models", "CfgNode", "get_embedding_function", "get_minibatches", "get_ray_bundle", "img2mse", "meshgrid_xy",
           "mse2psnr", "positional_encoding", "dump_rays", "GaussianSmoothing", "predict_and_render_radiance",
           "run_one_iter_of_nerf", "render_frames", "load_flame_data", "load_llff_data", "get_precision", "set_precision",
           "FusedFitter"]

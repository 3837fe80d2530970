"""Gradients for training (train_transformed_rays.py:389 `loss.backward()`) and for fitting a frozen avatar to images.

Forward: the fused sm_90a render kernel in its training variant (nfb_render_forward_train) — the same launch as
evaluation, which also leaves the FP16 activations of every layer, the sample depths and the per-sample colours in
buffers owned by the renderer.  Backward: nfb_render_backward_ex (csrc/nfb_train.cu) — compositing backward, the dX chain
and the weight-gradient GEMMs on wgmma, then the chain rule through the kernel's weight folding.  No torch.autograd
graph and no library GEMM is involved; the resampled depths carry no gradient, as in the reference
(`z_samples.detach()`, train_utils.py:124), and `layers_dir.3.*` receives None (unused by the forward, models.py:257).

Like the reference's autograd, every floating-point input that requires grad gets a gradient: the rays (origins and
directions; the near/far columns get zero), the expression, the latent code, the background and the ablation directions
(dir_z).  When no parameter requires grad (a frozen avatar), the backward runs in input-only mode and forms no parameter
gradient, which is most of its cost."""
import torch

from ._engine import PARAM_ORDER

_N_IN = 9  # inputs before the parameters: eng, args, has_fine, rays, frame_index, expr, latent, background, dir_z


class _RenderFn(torch.autograd.Function):
    """A training render and its backward.  frame_index None: one frame (expr [76], latent [32]; nfb_set_frame,
    nfb_render_forward_train, nfb_render_backward_ex); otherwise ray i is conditioned on frame frame_index[i] of expr [F,76] and
    latent [F,32] (nfb_set_frames, nfb_render_forward_frames_train, nfb_render_backward_frames)."""
    @staticmethod
    def forward(ctx, eng, args, has_fine, rays, frame_index, expr, latent, background, dir_z, *params):
        if frame_index is None:
            eng.set_frame(expr, latent)
        else:
            eng.set_frames(expr, latent)
        out = eng.render(rays[:, :3], rays[:, 3:6], train=True, background=background, dir_z=dir_z, frame_index=frame_index, **args)
        ctx.eng = eng
        ctx.keep = out.get("_keep")  # the chunked backward (include/nfb.h) re-reads the forward's inputs
        ctx.token = eng.train_token
        ctx.has_fine = has_fine
        ctx.frames = frame_index is not None
        ctx.shapes = dict(rays=rays.shape, expr=expr.shape, latent=latent.shape,
                          background=background.shape if background is not None else None,
                          dir_z=dir_z.shape if dir_z is not None else None)
        ctx.save_for_backward(*params)
        ctx.set_materialize_grads(False)
        res = (out["rgb_coarse"], out["disp_coarse"], out["acc_coarse"],
               out.get("rgb_fine"), out.get("disp_fine"), out.get("acc_fine"), out["w_last"])
        return tuple(r if r is not None else rays.new_zeros(0) for r in res)

    @staticmethod
    def backward(ctx, *gouts):
        eng = ctx.eng
        if ctx.token != eng.train_token:
            raise RuntimeError("the renderer keeps the saved state of ONE training forward; call backward() before the "
                               "next training-mode render on the same device")
        params = ctx.saved_tensors
        npar = len(PARAM_ORDER)
        if all(g is None for g in gouts):
            return (None,) * (_N_IN + len(params))
        gouts = [g if (g is not None and g.numel() > 0) else None for g in gouts]
        need = ctx.needs_input_grad
        want_params = any(need[_N_IN:])
        inputs = []
        if need[3]:
            inputs += ["ray_origins", "ray_directions"]
        if need[5]:
            inputs.append("expression")
        if need[7]:
            inputs.append("background")
        if need[8]:
            inputs.append("dir_z")
        # the single-frame backward always asks for d latent (an input-only one then keeps its PE-only weight-gradient launch); the
        # multi-frame one only when the latents require grad
        grads_c, grads_f, glat, ing = eng.backward(gouts, params[:npar], params[npar:2 * npar] if ctx.has_fine else None,
                                                   want_latent=need[6] or not ctx.frames, want_params=want_params, inputs=inputs,
                                                   frames=ctx.frames)
        gpar = (tuple(grads_c) + (tuple(grads_f) if ctx.has_fine else ())) if want_params else (None,) * len(params)
        g_rays = None
        if need[3]:
            g_rays = torch.zeros(ctx.shapes["rays"], device=eng.device, dtype=torch.float32)
            g_rays[:, 0:3] = ing["ray_origins"]
            g_rays[:, 3:6] = ing["ray_directions"]
        g_expr = ing["expression"].reshape(ctx.shapes["expr"]) if need[5] else None
        g_lat = glat.reshape(ctx.shapes["latent"]) if need[6] else None
        g_bg = ing["background"].reshape(ctx.shapes["background"]) if need[7] else None
        g_dz = ing["dir_z"].reshape(ctx.shapes["dir_z"]) if need[8] else None
        return (None, None, None, g_rays, None, g_expr, g_lat, g_bg, g_dz) + gpar


def render_with_grad(eng, rays, model_coarse, model_fine, expressions, latent_code, args, frame_index=None):
    """args: the keyword arguments of Renderer.render; its `background` and `dir_z` tensors become inputs of the graph.
    frame_index [N]: a multi-frame render over expressions [F,76] and latent_code [F,32]."""
    sd_c = dict(model_coarse.named_parameters())
    params = [sd_c[k] for k in PARAM_ORDER]
    has_fine = model_fine is not None
    if has_fine:
        sd_f = dict(model_fine.named_parameters())
        params += [sd_f[k] for k in PARAM_ORDER]
    args = dict(args)
    background, dir_z = args.pop("background", None), args.pop("dir_z", None)
    res = _RenderFn.apply(eng, args, has_fine, rays, frame_index, expressions, latent_code, background, dir_z, *params)
    return tuple(r if r.numel() > 0 else None for r in res)

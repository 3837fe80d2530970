"""Gradients for training (train_transformed_rays.py:389 `loss.backward()`).

Forward: the fused sm_90a render kernel in its training variant (nfb_render_forward_train) — the same launch as
evaluation, which also leaves the FP16 activations of every layer, the sample depths and the per-sample colours in
buffers owned by the renderer.  Backward: nfb_render_backward (csrc/nfb_train.cu) — compositing backward, the dX chain
and the weight-gradient GEMMs on wgmma, then the chain rule through the kernel's weight folding.  No torch.autograd
graph and no library GEMM is involved; the resampled depths carry no gradient, as in the reference
(`z_samples.detach()`, train_utils.py:124), and `layers_dir.3.*` receives None (unused by the forward, models.py:257)."""
import torch

from ._engine import PARAM_ORDER


class _RenderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, eng, rays, args, has_fine, expr, latent, *params):
        out = eng.render(rays[:, :3], rays[:, 3:6], train=True, **args)
        ctx.eng = eng
        ctx.keep = out.get("_keep")  # the chunked backward (include/nfb.h) re-reads the forward's inputs
        ctx.token = eng.train_token
        ctx.has_fine = has_fine
        ctx.latent_shape = latent.shape
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
            return (None,) * (6 + len(params))
        gouts = [g if (g is not None and g.numel() > 0) else None for g in gouts]
        grads_c, grads_f, glat = eng.backward(gouts, params[:npar], params[npar:2 * npar] if ctx.has_fine else None)
        gpar = list(grads_c) + (list(grads_f) if ctx.has_fine else [])
        return (None, None, None, None, None, glat.reshape(ctx.latent_shape)) + tuple(gpar)


def render_with_grad(eng, rays, model_coarse, model_fine, expressions, latent_code, args):
    sd_c = dict(model_coarse.named_parameters())
    params = [sd_c[k] for k in PARAM_ORDER]
    has_fine = model_fine is not None
    if has_fine:
        sd_f = dict(model_fine.named_parameters())
        params += [sd_f[k] for k in PARAM_ORDER]
    res = _RenderFn.apply(eng, rays, args, has_fine, expressions, latent_code, *params)
    return tuple(r if r.numel() > 0 else None for r in res)

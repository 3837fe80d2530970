"""Model classes of the render path.  Only ConditionalBlendshapePaperNeRFModel — the class 88/108 shipped configs
use (SURVEY.md §2 row 4) — is provided; its parameters, state_dict keys and shapes equal the reference's
(nerf/models.py:189-234) so existing checkpoints and optimizers work unchanged."""
import torch


class ConditionalBlendshapePaperNeRFModel(torch.nn.Module):
    """Holds the FP32 master weights.  `run_one_iter_of_nerf` never calls forward(): the fused sm_90a kernel
    reads a packed FP16 copy of these parameters (re-packed automatically when they change).  forward() is
    kept for callers that evaluate the MLP on pre-encoded rows; it is plain torch and not the hot path."""

    def __init__(self, num_layers=8, hidden_size=256, skip_connect_every=4, num_encoding_fn_xyz=6,
                 num_encoding_fn_dir=4, include_input_xyz=True, include_input_dir=True, use_viewdirs=True,
                 include_expression=True, latent_code_dim=32):
        super().__init__()
        self.dim_xyz = (3 if include_input_xyz else 0) + 2 * 3 * num_encoding_fn_xyz
        self.dim_dir = (3 if include_input_dir else 0) + 2 * 3 * num_encoding_fn_dir
        self.dim_expression = 76 if include_expression else 0
        self.dim_latent_code = latent_code_dim
        self.use_viewdirs = use_viewdirs
        d_in = self.dim_xyz + self.dim_expression + self.dim_latent_code
        L = torch.nn.Linear
        self.layers_xyz = torch.nn.ModuleList([L(d_in, 256), L(256, 256), L(256, 256), L(d_in + 256, 256),
                                               L(256, 256), L(256, 256)])
        self.fc_feat = L(256, 256)
        self.fc_alpha = L(256, 1)
        self.layers_dir = torch.nn.ModuleList([L(256 + self.dim_dir, 128), L(128, 128), L(128, 128), L(128, 128)])
        self.fc_rgb = L(128, 3)
        self.relu = torch.nn.functional.relu

    def fused_supported(self):
        return (self.dim_xyz, self.dim_dir, self.dim_expression, self.dim_latent_code, self.use_viewdirs) == \
            (63, 24, 76, 32, True)

    def forward(self, x, expr=None, latent_code=None, **kwargs):
        xyz, dirs = x[..., :self.dim_xyz], x[..., self.dim_xyz:]
        rows = xyz.shape[0]
        cond = [xyz]
        if self.dim_expression > 0:
            cond.append((expr * 1 / 3).reshape(1, -1).expand(rows, -1))
        cond.append(latent_code.reshape(1, -1).expand(rows, -1))
        initial = torch.cat(cond, dim=1)
        h = initial
        for i, layer in enumerate(self.layers_xyz):
            h = self.relu(layer(torch.cat((initial, h), dim=-1) if i == 3 else h))
        feat = self.fc_feat(h)
        alpha = self.fc_alpha(feat)
        g = self.relu(self.layers_dir[0](torch.cat((feat, dirs), dim=-1) if self.use_viewdirs else feat))
        g = self.relu(self.layers_dir[1](g))
        g = self.relu(self.layers_dir[2](g))  # layers_dir[3] is allocated but unused, as in the reference
        return torch.cat((self.fc_rgb(g), alpha), dim=-1)

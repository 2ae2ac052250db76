"""TEST INFRASTRUCTURE ONLY — nn.Module wrapper giving the oracle the ``EGNNDynamics`` call contract
(reference dynamics.py:87), so the DDPM samplers can be driven on CPU: used by the wrapper parity tests
and by bench.py's CPU-baseline / ``--impl reference`` legs (kind "port": the benchmark does not need the
reference checkout)."""
import torch.nn as nn

from . import egnn_oracle


class OracleDynamics(nn.Module):
    def __init__(self, cfg, state_dict, device='cpu'):
        super().__init__()
        self.cfg, self.device = cfg, device
        self.sd = {k: v.to(device) for k, v in state_dict.items()}      # moved once, not per call
        self.update_pocket_coords = cfg.update_pocket_coords
        self.n_dims = cfg.n_dims
        self.calls = 0

    def forward(self, xh_atoms, xh_residues, t, mask_atoms, mask_residues):
        self.calls += 1
        return egnn_oracle.denoiser_forward(self.cfg, self.sd, xh_atoms, xh_residues, t, mask_atoms, mask_residues,
                                            device=self.device)

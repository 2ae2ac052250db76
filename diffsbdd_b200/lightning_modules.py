"""``LigandPocketDDPM`` façade: the API surface ``generate_ligands.py`` / ``inpaint.py`` / ``optimize.py`` use.

reference: lightning_modules.py — constructor / model assembly (:31-173), ``prepare_pocket`` (:714-752),
``generate_ligands`` (:754-872).  Kept: class name, constructor signature, ``load_from_checkpoint``,
``.ddpm`` (with the reference's DDPM class identities — ``generate_ligands`` dispatches on the exact type,
lightning_modules.py:814, :837), ``.x_dims/.atom_nf/.aa_nf``, ``lig_type_encoder/decoder``,
``pocket_type_encoder/decoder``, ``dataset_info``; the likelihood evaluation ``forward`` / ``validation_step`` /
``test_step`` (:217-302, :365-380).  Not built (out of scope, SURVEY.md §2 rows 5-7, 12): training steps, W&B logging,
molecule metrics, visualisation.  PDB parsing (BioPython) and
molecule building (RDKit/OpenBabel, the reference's ``analysis`` package) are imported lazily and only by
``generate_ligands``; the tensor-level path ``generate_ligand_tensors`` needs neither.

Works without pytorch_lightning (absent offline): then the base class is ``torch.nn.Module`` and
``load_from_checkpoint`` is implemented here with the same checkpoint layout Lightning writes
({'state_dict', 'hyper_parameters'}).
"""
from __future__ import annotations

from argparse import Namespace

import numpy as np
import torch
import torch.nn.functional as F

from . import seeded
from .conditional_model import ConditionalDDPM, SimpleConditionalDDPM
from .dynamics import EGNNDynamics
from .en_diffusion import EnVariationalDiffusion, check_sampler, follows_dynamics_determinism, scatter_mean, num_nodes_to_batch_mask

try:  # pragma: no cover - not installed in the offline image
    import pytorch_lightning as pl
    _Base = pl.LightningModule
except Exception:  # noqa: BLE001
    pl = None
    _Base = torch.nn.Module

FLOAT_TYPE = torch.float32   # reference constants.py:8-9
INT_TYPE = torch.int64

_ELEMENTS = ['C', 'N', 'O', 'S', 'B', 'Br', 'Cl', 'P', 'I', 'F']
_AMINO = ['A', 'C', 'D', 'E', 'F', 'G', 'H', 'I', 'K', 'L', 'M', 'N', 'P', 'Q', 'R', 'S', 'T', 'V', 'W', 'Y']


def _vocab(symbols):
    return {s: i for i, s in enumerate(symbols)}, list(symbols)


def _dataset_info(name):
    """Type vocabularies of reference constants.py:96-100, :154-158, :169-173 (chemistry tables omitted)."""
    if name in ('crossdock', 'bindingmoad'):
        ae, ad = _vocab(_ELEMENTS)
        re_, rd = _vocab(_AMINO)
    elif name == 'crossdock_full':
        ae, ad = _vocab(_ELEMENTS + ['others'])
        re_, rd = _vocab(_ELEMENTS + ['others'])
    else:
        raise KeyError(name)
    return {'atom_encoder': ae, 'atom_decoder': ad, 'aa_encoder': re_, 'aa_decoder': rd}


def _get(ns, key, default=None):
    return ns.__dict__.get(key, default) if isinstance(ns, Namespace) else ns.get(key, default)


class LigandPocketDDPM(_Base):
    def __init__(self, outdir, dataset, datadir, batch_size, lr, egnn_params: Namespace, diffusion_params,
                 num_workers, augment_noise, augment_rotation, clip_grad, eval_epochs, eval_params,
                 visualize_sample_epoch, visualize_chain_epoch, auxiliary_loss, loss_params, mode, node_histogram,
                 pocket_representation='CA', virtual_nodes=False):
        super().__init__()
        if pl is not None:
            self.save_hyperparameters()
        ddpm_models = {'joint': EnVariationalDiffusion, 'pocket_conditioning': ConditionalDDPM,
                       'pocket_conditioning_simple': SimpleConditionalDDPM}
        assert mode in ddpm_models
        assert pocket_representation in {'CA', 'full-atom'}
        self.mode, self.pocket_representation = mode, pocket_representation
        self.dataset_name, self.datadir, self.outdir = dataset, datadir, outdir
        self.batch_size, self.lr = batch_size, lr
        self.loss_type = _get(diffusion_params, 'diffusion_loss_type')
        self.auxiliary_loss = auxiliary_loss
        self.T = _get(diffusion_params, 'diffusion_steps')
        self.dataset_info = _dataset_info(dataset)
        self.lig_type_encoder = dict(self.dataset_info['atom_encoder'])
        self.lig_type_decoder = list(self.dataset_info['atom_decoder'])
        if pocket_representation == 'CA':
            self.pocket_type_encoder = dict(self.dataset_info['aa_encoder'])
            self.pocket_type_decoder = list(self.dataset_info['aa_decoder'])
        else:
            # full-atom pockets use the SAME vocabulary objects as the ligand (lightning_modules.py:90-97): with
            # virtual_nodes the appended 'Ne' type therefore also widens aa_nf, as reference checkpoints expect
            self.pocket_type_encoder = self.lig_type_encoder
            self.pocket_type_decoder = self.lig_type_decoder
        self.virtual_nodes = virtual_nodes
        self.max_num_nodes = len(node_histogram) - 1
        symbol = 'Ne'
        if virtual_nodes:                                  # lightning_modules.py:119-131
            self.lig_type_encoder[symbol] = len(self.lig_type_encoder)
            self.virtual_atom = self.lig_type_encoder[symbol]
            self.lig_type_decoder.append(symbol)
            self.dataset_info['atom_encoder'] = self.lig_type_encoder
            self.dataset_info['atom_decoder'] = self.lig_type_decoder
        self.atom_nf, self.aa_nf, self.x_dims = len(self.lig_type_decoder), len(self.pocket_type_decoder), 3

        net_dynamics = EGNNDynamics(                       # lightning_modules.py:137-160
            atom_nf=self.atom_nf, residue_nf=self.aa_nf, n_dims=self.x_dims,
            joint_nf=_get(egnn_params, 'joint_nf'),
            device=_get(egnn_params, 'device', 'cuda') if torch.cuda.is_available() else 'cpu',
            hidden_nf=_get(egnn_params, 'hidden_nf'), act_fn=torch.nn.SiLU(),
            n_layers=_get(egnn_params, 'n_layers'), attention=_get(egnn_params, 'attention'),
            tanh=_get(egnn_params, 'tanh'), norm_constant=_get(egnn_params, 'norm_constant'),
            inv_sublayers=_get(egnn_params, 'inv_sublayers'), sin_embedding=_get(egnn_params, 'sin_embedding'),
            normalization_factor=_get(egnn_params, 'normalization_factor'),
            aggregation_method=_get(egnn_params, 'aggregation_method'),
            edge_cutoff_ligand=_get(egnn_params, 'edge_cutoff_ligand'),
            edge_cutoff_pocket=_get(egnn_params, 'edge_cutoff_pocket'),
            edge_cutoff_interaction=_get(egnn_params, 'edge_cutoff_interaction'),
            update_pocket_coords=(mode == 'joint'),
            reflection_equivariant=_get(egnn_params, 'reflection_equivariant'),
            edge_embedding_dim=_get(egnn_params, 'edge_embedding_dim'))
        self.ddpm = ddpm_models[mode](                     # lightning_modules.py:162-174
            dynamics=net_dynamics, atom_nf=self.atom_nf, residue_nf=self.aa_nf, n_dims=self.x_dims,
            timesteps=_get(diffusion_params, 'diffusion_steps'),
            noise_schedule=_get(diffusion_params, 'diffusion_noise_schedule'),
            noise_precision=_get(diffusion_params, 'diffusion_noise_precision'),
            loss_type=_get(diffusion_params, 'diffusion_loss_type'),
            norm_values=_get(diffusion_params, 'normalize_factors'),
            size_histogram=node_histogram,
            virtual_node_idx=self.lig_type_encoder[symbol] if virtual_nodes else None)

    # ---- checkpoint contract (Lightning layout) -------------------------------------------------------------
    if pl is None:
        @classmethod
        def load_from_checkpoint(cls, checkpoint_path, map_location=None, strict=True, **overrides):
            ckpt = torch.load(checkpoint_path, map_location=map_location, weights_only=False)
            hparams = dict(ckpt.get('hyper_parameters', {}))
            hparams.update(overrides)
            model = cls(**hparams)
            model.load_state_dict(ckpt['state_dict'], strict=strict)
            if map_location is not None and not isinstance(map_location, dict):
                model.to(map_location)
            return model

        @property
        def device(self):
            return next(self.parameters()).device

    # ---- pocket preparation (lightning_modules.py:714-752) ----------------------------------------------------
    def prepare_pocket_from_arrays(self, pocket_coord, pocket_types, repeats=1):
        """Tensor-level core of ``prepare_pocket``: coordinates [n,3] and integer types [n] -> pocket dict."""
        pocket_coord = torch.as_tensor(np.asarray(pocket_coord), device=self.device, dtype=FLOAT_TYPE)
        pocket_types = torch.as_tensor(np.asarray(pocket_types), device=self.device, dtype=INT_TYPE)
        one_hot = F.one_hot(pocket_types, num_classes=len(self.pocket_type_encoder))
        n = len(pocket_coord)
        return {'x': pocket_coord.repeat(repeats, 1), 'one_hot': one_hot.repeat(repeats, 1),
                'size': torch.tensor([n] * repeats, device=self.device, dtype=INT_TYPE),
                'mask': torch.repeat_interleave(torch.arange(repeats, device=self.device, dtype=INT_TYPE), n)}

    def prepare_pocket(self, biopython_residues, repeats=1):
        if self.pocket_representation == 'CA':
            from Bio.PDB.Polypeptide import three_to_one
            coords = np.array([res['CA'].get_coord() for res in biopython_residues])
            types = [self.pocket_type_encoder[three_to_one(res.get_resname())] for res in biopython_residues]
        else:
            atoms = [a for res in biopython_residues for a in res.get_atoms()
                     if (a.element.capitalize() in self.pocket_type_encoder or a.element != 'H')]
            coords = np.array([a.get_coord() for a in atoms])
            types = [self.pocket_type_encoder[a.element.capitalize()] for a in atoms]
        return self.prepare_pocket_from_arrays(coords, types, repeats)

    # ---- generation (lightning_modules.py:754-872) -------------------------------------------------------------
    @follows_dynamics_determinism
    @torch.no_grad()
    def generate_ligand_tensors(self, pocket, num_nodes_lig=None, timesteps=None, n_nodes_bias=0, n_nodes_min=0,
                                seeds=None, sampler='ddpm', eta=0.0, **kwargs):
        """Everything ``generate_ligands`` does between pocket preparation and molecule building
        (lightning_modules.py:785-852): returns (xh_lig, xh_pocket, lig_mask, pocket_mask) in the original
        pocket frame.  ``seeds``: one int64 per sample (seeded.py); the ligand size prior and every sampler draw then come
        from the sample's own seed (the size by inverse CDF over p(n_lig | n_pocket)).  ``sampler`` / ``eta``: the reverse
        step of ConditionalDDPM.sample_given_pocket.  A joint model refuses a few-step sampler here: this route runs its
        RePaint inpainting with the 'ddpm' step.  Few-step generation for a fixed pocket with a joint model is
        ``self.ddpm.inpaint(ligand, pocket, lig_fixed=zeros, pocket_fixed=ones, sampler=..., eta=...)`` (DESIGN §14)."""
        check_sampler(sampler, eta)
        if sampler != 'ddpm' and type(self.ddpm) == EnVariationalDiffusion:
            raise ValueError(f"sampler={sampler!r} is not supported for a joint model: it generates through RePaint inpainting, "
                             f"which runs the 'ddpm' step only here (use ddpm.inpaint with every pocket node fixed and sampler=...)")
        self.ddpm.eval()
        seeds = seeded.as_seeds(seeds, len(pocket['size']), pocket['x'].device)
        pocket_com_before = scatter_mean(pocket['x'], pocket['mask'], dim=0)
        if num_nodes_lig is None and seeds is not None:
            num_nodes_lig = seeded.size_prior(self.ddpm.size_distribution.prob, pocket['size'], seeds)
        elif num_nodes_lig is None:
            num_nodes_lig = self.ddpm.size_distribution.sample_conditional(n1=None, n2=pocket['size'])
        num_nodes_lig = torch.clamp(num_nodes_lig + n_nodes_bias, min=n_nodes_min)
        if type(self.ddpm) == EnVariationalDiffusion:
            # joint model: inpaint the ligand with every pocket node fixed (lightning_modules.py:814-835)
            lig_mask = num_nodes_to_batch_mask(len(num_nodes_lig), num_nodes_lig, self.device)
            ligand = {'x': torch.zeros((len(lig_mask), self.x_dims), device=self.device, dtype=FLOAT_TYPE),
                      'one_hot': torch.zeros((len(lig_mask), self.atom_nf), device=self.device, dtype=FLOAT_TYPE),
                      'size': num_nodes_lig, 'mask': lig_mask}
            lig_fixed = torch.zeros(len(lig_mask), device=self.device)
            pocket_fixed = torch.ones(len(pocket['mask']), device=self.device)
            xh_lig, xh_pocket, lig_mask, pocket_mask = self.ddpm.inpaint(
                ligand, pocket, lig_fixed, pocket_fixed, timesteps=timesteps, seeds=seeds, **kwargs)
        elif type(self.ddpm) == ConditionalDDPM:
            xh_lig, xh_pocket, lig_mask, pocket_mask = self.ddpm.sample_given_pocket(
                pocket, num_nodes_lig, timesteps=timesteps, seeds=seeds, sampler=sampler, eta=eta)
        else:
            raise NotImplementedError
        pocket_com_after = scatter_mean(xh_pocket[:, :self.x_dims], pocket_mask, dim=0)
        shift = pocket_com_before - pocket_com_after
        xh_pocket[:, :self.x_dims] += shift[pocket_mask]
        xh_lig[:, :self.x_dims] += shift[lig_mask]
        return xh_lig, xh_pocket, lig_mask, pocket_mask

    def generate_ligands(self, pdb_file, n_samples, pocket_ids=None, ref_ligand=None, num_nodes_lig=None,
                         sanitize=False, largest_frag=False, relax_iter=0, timesteps=None, n_nodes_bias=0,
                         n_nodes_min=0, **kwargs):
        assert (pocket_ids is None) ^ (ref_ligand is None)
        try:
            from Bio.PDB import PDBParser
            import utils                                                   # reference utils.py (repo root)
            from analysis.molecule_builder import build_molecule, process_molecule
        except ImportError as e:  # pragma: no cover
            raise ImportError('generate_ligands needs BioPython + the reference chemistry stack (RDKit/OpenBabel, '
                              '`analysis` and `utils` of the DiffSBDD repo on sys.path); use '
                              'generate_ligand_tensors() for the tensor-level path') from e
        pdb_struct = PDBParser(QUIET=True).get_structure('', pdb_file)[0]
        if pocket_ids is not None:
            residues = [pdb_struct[x.split(':')[0]][(' ', int(x.split(':')[1]), ' ')] for x in pocket_ids]
        else:
            residues = utils.get_pocket_from_ligand(pdb_struct, ref_ligand)
        pocket = self.prepare_pocket(residues, repeats=n_samples)
        xh_lig, _, lig_mask, _ = self.generate_ligand_tensors(
            pocket, num_nodes_lig, timesteps, n_nodes_bias, n_nodes_min, **kwargs)
        x = xh_lig[:, :self.x_dims].detach().cpu()
        atom_type = xh_lig[:, self.x_dims:].argmax(1).detach().cpu()
        lig_mask = lig_mask.cpu()
        molecules = []
        for mol_pc in zip(utils.batch_to_list(x, lig_mask), utils.batch_to_list(atom_type, lig_mask)):
            mol = build_molecule(*mol_pc, self.dataset_info, add_coords=True)
            mol = process_molecule(mol, add_hydrogens=False, sanitize=sanitize, relax_iter=relax_iter,
                                   largest_frag=largest_frag)
            if mol is not None:
                molecules.append(mol)
        return molecules

    # ---- likelihood evaluation (lightning_modules.py:217-302, :365-380) ---------------------------------------------
    def get_ligand_and_pocket(self, data):
        """Batch dict of the reference's datasets -> (ligand, pocket) dicts on this module's device."""
        ligand = {'x': data['lig_coords'].to(self.device, FLOAT_TYPE),
                  'one_hot': data['lig_one_hot'].to(self.device, FLOAT_TYPE),
                  'size': data['num_lig_atoms'].to(self.device, INT_TYPE),
                  'mask': data['lig_mask'].to(self.device, INT_TYPE)}
        if self.virtual_nodes:
            ligand['num_virtual_atoms'] = data['num_virtual_atoms'].to(self.device, INT_TYPE)
        pocket = {'x': data['pocket_coords'].to(self.device, FLOAT_TYPE),
                  'one_hot': data['pocket_one_hot'].to(self.device, FLOAT_TYPE),
                  'size': data['num_pocket_nodes'].to(self.device, INT_TYPE),
                  'mask': data['pocket_mask'].to(self.device, INT_TYPE)}
        return ligand, pocket

    def forward(self, data):
        """Per-complex negative log-likelihood bound -log p(x, h, N) (the VLB / evaluation branch of the reference) and the
        batch means of its terms.  Training (the l2 loss, the Lennard-Jones auxiliary term) is not built."""
        if self.training:
            raise NotImplementedError('training is not built in diffsbdd_b200 (no backward kernels); call eval() first')
        ligand, pocket = self.get_ligand_and_pocket(data)
        delta_log_px, error_t_lig, error_t_pocket, SNR_weight, loss_0_x_ligand, loss_0_x_pocket, loss_0_h, \
            neg_log_const_0, kl_prior, log_pN, _t_int, _xh_lig_hat, info = self.ddpm(ligand, pocket, return_info=True)
        # the loss terms are negative log-likelihoods; SNR_weight = 1 - SNR(s - t) is negative
        loss_t = -self.T * 0.5 * SNR_weight * (error_t_lig + error_t_pocket)
        loss_0 = loss_0_x_ligand + loss_0_x_pocket + loss_0_h + neg_log_const_0
        nll = loss_t + loss_0 + kl_prior - delta_log_px
        if not self.virtual_nodes:          # -log p(x, h, N) = -log p(x, h | N) - log p(N); constant N with virtual nodes
            nll = nll - log_pN
        for key, val in (('error_t_lig', error_t_lig), ('error_t_pocket', error_t_pocket), ('SNR_weight', SNR_weight),
                         ('loss_0', loss_0), ('kl_prior', kl_prior), ('delta_log_px', delta_log_px),
                         ('neg_log_const_0', neg_log_const_0), ('log_pN', log_pN)):
            info[key] = val.mean(0)
        return nll, info

    def log_metrics(self, metrics_dict, split, batch_size=None, **kwargs):
        if pl is None or getattr(self, '_trainer', None) is None:
            return                          # logging needs a Lightning trainer
        for m, value in metrics_dict.items():
            self.log(f'{m}/{split}', value, batch_size=batch_size, **kwargs)

    def _shared_eval(self, data, prefix, *args):
        nll, info = self.forward(data)
        info['loss'] = nll.mean(0)
        self.log_metrics(info, prefix, batch_size=len(data['num_lig_atoms']), sync_dist=True)
        return info

    @torch.no_grad()
    def validation_step(self, data, *args):
        return self._shared_eval(data, 'val', *args)

    @torch.no_grad()
    def test_step(self, data, *args):
        return self._shared_eval(data, 'test', *args)

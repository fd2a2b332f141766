"""``ResShiftSampler`` — the orchestration surface of the reference's ``sampler.py`` (reference
sampler.py:26-308) over the H100-native hot path.

Same constructor and methods (``sample_func``, ``inference``); models are still built from the yaml
``target:`` strings (reference utils/util_common.py:19-29), so pointing ``model.target`` /
``diffusion.target`` at ``resshift_b200.models.*`` (or putting ``resshift_b200/overlay`` first on
PYTHONPATH, see INTEGRATION.md) is all that changes.  The VQ-GAN autoencoder is whatever the config names
(a PyTorch module; bookends stay in PyTorch).  Multi-GPU follows the reference: one process per GPU,
contiguous batch slices per rank (sampler.py:273-277), same seed on every rank; on top of that rank 0 can
broadcast the weights over NCCL (``broadcast_weights``) and results can be gathered (``gather_results``).
``shard_tiles=True`` deals the tiles of each chunk across the ranks instead, bit-identical to one GPU (DESIGN.md §6);
a chunk with fewer units than ranks runs each unit on a team of ranks that splits its VQ-GAN bottleneck attention.
``devices=`` (or ``RS_DEVICES``) does the same inside one process: a pool of model replicas, one per listed GPU, each
driven by its own thread (resshift_b200.device_pool).
"""
from __future__ import annotations

import importlib
import inspect
import math
import os
import random
import re
from contextlib import nullcontext
from pathlib import Path
from typing import Any, NamedTuple, Optional

import numpy as np
import torch
import torch.distributed as dist
import torch.nn.functional as F

from .device_pool import DevicePool, Replica, pool_devices
from .parallel import gather_counts, row_exchange, team_group, unit_schedule


# --------------------------------------------------------------------------------------------------
# tiny config helpers (the reference uses OmegaConf, which is not a dependency here)
# --------------------------------------------------------------------------------------------------
class Cfg(dict):
    """dict with attribute access, enough of OmegaConf's DictConfig for the sampler."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v

    @staticmethod
    def wrap(obj):
        if isinstance(obj, dict):
            return Cfg({k: Cfg.wrap(v) for k, v in obj.items()})
        if isinstance(obj, list):
            return [Cfg.wrap(v) for v in obj]
        return obj


def load_yaml(path) -> Cfg:
    """yaml -> Cfg with ``${a.b.c}`` interpolation (the only OmegaConf feature the shipped configs use)."""
    import yaml
    raw = yaml.safe_load(Path(path).read_text())

    def lookup(dotted):
        node = raw
        for part in dotted.split("."):
            node = node[part]
        return node

    def resolve(node):
        if isinstance(node, dict):
            return {k: resolve(v) for k, v in node.items()}
        if isinstance(node, list):
            return [resolve(v) for v in node]
        if isinstance(node, str):
            m = re.fullmatch(r"\$\{([^}]+)\}", node.strip())
            if m:
                return resolve(lookup(m.group(1)))
        return node

    return Cfg.wrap(resolve(raw))


# yaml `target:` strings of the reference that this package implements natively: an unmodified reference config
# (configs/*.yaml) builds this package's classes (INTEGRATION.md); anything else is imported as written
_NATIVE_TARGETS = {
    "models.unet.UNetModelSwin": "resshift_b200.models.unet.UNetModelSwin",
    "models.unet.UNetModel": "resshift_b200.models.unet.UNetModel",
    "models.unet.UNetModelConv": "resshift_b200.models.unet.UNetModelConv",
    "models.script_util.create_gaussian_diffusion": "resshift_b200.models.script_util.create_gaussian_diffusion",
    "ldm.models.autoencoder.VQModelTorch": "resshift_b200.models.autoencoder.VQModelTorch",
    "ldm.models.autoencoder.AutoencoderKLTorch": "resshift_b200.models.autoencoder.AutoencoderKLTorch",
}


def _plain(obj):
    """Cfg / OmegaConf containers -> plain dict / list (constructor kwargs)."""
    if isinstance(obj, dict) or hasattr(obj, "items"):
        return {k: _plain(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)) or type(obj).__name__ == "ListConfig":
        return [_plain(v) for v in obj]
    return obj


def instantiate_from_config(config):
    """reference utils/util_common.py:19-29"""
    if "target" not in config:
        raise KeyError("Expected key `target` to instantiate.")
    target = _NATIVE_TARGETS.get(config["target"], config["target"])
    module, cls = target.rsplit(".", 1)
    return getattr(importlib.import_module(module), cls)(**_plain(config.get("params", dict())))


def make_configs(ucfg, dcfg, autoencoder: Optional[dict] = None, state_dict: Any = None) -> Cfg:
    """Programmatic equivalent of a configs/*.yaml for this package's targets."""
    from .config import UNetModelConfig, UNetModelConvConfig
    target = ("UNetModel" if isinstance(ucfg, UNetModelConfig) else
              "UNetModelConv" if isinstance(ucfg, UNetModelConvConfig) else "UNetModelSwin")
    return Cfg.wrap({
        "model": {"target": f"resshift_b200.models.unet.{target}", "ckpt_path": state_dict, "params": ucfg.to_kwargs()},
        "diffusion": {"target": "resshift_b200.models.script_util.create_gaussian_diffusion", "params": dcfg.to_kwargs()},
        "autoencoder": autoencoder,
    })


def reload_model(model, ckpt):
    """reference utils/util_net.py:86-98: copy every key of the MODEL's state_dict from the checkpoint."""
    keys = list(ckpt.keys())
    module_flag = keys[0].startswith("module.")
    compile_flag = "_orig_mod" in keys[0]
    for k, v in model.state_dict().items():
        tk = k
        if compile_flag and "_orig_mod." not in k:
            tk = "_orig_mod." + tk
        if module_flag and not k.startswith("module"):
            tk = "module." + tk
        assert tk in ckpt, f"checkpoint lacks {tk}"
        v.copy_(ckpt[tk])


def tile_starts(length: int, patch: int, stride: int):
    """Start offsets of the overlapping tiles along one axis — the same list, in the same order, as the reference's
    ImageSpliterTh.extract_starts (utils/util_image.py:923-932): multiples of `stride`, the last ones pulled back so
    that every tile lies inside the image, duplicates dropped."""
    if length <= patch:
        return [0]
    out = []
    for s0 in range(0, length, stride):
        s1 = min(s0, length - patch)
        if s1 not in out:
            out.append(s1)
    return out


def plan_tiles(h: int, w: int, patch: int, stride: int, chop_bs: int):
    """Host-side plan of the tiled pass, identical to iterating the reference's ImageSpliterTh(im, patch, stride, sf,
    extra_bs=chop_bs) (utils/util_image.py:889-960): (row starts, column starts, tile height, tile width, groups) where
    `groups` lists, per sample_func call, the (h_start, w_start) of the tiles stacked on the batch axis."""
    hs_list, ws_list = tile_starts(h, patch, stride), tile_starts(w, patch, stride)
    starts = [(hs, ws) for hs in hs_list for ws in ws_list]
    k = max(1, int(chop_bs))
    return hs_list, ws_list, min(patch, h), min(patch, w), [starts[i:i + k] for i in range(0, len(starts), k)]


class UnitNoise(NamedTuple):
    """The random numbers of one work unit, drawn ahead of it in one-GPU order (ResShiftSampler._unit_noises): the
    loop's T+1 noise tensors [T+1, n, c, h, w] on the device, and the first stage's posterior noise [n, c, h, w] on the
    CPU for an autoencoder that samples one (AutoencoderKLTorch), else None."""
    loop: torch.Tensor
    posterior: Optional[torch.Tensor]


def _unsupported_posterior(autoencoder) -> bool:
    """Whether ``autoencoder.encode`` samples a posterior (it takes ``sample_posterior``, as the reference's KL first
    stages do) without accepting that noise from the caller: its draws would follow the units a rank runs."""
    if autoencoder is None or getattr(autoencoder, "samples_posterior", False):
        return False
    try:
        return "sample_posterior" in inspect.signature(autoencoder.encode).parameters
    except (TypeError, ValueError):
        return False


def tile_counts(units, schedule, world: int):
    """counts[g][r]: tiles of shape group g that executor r keeps, for ResShiftSampler._plan_units ``units`` run by
    ``schedule`` (parallel.unit_schedule) — what parallel.gather_counts needs on every rank."""
    counts = [[0] * world for _ in range(units[-1][0] + 1)]
    for (g, starts, _, _), (a, _) in zip(units, schedule):
        counts[g][a] += len(starts)
    return counts


class BaseSampler:
    def __init__(self, configs, sf=4, use_amp=True, chop_size=128, chop_stride=128, chop_bs=1, padding_offset=16,
                 seed=10000):
        self.configs = configs
        self.sf, self.chop_size, self.chop_stride, self.chop_bs = sf, chop_size, chop_stride, chop_bs
        self.seed, self.use_amp, self.padding_offset = seed, use_amp, padding_offset
        self.setup_dist()
        self.setup_seed()
        self.build_model()

    def setup_seed(self, seed=None):
        seed = self.seed if seed is None else seed
        random.seed(seed)
        np.random.seed(seed)
        torch.manual_seed(seed)
        torch.cuda.manual_seed_all(seed)

    def setup_dist(self):
        """One process per GPU (torchrun); reference sampler.py:66-77."""
        if not torch.cuda.is_available():
            raise RuntimeError("resshift_b200 needs a CUDA device (no CPU fallback)")
        world = int(os.environ.get("WORLD_SIZE", "1"))
        if world > 1:
            rank = int(os.environ["LOCAL_RANK"])
            torch.cuda.set_device(rank % torch.cuda.device_count())
            if not dist.is_initialized():
                dist.init_process_group(backend="nccl", init_method="env://")
        self.num_gpus = world
        self.rank = int(os.environ.get("LOCAL_RANK", "0")) if world > 1 else 0

    def write_log(self, log_str):
        if self.rank == 0:
            print(log_str, flush=True)

    def build_model(self):
        self.base_diffusion = instantiate_from_config(self.configs.diffusion)
        ckpt = self.configs.model.ckpt_path
        assert ckpt is not None
        ae_cfg = self.configs.get("autoencoder", None)
        ae_ckpt = None if ae_cfg is None else ae_cfg.get("ckpt_path", None)
        self.model, self.autoencoder = self._instantiate_models(ckpt, ae_ckpt)

    def _instantiate_models(self, ckpt, ae_ckpt):
        """The denoiser (frozen) and the autoencoder (None when the configs have none) of the configs on the current
        device, in eval mode, with the checkpoints ``ckpt`` / ``ae_ckpt`` (a path or a state dict; ``ae_ckpt`` may be
        None) loaded."""
        model = instantiate_from_config(self.configs.model).cuda()
        self.load_model(model, ckpt)
        self.freeze_model(model)
        model.eval()
        autoencoder = None
        if self.configs.get("autoencoder", None) is not None:
            autoencoder = instantiate_from_config(self.configs.autoencoder).cuda()
            if ae_ckpt is not None:
                self.load_model(autoencoder, ae_ckpt)
            autoencoder.eval()
        return model, autoencoder

    def load_model(self, model, ckpt_path):
        if isinstance(ckpt_path, dict):
            state = ckpt_path
        else:
            state = torch.load(ckpt_path, map_location=f"cuda:{torch.cuda.current_device()}")
        if "state_dict" in state:
            state = state["state_dict"]
        with torch.no_grad():
            reload_model(model, state)

    def freeze_model(self, net):
        for p in net.parameters():
            p.requires_grad = False

    # -- NCCL plumbing the north-star asks for (the reference has each rank read the checkpoint) --------
    def broadcast_weights(self, src: int = 0):
        """One flat NCCL broadcast of every parameter from rank `src` (resshift_b200.parallel), then repack."""
        if self.num_gpus > 1:
            from .parallel import broadcast_state_dict
            broadcast_state_dict({k: p.data for k, p in self.model.named_parameters()}, src=src)
            self.model.pack_weights(force=True)

    def gather_results(self, local: torch.Tensor, batch: Optional[int] = None) -> Optional[torch.Tensor]:
        """All ranks call; every rank gets the global batch in order (NCCL all_gather over NVLink).  `batch` = global
        batch size; shards follow the reference's ceil(bs / world) slicing (sampler.py:273-277), so trailing ranks may
        hold fewer images or none (resshift_b200.parallel.gather_shards pads and trims)."""
        if self.num_gpus == 1:
            return local
        from .parallel import gather_shards
        return gather_shards(local.contiguous(), local.shape[0] * self.num_gpus if batch is None else batch)


class ResShiftSampler(BaseSampler):
    def __init__(self, configs, sf=4, use_amp=True, chop_size=128, chop_stride=128, chop_bs=1, padding_offset=16,
                 seed=10000, shard_tiles=None, devices=None):
        """``shard_tiles``: deal the tiles of each chunk of images across the ranks instead of slicing the chunk by
        image (``_run_rank``); ``None`` reads ``RS_SHARD_TILES`` (default 0), so unmodified reference scripts can turn
        it on.

        ``devices``: run ``inference`` on a pool of GPUs from this one process: ``"all"``, ``"0,2,3"`` or a list of
        indices; the first is the primary (models, noise, assembly, output).  ``None`` reads ``RS_DEVICES`` (unset: no
        pool).  The same device may be listed more than once: every entry is one model replica with its own stream.
        Refused with ``WORLD_SIZE > 1``, on devices that differ in SM count or compute capability, and for
        configurations that take the generic per-step route."""
        self.devices = pool_devices(devices)
        if shard_tiles is None:
            shard_tiles = os.environ.get("RS_SHARD_TILES", "0") not in ("", "0")
        self.shard_tiles = bool(shard_tiles)
        self._team_groups = {}                  # rank tuple -> process group of an attention team (parallel.team_group)
        with torch.cuda.device(self.devices[0]) if self.devices else nullcontext():
            super().__init__(configs, sf=sf, use_amp=use_amp, chop_size=chop_size, chop_stride=chop_stride,
                             chop_bs=chop_bs, padding_offset=padding_offset, seed=seed)
        self.pool = self._build_pool() if self.devices else None

    def _build_pool(self):
        """One replica per entry of ``self.devices``: the first uses this sampler's models, every other one gets the
        denoiser and the VQ-GAN built from the same configs on its device, with this sampler's parameters copied over
        device to device (each replica owns its library handles; modules holding them are never deep-copied)."""
        self._check_shardable("a device pool")
        replicas = []
        for k, d in enumerate(self.devices):
            if k == 0:
                model, autoencoder = self.model, self.autoencoder
            else:
                with torch.cuda.device(d):
                    model, autoencoder = self._instantiate_models(self.model.state_dict(), self.autoencoder.state_dict())
            replicas.append(Replica(k, d, model, autoencoder, primary=self.devices[0]))
        for d in sorted(set(self.devices)):                       # the parameter copies
            torch.cuda.synchronize(d)
        return DevicePool(replicas)

    def sample_func(self, y0, noise_repeat=False, mask=False):
        """y0: [n, c, h, w] in [-1, 1] -> [n, c, h*sf, w*sf] in [-1, 1] (reference sampler.py:119-165)."""
        if noise_repeat:
            self.setup_seed()
        if mask is False:      # reference quirk (`mask=False` default is "not None"); real callers pass None
            mask = None
        return self._pad_crop(y0, mask, lambda y, model_kwargs: self.base_diffusion.p_sample_loop(
            y=y, model=self.model, first_stage_model=self.autoencoder, noise=None, noise_repeat=noise_repeat,
            clip_denoised=(self.autoencoder is None), denoised_fn=None, model_kwargs=model_kwargs, progress=False))

    def _pad_crop(self, y0, mask, run):
        """``run(y0, model_kwargs)`` on y0 (and mask) reflect-padded to multiples of padding_offset, its result cropped to
        the input's size times sf and clamped to [-1, 1] (reference sampler.py:130-165)."""
        offset = self.padding_offset
        ori_h, ori_w = y0.shape[2:]
        flag_pad = not (ori_h % offset == 0 and ori_w % offset == 0)
        if flag_pad:
            pad_h = math.ceil(ori_h / offset) * offset - ori_h
            pad_w = math.ceil(ori_w / offset) * offset - ori_w
            y0 = F.pad(y0, pad=(0, pad_w, 0, pad_h), mode="reflect")
            if mask is not None:
                mask = F.pad(mask, pad=(0, pad_w, 0, pad_h), mode="reflect")
        results = run(y0, {"lq": y0} if mask is None else {"lq": y0, "mask": mask})
        if flag_pad:
            results = results[:, :, :ori_h * self.sf, :ori_w * self.sf]
        return results.clamp_(-1.0, 1.0)

    def _autocast(self):
        return torch.autocast("cuda") if self.use_amp else nullcontext()

    # ---------------------------------------------------------------------------------------------
    def _sample_tiled(self, im_lq, mask=None, noise_repeat=False):
        """[b, c, h, w] in [-1, 1] -> super-resolved [b, c, h*sf, w*sf] in [-1, 1]; inputs larger than chop_size are cut
        into overlapping chop_size tiles at the reference's start offsets (utils/util_image.py:923-932), `chop_bs` tiles
        are stacked on the batch axis per call exactly like ImageSpliterTh.__next__ (:940-960, `extra_bs`) — so the
        noise drawn per call matches the reference's — and overlaps are averaged (update / gather :962-979) by
        rs_op_tile_gather in the reference's accumulation order."""
        b, c, h, w = im_lq.shape
        if self._one_tile(h, w):
            with self._autocast():
                return self.sample_func(im_lq, noise_repeat=noise_repeat, mask=mask).float()
        tiles = []
        for unit in self._plan_units([(h, w)]):
            pch, mch = self._unit_input([im_lq], [mask], unit)
            with self._autocast():
                res = self.sample_func(pch, noise_repeat=noise_repeat, mask=mch).float()
            tiles.extend(torch.split(res, b, dim=0))
        return self._assemble(torch.stack(tiles), h, w)

    def _one_tile(self, h, w):
        """Whether an [h, w] input runs whole, in one sample_func call, rather than tiled (reference sampler.py:186)."""
        return not (h > self.chop_size or w > self.chop_size)

    # -- the sample_func calls of a chunk as work units, scheduled across ranks or replicas, bit-identical to one GPU --
    def _plan_units(self, shapes):
        """Work units of a chunk whose shape groups have LQ sizes ``shapes`` [(h, w)], in the order a one-GPU run makes
        its sample_func calls: (group, tile starts, tile h, tile w).  An image that fits in one tile is one unit with
        the single start (0, 0)."""
        units = []
        for g, (h, w) in enumerate(shapes):
            _, _, th, tw, groups = plan_tiles(h, w, self.chop_size, self.chop_stride, self.chop_bs)
            units += [(g, starts, th, tw) for starts in groups]
        return units

    def _schedule(self, n_units, world):
        """parallel.unit_schedule of a chunk of ``n_units`` units on ``world`` executors.  Teams need executors that can
        exchange attention rows (the ranks of a process group, or a pool's replicas in process) and an autoencoder that
        can split its attention (VQModelTorch.attention_team)."""
        teams = (self.pool is not None or dist.is_initialized()) and hasattr(self.autoencoder, "attention_team")
        return unit_schedule(n_units, world, teams)

    def _run_rank(self, lqs, masks, noise_repeat, units, schedule, rank):
        """One rank's part of a chunk in shard mode.  ``lqs`` / ``masks``: per shape group, [b, 3, h, w] in [-1, 1] and
        [b, 1, h, w] or None; ``units``: their _plan_units; ``schedule``: the executors [a, e) of each unit
        (_schedule).  The rank walks every unit and draws its noise (_unit_noises), so the CUDA generator is where a
        one-GPU run has it, and runs the units whose range contains ``rank``: under the autoencoder's attention_team
        when the range has more than one rank, with the query rows exchanged inside the team's process group, so every
        member ends with the whole unit.  Nothing else in the chain draws random numbers.  Returns, per group, the tiles
        of the units this rank keeps (rank == a) [n, b, 3, th*sf, tw*sf] in plan order (n may be 0).  With teams in the
        schedule every rank of the default group must call this."""
        self._check_shardable()
        if any(lq is None for lq in lqs):
            raise ValueError("shard_tiles needs the LQ image of every group")
        for a, e in schedule:                        # every rank creates every multi-rank team's group, in team order
            if e - a > 1:
                team_group(tuple(range(a, e)), self._team_groups)
        kept = [None] * len(units)
        for i, noises, spec in self._unit_noises(lqs, noise_repeat, units):
            a, e = schedule[i]
            if not a <= rank < e:
                continue
            team = None
            if e - a > 1:
                team = (rank - a, e - a, row_exchange(team_group(tuple(range(a, e)), self._team_groups), e - a, rank - a))
            res = self._run_unit(*self._unit_input(lqs, masks, units[i]), noises, spec, team=team)
            if rank == a:
                kept[i] = res
        return self._stack_shares(kept, lqs, units)

    def _latent_spec(self, n, h, w, dtype):
        """Shape and dtype of z_y = encode_first_stage(y, up_sample=True) for an [n, 3, h, w] input (after the
        padding_offset reflect-pad) of dtype ``dtype``, derived from the configs without running the encoder: the first
        stage (VQ or KL: both have ``embed_dim`` latent channels) keeps the data dtype (encode_first_stage) and
        downsamples by 2^(len(ch_mult) - 1)."""
        sf = self.base_diffusion.sf
        ae = self.configs.autoencoder.params
        f = 2 ** (len(ae.ddconfig.ch_mult) - 1)
        return (n, int(ae.embed_dim), int(h * sf) // f, int(w * sf) // f), dtype

    def _check_shardable(self, mode="shard_tiles"):
        if _unsupported_posterior(self.autoencoder):
            raise RuntimeError(
                f"{mode} needs every random number of a unit drawn ahead of it in one-GPU order; this autoencoder "
                f"({type(self.autoencoder).__name__}) samples its posterior inside encode and cannot take that noise "
                "(use resshift_b200.models.autoencoder.AutoencoderKLTorch)")
        if not self.base_diffusion._native_ok(self.model, clip_denoised=(self.autoencoder is None), denoised_fn=None,
                                              model_kwargs={"lq": None}):
            raise RuntimeError(
                f"{mode} needs the fused sampling loop, whose noise can be drawn ahead of the encoder; this "
                "configuration takes the generic per-step route (no autoencoder, so x0 is clipped; a model other than "
                "this package's UNetModelSwin, UNetModel or UNetModelConv; or T outside 2..64)")

    def _sample_unit(self, y0, mask, noises, spec, replica):
        """sample_func with its noise given (a UnitNoise): reflect-pad, encode_first_stage(up_sample=True) with the
        posterior noise, sample_latent(noises=), decode_first_stage, crop, clamp — the same steps, in the same order.
        ``spec`` is the z_y shape and dtype the noise was drawn for; it must be the real one.  ``replica``: a device_pool.Replica whose models run the unit, or
        None for this sampler's."""
        model, autoencoder = (self.model, self.autoencoder) if replica is None else (replica.model, replica.autoencoder)
        diff = self.base_diffusion

        def run(y, model_kwargs):
            z_y = diff.encode_first_stage(y, autoencoder, up_sample=True, posterior_noise=noises.posterior)
            assert (tuple(z_y.shape), z_y.dtype, z_y.is_contiguous()) == (spec[0], spec[1], True), \
                f"derived z_y {spec} != real {tuple(z_y.shape)} {z_y.dtype}"
            final = diff.sample_latent(z_y, model, model_kwargs, noises=noises.loop)
            with torch.no_grad():
                return diff.decode_first_stage(final, first_stage_model=autoencoder)
        return self._pad_crop(y0, mask, run)

    def _unit_noises(self, lqs, noise_repeat, units):
        """Yields (unit index, UnitNoise, z_y spec) for every unit of ``units`` in order: its T+1 noise tensors drawn as
        GaussianDiffusion.draw_noises does (after setup_seed with noise_repeat, as sample_func does), on the device of
        ``lqs``, so that the CUDA generator is where a one-GPU run has it whichever units run here.  For an
        autoencoder that samples its posterior (AutoencoderKLTorch), the unit's posterior noise is drawn too, as its
        encode would draw it (torch.randn on the CPU generator, after that setup_seed), so that generator also follows
        the one-GPU run."""
        offset = self.padding_offset
        posterior = getattr(self.autoencoder, "samples_posterior", False)
        for i, (g, starts, th, tw) in enumerate(units):
            lq = lqs[g]
            with self._autocast():
                if noise_repeat:
                    self.setup_seed()
                spec = self._latent_spec(lq.shape[0] * len(starts), math.ceil(th / offset) * offset,
                                         math.ceil(tw / offset) * offset, lq.dtype)
                post = torch.randn(spec[0]) if posterior else None
                noises = self.base_diffusion.draw_noises(torch.empty(spec[0], dtype=spec[1], device=lq.device),
                                                         noise_repeat=noise_repeat)
            yield i, UnitNoise(noises, post), spec

    @staticmethod
    def _unit_input(lqs, masks, unit):
        """The LQ tiles (and mask tiles or None) of one unit stacked on the batch axis, as sample_func receives them."""
        g, starts, th, tw = unit
        lq, mask = lqs[g], masks[g]
        pch = torch.cat([lq[:, :, hs:hs + th, ws:ws + tw] for hs, ws in starts], dim=0)
        mch = None if mask is None else torch.cat([mask[:, :, hs:hs + th, ws:ws + tw] for hs, ws in starts], dim=0)
        return pch, mch

    def _run_unit(self, pch, mch, noises, spec, team=None, replica=None):
        """One unit: _sample_unit under autocast (and under the autoencoder's attention_team with ``team``), as fp32.
        ``replica``: the device_pool.Replica that runs it (its models, on the current device and stream)."""
        autoencoder = self.autoencoder if replica is None else replica.autoencoder
        with self._autocast(), autoencoder.attention_team(*team) if team is not None else nullcontext():
            return self._sample_unit(pch, mch, noises, spec, replica).float()

    def _stack_shares(self, results, lqs, units):
        """Per group, the tiles of the units with an output in ``results`` (per unit, [n * b, 3, th*sf, tw*sf] or None)
        stacked [n, b, 3, th*sf, tw*sf] in plan order (n may be 0)."""
        out, empty = [[] for _ in lqs], {}
        for (g, _, th, tw), res in zip(units, results):
            empty[g] = (0,) + tuple(lqs[g].shape[:2]) + (th * self.sf, tw * self.sf)
            if res is not None:
                out[g].extend(torch.split(res, lqs[g].shape[0], dim=0))
        return [torch.stack(t) if t else torch.empty(empty[g], device=lq.device)
                for g, (t, lq) in enumerate(zip(out, lqs))]

    def _assemble(self, tiles, h, w):
        """All tiles of one shape group [T, b, c, th*sf, tw*sf], in plan order -> [b, c, h*sf, w*sf]: the tile of an
        image that runs whole, else the overlaps averaged by rs_op_tile_gather in the reference's accumulation order."""
        if self._one_tile(h, w):
            return tiles[0]
        from . import _lib
        sf = self.sf
        hs_list = tile_starts(h, self.chop_size, self.chop_stride)
        ws_list = tile_starts(w, self.chop_size, self.chop_stride)
        tiles_t = tiles.contiguous()
        b, c, th, tw = tiles_t.shape[1:]
        out = torch.empty(b, c, h * sf, w * sf, dtype=torch.float32, device=tiles_t.device)
        ys = torch.tensor([v * sf for v in hs_list], dtype=torch.int32, device=tiles_t.device)
        xs = torch.tensor([v * sf for v in ws_list], dtype=torch.int32, device=tiles_t.device)
        _lib.check(_lib.lib.rs_op_tile_gather(tiles_t.data_ptr(), b, c, h * sf, w * sf, th, tw, len(hs_list), len(ws_list),
                                              ys.data_ptr(), xs.data_ptr(), out.data_ptr(), _lib.current_stream()))
        return out

    def _process(self, im_lq, mask=None, noise_repeat=False, mask_back=True):
        """[b, c, h, w] in [-1, 1] -> [b, c, h*sf, w*sf] in [0, 1] (reference sampler.py:176-223)."""
        im_sr = self._sample_tiled(im_lq, mask=mask, noise_repeat=noise_repeat)
        im_sr = im_sr * 0.5 + 0.5
        if mask_back and mask is not None:
            m = mask * 0.5 + 0.5
            im_sr = im_sr * m + (im_lq * 0.5 + 0.5) * (1 - m)
        return im_sr

    def _process_u8(self, lq_u8, mask_u8=None, noise_repeat=False, mask_back=True, bgr=True):
        """uint8 edges fused on the device (SURVEY.md §8f rank 3): lq_u8 [b, h, w, 3] (RGB) and optional mask_u8 [b, h, w, 1]
        -> uint8 [b, h*sf, w*sf, 3] in BGR (what cv2.imwrite takes) or RGB order.  Ingest = (v / 255 - 0.5) / 0.5
        (reference datapipe default transform); emit = clamp, * 0.5 + 0.5, mask-back blend, round(v * 255)
        (sampler.py:218-223 + utils/util_image.tensor2img :216-273)."""
        lq, mask = self._ingest_u8(lq_u8, mask_u8)
        sr = self._sample_tiled(lq, mask=mask, noise_repeat=noise_repeat)
        return self._emit_u8(sr, lq, mask, mask_back=mask_back, bgr=bgr)

    @staticmethod
    def _ingest_u8(lq_u8, mask_u8=None):
        from . import _lib
        b, h, w, _ = lq_u8.shape
        lq = torch.empty(b, 3, h, w, dtype=torch.float32, device=lq_u8.device)
        _lib.check(_lib.lib.rs_op_ingest_u8(lq_u8.contiguous().data_ptr(), b, h, w, 3, lq.data_ptr(), _lib.current_stream()))
        mask = None
        if mask_u8 is not None:
            mask = torch.empty(b, 1, h, w, dtype=torch.float32, device=lq_u8.device)
            _lib.check(_lib.lib.rs_op_ingest_u8(mask_u8.contiguous().data_ptr(), b, h, w, 1, mask.data_ptr(), _lib.current_stream()))
        return lq, mask

    def _emit_u8(self, sr, lq, mask, mask_back=True, bgr=True):
        from . import _lib
        sr = sr.contiguous()
        b, _, h, w = lq.shape
        out = torch.empty(b, h * self.sf, w * self.sf, 3, dtype=torch.uint8, device=lq.device)
        blend = mask_back and mask is not None
        if blend and self.sf != 1:
            raise ValueError("mask-back needs sf == 1 (as in the reference's inpainting tasks)")
        _lib.check(_lib.lib.rs_op_emit_u8(sr.data_ptr(), lq.data_ptr() if blend else None, mask.data_ptr() if blend else None,
                                          b, h * self.sf, w * self.sf, int(bgr), out.data_ptr(), _lib.current_stream()))
        return out

    def inference(self, in_path, out_path, mask_path=None, mask_back=True, bs=1, noise_repeat=False):
        """File / folder driver (reference sampler.py:167-308).  Image I/O through OpenCV.  With ``shard_tiles`` every
        rank reads the whole chunk and runs its part of the chunk's unit schedule (_run_rank); rank 0 assembles and writes.
        With a device pool the chunk's units run on the pool's replicas (_inference_pool)."""
        import cv2
        if self.shard_tiles:
            self._check_shardable()
        in_path, out_path = Path(in_path), Path(out_path)
        if self.rank == 0:
            assert in_path.exists()
            out_path.mkdir(parents=True, exist_ok=True)
        if self.num_gpus > 1:
            dist.barrier()

        def read(p, gray=False):
            im = cv2.imread(str(p), cv2.IMREAD_GRAYSCALE if gray else cv2.IMREAD_COLOR)
            if im is None:
                raise FileNotFoundError(p)
            im = im[:, :, None] if gray else cv2.cvtColor(im, cv2.COLOR_BGR2RGB)
            return torch.from_numpy(np.ascontiguousarray(im))                 # uint8 HWC; normalised on the device

        exts = {".png", ".jpg", ".jpeg", ".bmp"}
        files = sorted(p for p in in_path.rglob("*") if p.suffix.lower() in exts) if in_path.is_dir() else [in_path]
        self.write_log(f"Find {len(files)} images in {in_path}")
        def read_group(group):
            paths, ims = zip(*group)
            lq = torch.stack(ims).cuda()
            mask = None
            if mask_path is not None:
                mp = Path(mask_path)
                mask = torch.stack([read(mp / p.name if mp.is_dir() else mp, gray=True) for p in paths]).cuda()
            return paths, lq, mask

        for i0 in range(0, len(files), bs):
            chunk = files[i0:i0 + bs]
            if self.pool is not None:
                self._inference_pool(_same_shape_groups(chunk, read), read_group, out_path, mask_back, noise_repeat)
            elif self.shard_tiles:
                self._inference_shards(_same_shape_groups(chunk, read), read_group, out_path, mask_back, noise_repeat)
            else:
                micro = math.ceil(bs / self.num_gpus)                     # reference sampler.py:273-277
                mine = chunk[self.rank * micro:(self.rank + 1) * micro]
                for group in _same_shape_groups(mine, read):
                    paths, lq, mask = read_group(group)
                    sr = self._process_u8(lq, mask_u8=mask, noise_repeat=noise_repeat, mask_back=mask_back, bgr=True).cpu().numpy()
                    for p, im in zip(paths, sr):
                        cv2.imwrite(str(out_path / f"{p.stem}.png"), im)
            if self.num_gpus > 1:
                dist.barrier()
        self.write_log(f"Processing done, enjoy the results in {out_path}")

    def _inference_shards(self, groups, read_group, out_path, mask_back, noise_repeat):
        """One chunk in shard_tiles mode: this rank's part of the unit schedule, one gather per shape group, assembly and
        writing on rank 0."""
        paths, lqs, masks = self._read_chunk(groups, read_group)
        units = self._plan_units([tuple(lq.shape[2:]) for lq in lqs])
        schedule = self._schedule(len(units), self.num_gpus)
        shares = self._run_rank(lqs, masks, noise_repeat, units, schedule, self.rank)
        for g, counts in enumerate(tile_counts(units, schedule, self.num_gpus)):
            tiles = gather_counts(shares[g], counts)
            if self.rank == 0:
                self._write_group(paths[g], tiles, lqs[g], masks[g], out_path, mask_back)

    def _inference_pool(self, groups, read_group, out_path, mask_back, noise_repeat):
        """One chunk on the device pool: read and ingest on the primary, every unit's noise drawn there in one-GPU
        order, the units run on the replicas (device_pool.DevicePool.run), then assembly and writing on the primary."""
        with torch.cuda.device(self.pool.primary):
            paths, lqs, masks = self._read_chunk(groups, read_group)
            units = self._plan_units([tuple(lq.shape[2:]) for lq in lqs])
            tiles = self._stack_shares(self.pool.run(self, lqs, masks, noise_repeat, units), lqs, units)
            for g, lq in enumerate(lqs):
                self._write_group(paths[g], tiles[g], lq, masks[g], out_path, mask_back)

    def _read_chunk(self, groups, read_group):
        """Per shape group of a chunk: the paths, the LQ images [b, 3, h, w] and the masks [b, 1, h, w] or None, in
        [-1, 1] on the current device."""
        paths, lqs, masks = [], [], []
        for group in groups:
            p, lq_u8, mask_u8 = read_group(group)
            lq, mask = self._ingest_u8(lq_u8, mask_u8)
            paths.append(p)
            lqs.append(lq)
            masks.append(mask)
        return paths, lqs, masks

    def _write_group(self, paths, tiles, lq, mask, out_path, mask_back):
        """Assembles one shape group from all its tiles (plan order) and writes its PNGs."""
        import cv2
        sr = self._emit_u8(self._assemble(tiles, *lq.shape[2:]), lq, mask, mask_back=mask_back, bgr=True)
        for p, im in zip(paths, sr.cpu().numpy()):
            cv2.imwrite(str(out_path / f"{p.stem}.png"), im)


def _same_shape_groups(paths, read):
    groups = {}
    for p in paths:
        im = read(p)
        groups.setdefault(tuple(im.shape), []).append((p, im))
    return list(groups.values())

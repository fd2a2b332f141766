"""``ResShiftSampler`` — the orchestration surface of the reference's ``sampler.py`` (reference
sampler.py:26-308) over the H100-native hot path.

Same constructor and methods (``sample_func``, ``inference``); models are still built from the yaml
``target:`` strings (reference utils/util_common.py:19-29), so pointing ``model.target`` /
``diffusion.target`` at ``resshift_b200.models.*`` (or putting ``resshift_b200/overlay`` first on
PYTHONPATH, see INTEGRATION.md) is all that changes.  The VQ-GAN autoencoder is whatever the config names
(a PyTorch module; bookends stay in PyTorch).  Multi-GPU follows the reference: one process per GPU,
contiguous batch slices per rank (sampler.py:273-277), same seed on every rank; on top of that rank 0 can
broadcast the weights over NCCL (``broadcast_weights``) and results can be gathered (``gather_results``).
"""
from __future__ import annotations

import importlib
import math
import os
import random
import re
from contextlib import nullcontext
from pathlib import Path
from typing import Any, Optional

import numpy as np
import torch
import torch.distributed as dist
import torch.nn.functional as F


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
    "models.script_util.create_gaussian_diffusion": "resshift_b200.models.script_util.create_gaussian_diffusion",
    "ldm.models.autoencoder.VQModelTorch": "resshift_b200.models.autoencoder.VQModelTorch",
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
    return Cfg.wrap({
        "model": {"target": "resshift_b200.models.unet.UNetModelSwin", "ckpt_path": state_dict, "params": ucfg.to_kwargs()},
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
        model = instantiate_from_config(self.configs.model).cuda()
        ckpt = self.configs.model.ckpt_path
        assert ckpt is not None
        self.load_model(model, ckpt)
        self.freeze_model(model)
        self.model = model.eval()
        if self.configs.get("autoencoder", None) is not None:
            ae_cfg = self.configs.autoencoder
            autoencoder = instantiate_from_config(ae_cfg).cuda()
            if ae_cfg.get("ckpt_path", None) is not None:
                self.load_model(autoencoder, ae_cfg.ckpt_path)
            self.autoencoder = autoencoder.eval()
        else:
            self.autoencoder = None

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
    def sample_func(self, y0, noise_repeat=False, mask=False):
        """y0: [n, c, h, w] in [-1, 1] -> [n, c, h*sf, w*sf] in [-1, 1] (reference sampler.py:119-165)."""
        if noise_repeat:
            self.setup_seed()
        offset = self.padding_offset
        ori_h, ori_w = y0.shape[2:]
        flag_pad = not (ori_h % offset == 0 and ori_w % offset == 0)
        if flag_pad:
            pad_h = math.ceil(ori_h / offset) * offset - ori_h
            pad_w = math.ceil(ori_w / offset) * offset - ori_w
            y0 = F.pad(y0, pad=(0, pad_w, 0, pad_h), mode="reflect")
            if mask is not None and mask is not False:
                mask = F.pad(mask, pad=(0, pad_w, 0, pad_h), mode="reflect")
        if mask is False:      # reference quirk (`mask=False` default is "not None"); real callers pass None
            mask = None
        model_kwargs = {"lq": y0} if mask is None else {"lq": y0, "mask": mask}
        results = self.base_diffusion.p_sample_loop(
            y=y0, model=self.model, first_stage_model=self.autoencoder, noise=None, noise_repeat=noise_repeat,
            clip_denoised=(self.autoencoder is None), denoised_fn=None, model_kwargs=model_kwargs,
            progress=False)
        if flag_pad:
            results = results[:, :, :ori_h * self.sf, :ori_w * self.sf]
        return results.clamp_(-1.0, 1.0)

    # ---------------------------------------------------------------------------------------------
    def _sample_tiled(self, im_lq, mask=None, noise_repeat=False):
        """[b, c, h, w] in [-1, 1] -> super-resolved [b, c, h*sf, w*sf] in [-1, 1]; inputs larger than chop_size are cut
        into overlapping chop_size tiles at the reference's start offsets (utils/util_image.py:923-932), `chop_bs` tiles
        are stacked on the batch axis per call exactly like ImageSpliterTh.__next__ (:940-960, `extra_bs`) — so the
        noise drawn per call matches the reference's — and overlaps are averaged (update / gather :962-979) by
        rs_op_tile_gather in the reference's accumulation order."""
        from . import _lib
        ctx = torch.autocast("cuda") if self.use_amp else nullcontext()
        b, c, h, w = im_lq.shape
        if not (h > self.chop_size or w > self.chop_size):
            with ctx:
                return self.sample_func(im_lq, noise_repeat=noise_repeat, mask=mask).float()
        sf = self.sf
        hs_list, ws_list, th, tw, groups = plan_tiles(h, w, self.chop_size, self.chop_stride, self.chop_bs)
        tiles = []
        for group in groups:
            pch = torch.cat([im_lq[:, :, hs:hs + th, ws:ws + tw] for hs, ws in group], dim=0)
            mch = None if mask is None else torch.cat([mask[:, :, hs:hs + th, ws:ws + tw] for hs, ws in group], dim=0)
            with ctx:
                res = self.sample_func(pch, noise_repeat=noise_repeat, mask=mch).float()
            tiles.extend(torch.split(res, b, dim=0))
        tiles_t = torch.stack(tiles).contiguous()                                   # [T, b, c, th*sf, tw*sf]
        out = torch.empty(b, tiles_t.shape[2], h * sf, w * sf, dtype=torch.float32, device=im_lq.device)
        ys = torch.tensor([v * sf for v in hs_list], dtype=torch.int32, device=im_lq.device)
        xs = torch.tensor([v * sf for v in ws_list], dtype=torch.int32, device=im_lq.device)
        _lib.check(_lib.lib.rs_op_tile_gather(tiles_t.data_ptr(), b, tiles_t.shape[2], h * sf, w * sf, th * sf, tw * sf,
                                              len(hs_list), len(ws_list), ys.data_ptr(), xs.data_ptr(), out.data_ptr(),
                                              _lib.current_stream()))
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
        from . import _lib
        b, h, w, _ = lq_u8.shape
        lq = torch.empty(b, 3, h, w, dtype=torch.float32, device=lq_u8.device)
        _lib.check(_lib.lib.rs_op_ingest_u8(lq_u8.contiguous().data_ptr(), b, h, w, 3, lq.data_ptr(), _lib.current_stream()))
        mask = None
        if mask_u8 is not None:
            mask = torch.empty(b, 1, h, w, dtype=torch.float32, device=lq_u8.device)
            _lib.check(_lib.lib.rs_op_ingest_u8(mask_u8.contiguous().data_ptr(), b, h, w, 1, mask.data_ptr(), _lib.current_stream()))
        sr = self._sample_tiled(lq, mask=mask, noise_repeat=noise_repeat).contiguous()
        out = torch.empty(b, h * self.sf, w * self.sf, 3, dtype=torch.uint8, device=lq_u8.device)
        blend = mask_back and mask is not None
        if blend and self.sf != 1:
            raise ValueError("mask-back needs sf == 1 (as in the reference's inpainting tasks)")
        _lib.check(_lib.lib.rs_op_emit_u8(sr.data_ptr(), lq.data_ptr() if blend else None, mask.data_ptr() if blend else None,
                                          b, h * self.sf, w * self.sf, int(bgr), out.data_ptr(), _lib.current_stream()))
        return out

    def inference(self, in_path, out_path, mask_path=None, mask_back=True, bs=1, noise_repeat=False):
        """File / folder driver (reference sampler.py:167-308).  Image I/O through OpenCV."""
        import cv2
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
        for i0 in range(0, len(files), bs):
            chunk = files[i0:i0 + bs]
            micro = math.ceil(bs / self.num_gpus)                     # reference sampler.py:273-277
            mine = chunk[self.rank * micro:(self.rank + 1) * micro]
            for group in _same_shape_groups(mine, read):
                paths, ims = zip(*group)
                lq = torch.stack(ims).cuda()
                mask = None
                if mask_path is not None:
                    mp = Path(mask_path)
                    mask = torch.stack([read(mp / p.name if mp.is_dir() else mp, gray=True) for p in paths]).cuda()
                sr = self._process_u8(lq, mask_u8=mask, noise_repeat=noise_repeat, mask_back=mask_back, bgr=True).cpu().numpy()
                for p, im in zip(paths, sr):
                    cv2.imwrite(str(out_path / f"{p.stem}.png"), im)
            if self.num_gpus > 1:
                dist.barrier()
        self.write_log(f"Processing done, enjoy the results in {out_path}")


def _same_shape_groups(paths, read):
    groups = {}
    for p in paths:
        im = read(p)
        groups.setdefault(tuple(im.shape), []).append((p, im))
    return list(groups.values())

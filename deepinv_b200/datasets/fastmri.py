"""FastMRI slice reader (drop-in for deepinv/datasets/fastmri.py:163-520 `FastMRISliceDataset` and the mask / scaling part of
`MRISliceTransform`, :563-749).

Same constructor keywords, sample enumeration (`slice_index`: "all" | int | tuple | "middle" | "middle+i" | "random",
`subsample_volumes`, `filter_id`, `SliceSampleID`), `__len__` / `__getitem__` contract — `(target, kspace[, params])` with k-space
as planar fp32 `(2, (N,) H, W)`, target `(1, h, w)` or nan, `params["mask"]` when the file carries one — as the reference.

Volumes: fastMRI `.h5` files when `h5py` is importable (like the reference, which raises the ImportError otherwise), and
"HDF5-shaped" `.npz` volumes with the same keys (`kspace` complex64 (D, (N,) H, W), optional `reconstruction_rss` /
`reconstruction_esc` (D, h, w), optional `mask` (W,), optional `attrs__num_low_frequency`) — the container this image can read.

GPU path: `load_batch(indices, device)` stages the raw INTERLEAVED complex slices in one pinned host buffer, moves them
with a single asynchronous copy and de-interleaves on the device (`dinvk_interleaved_to_planar`): the reference's host-side
`view_as_real + moveaxis + contiguous` pass per slice (mixins.py:148-156) and the per-sample H2D copies of a default
DataLoader do not exist; file masks come back as a `(B, W)` device tensor (`line_mask` expands them to the `(B, 2, H, W)` view
`MRI(mask=...)` takes, zero pattern exact).
"""
from __future__ import annotations

import os
import warnings
from collections import defaultdict
from pathlib import Path
from typing import Any, Callable, NamedTuple

import numpy as np
import torch

try:  # the reference keeps the ImportError and raises it at construction (fastmri.py:31-38, :355)
    import h5py
except ImportError as _e:  # pragma: no cover
    h5py = _e


class _NpzVolume:
    """read-only view of an HDF5-shaped .npz volume (keys as in fastMRI files; attributes as `attrs__<name>` entries)"""

    def __init__(self, fname):
        self._z = np.load(fname, mmap_mode="r", allow_pickle=False)
        self.attrs = {k[len("attrs__"):]: self._z[k] for k in self._z.files if k.startswith("attrs__")}

    def keys(self):
        return [k for k in self._z.files if not k.startswith("attrs__")]

    def __contains__(self, k):
        return k in self.keys()

    def __getitem__(self, k):
        return self._z[k]

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self._z.close()


def _open(fname):
    fname = Path(fname)
    if fname.suffix == ".npz":
        return _NpzVolume(fname)
    if isinstance(h5py, ImportError):
        raise h5py
    return h5py.File(fname, "r")


def from_torch_complex(z: torch.Tensor) -> torch.Tensor:
    """(B, ...) complex -> (B, 2, ...) planar real (mixins.py:148-156)"""
    return torch.view_as_real(z).moveaxis(-1, 1).contiguous()


class MRISliceTransform:
    """mask handling and scalar normalisation of `deepinv.datasets.MRISliceTransform` (fastmri.py:563-749): a file mask (W,)
    becomes (1, H, W); a mask generator draws a mask per slice (seeded by the slice id when `seed_mask_generator`) and is
    applied to the k-space; `normalize=<number>` scales by normalize / kspace.max().  Coil-map estimation (ESPIRiT), noise
    pre-whitening and the ACS-percentile normalisation are outside the hot path and raise."""

    def __init__(self, mask_generator=None, seed_mask_generator: bool = True, estimate_coil_maps=False, acs=None,
                 espirit_crop=False, prewhiten=False, normalize=False):
        if estimate_coil_maps or prewhiten or normalize is True:
            raise NotImplementedError("deepinv_b200.datasets.MRISliceTransform: coil-map estimation, pre-whitening and ACS "
                                      "normalisation are not part of the accelerated path (SURVEY §8: out of scope)")
        self.mask_generator, self.seed_mask_generator, self.normalize = mask_generator, seed_mask_generator, normalize

    def generate_mask(self, kspace: torch.Tensor, seed) -> torch.Tensor:
        if isinstance(seed, str):  # the reference hashes the string id into an integer seed (fastmri.py:645-650)
            seed = int.from_bytes(seed.encode(), "little") % (2 ** 31)
        return self.mask_generator.step(seed=seed if self.seed_mask_generator else None, img_size=kspace.shape[-2:],
                                        batch_size=0)["mask"]

    def __call__(self, target, kspace, mask=None, seed=None, metadata=None, **kwargs):
        if self.normalize:
            kspace = kspace / kspace.max() * self.normalize
        params = {}
        if mask is not None:
            params["mask"] = mask.unsqueeze(0).repeat(kspace.shape[-2], 1).unsqueeze(0).float()  # (W,) -> (1, H, W)
        if self.mask_generator is not None:
            params["mask"] = self.generate_mask(kspace, seed)
            kspace = kspace * params["mask"]
        return target, kspace, params


class FastMRISliceDataset(torch.utils.data.Dataset):
    class SliceSampleID(NamedTuple):
        fname: Path
        slice_ind: int
        metadata: dict[str, Any]

    @staticmethod
    def torch_shuffle(x: list, generator: torch.Generator | None = None) -> list:
        return [x[i] for i in torch.randperm(len(x), generator=generator).tolist()]

    def __init__(self, root=None, target_root=None, load_metadata_from_cache: bool = False, save_metadata_to_cache: bool = False,
                 metadata_cache_file="dataset_cache.pkl", slice_index="all", subsample_volumes: float | None = 1.0,
                 transform: Callable | None = None, filter_id: Callable | None = None, rng: torch.Generator | None = None):
        if load_metadata_from_cache or save_metadata_to_cache:
            raise NotImplementedError("metadata caching (pickle files) is not part of this reader")
        if root is None or not os.path.isdir(root):
            raise ValueError(f"The `root` folder doesn't exist. Please set `root` properly. Current value `{root}`.")
        self.root = Path(root)
        self.transform = transform if transform is not None else MRISliceTransform()
        self.target_root = Path(target_root) if target_root is not None else None
        all_fnames = sorted(list(self.root.glob("*.h5")) + list(self.root.glob("*.npz")))
        if any(f.suffix == ".h5" for f in all_fnames) and isinstance(h5py, ImportError):
            raise h5py
        samples = defaultdict(list)
        for fname in all_fnames:
            try:
                metadata = self._retrieve_metadata(fname)
            except OSError:  # pragma: no cover
                warnings.warn(f"Corrupted volume {fname.name} detected in FastMRI dataset. Skipping...")
                continue
            for slice_ind in range(metadata["num_slices"]):
                samples[str(fname)].append(self.SliceSampleID(fname, slice_ind, metadata))
        if slice_index != "all":
            for fname, samps in samples.items():
                if isinstance(slice_index, int):
                    chosen = samps[slice_index]
                elif isinstance(slice_index, (tuple, list)):
                    chosen = [samps[i] for i in slice_index]
                elif "middle" in slice_index:
                    i = slice_index.split("+")[-1]
                    i = int(i) if "+" in slice_index and i.isdigit() else 0
                    chosen = samps[len(samps) // 2 - i: len(samps) // 2 + i + 1]
                elif slice_index == "random":
                    chosen = self.torch_shuffle(samps, generator=rng)[0]
                else:
                    raise ValueError('slice_index must be "all", "random", "middle", "middle+i", int or tuple.')
                samples[fname] = chosen if isinstance(chosen, list) else [chosen]
        if subsample_volumes is not None and subsample_volumes < 1.0:
            keep = self.torch_shuffle(list(samples.keys()), generator=rng)[: round(len(all_fnames) * subsample_volumes)]
            samples = {k: samples[k] for k in keep}
        self.samples = [s for ss in samples.values() for s in ss]
        if filter_id is not None:
            self.samples = list(filter(filter_id, self.samples))

    @staticmethod
    def _retrieve_metadata(fname) -> dict[str, Any]:
        with _open(fname) as hf:
            shape = hf["kspace"].shape
            md = {"width": shape[-1], "height": shape[-2], "num_slices": shape[0]}
            if len(shape) == 4:
                md["coils"] = shape[1]
            if "num_low_frequency" in hf.attrs:
                md["acs"] = int(hf.attrs["num_low_frequency"])
        return md

    def __len__(self) -> int:
        return len(self.samples)

    @staticmethod
    def _target(f, slice_ind):
        key = "reconstruction_esc" if "reconstruction_esc" in f.keys() else "reconstruction_rss"
        return torch.from_numpy(np.asarray(f[key][slice_ind])).unsqueeze(0)

    def _read(self, idx):
        """raw slice: complex (N,) H, W array, target tensor or None, file mask tensor or None"""
        fname, slice_ind, metadata = self.samples[idx]
        with _open(fname) as hf:
            ks = np.ascontiguousarray(hf["kspace"][slice_ind])
            if any("reconstruction" in k for k in hf.keys()):
                target = self._target(hf, slice_ind)
            elif self.target_root is not None:
                with _open(self.target_root / Path(fname).name) as hf2:
                    target = self._target(hf2, slice_ind)
            else:
                target = None
            mask = torch.as_tensor(np.asarray(hf["mask"])) if "mask" in hf else None
        return ks, target, mask

    def __getitem__(self, idx: int):
        fname, slice_ind, metadata = self.samples[idx]
        ks, target, mask = self._read(idx)
        kspace = from_torch_complex(torch.from_numpy(ks).to(torch.complex64).unsqueeze(0)).squeeze(0)  # (2, (N,) H, W)
        params = {} if mask is None else {"mask": mask}
        if self.transform is not None:
            target, kspace, params = self.transform(target, kspace, seed=str(fname) + str(slice_ind), metadata=metadata, **params)
        return (target if target is not None else torch.nan, kspace) + ((params,) if params else ())

    # ---- GPU path -----------------------------------------------------------------------------------------------------
    def load_batch(self, indices, device, non_blocking: bool = True) -> dict:
        """slices `indices` (same k-space shape) -> {"y": (B, 2, (N,) H, W) fp32 on `device`, "mask": (B, W) fp32 or None,
        "target": list of host tensors / None}.  One pinned staging buffer, one H2D copy, de-interleave on the device."""
        from .. import ops

        raws = [self._read(i) for i in indices]
        shape = raws[0][0].shape
        if any(r[0].shape != shape for r in raws):
            raise ValueError("load_batch: the slices have different k-space shapes; batch slices of one geometry")
        stage = torch.empty((len(raws), *shape), dtype=torch.complex64)
        pin = torch.cuda.is_available()
        if pin:
            stage = stage.pin_memory()
        view = stage.numpy()
        for b, (ks, _, _) in enumerate(raws):
            view[b] = ks  # raw interleaved complex64, no layout change on the host
        y = ops.interleaved_to_planar(stage.to(device, non_blocking=non_blocking))
        masks = [r[2] for r in raws]
        mask = None
        if all(m is not None for m in masks):
            mask = torch.stack([m.float() for m in masks])
            mask = (mask.pin_memory() if pin else mask).to(device, non_blocking=non_blocking)
        return {"y": y, "mask": mask, "target": [r[1] for r in raws]}

    @staticmethod
    def line_mask(mask_w: torch.Tensor, H: int) -> torch.Tensor:
        """(B, W) column masks -> the (B, 2, H, W) tensor `MRI(mask=...)` takes (values unchanged: exact zero pattern)"""
        B, W = mask_w.shape
        return mask_w[:, None, None, :].expand(B, 2, H, W).contiguous()

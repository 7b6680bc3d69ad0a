"""Raw CT volumes -> normalised target_size^3 cubes -- the reference's
`data_generator/synthetic_dataset/process_raw_data.py`, with its scipy zooms on the GPU.

    python -m r2_gaussian_b200.process_raw_data [--metadata data_generator/raw_metadata.py]
        [--output data_generator/volume_gt] [--target_size 256]

The metadata file is Python defining `raw_info`, a list of cases in the reference's format (it is loaded with
importlib, so the reference's own `raw_metadata.py` works as it is).  Each case becomes `<output>/<output_name>.npy`
(float32); a case whose file already exists is skipped.  The chains, per `file_type`:
  * `raw`: np.fromfile(dtype).reshape(shape[::-1]).transpose(2, 1, 0); min / max normalisation in float64; `reshape`
    ("crop", "expand" or None, see `reshape_plan`); clip to [0, 1], `transpose`, and a z flip with `z_invert`.
  * `tif`: tifffile.imread, normalised as numpy does it (no initial transpose), then as `raw`.
  * `dcm`: the sorted `*.dcm` files of `raw_path` read with pydicom, pixel_array * RescaleSlope + RescaleIntercept in
    float64, stacked on the last axis, z flipped, clipped to [-1000, 2000], normalised and resized straight to the cube
    (the reference ignores the spacing here, and so does this), clipped to [0, 1], x and y flipped with `xy_invert`.
The `reshape` modes first resample to unit spacing: new shape np.round(shape * spacing) (half to even), factors
new shape / shape; then "crop" centre-crops to the shortest axis and "expand" zero-pads to the longest; then the cube
is resized to target_size^3 if any factor is not 1.  Every zoom is `resample.zoom_placed` (scipy.ndimage.zoom, order 3,
mode "nearest", on the GPU) and every placement -- normalisation, dtype conversion, expand or crop -- happens inside the
zoom's fill pass: a raw file goes to the device in its own dtype, and the normalised or cubed volume never exists on
its own.  Everything else (min / max, the clips, permutations and flips) is exact float64 arithmetic on the host and
gives numpy's bits.  The chains are written over a zoom callable, `zoom(source, factors, place)`, so they run with any
implementation of that signature.

Differences from the reference: each of these is refused with a message naming the case, where the reference raises a
bare KeyError, writes NaNs or reads garbage -- a missing metadata key, an unknown `file_type` or `reshape`, a `.raw` file
whose size is not prod(shape) * itemsize, a constant volume (min = max: normalising divides by zero) or one with
non-finite values, a `.tif` that is not uint8, uint16, uint32 or float64 (numpy's arithmetic on other types is not
restated), a case that needs `pydicom` or `tifffile` when it is not installed.  All metadata keys are checked before any
case is processed.  A `dcm` case needs no `thickness` key (the reference reads it and never uses it).  Dependencies:
numpy and torch with this package's CUDA library; `pydicom` and `tifffile` only for the cases that need them.
"""
from __future__ import annotations

import argparse
import glob
import importlib.util
import os

import numpy as np

from .resample import Place

_KEYS = {"raw": ("raw_path", "dtype", "shape", "spacing", "reshape", "transpose", "z_invert"),
         "tif": ("raw_path", "spacing", "reshape", "transpose", "z_invert"),
         "dcm": ("raw_path", "xy_invert")}
_RESHAPE = (None, "crop", "expand")
_TIF_DTYPES = (np.uint8, np.uint16, np.uint32, np.float64)


def _name(case) -> str:
    return str(case.get("output_name", "?"))


def check_case(case) -> None:
    """Refuse a case whose keys are missing or whose file_type / reshape is unknown, naming it."""
    for key in ("output_name", "file_type"):
        if key not in case:
            raise ValueError(f"case {_name(case)}: metadata has no {key!r}")
    ftype = case["file_type"]
    if ftype not in _KEYS:
        raise ValueError(f"case {_name(case)}: unsupported file_type {ftype!r} (raw, tif or dcm)")
    missing = [k for k in _KEYS[ftype] if k not in case]
    if missing:
        raise ValueError(f"case {_name(case)}: metadata has no {', '.join(repr(k) for k in missing)}")
    if ftype != "dcm" and case["reshape"] not in _RESHAPE:
        raise ValueError(f"case {_name(case)}: unsupported reshape {case['reshape']!r} (None, 'crop' or 'expand')")


def normalising_place(vol: np.ndarray, name: str) -> Place:
    """The placement that normalises `vol` by its min and max, refused for a constant or non-finite volume."""
    lo, hi = float(vol.min()), float(vol.max())
    if not (np.isfinite(lo) and np.isfinite(hi)):
        raise ValueError(f"case {name}: the volume has non-finite values (min {lo}, max {hi})")
    if lo == hi:
        raise ValueError(f"case {name}: the volume is constant ({lo}); normalising it would divide by zero")
    return Place(tuple(vol.shape), (0, 0, 0), lo, hi)


def cube_place(shape, mode: str) -> Place:
    """expand_to_cube (zero padding to the longest axis, the odd voxel at the end) or crop_to_cube (centre crop to the
    shortest) of a volume of `shape`, as a placement."""
    if mode == "expand":
        m = max(shape)
        return Place((m, m, m), tuple((m - s) // 2 for s in shape))
    m = min(shape)
    return Place((m, m, m), tuple(-((s - m) // 2) for s in shape))


def reshape_plan(shape, spacing, target_size: int, mode):
    """The reference's reshape_vol as zoom calls: a list of (factors, place-of-previous-result) steps after the
    first, and the first step's factors.  With a mode: resample to unit spacing, then crop / expand and resize."""
    if mode is None:
        return [tuple(target_size / s for s in shape)], []
    new_shape = np.round(np.array(shape) * np.array(list(spacing), dtype=np.float64))
    factors = tuple(float(f) for f in new_shape / np.array(shape))
    resampled = tuple(int(round(n * f)) for n, f in zip(shape, factors))
    cube = cube_place(resampled, mode)
    m = cube.shape[0]
    return [factors, (target_size / m,) * 3], [cube]


def reshape_vol(source, place: Place, spacing, target_size: int, mode, zoom):
    """Zoom chain of `reshape_vol` on the placed source: the first zoom applies `place`, later ones their cube."""
    factors, places = reshape_plan(place.shape, spacing, target_size, mode)
    vol = zoom(source, factors[0], place)
    for f, p in zip(factors[1:], places):
        vol = zoom(vol, f, p)
    return vol


def _to_host(vol) -> np.ndarray:
    return vol.cpu().numpy() if hasattr(vol, "cpu") else np.asarray(vol)


def _finish(vol, case) -> np.ndarray:
    out = _to_host(vol).clip(0.0, 1.0)
    out = out.transpose(case["transpose"])
    return out[:, :, ::-1] if case["z_invert"] else out


def read_raw(case) -> np.ndarray:
    dtype = np.dtype(case["dtype"])
    shape = [int(s) for s in case["shape"]]
    size = os.path.getsize(case["raw_path"])
    if size != int(np.prod(shape)) * dtype.itemsize:
        raise ValueError(f"case {_name(case)}: {case['raw_path']} has {size} bytes, shape {shape} of {dtype} needs "
                         f"{int(np.prod(shape)) * dtype.itemsize}")
    data = np.fromfile(case["raw_path"], dtype=dtype).reshape(shape[::-1]).transpose(2, 1, 0)
    # uint8 / uint16 go to the device as they are; any other type becomes float64 here, exactly as astype(float)
    return data if dtype in (np.uint8, np.uint16, np.float64) else data.astype(np.float64)


def _import(module: str, case):
    try:
        return importlib.import_module(module)
    except ImportError as e:
        raise RuntimeError(f"case {_name(case)}: reading it needs the {module!r} package, which is not installed") from e


def process_raw(case, target_size: int, zoom) -> np.ndarray:
    data = read_raw(case)
    place = normalising_place(data, _name(case))
    return _finish(reshape_vol(data, place, case["spacing"], target_size, case["reshape"], zoom), case)


def process_tif(case, target_size: int, zoom) -> np.ndarray:
    data = np.asarray(_import("tifffile", case).imread(case["raw_path"]))
    if data.ndim != 3 or data.dtype not in _TIF_DTYPES:
        raise ValueError(f"case {_name(case)}: {case['raw_path']} is a {data.dtype} array of shape {data.shape}; "
                         "a 3-D uint8, uint16, uint32 or float64 volume is expected")
    if data.dtype == np.uint32:
        data = data.astype(np.float64)      # exact; (d - min) / (max - min) then gives numpy's uint32 bits
    place = normalising_place(data, _name(case))
    return _finish(reshape_vol(data, place, case["spacing"], target_size, case["reshape"], zoom), case)


def read_dcm(case) -> np.ndarray:
    pydicom = _import("pydicom", case)
    paths = sorted(glob.glob(os.path.join(case["raw_path"], "*.dcm")))
    if not paths:
        raise ValueError(f"case {_name(case)}: no .dcm files in {case['raw_path']}")
    slices = []
    for p in paths:
        ds = pydicom.dcmread(p)
        slices.append(np.array(ds.pixel_array).astype(float) * float(ds.RescaleSlope) + float(ds.RescaleIntercept))
    return np.stack(slices, axis=-1)[:, :, ::-1].clip(-1000, 2000)


def process_dcm(case, target_size: int, zoom) -> np.ndarray:
    vol = read_dcm(case)
    place = normalising_place(vol, _name(case))
    out = _to_host(reshape_vol(vol, place, None, target_size, None, zoom)).clip(0.0, 1.0)
    return out[::-1, ::-1, :] if case["xy_invert"] else out


PROCESS = {"raw": process_raw, "tif": process_tif, "dcm": process_dcm}


def load_metadata(path: str) -> list:
    spec = importlib.util.spec_from_file_location("metadata", path)
    module = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(module)
    return module.raw_info


def run(metadata: str, output: str, target_size: int = 256, zoom=None) -> list:
    """Process every case of `metadata` whose `<output>/<output_name>.npy` does not exist yet; return the paths
    written.  `zoom(source, factors, place)` defaults to the GPU's `resample.zoom_placed`."""
    if target_size < 1:
        raise ValueError(f"--target_size must be at least 1, got {target_size}")
    raw_info = load_metadata(metadata)
    for case in raw_info:
        check_case(case)
    os.makedirs(output, exist_ok=True)
    written = []
    for case in raw_info:
        path = os.path.join(output, f"{case['output_name']}.npy")
        if os.path.exists(path):
            continue
        if zoom is None:
            import torch

            if not torch.cuda.is_available():
                raise RuntimeError("process_raw_data needs a CUDA device: the zooms run on the GPU, with no CPU "
                                   "fallback")
            from .resample import zoom_placed as zoom
        print(f"Processing {case['output_name']}")
        vol = PROCESS[case["file_type"]](case, target_size, zoom)
        np.save(path, vol.astype(np.float32))
        written.append(path)
    return written


def main(argv=None) -> list:
    ap = argparse.ArgumentParser(description="Normalise raw CT volumes into cubes")
    ap.add_argument("--metadata", default="data_generator/raw_metadata.py", type=str, help="Path to metadata.")
    ap.add_argument("--output", default="data_generator/volume_gt", type=str, help="Path to output folder.")
    ap.add_argument("--target_size", default=256, type=int, help="Target volume size (a cube)")
    a = ap.parse_args(argv)
    return run(a.metadata, a.output, a.target_size)


if __name__ == "__main__":
    main()

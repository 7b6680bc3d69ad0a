"""Exercise the less-travelled kernel paths (radix binning, capacity overflow + re-run, exports, backward) on small inputs so that
the script can run under compute-sanitizer.  Prints OK lines; any CUDA error aborts."""
import os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import util
from r2_gaussian_b200 import scene, _C

def voxel(P, nV, kind="trained", bwd=True, hint=None):
    cloud = scene.make_cloud(P, kind=kind, seed=3)
    key = _C.voxel_key(torch.device("cuda", 0), P, *nV, 2.0)
    if hint is not None:
        _C._Workspace.hints[key] = hint          # force a capacity overflow on the first attempt
    f = util.ours_voxel_forward(cloud, nV, (2.0, 2.0, 2.0), (0.0, 0.0, 0.0))
    torch.cuda.synchronize()
    o = util.oracle_voxel_forward(cloud, nV, (2.0, 2.0, 2.0), (0.0, 0.0, 0.0))
    err = np.abs(f["vol"].astype(np.float64) - o["vol"]).max() / max(np.abs(o["vol"]).max(), 1e-30)
    assert int(f["R"]) == o["R"] and err < 1e-5, (int(f["R"]), o["R"], err)
    if bwd:
        dL = np.random.RandomState(1).randn(*nV).astype(np.float32)
        util.ours_voxel_backward(cloud, nV, (2.0, 2.0, 2.0), (0.0, 0.0, 0.0), f, dL)
        torch.cuda.synchronize()
    print("voxel", P, nV, "R", o["R"], "err", err, "OK", flush=True)

def raster(P, n, kind="trained", hint=None):
    cloud = scene.make_cloud(P, kind=kind, seed=4)
    view = scene.make_view(scene.cone_beam_scanner(n, 64), 0.7)
    key = _C.raster_key(torch.device("cuda", 0), P, n, n)
    if hint is not None:
        _C._Workspace.hints[key] = hint
    f = util.ours_raster_forward(cloud, view)
    torch.cuda.synchronize()
    o = util.oracle_raster_forward(cloud, view)
    err = np.abs(f["image"].astype(np.float64) - o["image"]).max() / max(np.abs(o["image"]).max(), 1e-30)
    assert int(f["R"]) == o["R"] and err < 1e-5, (int(f["R"]), o["R"], err)
    dL = np.random.RandomState(2).randn(n, n).astype(np.float32)
    util.ours_raster_backward(cloud, view, f, dL)
    torch.cuda.synchronize()
    print("raster", P, n, "R", o["R"], "err", err, "OK", flush=True)

raster(3000, 128)
raster(3000, 128, hint=4096)                 # direct binning, overflow then re-run
raster(1500, 1040)                           # 4225 tiles: radix path
raster(1500, 1040, hint=4096)                # radix path, overflow then re-run
voxel(1500, (32, 32, 32))
voxel(1500, (32, 32, 32), hint=4096)
voxel(1200, (144, 136, 136))                 # 5202 tiles, 125 supertiles: two-level binning
voxel(1200, (144, 136, 136), hint=4096)
voxel(20000, (96, 96, 96), kind="init")      # 1728 tiles, many instances per tile (multi-chunk tiles)
print("ALL OK")

"""FDK's windowed ramp filters on the GPU (fdk(filter=...) over r2x_fdk's filter field, fdk_window_kernel) against the
float64 oracle tests/fdk_window_oracle.py: every filter with both beams and every redundancy weighting, the filter
alone and the volume at the row widths where the kernel's work split and shared-memory opt-in change, bitwise
reproducibility, Ram-Lak through the keyword bit for bit the default, and the filters end to end on a noisy scene
(`recon_volume`, `recon --fdk_filter`, `initialize_pcd --recon_method fdk --fdk_filter`)."""
import math
import re

import numpy as np
import pytest
import yaml

import ct_edge_cases as ct
import fdk_cases as fc
import fdk_window_oracle as fwo
from test_fdk_window_cpu import WINDOWED, first_window_opt_in_width

pytestmark = pytest.mark.gpu

FDK_BOUND = 1e-4       # max error over max |want|, as for the unwindowed FDK


def _torch():
    import torch

    return torch


def _bits(t):
    return t.contiguous().view(_torch().int32)


def _rel_err(got, want) -> float:
    return float(np.abs(np.asarray(got, np.float64) - want).max() / np.abs(want).max())


def _scanner(mode, weighting):
    """A 10 x 20 detector, a non-cubic off-centre grid, and the detector offset each weighting takes: both axes for
    plain, vertical only for Parker, horizontal (and vertical) for half fan."""
    sc = ct._scanner(mode, (10, 20), (9, 10, 8), (1.3, 1.5, 1.1), (0.05, -0.1, 0.08))
    t_u, t_v = {"plain": (1.7, -0.6), "parker": (0.0, 0.4), "half_fan": (-3.4, 0.3)}[weighting]
    return ct._offset(sc, t_u, t_v)


def _angles(mode, weighting):
    if weighting == "parker":
        return np.linspace(0.0, math.radians(240.0 if mode == "cone" else 200.0), 15)[:-1] + 0.3
    return fc.full_scan(16) + 0.2


@pytest.mark.parametrize("weighting", ["plain", "parker", "half_fan"])
@pytest.mark.parametrize("mode", ["cone", "parallel"])
@pytest.mark.parametrize("name", fwo.FILTERS)
def test_cuda_matches_oracle(name, mode, weighting):
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk

    sc, angles = _scanner(mode, weighting), _angles(mode, weighting)
    projs = np.random.RandomState(len(name) + 7 * len(weighting)).uniform(0.0, 1.0, (len(angles), 10, 20))
    projs = projs.astype(np.float32)
    kw = dict(short_scan=weighting == "parker", use_offDetector=True, half_fan=weighting == "half_fan")
    got = fdk(torch.tensor(projs, device="cuda"), angles, sc, filter=name, **kw).cpu().numpy()
    want = fwo.fdk_scene(projs, angles, sc, name, **kw)
    assert got.shape == (9, 10, 8)
    assert _rel_err(got, want) <= FDK_BOUND, (_rel_err(got, want), name, mode, weighting)


def test_ram_lak_keyword_is_the_default_and_windows_are_reproducible():
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk

    sc = fc.scanner("cone", 64, 40)
    angles = fc.full_scan(30)
    projs = torch.rand(30, 64, 64, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    plain = fdk(projs, angles, sc)
    assert _bits(fdk(projs, angles, sc, filter="ram_lak")).equal(_bits(plain))
    assert _bits(fdk(projs, angles, dict(sc, filter="hann"), filter="ram_lak")).equal(_bits(plain))
    for name in WINDOWED:
        a, b = fdk(projs, angles, sc, filter=name), fdk(projs, angles, sc, filter=name)
        assert _bits(a).equal(_bits(b)), name                           # bitwise, signed zeros included
        assert not a.equal(plain), name
        # the scanner's filter is taken with the keyword, and the keyword wins over it
        assert _bits(fdk(projs, angles, dict(sc, filter="cosine"), filter=name)).equal(_bits(a)), name
    with pytest.raises(ValueError, match="filter"):
        fdk(projs, angles, dict(sc, filter="hann"))


def _raw_fdk(projs, angles, sc, name):
    """r2x_fdk on a centred detector with `name`'s filter field: (volume, the filtered views it left in scratch)."""
    torch = _torch()
    from r2_gaussian_b200 import _lib, scene
    from r2_gaussian_b200.fdk import FILTERS

    lib = _lib.load()
    views = [scene.make_view(sc, float(a)) for a in angles]
    N, H, W = projs.shape
    nx, ny, nz = sc["nVoxel"]
    vm = torch.tensor(np.stack([v.viewmatrix.reshape(16) for v in views]), device="cuda")
    pm = torch.tensor(np.stack([v.projmatrix.reshape(16) for v in views]), device="cuda")
    p = torch.tensor(projs, device="cuda")
    vol = torch.empty(nx, ny, nz, device="cuda")
    nbytes = int(lib.r2x_fdk_scratch_bytes(N, H, W))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    assert scratch.data_ptr() % 256 == 0                        # r2x_fdk's filtered views start at the scratch
    rc = lib.r2x_fdk(torch.cuda.current_stream().cuda_stream, N, H, W, p.data_ptr(), vm.data_ptr(), pm.data_ptr(),
                     float(views[0].tanfovx), float(views[0].tanfovy), int(views[0].mode), 0.0, 0.0,
                     FILTERS.index(name) << 8, None, 0.0, float(sc["DSO"]), nx, ny, nz, *sc["sVoxel"], *sc["offOrigin"],
                     vol.data_ptr(), scratch.data_ptr(), nbytes)
    _lib.check(rc, "r2x_fdk")
    q = scratch[:N * H * W * 4].view(torch.float32).view(N, H, W)
    return vol.cpu().numpy(), q.cpu().numpy()


def _widths():
    T, Wo = ct.K["FDK_FILTER_THREADS"], first_window_opt_in_width()
    return [1, 2, 3, T - 1, T, T + 1, Wo - 1, Wo, ct.K["FDK_MAX_W"]]


@pytest.mark.parametrize("W", _widths())
@pytest.mark.parametrize("name", WINDOWED)
def test_single_rows_at_every_launch_switch(name, W):
    """One detector row, two views: the filter alone on noise, and the volume (on the smooth rows of
    ct_edge_cases.fdk_inputs above 64 pixels, whose backprojection stays within the bar at any width)."""
    sc = ct._scanner("cone", (1, W), (5, 6, 7))
    angles = fc.full_scan(2) + 0.2
    case = ct.Case(f"w{W}", "fdk", "", (), sc, angles, W)
    noise = ct.fdk_inputs(case, smooth=False)
    _, q = _raw_fdk(noise, angles, sc, name)
    v0 = ct.views(case)[0]
    want_q = fwo.filter_projections(noise, name, v0.tanfovx, v0.tanfovy, v0.mode, float(sc["DSO"]))
    assert _rel_err(q, want_q) <= FDK_BOUND, ("filter", _rel_err(q, want_q))
    projs = ct.fdk_inputs(case)
    vol, _ = _raw_fdk(projs, angles, sc, name)
    want = fwo.fdk_scene(projs, angles, sc, name)
    assert _rel_err(vol, want) <= FDK_BOUND, ("volume", _rel_err(vol, want))


# ---- a noisy generate_data scene ------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def noisy_scene(tmp_path_factory):
    """test_tv_recon_gpu's scene: 24 train and 6 test views of 96^2 of the round-trip volume on a 48^3 grid, Poisson
    (1e5) + Gaussian noise."""
    from r2_gaussian_b200 import generate_data
    from test_projector_gpu import _write_inputs

    tmp = tmp_path_factory.mktemp("window_scene")
    yml, vol_path, *_ = _write_inputs(tmp, noise=True)
    return generate_data.main(["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24", "--n_test", "6",
                               "--output", str(tmp / "data")])


def test_hann_beats_ram_lak_on_the_noisy_scene(noisy_scene):
    torch = _torch()
    from r2_gaussian_b200 import recon
    from r2_gaussian_b200.dataset import read_blender
    from r2_gaussian_b200.metrics import metric_vol

    info = read_blender(noisy_scene, eval=False)
    b = torch.tensor(np.stack([c.image for c in info.train_cameras]), dtype=torch.float32, device="cuda")
    angles = [c.angle for c in info.train_cameras]
    psnr = {name: metric_vol(info.vol, recon.recon_volume(b, angles, info.scanner_cfg, "fdk", fdk_filter=name)
                             .cpu().numpy(), "psnr")[0] for name in fwo.FILTERS}
    print(f"fdk psnr_3d by filter: {psnr}")
    assert psnr["hann"] > psnr["ram_lak"], psnr


def test_command_lines_end_to_end(noisy_scene, tmp_path, capsys):
    from r2_gaussian_b200 import initialize_pcd, recon

    out = tmp_path / "trad"
    report = recon.main(["-s", noisy_scene, "-m", str(out), "--methods", "fdk,sart", "--fdk_filter", "hann"])
    with open(out / "fdk" / "eval_3d.yml") as f:
        per = yaml.safe_load(f)
    assert per["filter"] == "hann" and per == report["fdk"]
    with open(out / "sart" / "eval_3d.yml") as f:
        assert "filter" not in yaml.safe_load(f)
    plain = recon.main(["-s", noisy_scene, "-m", str(tmp_path / "rl"), "--methods", "fdk", "--fdk_filter", "ram_lak"])
    assert "filter" not in plain["fdk"]
    print(f"recon fdk psnr_3d: hann {per['psnr_3d']:.3f}, ram_lak {plain['fdk']['psnr_3d']:.3f}")

    psnr = {}
    for name in ("ram_lak", "hann"):
        capsys.readouterr()
        init = initialize_pcd.main(["--data", noisy_scene, "--recon_method", "fdk", "--fdk_filter", name,
                                    "--n_points", "2000", "--evaluate", "--output", str(tmp_path / f"init_{name}.npy")])
        pts = np.load(init)
        assert pts.shape == (2000, 4) and np.isfinite(pts).all()
        found = re.findall(r"3D PSNR for initial Gaussians: (\S+)", capsys.readouterr().out)
        assert len(found) == 1 and math.isfinite(float(found[0])), found
        psnr[name] = float(found[0])
    print(f"initial-cloud 3D PSNR: {psnr}")

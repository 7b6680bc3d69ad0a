"""`python -m r2_gaussian_b200.test` and the device metrics without a GPU: settings merge and `cfg_args` parsing,
iteration discovery and its refusals, the NIfTI-1 writer read back with an independent header parser, and the
metrics' refusal of CPU tensors before any CUDA call."""
import builtins
import gzip
import os
import struct

import numpy as np
import pytest
import torch

from r2_gaussian_b200 import metrics, trainer
from r2_gaussian_b200 import test as evaltest


def _trained_dir(tmp_path, use_offDetector=False, json_too=True):
    m = tmp_path / "model"
    m.mkdir()
    extra = {"test_iterations": [7], "save_iterations": [7], "quiet": False}
    if use_offDetector:
        extra["use_offDetector"] = True
    trainer.write_cfg_args(str(m), trainer.ModelParams(source_path="/scenes/a", model_path=str(m), eval=True),
                           trainer.PipelineParams(compute_cov3D_python=True), trainer.OptimizationParams(), extra)
    if not json_too:
        os.remove(m / "cfg_args.json")
    return m


def _save_iteration(m, n, pickle=True):
    d = m / "point_cloud" / f"iteration_{n}"
    d.mkdir(parents=True)
    if pickle:
        (d / "point_cloud.pickle").write_bytes(b"")
    return d


# ---- settings -----------------------------------------------------------------------------------------------------------

def test_cfg_args_is_read_without_eval(tmp_path, monkeypatch):
    m = _trained_dir(tmp_path, use_offDetector=True, json_too=False)

    def no_eval(*a, **k):
        raise AssertionError("eval called")
    monkeypatch.setattr(builtins, "eval", no_eval)
    s = evaltest.load_settings(str(m))
    assert s["source_path"] == "/scenes/a" and s["compute_cov3D_python"] is True and s["use_offDetector"] is True
    assert s["test_iterations"] == [7] and s["max_num_gaussians"] == 500_000 and s["densify_scale_threshold"] == 0.1
    with pytest.raises(ValueError):
        evaltest.parse_cfg_args("Namespace(a=__import__('os').getcwd())")
    with pytest.raises(ValueError):
        evaltest.parse_cfg_args("print(1)")


def test_json_settings_and_the_flat_run_options_are_merged(tmp_path):
    m = _trained_dir(tmp_path, use_offDetector=True)
    s = evaltest.load_settings(str(m))
    assert s["source_path"] == "/scenes/a" and s["compute_cov3D_python"] is True
    assert s["use_offDetector"] is True                      # recorded only in the flat file
    (tmp_path / "plain").mkdir()
    assert "use_offDetector" not in evaltest.load_settings(str(_trained_dir(tmp_path / "plain")))


def test_no_settings_file_is_refused_naming_both_paths(tmp_path):
    with pytest.raises(FileNotFoundError) as e:
        evaltest.load_settings(str(tmp_path))
    assert str(tmp_path / "cfg_args.json") in str(e.value) and str(tmp_path / "cfg_args") in str(e.value)


def test_the_command_line_wins_over_the_file(tmp_path):
    m = _trained_dir(tmp_path)
    a, s = evaltest.parse_args(["-m", str(m)])
    assert s["source_path"] == "/scenes/a" and s["compute_cov3D_python"] is True and not s.get("use_offDetector")
    assert a.iteration == -1 and not (a.skip_render_train or a.skip_render_test or a.skip_recon or a.quiet)
    a, s = evaltest.parse_args(["-m", str(m), "-s", "/scenes/b", "--use_offDetector", "--debug", "--iteration", "3",
                                "--skip_recon", "--quiet"])
    assert s["source_path"] == "/scenes/b" and s["use_offDetector"] is True and s["debug"] is True
    assert a.iteration == 3 and a.skip_recon and a.quiet


def test_a_missing_model_directory_is_refused_naming_it(tmp_path, capsys):
    missing = tmp_path / "nowhere"
    with pytest.raises(SystemExit):
        evaltest.main(["-m", str(missing)])
    assert str(missing) in capsys.readouterr().err


# ---- iterations ---------------------------------------------------------------------------------------------------------

def test_iteration_minus_one_picks_the_largest_saved_iteration(tmp_path):
    m = _trained_dir(tmp_path)
    for n in (7, 1000, 30):
        _save_iteration(m, n)
    (m / "point_cloud" / "iteration_x").mkdir()
    (m / "point_cloud" / "iteration_99999").write_text("a file, not a saved iteration")
    it, path = evaltest.resolve_iteration(str(m), -1)
    assert it == 1000 and path == str(m / "point_cloud" / "iteration_1000" / "point_cloud.pickle")
    assert evaltest.resolve_iteration(str(m), 30)[0] == 30


def test_missing_iterations_and_pickles_are_refused_naming_the_path(tmp_path, capsys):
    m = _trained_dir(tmp_path)
    with pytest.raises(FileNotFoundError, match=str(m / "point_cloud")):
        evaltest.resolve_iteration(str(m), -1)
    (m / "point_cloud").mkdir()
    with pytest.raises(FileNotFoundError, match=str(m / "point_cloud")):
        evaltest.resolve_iteration(str(m), -1)
    _save_iteration(m, 5, pickle=False)
    with pytest.raises(FileNotFoundError, match=str(m / "point_cloud" / "iteration_5" / "point_cloud.pickle")):
        evaltest.resolve_iteration(str(m), -1)
    with pytest.raises(FileNotFoundError, match=str(m / "point_cloud" / "iteration_6")):
        evaltest.resolve_iteration(str(m), 6)
    with pytest.raises(SystemExit) as e:
        evaltest.main(["-m", str(m), "--iteration", "6"])
    assert str(m / "point_cloud" / "iteration_6") in str(e.value)


# ---- NIfTI-1 ------------------------------------------------------------------------------------------------------------

def _read_nifti(path):
    """An independent reading of the NIfTI-1 fields the writer promises."""
    raw = gzip.open(path, "rb").read()
    h = raw[:348]
    f = {"sizeof_hdr": struct.unpack_from("<i", h, 0)[0],
         "dim": struct.unpack_from("<8h", h, 40),
         "datatype": struct.unpack_from("<h", h, 70)[0], "bitpix": struct.unpack_from("<h", h, 72)[0],
         "pixdim": struct.unpack_from("<8f", h, 76),
         "vox_offset": struct.unpack_from("<f", h, 108)[0],
         "scl_slope": struct.unpack_from("<f", h, 112)[0],
         "qform_code": struct.unpack_from("<h", h, 252)[0], "sform_code": struct.unpack_from("<h", h, 254)[0],
         "quatern": struct.unpack_from("<3f", h, 256), "qoffset": struct.unpack_from("<3f", h, 268),
         "srow": np.array(struct.unpack_from("<12f", h, 280)).reshape(3, 4),
         "magic": h[344:348]}
    return f, raw


@pytest.mark.parametrize("shape", [(5, 7, 3), (1, 1, 1), (20, 36, 28)])
def test_nifti_header_fields_and_data(tmp_path, shape):
    vol = np.random.RandomState(3).standard_normal(shape).astype(np.float32)
    vol.flat[0] = np.float32(-0.0)
    path = tmp_path / "v.nii.gz"
    evaltest.write_nifti(str(path), vol)
    f, raw = _read_nifti(path)
    nx, ny, nz = shape
    assert f["sizeof_hdr"] == 348 and f["magic"] == b"n+1\0" and f["vox_offset"] == 352.0
    assert f["dim"][:4] == (3, ny, nx, nz) and f["datatype"] == 16 and f["bitpix"] == 32
    assert f["pixdim"][:4] == (1.0, 1.0, 1.0, 1.0)
    assert f["qform_code"] == 1 and f["sform_code"] == 1
    assert np.array_equal(f["srow"], [[-1, 0, 0, 0], [0, -1, 0, 0], [0, 0, 1, 0]])
    # qform: quaternion (0, 0, 1) is a rotation of 180 degrees about z, qfac 1 -> diag(-1, -1, 1); zero offset
    b, c, d = f["quatern"]
    a = np.sqrt(max(0.0, 1 - b * b - c * c - d * d))
    R = np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                  [2 * (b * c + a * d), a * a + c * c - b * b - d * d, 2 * (c * d - a * b)],
                  [2 * (b * d - a * c), 2 * (c * d + a * b), a * a + d * d - b * b - c * c]])
    assert np.array_equal(R, np.diag([-1.0, -1.0, 1.0])) and f["qoffset"] == (0.0, 0.0, 0.0)
    assert len(raw) == 352 + vol.size * 4 and raw[348:352] == b"\0\0\0\0"
    data = np.frombuffer(raw[352:], "<f4")
    want = np.ascontiguousarray(vol.transpose(2, 0, 1))
    assert np.array_equal(data.view(np.uint32), want.reshape(-1).view(np.uint32))
    # dim[1] is the fastest axis: ITK's x is the volume's second axis
    assert np.array_equal(data.reshape(nz, nx, ny)[:, :, :], want)


# ---- the device metrics and the shared cameras --------------------------------------------------------------------------

def test_device_metrics_refuse_cpu_tensors_before_any_cuda_call(monkeypatch):
    def no_cuda(*a, **k):
        raise AssertionError("a CUDA call was made")
    monkeypatch.setattr("r2_gaussian_b200._lib.load", no_cuda)
    monkeypatch.setattr(torch.cuda, "current_stream", no_cuda)
    monkeypatch.setattr(torch.cuda, "synchronize", no_cuda)
    v = torch.rand(4, 5, 6)
    for fn in (metrics.volume_metrics, metrics.projection_metrics):
        with pytest.raises(RuntimeError, match="expected CUDA tensors"):
            fn(v, v.clone())
        with pytest.raises(RuntimeError, match="expected CUDA tensors"):
            fn(v.double(), v.double())
        with pytest.raises(TypeError, match="torch tensors"):
            fn(v.numpy(), v.numpy())


def test_evaluation_cameras_without_corrections_are_the_scene_cameras():
    class _Scene:
        train, test = [object(), object()], [object()]

        def getTrainCameras(self):
            return self.train

        def getTestCameras(self):
            return self.test
    sc = _Scene()
    (n0, c0), (n1, c1) = trainer.evaluation_cameras(sc)
    assert (n0, n1) == ("train", "test") and c0 is sc.train and c1 is sc.test

"""r2_gaussian_b200 -- H100-native X-ray Gaussian rasterizer + voxelizer (the R2-Gaussian hot path).

Layout
  csrc/             hand-written sm_90a CUDA kernels + the C ABI (include/r2x.h) -> libr2xray.so
  _lib, _C          ctypes binding; the reference extension's five entry points over the C ABI
  rasterization, voxelization
                    the reference's Python surface (settings NamedTuples, nn.Modules, autograd bridges)
  render_query      render() / query() mirrors
  engine            persistent-workspace asynchronous forward engines (throughput paths)
  sharded           Gaussian-sharded multi-GPU helpers (one all-reduce of the image / volume)
  scene             synthetic scanner geometry, cameras and Gaussian clouds
"""
__version__ = "0.1.0"

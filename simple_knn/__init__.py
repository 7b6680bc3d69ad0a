"""Drop-in for the reference's `simple_knn` extension package (un-vendored submodule
`r2_gaussian/submodules/simple-knn`): `from simple_knn._C import distCUDA2` resolves to the sm_90a kernel of
this repository (r2_gaussian_b200/csrc/r2x_knn.cu)."""

"""Drop-in for the reference's ``simple_knn`` package (submodules/simple-knn): ``from simple_knn._C import distCUDA2``
(wildgaussians/method.py:25) resolves to this repo's sm_90a implementation (csrc/knn.cu) when ``wild-gaussians_b200`` is on
``sys.path``."""

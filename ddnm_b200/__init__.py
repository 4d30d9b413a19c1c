"""ddnm_b200 — H100-native DDNM sampling engine (hand-written sm_90a CUDA behind a C ABI).

Public surface mirrors the reference's hot path (wyhuai/DDNM):
  ddnm_b200.model.Model                      <- guided_diffusion/models.py::Model  (``et = model(xt, t)``)
  ddnm_b200.operators.*                      <- functions/svd_operators.py  (A, A_pinv, Lambda, Lambda_noise)
  ddnm_b200.sampler.ddnm_diffusion / ddnm_plus_diffusion  <- functions/svd_ddnm.py
"""
__all__ = ["model", "operators", "sampler"]

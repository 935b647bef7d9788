"""kubeflow_b200 — H100-native engine for Katib's Bayesian-optimisation suggestion path.

Hot path (CUDA, sm_90a, behind the C ABI in include/kbo.h):  Gram -> Cholesky -> alpha -> L^-1 ->
candidate sweep (K*, posterior mean, wgmma variance contraction) -> EI/LCB/PI -> first-index argmax.
Host side (Python, mirrors the reference-side interfaces):  gp.GPEngine (tell/ask at fixed θ),
optimizer.Optimizer (skopt-style), suggestion/ (api.v1.beta1 Suggestion gRPC service).
"""
__version__ = "0.1.0"

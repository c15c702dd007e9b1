"""distributed_cluster_gpus_b200 — H100-native (sm_90a) batched discrete-event engine.

Drop-in for ONE path of filrg/distributed_cluster_GPUs: the multi-DC event loop of
simcore/simulator_paper_multi.py, run as tens of thousands of independent Monte-Carlo replicas per GPU.
See DESIGN.md (path, boundary, kernels) and INTEGRATION.md (how a reference checkout binds to it).
"""
__version__ = "0.1.0"

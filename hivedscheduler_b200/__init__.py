"""hivedscheduler_b200 — CUDA-native (H100, sm_90a) implementation of HiveD's scheduling hot path
(microsoft/hivedscheduler pkg/algorithm) behind the reference's own plugin boundary.

Only what the path needs lives here: ``csrc/`` (CUDA kernels + the C ABI of include/hived.h),
``algorithm`` (host-side mirror of internal.SchedulerAlgorithm), ``config`` (api.Config mirror and
the synthetic clusters) and ``trace`` (seeded event traces of the benchmark configs).
"""
__all__ = ["algorithm", "config", "_cabi"]

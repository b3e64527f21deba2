"""
gordo_components_b200 -- H100-native (sm_90a) implementation of gordo's per-machine
autoencoder train-and-score hot path, behind gordo's own sklearn-style model API.

Drop-in: replace the ``gordo.`` prefix of the model classes in a gordo model definition
with ``gordo_components_b200.`` -- e.g.

    gordo_components_b200.machine.model.anomaly.diff.DiffBasedAnomalyDetector:
      base_estimator:
        gordo_components_b200.machine.model.models.KerasAutoEncoder:
          kind: feedforward_hourglass

All arithmetic runs in hand-written CUDA kernels reached through the C ABI declared in
``include/gordo_b200.h``; there is no CPU fallback.
"""
__version__ = "0.1.0"

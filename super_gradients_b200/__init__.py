"""super_gradients_b200 -- H100 (sm_90a) native hot path of SuperGradients (YOLO-NAS / ResNet conv fwd+bwd,
DFL + IoU loss, batched NMS, data-parallel training) behind the reference's registry / models.get / Trainer API.

The compute path is libsgb200.so (hand-written CUDA, C ABI in include/sgb200.h); there is no CPU fallback.
"""
__version__ = "0.1.0"

"""unsupervised_detection_b200: H100 (sm_90a) CUDA adversarial motion-segmentation hot path (drop-in for the
train/inference step of antonilo/unsupervised_detection).  See DESIGN.md."""
__version__ = '0.1.0'

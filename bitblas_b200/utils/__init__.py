"""``auto_detect_nvidia_target`` kept by name (bitblas/utils/target_detector.py:82-105).  The reference maps
`nvidia-smi` output to a TVM target tag; here the only target is sm_90a (H100)."""
import torch


def auto_detect_nvidia_target(gpu_id: int = 0) -> str:
    if torch.cuda.is_available():
        major, minor = torch.cuda.get_device_capability(gpu_id)
        if (major, minor) != (9, 0):
            raise RuntimeError(f"bitblas_b200 targets sm_90a (H100); found compute capability {major}.{minor}")
        return "cuda -arch=sm_90a"
    return "cuda -arch=sm_90a"


def get_default_cache_path():
    from ..cache import get_database_path
    return get_database_path()

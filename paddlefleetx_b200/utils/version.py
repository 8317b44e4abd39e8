"""Version checks (reference ppfleetx/utils/version.py gates on the Paddle version; here: torch / CUDA / device arch)."""
import torch

from .log import logger

MIN_TORCH = (2, 6)


def version_check():
    ver = tuple(int(x) for x in torch.__version__.split("+")[0].split(".")[:2])
    if ver < MIN_TORCH:
        raise RuntimeError(f"paddlefleetx_b200 needs torch >= {MIN_TORCH[0]}.{MIN_TORCH[1]}, found {torch.__version__}")
    if torch.cuda.is_available():
        major, minor = torch.cuda.get_device_capability()
        if (major, minor) != (9, 0):
            logger.warning(f"kernels are built for sm_90a only; this device is sm_{major}{minor} — native ops will refuse to load")
    return True

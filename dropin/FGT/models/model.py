"""Shadow of /root/reference/FGT/models/model.py: put `dropin/` first on sys.path and the unchanged
driver (tool/video_inpainting.py:217-230) instantiates the H100-native model instead."""
from fgt_b200.fgt_model import FGT, Model  # noqa: F401

"""Shadow of /root/reference/RAFT/__init__.py: `from RAFT import RAFT` (tool/video_inpainting.py:26)
yields the H100-native model constructor (the basic or the small model, as args.small says); other
submodules (RAFT.utils, ...) still resolve from the reference's RAFT/ directory further down sys.path."""
import pkgutil

__path__ = pkgutil.extend_path(__path__, __name__)
from fgt_b200.raft_small import make_raft as RAFT  # noqa: E402,F401

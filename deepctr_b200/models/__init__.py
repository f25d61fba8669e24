from .deepfm import DeepFM
from .xdeepfm import xDeepFM
from .dcn import DCN
from .autoint import AutoInt
from .sequence import DIN, BST
from .nfm import NFM
from .afm import AFM
from .fibinet import FiBiNET

__all__ = ["DeepFM", "xDeepFM", "DCN", "AutoInt", "DIN", "NFM", "AFM", "FiBiNET", "BST"]

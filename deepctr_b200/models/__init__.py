from .deepfm import DeepFM
from .xdeepfm import xDeepFM
from .dcn import DCN
from .autoint import AutoInt
from .sequence import DIN, BST
from .nfm import NFM
from .afm import AFM
from .fibinet import FiBiNET
from .fwfm import FwFM
from .deepfefm import DeepFEFM
from .pnn import PNN
from .ifm import IFM
from .difm import DIFM
from .onn import ONN
from .edcn import EDCN
from .ccpm import CCPM
from .flen import FLEN

__all__ = ["DeepFM", "xDeepFM", "DCN", "AutoInt", "DIN", "NFM", "AFM", "FiBiNET", "BST", "FwFM", "DeepFEFM", "PNN",
           "IFM", "DIFM", "ONN", "EDCN", "CCPM", "FLEN"]

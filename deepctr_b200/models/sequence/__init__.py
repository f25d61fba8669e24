from .din import DIN
from .bst import BST

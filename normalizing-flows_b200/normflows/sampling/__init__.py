from . import hais
from .hais import HAIS

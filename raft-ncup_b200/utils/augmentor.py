"""Drop-in for `core/utils/augmentor.py`: `FlowAugmentor` and `SparseFlowAugmentor`, run on the GPU."""
from rnc.augment import FlowAugmentor, SparseFlowAugmentor  # noqa: F401

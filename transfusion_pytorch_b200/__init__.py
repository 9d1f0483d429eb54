"""transfusion_pytorch_b200 - H100-native (sm_90a) Transfusion training / sampling hot path behind the
public API of lucidrains/transfusion-pytorch (`transfusion_pytorch/__init__.py:1-6`)."""
from .transfusion import Transfusion, Transformer, LossBreakdown, SelfMaskedRepTraining, print_modality_sample, create_dataloader

__all__ = ['Transfusion', 'Transformer', 'LossBreakdown', 'SelfMaskedRepTraining', 'print_modality_sample', 'create_dataloader']

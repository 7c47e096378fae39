"""seist_b200 — CUDA-native (sm_90a, H100) implementation of the SeisT forward/backward hot path.

Public surface mirrors the reference's (senli1073/SeisT):
  seist_b200.models   — register_model / create_model / get_model_list / save_checkpoint /
                        load_checkpoint, the seist_* creators and the loss classes
                        (reference: models/__init__.py, models/_factory.py, models/loss.py)
  seist_b200.config   — Config registry (reference: config.py)
  seist_b200.train    — the data-parallel training step (reference: training/train.py:75-121)
"""
__version__ = "0.1.0"

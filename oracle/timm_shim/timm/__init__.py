"""Minimal stand-in for `timm` (not installed here). TEST INFRASTRUCTURE ONLY.

The reference imports exactly one symbol from timm: `timm.models.layers.DropPath`
(models/seist.py:7, timm==0.9.2 pinned in requirements.txt:14).
"""

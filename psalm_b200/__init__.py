"""psalm_b200 — H100 (sm_90a) implementation of the PSALM segmentation inference hot path
(`PSALM.eval_seg`, reference psalm/model/language_model/llava_phi.py:1317).  See DESIGN.md."""
__version__ = "0.1.0"

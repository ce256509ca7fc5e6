"""Drop-in boundary package: the slice of the reference's `basicsr` import surface that its inference
entry point uses (inference_femasr.py:9-11), backed by the H100-native engine in `femasr_b200`.
Unlike the reference's basicsr/__init__.py:3-9 nothing here imports training code, timm or pyiqa."""
__version__ = "0.1.0+b200"

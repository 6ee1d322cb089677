"""torch.hub entry points of GenPercept v1 on the native engine (genpercept_b200/hub.py):

    torch.hub.load("/path/to/this/checkout", "GenPercept_Depth", source="local", local_dir="/path/to/weights")
"""
dependencies = ["torch", "numpy", "PIL", "safetensors"]

from genpercept_b200.hub import GenPercept_Depth, GenPercept_Normal, GenPercept_Segmentation  # noqa: E402,F401

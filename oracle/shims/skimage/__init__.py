"""ORACLE SHIM: the one scikit-image function the reference's data.py uses (skimage.transform.rotate), see transform.py."""

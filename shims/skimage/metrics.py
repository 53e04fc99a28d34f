"""skimage.metrics shim: structural_similarity for the one argument set evaluate.py:67 passes, on the GPU (hrviton_b200.metrics.ssim,
fp64).  Any other argument combination raises NotImplementedError.  A real skimage, when installed, comes first on sys.path and wins."""

_SUPPORTED = {"data_range": 255, "gaussian_weights": True, "use_sample_covariance": False}


def structural_similarity(*a, **k):
    if len(a) != 2 or k != _SUPPORTED or getattr(a[0], "ndim", None) != 2 or getattr(a[1], "ndim", None) != 2:
        raise NotImplementedError("skimage shim: structural_similarity runs only as evaluate.py calls it: (im1, im2) 2-D grayscale, "
                                  "data_range=255, gaussian_weights=True, use_sample_covariance=False; got %d positional arguments "
                                  "and %s" % (len(a), sorted(k.items())))
    import hrv_loader
    hrv_loader.load()
    from hrviton_b200 import metrics
    return float(metrics.ssim(a[0], a[1], data_range=255))

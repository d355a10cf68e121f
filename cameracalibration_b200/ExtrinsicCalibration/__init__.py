from .extrinsicCalib import CenterImage, ExCalibrator, ScaleImage  # noqa: F401

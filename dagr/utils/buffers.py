from dagr_b200.utils.buffers import bbox_t_to_ndarray, compile, format_data, records_from_device, save_detections, to_npy  # noqa: F401
from dagr_b200.evaluation import DetectionBuffer  # noqa: F401

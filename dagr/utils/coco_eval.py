from dagr_b200.evaluation import evaluate_detection  # noqa: F401

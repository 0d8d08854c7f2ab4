from .pipelines import PIPELINES, Compose, build_test_pipeline, run_test_pipeline  # noqa: F401

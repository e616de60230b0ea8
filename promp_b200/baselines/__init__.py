"""Device-backed baselines: the fit / predict of LinearFeatureBaseline and LinearTimeBaseline run inside
promp_process_samples (one Gram + Cholesky per task on the GPU); ZeroBaseline selects the no-baseline path of the same
kernel.  Any other object with fit / predict is accepted by MetaSampleProcessor and runs on the host."""
from promp_b200.baselines.linear_baseline import LinearFeatureBaseline, LinearTimeBaseline  # noqa: F401
from promp_b200.baselines.zero_baseline import ZeroBaseline  # noqa: F401

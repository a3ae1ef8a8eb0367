"""With the persistent ps resident on the same GPU, every cluster of a fused launch is resident from the start: each
claims steps, and each makes its first claim within one step time of the first cluster."""
import pytest

pytestmark = pytest.mark.gpu


def test_every_lane_resident_beside_the_ps():
    from bench_tools import lane_residency

    from dist_mnist_b200.parallel.ps import serve_geometry

    res = lane_residency.run(lanes=12, steps=20000, warmup=50, batch=32)
    lanes = res["lanes"]
    n_ctas, cluster = serve_geometry(35, 0, True, "fused")
    assert res["ps_ctas"] == n_ctas
    # every ps cluster takes one of the device's cluster slots
    assert lanes == min(12, res["fused_max_active_clusters_before_ps"] - n_ctas // cluster)
    claims = [c["steps"] for c in res["clusters"]]
    assert len(claims) == lanes and sum(claims) == 20000
    assert min(claims) > 0, claims
    step_us = res["us_per_step_per_lane"]
    late = [c for c in res["clusters"] if c["first_claim_us"] > step_us]
    assert not late, (step_us, late)

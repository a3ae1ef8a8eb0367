"""Launch geometry of the persistent ps serve kernel (ps.serve_geometry): beside a fused worker on the same GPU, the
fewest clusters of at most 8 CTAs that keep one item per CTA; unchanged otherwise."""
from dist_mnist_b200.models import mlp
from dist_mnist_b200.parallel.ps import serve_geometry
from dist_mnist_b200.parallel.sharding import build_layout


def test_beside_a_fused_worker_fewest_clusters_with_one_item_per_cta():
    assert serve_geometry(35, 0, True, "fused") == (35, 7)   # the flagship shard: 5 clusters of 7
    assert serve_geometry(18, 0, True, "fused") == (18, 6)   # row_split over 2 ps on one GPU
    assert serve_geometry(17, 0, True, "fused") == (18, 6)   # whole clusters: one CTA owns no item
    assert serve_geometry(5, 0, True, "fused") == (5, 5)
    assert serve_geometry(131, 0, True, "fused") == (40, 8)  # at most 40 CTAs beside a worker, as before


def test_other_topologies_unchanged():
    assert serve_geometry(35, 0, True, "graph") == (35, 1)
    assert serve_geometry(35, 0, False, "fused") == (35, 1)
    assert serve_geometry(300, 0, True, "graph") == (40, 1)
    assert serve_geometry(300, 0, False, "graph") == (128, 1)
    assert serve_geometry(35, 20, True, "fused") == (20, 1)   # an explicit ps_ctas is taken as it is
    assert serve_geometry(35, 64, True, "fused") == (35, 1)


def test_flagship_shard_keeps_one_item_per_cta():
    lay = build_layout(mlp.book_model(100), 1, "round_robin", engine="fused", ps_row_blocks=4)
    n_items = lay.shards[0].n_items
    n_ctas, cluster = serve_geometry(n_items, 0, True, "fused")
    assert (n_items, n_ctas, cluster) == (35, 35, 7)

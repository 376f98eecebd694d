"""The graph and settings of the visited-set tests (test_gpu_visited_stages, test_gpu_visited_smem): M = 4, ef = 16,
so that a search's first stage holds 256 entries and its full stage 1024."""
import numpy as np

from graphs import build_both

M, EFC, EF, K = 4, 48, 16, 10
ALWAYS, NEVER, AUTO = 1, 2, 0   # hnsw_b200_set_visited_stages modes


def move_at(ef):
    """insertions at which a search moves: 3/4 of a first stage of cap / 4"""
    cap = max(1024, 1 << (2 * (ef + 16) * 2 * M - 1).bit_length())
    return (cap // 4) * 3 // 4


def staged_graph(pkg, po, n, d, seed, max_elements=None):
    """(X, oracle, handle, top level): uniform f32 L2 rows built serially on the GPU and in the oracle, equal list for
    list, with the stages forced on"""
    X, o, h = build_both(pkg, po, np.float32, "DistL2", n, d, M, EFC, seed, max_elements=max_elements)
    h.set_visited_stages(ALWAYS)
    return X, o, h, int(o.export_points()[0].max())

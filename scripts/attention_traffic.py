"""CPU: bytes the 64-wide attention copies from L2 / HBM into shared memory per layer, for both kernels, from a GraphPlan
(the bench shape by default: 330 pairs of 200 + 200 nodes).  K / V blocks only (bf16x3, 1 KB per split of an 8-node
block); the Q rows (256 B per query node) are the same for both kernels.
  attention64_tc_kernel:  every non-empty 64-row query tile streams its partner's 64-key chunks, K x 3 splits in pass 1
                          and K + V x 3 splits in pass 2.
  attention64_res_kernel: every query protein copies its partner's chunks once, K + V x 3 splits.
usage: attention_traffic.py [pairs] [ligand nodes] [receptor nodes]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from equidock_public_b200 import hetero_graph as hg, synthetic
from equidock_public_b200.engine import GraphPlan

CHUNK = 8 * 1024   # one split of a 64-key chunk
RES_MAX_NODES = 248   # AT_RES_MAX_NODES in csrc/attn_tc.cu


def attention_traffic(plan):
    """(streaming bytes, resident bytes or None if the plan's proteins do not all fit) per layer."""
    seg, B = [int(v) for v in plan.seg_ptr_host], plan.n_pairs
    stream = resident = 0
    for s in range(2 * B):
        p = s + B if s < B else s - B
        j0, j1 = seg[p], seg[p + 1]
        nchunks = ((j1 + 7) // 8 - j0 // 8 + 7) // 8
        halves = (seg[s + 1] - seg[s] + 63) // 64
        stream += halves * nchunks * (3 + 6) * CHUNK
        resident += (halves > 0) * nchunks * 6 * CHUNK
    return stream, resident if plan.struct.max_segment_nodes <= RES_MAX_NODES else None


if __name__ == '__main__':
    B, nl, nr = (int(v) for v in (sys.argv[1:] + ['330', '200', '200'][len(sys.argv) - 1:]))
    plan = GraphPlan.from_graph(hg.batch_pairs(synthetic.to_torch_pairs(synthetic.synthetic_batch(B, nl, nr, 10, seed=0))),
                                'cpu', 10)
    st, res = attention_traffic(plan)
    tiles = sum((n + 63) // 64 for n in plan.n_lig_list + plan.n_rec_list)
    print(f'{B} pairs of {nl} + {nr} nodes, {tiles} query tiles of 64 rows, max_segment_nodes {plan.struct.max_segment_nodes}')
    print(f'attention64_tc_kernel  (streaming): {st / 1e6:8.1f} MB per layer ({st / tiles / 1024:.0f} KiB per tile)')
    print(f'attention64_res_kernel (resident):  ' + (f'{res / 1e6:8.1f} MB per layer ({st / res:.1f}x less)' if res is not None
                                                     else 'not used: a protein exceeds its capacity'))

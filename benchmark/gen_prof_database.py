"""Profile the cluster's collectives and GEMM rate and store the tables the cost model interpolates
(reference: benchmark/alpa/gen_prof_database.py -> alpa.mesh_profiling.profile_all / ProfilingResultDatabase).

    torchrun --nproc-per-node 8 benchmark/gen_prof_database.py --filename prof_database.pkl
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import alpa_b200 as alpa  # noqa: E402
from alpa_b200.mesh_profiling import ProfilingResultDatabase, profile_all  # noqa: E402

if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("--cluster-key", type=str, default="h100-nvswitch")
    parser.add_argument("--filename", type=str, default="prof_database.pkl")
    parser.add_argument("--max-comm-size-intra-node", type=int, default=28, help="log2 of the largest message in bytes")
    parser.add_argument("--max-comm-size-inter-node", type=int, default=26)
    parser.add_argument("--cache-filename", type=str, default="/tmp/alpa_b200_hlo_op_cost_dict.pkl")
    args = parser.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    alpa.init(cluster="distributed" if world > 1 else "local")
    cluster = alpa.get_global_cluster()
    db = profile_all(cluster, args.cluster_key, args.max_comm_size_intra_node, args.max_comm_size_inter_node,
                     cache_filename=args.cache_filename)
    if int(os.environ.get("RANK", "0")) == 0:
        old = ProfilingResultDatabase()
        if os.path.exists(args.filename):
            old.load(args.filename)
        old.update(db)
        old.save(args.filename)
        for key, res in old.data.items():
            print(key, res)
        print(f"Save profiling database to {args.filename}")
    alpa.shutdown()

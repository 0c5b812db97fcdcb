"""Inspect (and optionally edit) a profiling database written by gen_prof_database.py
(reference: benchmark/alpa/inspect_prof_database.py).

    python benchmark/inspect_prof_database.py --filename prof_database.pkl --cluster-key h100-nvswitch --mesh 1 8
    python benchmark/inspect_prof_database.py --filename prof_database.pkl --insert-dummy 2 8      # extrapolated entry
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from alpa_b200.mesh_profiling import ProfilingResultDatabase  # noqa: E402


def describe(db: ProfilingResultDatabase, cluster_key=None, mesh=None) -> str:
    lines = ["Meshes:", str(list(db.data.keys())), ""]
    keys = [k for k in db.data if (cluster_key is None or k[0] == cluster_key) and (mesh is None or tuple(k[1]) == mesh)]
    for key in keys:
        lines.append(f"{key}:")
        lines.append(str(db.data[key]))
    if not keys and (cluster_key or mesh):
        lines.append(f"no entry for cluster_key={cluster_key} mesh={mesh}")
    return "\n".join(lines)


if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("--filename", type=str, default="prof_database.pkl")
    parser.add_argument("--cluster-key", type=str, default=None)
    parser.add_argument("--mesh", type=int, nargs=2, default=None, metavar=("HOSTS", "DEVICES_PER_HOST"))
    parser.add_argument("--insert-dummy", type=int, nargs=2, default=None, metavar=("HOSTS", "DEVICES_PER_HOST"),
                        help="add an entry for an unmeasured mesh shape (copied from the closest measured one) and save")
    args = parser.parse_args()
    db = ProfilingResultDatabase()
    db.load(args.filename)
    if args.insert_dummy:
        key = args.cluster_key or next(iter(db.data))[0]
        db.insert_dummy_mesh_result(key, tuple(args.insert_dummy))
        db.save(args.filename)
        print(f"inserted {key} {tuple(args.insert_dummy)} and saved {args.filename}")
    print(describe(db, args.cluster_key, tuple(args.mesh) if args.mesh else None))

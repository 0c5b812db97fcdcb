#!/bin/bash
#SBATCH --job-name=alpa_b200_prerequisites
#SBATCH --nodes=1
#SBATCH --ntasks-per-node=1
#SBATCH --cpus-per-task=16
#SBATCH --time=00:20:00
# Checks the software stack on a compute node; needs no GPU.
set -euo pipefail
REPO=${REPO:-$PWD}
cd "$REPO"
python -V
python -c "import torch; print('torch', torch.__version__, 'cuda', torch.version.cuda, 'nccl', torch.cuda.nccl.version() if torch.cuda.is_available() else 'n/a')"
nvcc --version | tail -n 2
# compile every extension for sm_90a (cross-compiles without a GPU) and import the package
python -c "import __graft_entry__ as g; g.build(); import alpa_b200; print('alpa_b200', alpa_b200.__version__)"
python -m pytest tests -x -q -m "not gpu" -k "install or api_usage or shard_parallel" --timeout 900

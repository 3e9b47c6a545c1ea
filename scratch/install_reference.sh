#!/bin/bash
# scratch/install_reference.sh REFERENCE_CHECKOUT — copies the UNMODIFIED reference tree into baseline/_ref/ (git-ignored: it never enters the history).
# Used by (1) tests/test_gpu_rollout_policy.py — the reference's own DRL_GAT network inside the device-resident rollout — and (2)
# scratch/shmem_baseline.py — the reference's own ShmemVecEnv timed on the GPU machine's host cores (BASELINE.md section 3).  Both skip without it.
set -e
REF=$(cd "${1:?usage: scratch/install_reference.sh REFERENCE_CHECKOUT}" && pwd)
cd "$(dirname "$0")/.."
rm -rf baseline/_ref && mkdir -p baseline/_ref
cp -r "$REF"/*.py "$REF"/pct_envs "$REF"/wrapper baseline/_ref/
find baseline/_ref -name __pycache__ -type d -exec rm -rf {} +
echo "installed: $(find baseline/_ref -name '*.py' | wc -l) python files, $(du -sh baseline/_ref | cut -f1)"

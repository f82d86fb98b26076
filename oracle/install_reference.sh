#!/bin/bash
# Copy the original federated-pytorch-test scripts into oracle/_ref/src (git-ignored), where
# `bench.py --impl reference` (baseline/ref_shim.py) runs them.  The original is a directory of scripts
# without setup.py / pyproject, so it is copied, not pip-installed.
#
#   oracle/install_reference.sh /path/to/federated-pytorch-test
set -e
SRC="${1:?usage: oracle/install_reference.sh /path/to/federated-pytorch-test}"
cd "$(dirname "$0")/.."
rm -rf oracle/_ref
mkdir -p oracle/_ref
cp -r "$SRC/src" oracle/_ref/src
cp "$SRC/README.md" "$SRC/LICENSE" oracle/_ref/ 2>/dev/null || true
ls oracle/_ref/src

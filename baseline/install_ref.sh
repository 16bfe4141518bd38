#!/bin/sh
# Offline install of the UNMODIFIED reference (facebookresearch/audiocraft @ 896ec7c) into baseline/_ref.
#   baseline/install_ref.sh <path to the reference source tree>
# --no-deps: the reference's third-party dependencies (xformers, flashy, julius, av, ...) need not be installed;
# oracle/ref_import.py stubs the ones the import graph touches (the hot path itself never calls them).  Point pip at a local
# wheel directory with PIP_FIND_LINKS if the build tools are not installed.  baseline/_ref is git-ignored.
set -e
REF="${1:?usage: baseline/install_ref.sh <reference source tree>}"
REF="$(cd "$REF" && pwd)"
cd "$(dirname "$0")/.."
rm -rf baseline/_ref
python -m pip install --no-index --no-build-isolation --no-deps --target baseline/_ref "$REF"

#!/bin/bash
# Build / test driver -- counterpart of the reference's build.sh (build.sh:91-150 `unit_test`): native build, C++
# stress test under sanitizers, unit tests, and the end-to-end matrix: examples standalone and with np in {1, 2},
# checkpoint -> reload with a DIFFERENT worker count, one-batch edge cases. CPU / gloo only (the CI box has no GPU);
# GPU tests: `./build.sh gpu` on an H100 machine.
set -euo pipefail
cd "$(dirname "$0")"
PY=${PYTHON:-python}
cmd=${1:-all}

build() { $PY -c "import __graft_entry__ as g; g.build()"; }

unit() { $PY -m pytest tests -x -q -m "not gpu"; }

torchrun_cpu() { # nproc script args...
  local n=$1; shift
  $PY -m torch.distributed.run --nnodes=1 --nproc-per-node "$n" --master-addr 127.0.0.1 --master-port $((29600 + RANDOM % 300)) "$@"
}

matrix() {
  local tmp; tmp=$(mktemp -d)
  $PY examples/make_sample_data.py --rows 400 --out "$tmp/train.csv"
  echo "== standalone, checkpoint"
  $PY examples/criteo_deepctr_network.py --cpu --data "$tmp/train.csv" --batch_size 100 --epochs 1 --checkpoint "$tmp/ck1_"
  for np in 1 2; do
    echo "== np=$np, load the checkpoint written by 1 worker, save again"
    torchrun_cpu $np examples/criteo_deepctr_network.py --cpu --data "$tmp/train.csv" --batch_size 100 --epochs 1 \
        --load "$tmp/ck1_1" --checkpoint "$tmp/ck_np${np}_"
  done
  echo "== np=1 loads the checkpoint written by np=2 (re-shard on load)"
  $PY examples/criteo_deepctr_network.py --cpu --data "$tmp/train.csv" --batch_size 100 --epochs 1 --load "$tmp/ck_np2_1"
  echo "== one-batch edge cases (batch 100 / 50 / 10 on 100 rows)"
  $PY examples/make_sample_data.py --rows 100 --out "$tmp/small.csv"
  for bs in 100 50 10; do
    OE_DEVICE=cpu $PY examples/criteo_lr_subclass.py --data "$tmp/small.csv" --batch_size $bs --epochs 1
  done
  rm -rf "$tmp"
  echo "MATRIX_OK"
}

case "$cmd" in
  build) build ;;
  unit) build; unit ;;
  matrix) build; matrix ;;
  gpu) build; $PY -m pytest tests -x -q -m gpu ;;
  all|test) build; unit; matrix ;;
  *) echo "usage: $0 [build|unit|matrix|gpu|all]"; exit 2 ;;
esac

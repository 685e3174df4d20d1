#!/bin/bash
# Canned experiment suites of the engine.  The three dataset suites reproduce the experiment grid of the reference launcher
# (src/runner.sh:12-38: {no attack, backdoor attack, attack + Robust LR} x {FMNIST, CIFAR-10, Fed-EMNIST}); the last suite adds the
# ResNet-18 / VGG-11 configs of BASELINE.json.
#
#   bash scripts/runner.sh [NGPUS] [SUITE ...]        SUITE in: fmnist cifar10 fedemnist b200   (default: all)
#
# NGPUS > 1 launches one rank per GPU with torchrun; runs are sequential (the reference backgrounds them on two GPUs).
set -euo pipefail
NG=${1:-1}; shift || true
SUITES=("$@"); [ ${#SUITES[@]} -eq 0 ] && SUITES=(fmnist cifar10 fedemnist b200)
cd "$(dirname "$0")/.."

launch() {
  if [ "$NG" -gt 1 ]; then
    python -m torch.distributed.run --nnodes=1 --nproc-per-node "$NG" --master-addr 127.0.0.1 --master-port 29600 federated.py "$@"
  else
    python federated.py "$@"
  fi
}

# attack / defence variants shared by every suite: "" = clean, attack, attack + RLR (threshold filled in per suite)
variants() {  # $1 = corrupt agents, $2 = RLR threshold
  echo ""
  echo "--num_corrupt=$1 --poison_frac=0.5"
  echo "--num_corrupt=$1 --poison_frac=0.5 --robustLR_threshold=$2"
}

declare -A COMMON=(
  [fmnist]="--data=fmnist --local_ep=2 --bs=256 --num_agents=10 --rounds=200"
  [cifar10]="--data=cifar10 --local_ep=2 --bs=256 --num_agents=40 --rounds=200"
  [fedemnist]="--data=fedemnist --num_agents=3383 --agent_frac=0.01 --local_ep=10 --bs=64 --rounds=500 --snap=5"
)
declare -A CORRUPT=([fmnist]=1 [cifar10]=4 [fedemnist]=338)
declare -A THETA=([fmnist]=4 [cifar10]=8 [fedemnist]=8)

echo 'Calling scripts!'
rm -rf logs   # like the reference; comment out to keep old logs
for suite in "${SUITES[@]}"; do
  if [ "$suite" = b200 ]; then
    launch --data=cifar10 --model=resnet18 --local_ep=2 --bs=256 --num_agents=8 --rounds=100 --num_corrupt=2 --poison_frac=0.5 --robustLR_threshold=4
    launch --data=cifar10 --model=vgg11 --aggr=comed --local_ep=2 --bs=256 --num_agents=8 --rounds=100
    continue
  fi
  while IFS= read -r extra; do
    # shellcheck disable=SC2086
    launch ${COMMON[$suite]} $extra
  done < <(variants "${CORRUPT[$suite]}" "${THETA[$suite]}")
done
echo 'All experiments are finished!'

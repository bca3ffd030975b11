#!/bin/bash
# Continue training a Hugging Face Llama checkpoint on your own corpus, then hand the result back to transformers.
#   HF=/models/llama-1b TOK=/models/llama-1b CORPUS="corpus/*.jsonl" examples/finetune_from_hf.sh
# Runs on the CPU with the debug model when HF is unset (a random donor is exported first), on an H100 with the real one.
set -euo pipefail
cd "$(dirname "$0")/.."
OUT="${OUT:-/tmp/prime_b200/finetune}"
mkdir -p "$OUT"
if [ -z "${HF:-}" ]; then   # no checkpoint at hand: make a tiny donor so that the whole path can be exercised anywhere
  python - <<PY
import torch
from prime_b200.models import hf
from prime_b200.models.llama import build_model
hf.save_hf_dir(build_model("debugmodel", dtype=torch.float32, seed=7), "$OUT/donor")
PY
  HF="$OUT/donor"; MODEL=debugmodel; SEQ=64; EXTRA="--optim.batch_size 8 --train.micro_bs 4 --optim.total_steps 20 --diloco.inner_steps 10"
  printf 'the quick brown fox jumps over the lazy dog. %.0s' {1..400} > "$OUT/corpus.txt"; CORPUS="$OUT/corpus.txt"; TOK=bytes
else
  MODEL="${MODEL:-1B}"; SEQ="${SEQ:-1024}"; EXTRA="${EXTRA:-}"
fi
# 1. text -> token shards (uint16 / uint32 + dtype sidecars) with the checkpoint's own tokenizer
python tools/tokenize_corpus.py --tokenizer "${TOK}" --out "$OUT/data" ${CORPUS}
# 2. train from the imported weights; validation loss every 10 steps; a checkpoint at the end
python -m diloco.train --name_model "$MODEL" --data.fake false --data.dataset_name_or_paths "$OUT/data" --data.seq_length "$SEQ" \
    --train.init_weights "$HF" --train.eval_interval 10 --data.eval_dataset_name_or_paths "$OUT/data" --ckpt.path "$OUT/ckpt" --ckpt.interval 1000000 $EXTRA "$@"
STEP=$(cat "$OUT/ckpt/latest")
# 3. offline: perplexity of the result, and an HF directory again
python -m prime_b200.eval ppl --ckpt "$OUT/ckpt/$STEP" --model "$MODEL" --data "$OUT/data" --seq "$SEQ" --batches 4 --batch-size 4
python -m prime_b200.models.hf export --ckpt "$OUT/ckpt/$STEP" --model "$MODEL" --out "$OUT/hf_out"
echo "fine-tuned model: $OUT/hf_out (transformers.AutoModelForCausalLM.from_pretrained)"

"""GPT training with pipeline + intra-operator parallelism (reference: examples/gpt2, benchmark_one_case_gpt_bert.py).

    python examples/gpt_pipeshard.py                                   # emulated 8-device cluster on CPU, tiny model
    torchrun --nproc-per-node 8 examples/gpt_pipeshard.py --model 2.6B # 8 x H100: 2 stages x (dp2, op2)
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import alpa_b200 as alpa  # noqa: E402
from alpa_b200.model.gpt_model import GPTConfig, GPTModel, config_from_spec, gpt_lm_loss  # noqa: E402
from alpa_b200.model.model_util import TrainState, adamw, functional_call, params_of  # noqa: E402

parser = argparse.ArgumentParser()
parser.add_argument("--model", default=None, help="name in GPT_SPECS (default: a tiny CPU model)")
parser.add_argument("--dp", type=int, default=2)
parser.add_argument("--op", type=int, default=2)
parser.add_argument("--pp", type=int, default=2)
parser.add_argument("--micro-batches", type=int, default=4)
args = parser.parse_args()
distributed = "WORLD_SIZE" in os.environ and int(os.environ["WORLD_SIZE"]) > 1
alpa.init(cluster="distributed") if distributed else alpa.init(cluster="local", num_devices=args.dp * args.op * args.pp)
device = "cuda" if torch.cuda.is_available() and distributed else "cpu"
if args.model:
    cfg = config_from_spec(args.model, add_manual_pipeline_markers=True, pipeline_mp_size=args.pp)
else:
    cfg = GPTConfig(vocab_size=512, hidden_size=128, num_hidden_layers=4, num_attention_heads=4,
                    max_position_embeddings=64, dtype=torch.float32, add_manual_pipeline_markers=True,
                    pipeline_mp_size=args.pp)
model = GPTModel(cfg, device=device)
state = TrainState.create(apply_fn=None, params=params_of(model), tx=adamw(1e-4, fused=device == "cuda"),
                          use_master_copy=device == "cuda")
B, S = 4 * args.micro_batches * args.dp, cfg.max_position_embeddings
batch = {"input_ids": torch.randint(1, cfg.vocab_size, (B, S)), "position_ids": torch.arange(S).repeat(B, 1),
         "labels": torch.randint(1, cfg.vocab_size, (B, S))}
method = alpa.get_3d_parallel_method(num_micro_batches=args.micro_batches, data_parallel=args.dp,
                                     operator_parallel=args.op, pipeline_parallel=args.pp)


@alpa.parallelize(method=method, donate_argnums=(0,))
def train_step(state, batch):
    def loss_fn(p):
        return gpt_lm_loss(functional_call(model, p, (batch["input_ids"], batch["position_ids"])), batch["labels"])
    loss, grads = alpa.value_and_grad(loss_fn)(state.params)
    return state.apply_gradients(grads=grads), loss


for step in range(3):
    state, loss = train_step(state, batch)
    print(f"step {step}: loss {float(loss._value):.4f}", flush=True)
ex = train_step.get_last_executable()
print(ex.get_instruction_text()[:1500] if hasattr(ex, "get_instruction_text") else "")
alpa.shutdown()

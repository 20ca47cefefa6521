#!/bin/bash
# Launch of LLaVA-1.5-7B LoRA-DPO (r=64, alpha=16, dropout 0.05): the flags of the reference recipe (its
# script/train/llava15_train_lora.sh), torchrun launcher, native ZeRO-2 over the adapter + projector buckets.
export PYTHONPATH=$PYTHONPATH:`realpath .`
task_name=llava15_7b_DPO
exp_name=llava15_rlaifv_lora
NGPU=${NGPU:-8}
CKPT=.ckpt/$task_name-$exp_name

MODEL=(--model_name_or_path liuhaotian/llava-v1.5-7b --vision_tower openai/clip-vit-large-patch14-336
       --mm_projector_type mlp2x_gelu --mm_vision_select_layer -2 --mm_use_im_start_end False
       --mm_use_im_patch_token False --fully_tune False --model_max_length 2048 --lora_enable True)
DATA=(--data_dir ./RLAIF-V-Dataset_logps/ --image_folder not_used --image_aspect_ratio pad --lazy_preprocess True
      --data_source_names '' --data_source_weights 1 --dataloader_num_workers 16)
DPO=(--task DPO --dpo_beta 0.1 --dpo_use_average False --dpo_token_weighted False --dpo_token_weight 1.0)
OPTIM=(--learning_rate 1e-5 --weight_decay 0.01 --warmup_ratio 0.05 --lr_scheduler_type "cosine" --max_steps 2672
       --num_train_epochs 10 --per_device_train_batch_size 1 --per_device_eval_batch_size 4
       --gradient_accumulation_steps 1 --gradient_checkpointing True --bf16 True --tf32 True
       --deepspeed ./script/zero2.json)
IO=(--output_dir $CKPT/checkpoints --logging_dir $CKPT/log --logging_steps 2 --evaluation_strategy "no"
    --save_strategy "steps" --save_steps 167 --save_total_limit 50 --report_to wandb --run_name $exp_name)

python -m torch.distributed.run --nnodes=1 --nproc-per-node $NGPU --master-addr 127.0.0.1 \
    --master-port ${MASTER_PORT:-29500} -m rlaifv_b200.train_llava15_lora \
    "${MODEL[@]}" "${DATA[@]}" "${DPO[@]}" "${OPTIM[@]}" "${IO[@]}"

# like the reference recipe, make every checkpoint directory self-contained for llava/model/builder.py
# (adapter files are already inside; add the model config and the projector weights)
for dir in $CKPT/checkpoints/checkpoint-*; do
    [ -d "$dir" ] || continue
    new_dir="$CKPT/checkpoints/RLAIFV7B-lora_$(basename "$dir")"
    mv "$dir" "$new_dir"
    cp "$CKPT/checkpoints/config.json" "$CKPT/checkpoints/non_lora_trainables.bin" "$new_dir/"
done

#!/bin/bash
# Launch of LLaVA-1.5-7B DPO: every flag of the reference recipe (its script/train/llava15_train.sh) is accepted
# with the same meaning; the launcher is torchrun (one process per GPU, NCCL over NVLink) and ZeRO-2 is native.
export PYTHONPATH=$PYTHONPATH:`realpath .`
task_name=llava15_7b_DPO
exp_name=llava15_rlaifv
NGPU=${NGPU:-8}
CKPT=.ckpt/$task_name-$exp_name

MODEL=(--model_name_or_path liuhaotian/llava-v1.5-7b --vision_tower openai/clip-vit-large-patch14-336
       --mm_projector_type mlp2x_gelu --mm_vision_select_layer -2 --mm_use_im_start_end False
       --mm_use_im_patch_token False --fully_tune True --model_max_length 2048)
DATA=(--data_dir ./RLAIF-V-Dataset_logps/ --image_folder not_used --image_aspect_ratio pad --lazy_preprocess True
      --data_source_names '' --data_source_weights 1 --dataloader_num_workers 16)
DPO=(--task DPO --dpo_beta 0.1 --dpo_use_average False --dpo_token_weighted False --dpo_token_weight 1.0)
OPTIM=(--learning_rate 5e-7 --weight_decay 0.01 --warmup_ratio 0.05 --lr_scheduler_type "cosine" --max_steps 2672
       --num_train_epochs 10 --per_device_train_batch_size 1 --per_device_eval_batch_size 4
       --gradient_accumulation_steps 1 --gradient_checkpointing True --bf16 True --tf32 True
       --deepspeed ./script/zero2.json)
IO=(--output_dir $CKPT/checkpoints --logging_dir $CKPT/log --logging_steps 2 --evaluation_strategy "no"
    --save_strategy "steps" --save_steps 167 --save_total_limit 50 --report_to wandb --run_name $exp_name)

python -m torch.distributed.run --nnodes=1 --nproc-per-node $NGPU --master-addr 127.0.0.1 \
    --master-port ${MASTER_PORT:-29500} -m rlaifv_b200.train_llava15 \
    "${MODEL[@]}" "${DATA[@]}" "${DPO[@]}" "${OPTIM[@]}" "${IO[@]}"

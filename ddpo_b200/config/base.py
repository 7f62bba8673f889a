"""Experiment configuration -- same keys and defaults as the reference's ``config/base.py:3-103``
(``base["sample"|"train"|"pg"]``) plus the dataset overrides this build exercises.  ``pretrained_model`` is
a label only: weights are random-init (no checkpoints offline); the U-Net shape comes from ``unet_config``."""

base = {
    "sample": {
        "loadpath": "f:models/{iteration}", "savepath": "f:samples/{iteration}", "load_epoch": "latest",
        "n_samples_per_device": 4, "pretrained_model": "stabilityai/stable-diffusion-2-base", "prompt_kwargs": {},
        "n_inference_steps": 50, "eta": 1.0, "resolution": 512, "max_samples": 50e3, "max_steps": None,
        "local_size": 1600, "guidance_scale": 5.0, "filter_field": "labels", "mask_mode": "streaming_percentile",
        "mask_param": 95, "identical_batch": False, "iteration": 0, "evaluate": False, "cache": "cache", "seed": None,
    },
    "train": {
        "modelpath": "f:models/{iteration}", "loadpath": "f:samples/{iteration}", "savepath": "f:models/{iteration+1}",
        "pretrained_model": "stabilityai/stable-diffusion-2-base", "finetuned_model": None, "load_epoch": "latest",
        "max_train_samples": None, "resolution": 512, "train_cfg": False, "guidance_scale": 5.0,
        "train_batch_size": 2, "num_train_epochs": 40, "max_train_steps": None, "learning_rate": 1e-5, "beta1": 0.9,
        "beta2": 0.999, "weight_decay": 1e-4, "epsilon": 1e-8, "max_grad_norm": 1.0, "iteration": 0,
        "weighted_batch": False, "weighted_dataset": False, "dtype": "float32", "cache": "cache", "verbose": False,
        "save_freq": 100, "per_prompt_weights": False, "seed": 0,
    },
    "pg": {
        "loadpath": "", "load_epoch": "latest", "modelpath": "models/pg", "savepath": "f:models/pg",
        "pretrained_model": "stabilityai/stable-diffusion-2-base", "resolution": 512, "filter_field": None,
        "guidance_scale": 5.0, "dtype": "float32", "cache": "cache", "verbose": False, "seed": 0, "iteration": 0,
        "sample_batch_size": 8, "num_sample_batches_per_epoch": 1, "n_inference_steps": 50, "identical_batch": False,
        "evaluate": False, "eta": 1.0,
        "train_batch_size": 2, "train_accumulation_steps": 1, "num_train_epochs": 200, "num_inner_epochs": 1,
        "ppo_clip_range": 1e-4, "train_cfg": True, "learning_rate": 1e-5, "beta1": 0.9, "beta2": 0.999,
        "weight_decay": 1e-4, "epsilon": 1e-8, "max_grad_norm": 1.0, "save_freq": 10, "optimizer": "adamw",
        "train_timestep_ratio": 1.0, "prompt_kwargs": {}, "per_prompt_stats_bufsize": 32,
        "per_prompt_stats_min_count": 16,
        # extension (not in the reference): timesteps of one minibatch stacked into one U-Net pass; 1 = the
        # reference's call sequence (ddpo_b200/pipeline/policy_gradient.py)
        "train_macro": 10,
        # extension: rank (4, 8 or 16) of LoRA adapters on the attention projections, trained with the U-Net frozen;
        # 0 = full fine-tuning, the reference's only mode
        "lora_rank": 0,
    },
}

_SPARSE_SAMPLE = {"max_samples": 1024, "mask_mode": "percentile", "mask_param": 90, "identical_batch": True}
_RWR_SAMPLE = {"max_samples": 10240, "mask_mode": "streaming_percentile", "mask_param": 0, "identical_batch": False}
_SPARSE_TRAIN = {"train_cfg": True, "num_train_epochs": 50, "save_freq": 20, "dtype": "float32"}
_RWR_TRAIN = {"train_cfg": True, "train_batch_size": 1, "num_train_epochs": 5, "save_freq": 20, "dtype": "float32",
              "weighted_dataset": True, "temperature": 1 / 5.0}

# dataset overrides with the reference's names and values (config/base.py:105-200, :300-340); logbase is local
# (the reference prefixes its GCS bucket, config/user.py)
compressed_animals = {
    "common": {"logbase": "logs/compressed-animals", "prompt_fn": "imagenet_animals", "filter_field": "jpeg"},
    "sample": dict(_SPARSE_SAMPLE), "train": dict(_SPARSE_TRAIN, train_batch_size=4), "pg": {},
}
neg_compressed_animals = {
    "common": {"logbase": "logs/neg-compressed-animals", "prompt_fn": "imagenet_animals", "filter_field": "neg_jpeg"},
    "sample": dict(_SPARSE_SAMPLE), "train": dict(_SPARSE_TRAIN, train_batch_size=1), "pg": {},
}
compressed_animals_rwr = {
    "common": {"logbase": "logs/rwr-compressed-animals", "prompt_fn": "imagenet_animals", "filter_field": "jpeg"},
    "sample": dict(_RWR_SAMPLE), "train": dict(_RWR_TRAIN), "pg": {},
}
neg_compressed_animals_rwr = {
    "common": {"logbase": "logs/rwr-neg-compressed-animals", "prompt_fn": "imagenet_animals", "filter_field": "neg_jpeg"},
    "sample": dict(_RWR_SAMPLE), "train": dict(_RWR_TRAIN), "pg": {},
}
# the reference's own dataset names (config/base.py:200-385); prompt files resolve to this repo's ``assets/``
_AESTHETIC_COMMON = {"prompt_fn": "from_file", "prompt_kwargs": {"loadpath": "assets/common_animals.txt"},
                     "filter_field": "aesthetic"}
a_animals = {
    "common": dict(_AESTHETIC_COMMON, logbase="logs/aesthetic_simple_animals"),
    "sample": dict(_SPARSE_SAMPLE), "train": dict(_SPARSE_TRAIN, train_batch_size=1),
    "pg": {"train_batch_size": 1, "train_accumulation_steps": 2},
}
a_animals_rwr = {
    "common": dict(_AESTHETIC_COMMON, logbase="logs/aesthetic_simple_animals_rwr_ppb"),
    "sample": dict(_RWR_SAMPLE),
    "train": dict(_RWR_TRAIN, train_batch_size=4, save_freq=10000000, per_prompt_weights=True), "pg": {},
}
a_dog_1 = {
    "common": {"logbase": "logs/aesthetic_dogs_sweep/one", "prompt_fn": "manual", "prompt_kwargs": {"prompts": ["a dog"]},
               "filter_field": "aesthetic"},
    "pg": {"per_prompt_stats_bufsize": None, "per_prompt_stats_min_count": None, "train_batch_size": 1,
           "train_accumulation_steps": 2},
}
a_dog_2 = {
    "common": {"logbase": "logs/aesthetic_dogs_sweep/imagenet", "prompt_fn": "imagenet_dogs", "prompt_kwargs": {},
               "filter_field": "aesthetic"},
    "pg": {"train_batch_size": 1, "train_accumulation_steps": 2},
}
llava_bertscore = {
    "common": {"logbase": "logs/llava-bertscore-2-simple-animals", "prompt_fn": "nouns_activities",
               "prompt_kwargs": {"nouns_path": "assets/common_animals.txt", "activities_path": "assets/activities_v0.txt"},
               "filter_field": "llava_bertscore"},
    "pg": {},
}
llava_counting = {
    "common": {"logbase": "logs/llava-counting-v0-8", "prompt_fn": "counting",
               "prompt_kwargs": {"nouns_path": "assets/very_simple_animals.txt", "number_range": (2, 8)},
               "filter_field": "llava_vqa"},
    "pg": {},
}
compressed_animals_nocfg = {
    "common": {"logbase": "logs/nocfg-compressed-animals", "prompt_fn": "imagenet_animals", "filter_field": "jpeg"},
    "sample": dict(_SPARSE_SAMPLE), "train": dict(_SPARSE_TRAIN, train_cfg=False, train_batch_size=2), "pg": {},
}
neg_compressed_animals_nocfg = {
    "common": {"logbase": "logs/nocfg-neg-compressed-animals", "prompt_fn": "imagenet_animals", "filter_field": "neg_jpeg"},
    "sample": dict(_SPARSE_SAMPLE), "train": dict(_SPARSE_TRAIN, train_cfg=False, train_batch_size=2), "pg": {},
}
# this repo's earlier names, kept as aliases (BASELINE.json configs 3 and 5)
aesthetic_animals = {
    "common": {"logbase": "logs/aesthetic-animals", "prompt_fn": "common_animals", "filter_field": "aesthetic"},
    "sample": dict(_SPARSE_SAMPLE), "train": dict(_SPARSE_TRAIN, train_batch_size=4), "pg": {},
}
llava_alignment = {
    "common": {"logbase": "logs/llava-alignment", "prompt_fn": "nouns_activities", "filter_field": "llava_bertscore"},
    "pg": {"per_prompt_stats_bufsize": 32},
}

"""Constants of the hot path, same names and values as the reference's config.py (file:line cited per block).
Only what the hot path, the dataset builders and the training steps read is mirrored."""
from types import SimpleNamespace

# OpenAI's pretrained implementation                                   (config.py:5-7)
CLIP_MODEL = 'openai/clip-vit-large-patch14-336'
CLIP_EMBED_DIM = 1024

# Pretraining data: metadata CSVs, image folders and the CLIP tokenizer   (config.py:11-19, 49)
PRETRAIN_METADATA_PATH = 'data/data_pretrain.csv'
IMAGE_PATH = 'data/streetview_outputs_cropped'
IMAGE_PATH_2 = 'data/streetview_part_2_data'
PRETRAIN_METADATA_PATH_YFCC = 'data/data_yfcc_augmented_non_contaminated.csv'
IMAGE_PATH_YFCC = 'data/images_mp_16/jpgs'
DRIVING_SIDE_PATH = 'data/driving_side/countries_driving_side.json'
# A local copy of CLIP_MODEL's tokenizer files (vocab.json, merges.txt): nothing is downloaded
CLIP_TOKENIZER_PATH = 'saved_models/clip_tokenizer'

# Fine-tuning data: metadata CSVs and image folders                     (config.py:10, 12, 17, 19, 22-23)
METADATA_PATH = 'data/data_duels.csv'
METADATA_PATH_YFCC = 'data/data_yfcc_augmented_non_contaminated.csv'
METADATA_PATH_LANDMARKS = 'data/data_landmarks_aug.csv'
IMAGE_PATH_LANDMARKS = 'data/benchmarks/google_landmark/jpgs'

# Geocells path                                                        (config.py:34-36)
GEOCELL_PATH = 'data/geocells_2203.csv'       # PIGEON
GEOCELL_PATH_YFCC = 'data/geocells_yfcc.csv'  # PIGEOTTO

# Country borders for Country_accuracy (a GeoJSON FeatureCollection supplied by the user)   (config.py:26)
COUNTRY_PATH = 'data/geocells/countries.geojson'

# Multi-task regression scalers (joblib StandardScaler)             (config.py:39-40)
SCALER_PATH = 'saved_models/scaler/regression.scaler'
SCALER_PATH_YFCC = 'saved_models/scaler/regression_yfcc.scaler'

# GeoGuessr score decay, in km                                         (config.py:52)
DECAY_CONSTANT = 1492.7

# Haversine smoothing constant                                         (config.py:54-56)
LABEL_SMOOTHING_CONSTANT = 65

# Models                                                               (config.py:58-69)
CURRENT_SAVE_PATH = 'saved_models/WorldCLIP_head_landmarks.model'
PRETRAINED_CLIP = 'saved_models/StreetviewCLIP.model'
CLIP_PRETRAINED_HEAD = 'saved_models/New_Base_smooth_avg_MT_Geo_SV.model'
PRETRAINED_CLIP_YFCC = 'saved_models/WorldCLIP.model'
CLIP_PRETRAINED_HEAD_YFCC = 'saved_models/WorldCLIP_head.model'
CLIP_PRETRAINED_HEAD_YFCC_LANDMARKS = 'saved_models/WorldCLIP_head_landmarks.model'

# Embedding                                                            (config.py:70-71)
EMBED_BATCH_SIZE_PER_GPU = 512

# Cluster refinement model                                             (config.py:73-90)
PROTO_PATH = 'data/data_prototypes_2203.csv'
DATASET_PATH = 'data/hf_SVCLIP_2203'
PROTO_MODEL_PATH = 'saved_models/refiner/proto.refiner'
PROTO_PATH_YFCC = 'data/data_prototypes_YFCC.csv'
DATASET_PATH_YFCC = 'data/hf_YFCC'
PROTO_MODEL_YFCC_PATH = 'saved_models/refiner/proto_YFCC.refiner'
PROTO_PATH_LANDMARKS = 'data/data_prototypes_landmarks.csv'
DATASET_PATH_LANDMARKS = 'data/hf_landmarks'
PROTO_MODEL_LANDMARKS_PATH = 'saved_models/refiner/proto_landmarks.refiner'

# Benchmarks: a JSON file supplied by the user, {name: {"meta": CSV path, "images": image folder prefix}}   (config.py:91)
BENCHMARKS = 'data/benchmarks/benchmarks.json'

# Evaluation batch size (TRAIN_ARGS.per_device_eval_batch_size)        (config.py:98)
EVAL_BATCH_SIZE = 256

# Fine-tuning arguments (the fields training/train_eval_loop.py reads from TRAIN_ARGS)   (config.py:94-109)
TRAIN_ARGS = SimpleNamespace(output_dir='saved_models', per_device_train_batch_size=256, per_device_eval_batch_size=256,
                             num_train_epochs=1000, learning_rate=2e-5, logging_steps=1, gradient_accumulation_steps=1,
                             seed=330)

# Pretraining arguments (the HF TrainingArguments fields `pretrain.CLIPPretrainer` reads; report_to='tensorboard' is not
# implemented: the log goes to trainer_state.json and the `pretrain` logger)
_PRETRAIN_COMMON = dict(overwrite_output_dir=True, do_train=True, do_eval=True, evaluation_strategy='steps', eval_steps=50,
                        per_device_train_batch_size=32, per_device_eval_batch_size=32, gradient_accumulation_steps=8,
                        weight_decay=0.001, adam_beta1=0.9, adam_beta2=0.98, adam_epsilon=1e-06, max_grad_norm=1.0,
                        max_steps=-1, lr_scheduler_type='linear', logging_first_step=False, logging_strategy='steps',
                        logging_steps=1, save_strategy='steps', save_steps=50, seed=42, dataloader_drop_last=True,
                        run_name=None, adafactor=False, report_to='tensorboard', skip_memory_metrics=True,
                        resume_from_checkpoint=None, warmup_steps=0)

# PIGEOTTO                                                             (config.py:112-143)
PRETAIN_ARGS_YFCC = SimpleNamespace(**_PRETRAIN_COMMON, output_dir='saved_models/pretrained_yfcc', learning_rate=5e-07,
                                    num_train_epochs=4, warmup_ratio=0.02)
# PIGEON                                                               (config.py:145-177)
PRETAIN_ARGS = SimpleNamespace(**_PRETRAIN_COMMON, output_dir='saved_models/pretrained', learning_rate=1e-06,
                               num_train_epochs=20, warmup_ratio=0.2)

"""Environment-driven paths, mirroring ssd/paths.py:19-63 (names consumed by bench/bench_helpers.py:8-11).

Unlike the reference, a missing SSD_HF_CACHE / SSD_DATASET_DIR does not raise at import time: synthetic
model directories (ssd_b200.synth) make the engine usable without any downloaded checkpoint."""
import os

CUDA_ARCH = os.environ.get("SSD_CUDA_ARCH", "9.0")  # H100, as the reference (paths.py:5)
HF_CACHE_DIR = os.environ.get("SSD_HF_CACHE", "/tmp/ssd_b200_models")
DATASET_DIR = os.environ.get("SSD_DATASET_DIR", "/tmp/ssd_b200_datasets")

DEFAULT_TARGET = os.environ.get(
    "SSD_TARGET_MODEL",
    f"{HF_CACHE_DIR}/models--meta-llama--Llama-3.1-8B-Instruct/snapshots/0e9e39f249a16976918f6564b8830bc894c89659")
DEFAULT_DRAFT = os.environ.get(
    "SSD_DRAFT_MODEL",
    f"{HF_CACHE_DIR}/models--meta-llama--Llama-3.2-1B-Instruct/snapshots/9213176726f574b556790deb65791e0c5aa438b6")
EAGLE3_SPECFORGE_70B = os.environ.get("SSD_EAGLE3_SPECFORGE_70B", f"{HF_CACHE_DIR}/models--lmsys--SGLang-EAGLE3-Llama-3.3-70B-Instruct-SpecForge")
EAGLE3_YUHUILI_8B = os.environ.get("SSD_EAGLE3_8B", f"{HF_CACHE_DIR}/models--yuhuili--EAGLE3-LLaMA3.1-Instruct-8B")
EAGLE3_QWEN_32B = os.environ.get("SSD_EAGLE3_QWEN_32B", f"{HF_CACHE_DIR}/models--RedHatAI--Qwen3-32B-speculator.eagle3")
DATASET_PATHS = {
    "humaneval": f"{DATASET_DIR}/humaneval/humaneval_data_10000.jsonl",
    "alpaca": f"{DATASET_DIR}/alpaca/alpaca_data_10000.jsonl",
    "c4": f"{DATASET_DIR}/c4/c4_data_10000.jsonl",
    "gsm": f"{DATASET_DIR}/gsm8k/gsm8k_data_10000.jsonl",
    "ultrafeedback": f"{DATASET_DIR}/ultrafeedback/ultrafeedback_data_10000.jsonl",
}

"""videollama2_b200 — H100 (sm_90a) engine for VideoLLaMA2's video->text path.

Host code is Python/PyTorch (memory, streams, torch.distributed); all arithmetic runs in libvl2.so
(hand-written CUDA: wgmma/TMA GEMM + attention, fused row kernels) through the C-ABI in include/vl2.h.

`model_init` / `mm_infer` mirror the reference's two user-facing calls (videollama2/__init__.py:14-36, 39-114): the
callers on either side of the accelerated path.  Everything heavy is imported lazily so that `import videollama2_b200`
works on a CPU-only box."""
from __future__ import annotations

import copy
from functools import partial

__version__ = "0.1.0"

# The default system turn of the Llama-2 / Mistral chat format the reference prepends for its Mistral-family models
# (videollama2/__init__.py:76-85); a constant of the prompt format, needed for identical prompts.
_LLAMA2_SYSTEM = (
    "<<SYS>>\nYou are a helpful, respectful and honest assistant. Always answer as helpfully as possible, while being "
    "safe.  Your answers should not include any harmful, unethical, racist, sexist, toxic, dangerous, or illegal content. "
    "Please ensure that your responses are socially unbiased and positive in nature."
    "\n"
    "If a question does not make any sense, or is not factually coherent, explain why instead of answering something "
    "not correct. If you don't know the answer to a question, please don't share false information.\n<</SYS>>")


def get_model_name_from_path(model_path: str) -> str:
    """mm_utils.py:305-311: last path component, `parent_checkpoint-N` for trainer checkpoints."""
    parts = model_path.strip("/").split("/")
    return parts[-2] + "_" + parts[-1] if parts[-1].startswith("checkpoint-") else parts[-1]


def model_init(model_path=None, device="cuda", **kwargs):
    """(model, processor, tokenizer) like the reference's model_init.  `model_path` must be a LOCAL checkpoint directory
    (no network here); `processor` maps 'image' / 'video' to the device-side preprocessing of already decoded frames
    (aspect_ratio=None, as the reference passes: resize + centre crop, no square padding)."""
    from .constants import NUM_FRAMES
    from .mm_utils import process_image, process_video
    from .model import load_pretrained_model
    if model_path is None:
        raise ValueError("model_init needs a local checkpoint directory (the reference's hub default cannot be fetched offline)")
    tokenizer, model, processor, _ = load_pretrained_model(model_path, None, get_model_name_from_path(model_path),
                                                           device=device, **kwargs)
    if tokenizer.pad_token is None and tokenizer.unk_token is not None:
        tokenizer.pad_token = tokenizer.unk_token
    num_frames = getattr(model.config, "num_frames", NUM_FRAMES)
    processors = {
        "image": partial(process_image, processor=processor, aspect_ratio=None, device=device),
        "video": partial(process_video, processor=processor, aspect_ratio=None, num_frames=num_frames, device=device),
    }
    return model, processors, tokenizer


def build_messages(instruct, modal: str, model_type: str):
    """The chat turns mm_infer hands to `tokenizer.apply_chat_template` (videollama2/__init__.py:54-88)."""
    from .constants import DEFAULT_IMAGE_TOKEN, DEFAULT_VIDEO_TOKEN
    if modal == "image":
        modal_token = DEFAULT_IMAGE_TOKEN
    elif modal == "video":
        modal_token = DEFAULT_VIDEO_TOKEN
    elif modal == "text":
        modal_token = ""
    else:
        raise ValueError(f"Unsupported modal: {modal}")
    if isinstance(instruct, str):
        message = [{"role": "user", "content": modal_token + "\n" + instruct}]
    elif isinstance(instruct, list):
        message = copy.deepcopy(instruct)
        message[0]["content"] = modal_token + "\n" + message[0]["content"]
    else:
        raise ValueError(f"Unsupported type of instruct: {type(instruct)}")
    system = []
    if model_type in ("videollama2", "videollama2_mistral", "videollama2_mixtral"):
        system = [{"role": "system", "content": _LLAMA2_SYSTEM}]
    return system + message, modal_token


def mm_infer(image_or_video, instruct, model, tokenizer, modal="video", **kwargs):
    """Inference API of the reference (videollama2/__init__.py:39-114) on the H100 engine: prompt construction and
    stopping criteria on the host (exact), vision + prefill + graph-replayed decode on the device.  Greedy by default;
    do_sample=True samples on the device (vl2_sample_token) with the reference's defaults: temperature 0.2, top_p 0.9 and
    GenerationConfig's top_k 50; torch.manual_seed makes the draws reproducible."""
    import torch
    from .mm_utils import KeywordsStoppingCriteria, tokenizer_multimodal_token
    message, modal_token = build_messages(instruct, modal, model.config.model_type)
    images = None
    if modal != "text":
        images = [(image_or_video.to(device=model.device, dtype=getattr(model, "dtype", torch.bfloat16)), modal)]
    prompt = tokenizer.apply_chat_template(message, tokenize=False, add_generation_prompt=True)
    input_ids = tokenizer_multimodal_token(prompt, tokenizer, modal_token, return_tensors="pt").unsqueeze(0).long()
    attention_masks = input_ids.ne(tokenizer.pad_token_id).long()
    stopping = KeywordsStoppingCriteria([tokenizer.eos_token], tokenizer, input_ids)
    do_sample = kwargs.get("do_sample", False)
    output_ids = model.generate(input_ids, attention_mask=attention_masks, images=images, do_sample=do_sample,
                                temperature=kwargs.get("temperature", 0.2 if do_sample else 0.0),
                                max_new_tokens=kwargs.get("max_new_tokens", 2048), top_p=kwargs.get("top_p", 0.9),
                                use_cache=True, stopping_criteria=[stopping], pad_token_id=tokenizer.eos_token_id)
    return tokenizer.batch_decode(output_ids, skip_special_tokens=True)[0].strip()

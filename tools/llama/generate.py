"""tools/llama/generate.py — the entry point BASELINE.json's north_star names. In the reference commit its
contents live in fish_speech/models/text2semantic/inference.py; this shim re-exports the H100-native
equivalents under the old path."""
from fish_speech_b200.models.text2semantic.inference import (  # noqa: F401
    GenerateRequest,
    GenerateResponse,
    WrappedGenerateResponse,
    decode_n_tokens,
    decode_one_token_ar,
    decode_to_audio,
    encode_audio,
    generate,
    generate_batch,
    generate_long,
    init_model,
    launch_thread_safe_queue,
    load_codec_model,
    main,
)

if __name__ == "__main__":
    main()

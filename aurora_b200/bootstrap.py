"""Deployment bootstrap: build the CUDA encoder + shard from environment variables and install them
behind the reference's module API.  Used as the daemon's boot hook:

    AURORA_B200_ENCODER_WEIGHTS=/models/bge-base-en/model.safetensors \\
    AURORA_B200_VOCAB=/models/bge-base-en/vocab.txt \\
    python -m aurora_b200.daemon --socket /run/aurora_b200.sock --boot aurora_b200.bootstrap:configure_from_env

Variables: AURORA_B200_MODEL (bge-base | bge-large | minilm-l6, default bge-base), AURORA_B200_ENCODER_WEIGHTS
(HuggingFace BertModel safetensors), AURORA_B200_VOCAB (WordPiece vocab.txt), AURORA_B200_DEVICE (0),
AURORA_B200_CAPACITY (rows to map in HBM at start, default 1048576; the shards grow as chunks arrive), AURORA_B200_DTYPE (row format of the shards: bf16, the
default, or int8 for half the HBM), AURORA_B200_SNAPSHOT (directory: restored at
start when present; see KnowledgeBase.save), AURORA_B200_MAX_TOKENS / AURORA_B200_MAX_SEQS (encoder workspace).
There is no CPU fallback: without a CUDA device or with a variable missing this raises.

With AURORA_B200_DEVICES (one owner process over several GPUs) every listed GPU holds an encoder replica as well as its
shard (bf16 and int8 shards; f32 shards take host vectors and get no replicas), and ingest encodes each shard's share on its own GPU.  Each replica takes the weights plus its own workspace,
sized by AURORA_B200_MAX_TOKENS / MAX_SEQS.  For bge-base at the defaults (32768 tokens, 2048 sequences), counted from
aur_encoder_open's allocations, that is 218 MB of weights, 511 MB of activations and 9 MB of pooled outputs per GPU.
"""

from __future__ import annotations

import os


def _model_config(name: str):
    from .encoder import BGE_BASE, BGE_LARGE, MINILM_L6

    table = {"bge-base": BGE_BASE, "bge-large": BGE_LARGE, "minilm-l6": MINILM_L6}
    if name not in table:
        raise ValueError(f"AURORA_B200_MODEL={name!r}: expected one of {sorted(table)}")
    return table[name]


def configure_from_env() -> None:
    from . import retriever
    from .encoder import EmbeddingClient, Encoder, TextEncoder, configure_embedding_client, from_hf_bert, read_safetensors
    from .wordpiece import NativeTokenizer

    missing = [v for v in ("AURORA_B200_ENCODER_WEIGHTS", "AURORA_B200_VOCAB") if not os.environ.get(v)]
    if missing:
        raise RuntimeError("aurora_b200 bootstrap: set " + ", ".join(missing))
    cfg = _model_config(os.environ.get("AURORA_B200_MODEL", "bge-base"))
    device = int(os.environ.get("AURORA_B200_DEVICE", "0"))
    capacity = int(os.environ.get("AURORA_B200_CAPACITY", str(1 << 20)))
    dtype = os.environ.get("AURORA_B200_DTYPE", "bf16")
    enc = Encoder(cfg, max_tokens=int(os.environ.get("AURORA_B200_MAX_TOKENS", "32768")),
                  max_seqs=int(os.environ.get("AURORA_B200_MAX_SEQS", "2048")), device=device)
    enc.load_weights(from_hf_bert(read_safetensors(os.environ["AURORA_B200_ENCODER_WEIGHTS"]), cfg))
    tok = NativeTokenizer(os.environ["AURORA_B200_VOCAB"], lower=os.environ.get("AURORA_B200_CASED", "0") != "1")   # C++, multi-threaded
    if tok.vocab_size != cfg.vocab:
        raise RuntimeError(f"vocabulary has {tok.vocab_size} entries, the model expects {cfg.vocab}")
    text_encoder = TextEncoder(enc, tok, max_len=cfg.max_pos)
    # the correlation path's embedding client (daemon ops embed / embed_batch / similarity_scores) on the same encoder
    configure_embedding_client(lambda: EmbeddingClient(enc, lambda text: tok.encode(text, cfg.max_pos)))
    snap = os.environ.get("AURORA_B200_SNAPSHOT")
    wal = os.environ.get("AURORA_B200_WAL", "1") != "0"      # mutation log beside the snapshot (replayed after a crash)

    # AURORA_B200_DEVICES = "all" or "0,1,2,...": this process owns one shard per listed GPU (engine.MultiIndex) and
    # one encoder on each of those GPUs (the weights are read once and copied device to device): every shard's share of
    # an ingest is encoded on its own GPU.  Queries are encoded on AURORA_B200_DEVICE.
    devs = os.environ.get("AURORA_B200_DEVICES", "").strip()
    factory = loader = None
    if devs:
        from . import _native as N
        from .engine import MultiIndex

        devices = list(range(N.load().aur_device_count())) if devs == "all" else [int(x) for x in devs.split(",")]
        if dtype != "f32":              # f32 shards take host vectors (TextEncoder.can_append): replicas would sit idle
            text_encoder.replicate(devices)
        factory = lambda dim, cap: MultiIndex(dim, cap, devices=devices, dtype=dtype)       # noqa: E731
        loader = lambda path, cap: MultiIndex.load(path, capacity=cap, devices=devices)     # noqa: E731

    def make():
        if snap and os.path.exists(os.path.join(snap, "meta.json")):
            kb = retriever.KnowledgeBase.load(snap, text_encoder, capacity=capacity, device=device, index_loader=loader)
        else:
            kb = retriever.KnowledgeBase(text_encoder, capacity=capacity, device=device, index_factory=factory, dtype=dtype)
        if snap and wal:
            os.makedirs(snap, exist_ok=True)
            kb.attach_wal(os.path.join(snap, "mutations.log"))
        return kb

    retriever.configure(factory=make)

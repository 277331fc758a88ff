"""OpenAI-style chat-completions server on the sm_90a hot path (SURVEY §8 f3).

Mirrors the request / response shapes of the reference's `serving/server.py` (`ChatCompletionRequest`
:84-95, content parts :45-62, `/chat/completions` :209-300: `data: {chunk}\n\n` server-sent events when
`stream` is set, one `chat.completion` object otherwise) on top of `generate_content(prompt, stream=...)`.
The reference serialises requests with a global lock; here non-streaming requests that arrive while the
engine is busy are grouped (up to `slots`) and decoded together by `LlavaLlamaModel.generate_batch`
(continuous batching over the shared paged pool, vila_b200/serving.py).  With --sample every non-streaming
request goes through generate_batch with its own temperature, top_p and seed, drawn on the device; streaming
requests stay on the single-stream greedy decoder.

    python -m vila_b200.server --model-path <dir> --port 8000
"""
from __future__ import annotations

import argparse
import asyncio
import base64
import json
import re
import time
import uuid
from io import BytesIO
from typing import Any, Dict, List, Literal, Optional, Union

from pydantic import BaseModel

IMAGE_B64 = re.compile(r"^data:image/(png|jpe?g);base64,(.*)$")
VIDEO_B64 = re.compile(r"^data:video/(mp4);base64,(.*)$")


class MediaURL(BaseModel):
    url: str


class TextContent(BaseModel):
    type: Literal["text"]
    text: str


class ImageContent(BaseModel):
    type: Literal["image_url"]
    image_url: MediaURL


class VideoContent(BaseModel):
    type: Literal["video_url"]
    video_url: MediaURL
    frames: Optional[int] = 8


class ChatMessage(BaseModel):
    role: Literal["user", "assistant"]
    content: Union[str, List[Union[TextContent, ImageContent, VideoContent]]]


class ChatCompletionRequest(BaseModel):
    model: str
    messages: List[ChatMessage]
    max_tokens: Optional[int] = 512
    top_p: Optional[float] = 0.9
    temperature: Optional[float] = 0.2
    stream: Optional[bool] = False
    use_cache: Optional[bool] = True
    num_beams: Optional[int] = 1
    client: Optional[dict] = None
    seed: Optional[int] = None


def load_image(url: str):
    from PIL import Image
    m = IMAGE_B64.match(url)
    if m is None:
        if url.startswith("http"):
            raise ValueError("remote image URLs need network access; send base64 data URLs")
        return Image.open(url).convert("RGB")
    return Image.open(BytesIO(base64.b64decode(m.groups()[1]))).convert("RGB")


def load_video(url: str) -> str:
    """A `video_url` -> a file on disk (serving/server.py:124-143: base64 mp4 data URL or http(s)
    download).  A path that exists locally is accepted as it is (no network on a serving box)."""
    import os
    import tempfile
    if url.startswith("http"):
        import requests
        payload = requests.get(url).content
    else:
        m = VIDEO_B64.match(url)
        if m is None:
            if os.path.exists(url):
                return url
            raise ValueError(f"Invalid video url: {url[:64]}")
        payload = base64.b64decode(m.groups()[1])
    path = os.path.join(tempfile.mkdtemp(prefix="vila_serving_"), f"{uuid.uuid5(uuid.NAMESPACE_DNS, url)}.mp4")
    with open(path, "wb") as f:
        f.write(payload)
    return path


def sample_frames_from_video(path: str, num_frames: int = 8) -> list:
    """The server's own sampling rule (serving/server.py:106-122), not `_load_video`'s: frame i of n sits at
    index int(total / n * i); unreadable frames are dropped; a directory of frames is sampled the same way."""
    import os
    from PIL import Image
    if os.path.isdir(path):
        files = sorted(os.path.join(path, f) for f in os.listdir(path))
        return [Image.open(files[int(len(files) / num_frames * i)]).convert("RGB") for i in range(num_frames)]
    import cv2
    cap = cv2.VideoCapture(path)
    total = int(cap.get(cv2.CAP_PROP_FRAME_COUNT))
    frames = []
    for i in range(num_frames):
        cap.set(cv2.CAP_PROP_POS_FRAMES, int(total / num_frames * i))
        ok, frame = cap.read()
        if ok:
            frames.append(Image.fromarray(cv2.cvtColor(frame, cv2.COLOR_BGR2RGB)))
    cap.release()
    return frames


def build_prompt(messages: List[ChatMessage], num_video_frames: int = 8) -> list:
    """messages -> the prompt list generate_content takes (serving/server.py:234-256): strings and text
    parts as they come, images decoded to PIL, a video replaced by its sampled frames (as images)."""
    prompt: list = []
    for message in messages:
        if isinstance(message.content, str):
            prompt.append(message.content)
            continue
        for part in message.content:
            if part.type == "text":
                prompt.append(part.text)
            elif part.type == "image_url":
                prompt.append(load_image(part.image_url.url))
            elif part.type == "video_url":
                prompt += sample_frames_from_video(load_video(part.video_url.url), part.frames or num_video_frames)
            else:
                raise NotImplementedError(f"Unsupported content type: {part.type}")
    return prompt


class Engine:
    """One model, one asyncio lock (the GPU is a single queue): streaming requests hold the lock while
    their generator runs; non-streaming requests waiting for it are batched together."""

    def __init__(self, model, model_name: str, slots: int = 8, kv_cache: str = "bf16", sample: bool = False):
        self.model, self.model_name, self.slots = model, model_name, slots
        self.kv_cache = kv_cache
        if sample and not hasattr(model, "generate_batch"):
            raise ValueError("sample=True needs a model with generate_batch (the batched engine draws the tokens)")
        self.sample = sample  # non-streaming requests: sampled on the batched engine with their own parameters
        self.lock = asyncio.Lock()
        self.pending: List[Any] = []

    def _gen_config(self, req: ChatCompletionRequest):
        gc = self.model.default_generation_config
        gc.max_new_tokens = req.max_tokens
        return gc

    async def complete(self, req: ChatCompletionRequest) -> Dict[str, Any]:
        if req.model != self.model_name:
            raise ValueError(f"The endpoint is configured to use the model {self.model_name}, "
                             f"but the request model is {req.model}")
        # checked before the request joins a batch: a bad value fails this request only
        params = self._sampling(req) if self.sample else None
        loop = asyncio.get_running_loop()
        fut = loop.create_future()
        self.pending.append((req, fut, params))
        async with self.lock:
            if not fut.done():  # this task drains the queue for everyone that piled up behind the lock
                batch, self.pending = self.pending[:self.slots], self.pending[self.slots:]
                try:
                    texts = await loop.run_in_executor(None, self._run_batch, [r for r, _, _ in batch],
                                                       [p for _, _, p in batch] if self.sample else None)
                except Exception as e:  # every request of the failed batch gets the error, none is left waiting
                    for _, f, _ in batch:
                        if not f.done():
                            f.set_exception(e)
                else:
                    for (_, f, _), t in zip(batch, texts):
                        if not f.done():
                            f.set_result(t)
        text = await fut
        return {"id": uuid.uuid4().hex, "object": "chat.completion", "created": int(time.time()),
                "model": req.model, "index": 0,
                "choices": [{"message": {"role": "assistant", "content": text}}]}

    def _run_batch(self, reqs: List[ChatCompletionRequest], sampling: Optional[list] = None) -> List[str]:
        """sampling: one SamplingParams per request (Engine(sample=True)), or None for greedy decoding"""
        m = self.model
        if sampling is None and (len(reqs) == 1 or not hasattr(m, "generate_batch")):
            return [m.generate_content(build_prompt(r.messages), generation_config=self._gen_config(r)) for r in reqs]
        prepared = [m._prepare_content(build_prompt(r.messages)) for r in reqs]
        # the default is not passed: a model whose generate_batch predates the kv_cache argument keeps working
        kw = {} if self.kv_cache == "bf16" else {"kv_cache": self.kv_cache}
        if sampling is not None:
            kw["sampling"] = sampling
        ids = m.generate_batch([{"input_ids": i, "media": md, "media_config": mc} for i, md, mc in prepared],
                               max_new_tokens=max(r.max_tokens or 512 for r in reqs), slots=self.slots, **kw)
        outs = []
        for r, g in zip(reqs, ids):
            outs.append(m.tokenizer.decode(g[:r.max_tokens or 512], skip_special_tokens=True).strip())
        return outs

    @staticmethod
    def _sampling(req: ChatCompletionRequest):
        """a request's SamplingParams: temperature None or 0 is greedy, top_p None is off; bad values raise"""
        from .sampling import SamplingParams
        return SamplingParams(temperature=float(req.temperature or 0.0),
                              top_p=float(req.top_p) if req.top_p is not None else 1.0, seed=req.seed)

    async def stream(self, req: ChatCompletionRequest):
        if req.model != self.model_name:
            raise ValueError(f"The endpoint is configured to use the model {self.model_name}, "
                             f"but the request model is {req.model}")
        async with self.lock:
            gen = self.model.generate_content(build_prompt(req.messages), generation_config=self._gen_config(req),
                                              stream=True)
            for chunk_id, new_text in enumerate(gen):
                if len(new_text):
                    chunk = {"id": str(chunk_id), "object": "chat.completion.chunk", "created": int(time.time()),
                             "model": req.model, "choices": [{"delta": {"content": new_text}}]}
                    yield f"data: {json.dumps(chunk)}\n\n"
                await asyncio.sleep(0)
            yield "data: [DONE]\n\n"


def create_app(model, model_name: str, slots: int = 8, kv_cache: str = "bf16", sample: bool = False):
    from fastapi import FastAPI
    from fastapi.responses import JSONResponse, StreamingResponse
    app = FastAPI()
    engine = Engine(model, model_name, slots, kv_cache, sample)
    app.state.engine = engine

    @app.get("/")
    async def read_root():
        return {"message": "vila_b200 chat-completions endpoint: POST /chat/completions"}

    @app.post("/chat/completions")
    async def chat_completions(request: ChatCompletionRequest):
        try:
            if request.stream:
                return StreamingResponse(engine.stream(request), media_type="text/event-stream")
            return await engine.complete(request)
        except Exception as e:  # the reference answers 500 with the message (server.py:302-306)
            return JSONResponse(status_code=500, content={"error": str(e)})

    return app


def main() -> None:
    import uvicorn

    import llava
    from llava.mm_utils import get_model_name_from_path
    ap = argparse.ArgumentParser()
    ap.add_argument("--host", type=str, default="0.0.0.0")
    ap.add_argument("--port", type=int, default=8000)
    ap.add_argument("--model-path", type=str, required=True)
    ap.add_argument("--slots", type=int, default=8)
    ap.add_argument("--decode-weights", choices=("bf16", "fp8", "w4a16"), default="bf16",
                    help="weights of the single-stream greedy decoder (fp8: e4m3 with per-row scales; w4a16: "
                         "4-bit with group-128 scales and zero points, lm_head e4m3), and of the engine that "
                         "batches queued requests; the prefill stays bf16)")
    ap.add_argument("--kv-cache", choices=("bf16", "fp8"), default="bf16",
                    help="K/V format of the engine that batches queued requests (fp8: e4m3 with one fp32 scale "
                         "per token and KV head, about half the bytes; the single-stream decoder stays bf16)")
    ap.add_argument("--sample", action="store_true",
                    help="sample non-streaming requests with their own temperature, top_p and seed on the batched "
                         "engine (vila_sample_batch, on the device), even a request that arrives alone; without it "
                         "every request is decoded greedily.  Streaming requests stay on the single-stream greedy "
                         "decoder either way")
    args = ap.parse_args()
    model = llava.load(args.model_path, decode_weights=args.decode_weights)
    uvicorn.run(create_app(model, get_model_name_from_path(args.model_path), args.slots, args.kv_cache, args.sample),
                host=args.host, port=args.port)


if __name__ == "__main__":
    main()

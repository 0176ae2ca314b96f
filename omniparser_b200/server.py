"""Serving layer with cross-request dynamic batching (SURVEY.md §8f-4).

The reference server (ref:omnitool/omniparserserver/omniparserserver.py:37-44) handles ``POST /parse/`` one request at a
time: ``Omniparser.parse(base64_image)`` -> ``{"som_image_base64", "parsed_content_list", "latency"}``.  On this path a
batch of 8 screenshots costs far less than 8 times one screenshot, so the throughput of a serving process is decided by
whether concurrent requests share a batch.  :class:`BatchingOmniparser` keeps the facade's interface (``parse(base64) ->
(png_b64, parsed_content_list)``, same config keys) and is safe to call from any number of threads: requests that arrive
within ``max_wait_ms`` of each other are parsed in ONE ``parse_screenshots`` call whatever their image sizes (they share
the detector's 640 x 640 canvas: one detector forward, one Florence-2 pass); PNG decode, the OCR pre-step, the overlay drawing and the PNG encode run on the
callers' own threads, outside the batch.  ``create_app`` builds the FastAPI application with the reference's routes and wire
format (base64 PNG in JSON both ways, ref:omnitool/gradio/agent/llm_utils/omniparserclient.py:17-23).

    python -m omniparser_b200.server --som_model_path weights/icon_detect_v3/model.pt \\
        --caption_model_path weights/icon_caption_florence --BOX_TRESHOLD 0.05
"""
import base64
import io
import threading
import time
from concurrent.futures import Future
from typing import Callable, Dict, Hashable, List, Optional, Sequence


class DynamicBatcher:
    """Groups concurrent ``submit(key, item)`` calls into batches per key.

    A batch is dispatched to ``run_batch(key, [items]) -> [results]`` (on the batcher's single worker thread) when it reaches
    ``max_batch`` items or when its oldest item has waited ``max_wait_s``.  Batches of one key keep arrival order; an
    exception raised by ``run_batch`` is delivered to every caller of that batch.  ``submit`` blocks until its result is
    ready.  One worker thread = one batch on the device at a time (the handles underneath serialise themselves anyway)."""

    def __init__(self, run_batch: Callable[[Hashable, List], Sequence], max_batch: int = 8, max_wait_s: float = 0.004):
        if max_batch < 1:
            raise ValueError("max_batch must be >= 1")
        self._run, self.max_batch, self.max_wait_s = run_batch, int(max_batch), float(max_wait_s)
        self._cv = threading.Condition()
        self._queues: Dict[Hashable, List] = {}     # key -> [(t_arrival, item, future)]
        self._closed = False
        self.stats = dict(batches=0, items=0, max_batch_seen=0)
        self._worker = threading.Thread(target=self._loop, name="b2p-batcher", daemon=True)
        self._worker.start()

    def submit(self, key: Hashable, item):
        fut: Future = Future()
        with self._cv:
            if self._closed:
                raise RuntimeError("batcher is closed")
            self._queues.setdefault(key, []).append((time.monotonic(), item, fut))
            self._cv.notify_all()
        return fut.result()

    def close(self):
        with self._cv:
            self._closed = True
            self._cv.notify_all()
        self._worker.join(timeout=5)

    def _pick(self, now):
        """-> (key, entries) of a batch that is due, or (None, seconds until the next one is)."""
        best, wait = None, None
        for key, q in self._queues.items():
            if not q:
                continue
            age = now - q[0][0]
            if len(q) >= self.max_batch or age >= self.max_wait_s or self._closed:
                if best is None or q[0][0] < self._queues[best][0][0]:
                    best = key
            else:
                left = self.max_wait_s - age
                wait = left if wait is None else min(wait, left)
        if best is None:
            return None, wait
        q = self._queues[best]
        take, self._queues[best] = q[:self.max_batch], q[self.max_batch:]
        return best, take

    def _loop(self):
        while True:
            with self._cv:
                while True:
                    key, got = self._pick(time.monotonic())
                    if key is not None:
                        break
                    if self._closed and not any(self._queues.values()):
                        return
                    self._cv.wait(timeout=got)
            items = [e[1] for e in got]
            try:
                results = self._run(key, items)
                if len(results) != len(items):
                    raise RuntimeError(f"run_batch returned {len(results)} results for {len(items)} items")
                for (_, _, fut), r in zip(got, results):
                    fut.set_result(r)
            except BaseException as exc:   # noqa: BLE001 -- delivered to the callers
                for _, _, fut in got:
                    if not fut.done():
                        fut.set_exception(exc)
            self.stats["batches"] += 1
            self.stats["items"] += len(items)
            self.stats["max_batch_seen"] = max(self.stats["max_batch_seen"], len(items))


class BatchingOmniparser:
    """``util/omniparser.py::Omniparser`` (ref:util/omniparser.py:7-32) with cross-request batching: same config keys and
    ``parse`` contract, results identical to :class:`omniparser_b200.omniparser.Omniparser` request by request.
    Extra config keys: ``max_batch`` (8), ``max_wait_ms`` (4), and those of the facade (``device``, ``detector_precision``,
    ``caption_precision``, ``tokenizer_path``, ``allow_id_captions``, ``ocr_fn``)."""

    def __init__(self, config: Dict, models=None):
        from .utils import get_caption_model_processor, get_yolo_model
        self.config = config
        device = config.get("device", "cuda")
        if models is None:
            som = get_yolo_model(model_path=config.get("som_model_path"), device=device, precision=config.get("detector_precision"))
            cmp_ = get_caption_model_processor(model_name=config["caption_model_name"], model_name_or_path=config["caption_model_path"],
                                               device=device, precision=config.get("caption_precision", "fp16x3"),
                                               tokenizer_path=config.get("tokenizer_path"), allow_id_captions=config.get("allow_id_captions"))
        else:
            som, cmp_ = models
        self.som_model, self.caption_model_processor = som, cmp_
        self._ocr = config.get("ocr_fn")
        self._batcher = DynamicBatcher(self._run_batch, int(config.get("max_batch", 8)), float(config.get("max_wait_ms", 4.0)) / 1e3)
        print("Omniparser initialized!!!")

    @property
    def stats(self):
        return dict(self._batcher.stats)

    def close(self):
        self._batcher.close()

    def _run_batch(self, key, items):
        from .utils import parse_screenshots
        imgs = [it["img"] for it in items]
        ocr = [(it["text"], it["ocr_bbox"]) for it in items]
        res = parse_screenshots(imgs, self.som_model, self.caption_model_processor, ocr, self.config["BOX_TRESHOLD"], 0.7, 640)
        return [r[0] for r in res]

    def parse(self, image_base64: str):
        import numpy as np
        from PIL import Image

        from . import som_overlay
        image = Image.open(io.BytesIO(base64.b64decode(image_base64)))
        print("image size:", image.size)
        r = max(image.size) / 3200                                   # ref:util/omniparser.py:21-27
        cfg = {"text_scale": 0.8 * r, "text_thickness": max(int(2 * r), 1), "text_padding": max(int(3 * r), 1), "thickness": max(int(3 * r), 1)}
        ocr = self._ocr
        if ocr is None:
            from .ocr import check_ocr_box as ocr
        (text, ocr_bbox), _ = ocr(image, display_img=False, output_bb_format="xyxy", easyocr_args={"text_threshold": 0.8}, use_paddleocr=False)
        img = np.asarray(image.convert("RGB"))
        if not ocr_bbox:
            print("no ocr bbox!!!")
        # queued by detector canvas: every request through this facade letterboxes to 640 x 640, so screenshots of any size
        # share a batch (parse_screenshots takes a batch of different sizes)
        elems = self._batcher.submit((640, 640), dict(img=img, text=list(text), ocr_bbox=ocr_bbox or None))
        print("len(filtered_boxes):", len(elems), -1)
        encoded, _, _ = som_overlay.som_outputs(img, [e["bbox"] for e in elems], True, **cfg,
                                                device=getattr(self.som_model, "device", None))
        return encoded, elems


def create_app(config: Dict, parser=None):
    """FastAPI application with the reference's routes: POST /parse/ {"base64_image"} -> {"som_image_base64",
    "parsed_content_list", "latency"}; GET /probe/.  Handlers are sync functions, so FastAPI runs them on its thread pool and
    concurrent requests meet in the batcher."""
    from fastapi import FastAPI
    from pydantic import BaseModel

    omniparser = parser if parser is not None else BatchingOmniparser(config)
    app = FastAPI()

    class ParseRequest(BaseModel):
        base64_image: str

    @app.post("/parse/")
    def parse(parse_request: ParseRequest):
        print("start parsing...")
        start = time.time()
        dino_labled_img, parsed_content_list = omniparser.parse(parse_request.base64_image)
        latency = time.time() - start
        print("time:", latency)
        return {"som_image_base64": dino_labled_img, "parsed_content_list": parsed_content_list, "latency": latency}

    @app.get("/probe/")
    def root():
        return {"message": "Omniparser API ready"}

    app.state.omniparser = omniparser
    return app


def parse_arguments(argv: Optional[Sequence[str]] = None):
    import argparse
    p = argparse.ArgumentParser(description="Omniparser API")        # flags of ref:omnitool/omniparserserver/omniparserserver.py:17-27
    p.add_argument("--som_model_path", type=str, default=None)
    p.add_argument("--caption_model_name", type=str, default="florence2")
    p.add_argument("--caption_model_path", type=str, default="../../weights/icon_caption_florence")
    p.add_argument("--device", type=str, default="cuda")
    p.add_argument("--BOX_TRESHOLD", type=float, default=0.05)
    p.add_argument("--host", type=str, default="127.0.0.1")
    p.add_argument("--port", type=int, default=8000)
    p.add_argument("--max_batch", type=int, default=8)
    p.add_argument("--max_wait_ms", type=float, default=4.0)
    return p.parse_args(argv)


if __name__ == "__main__":
    import uvicorn
    args = parse_arguments()
    uvicorn.run(create_app(vars(args)), host=args.host, port=args.port)

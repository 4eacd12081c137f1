"""REST front-end bound to the GPU-resident queue (SURVEY 8f N4).

Same 20 routes, request bodies and response shapes as the reference's `api.py` (routes A:365-935), so its clients keep
working; `create_app(db)` takes any `swarmdb_b200.SwarmsDB` (one GPU) or `ShardedSwarmsDB` rank.  Three defects of
the reference layer are FIXED here rather than reproduced (SURVEY section 4 lists them):

  * `POST /messages/broadcast` and `POST /groups/message` declare `response_model=List[str]` but return a dict
    (A:507/530, A:760/781): every call answers 500 there.  Here they have response models that match what is returned
    (`{"status", "message_id"}` / `{"status", "message_ids"}`).
  * route parameters called `status` shadow `fastapi.status`, so the 403 / 404 branches of three routes raise
    `AttributeError` (A:576+599, A:630+639, A:694+702).  Here the query parameter keeps its public name through an alias.
  * authorisation / not-found errors raised inside a `try` are re-wrapped as 500 (A:595-620).  Here an `HTTPException`
    always reaches the client unchanged.

Two read-only additions expose what the device knows: `GET /agents/{id}/load` (inbox size / unread count / priority
histogram from the rings) and `GET /queue` (queue-wide statistics) - N3.

    uvicorn swarmdb_b200.server:app            # builds the queue from the environment (see `Settings`)
"""
from __future__ import annotations

import os
import time
from collections import defaultdict, deque
from dataclasses import dataclass, field
from datetime import datetime, timedelta, timezone
from typing import Any, Deque, Dict, List, Optional, Union

from fastapi import Depends, FastAPI, Header, HTTPException, Query, Request
from fastapi import status as http
from fastapi.middleware.cors import CORSMiddleware
from fastapi.responses import JSONResponse
from fastapi.security import HTTPAuthorizationCredentials, HTTPBearer
from pydantic import BaseModel

from .core import GpuConfig, KafkaConfig, Message, MessagePriority, MessageStatus, MessageType, SwarmsDB

VERSION = "1.0.0"


@dataclass
class Settings:
    """Knobs of the reference server (A:39-52, A:59-73, A:86, A:312), read from the same environment variables."""
    environment: str = field(default_factory=lambda: os.getenv("API_ENV", "development"))
    jwt_secret: str = field(default_factory=lambda: os.getenv("JWT_SECRET", "supersecretkey"))
    jwt_algorithm: str = field(default_factory=lambda: os.getenv("JWT_ALGORITHM", "HS256"))
    token_minutes: int = field(default_factory=lambda: int(os.getenv("TOKEN_EXPIRE_MINUTES", "1440")))
    topic_prefix: str = field(default_factory=lambda: os.getenv("KAFKA_TOPIC_PREFIX", "agent_messaging_"))
    history_dir: str = field(default_factory=lambda: os.getenv("MESSAGE_HISTORY_DIR", "./message_history"))
    save_interval: int = field(default_factory=lambda: int(os.getenv("SAVE_INTERVAL_SECONDS", "300")))
    num_shards: int = field(default_factory=lambda: int(os.getenv("KAFKA_NUM_PARTITIONS", "1")))
    cors_origins: List[str] = field(default_factory=lambda: os.getenv("CORS_ORIGINS", "*").split(","))
    rate_limit_per_minute: int = field(default_factory=lambda: int(os.getenv("RATE_LIMIT_PER_MINUTE", "300")))


# ---- wire models (field names are the public contract of the reference API) ---------------------------------------
Content = Union[str, Dict[str, Any], List[Any]]


class Credentials(BaseModel):
    username: str
    password: str


class TokenOut(BaseModel):
    access_token: str
    token_type: str


class SendIn(BaseModel):
    content: Content
    receiver_id: Optional[str] = None
    message_type: MessageType = MessageType.CHAT
    priority: MessagePriority = MessagePriority.NORMAL
    metadata: Optional[Dict[str, Any]] = None
    visible_to: Optional[List[str]] = None
    supersede: bool = False                # a newer superseding send of the sender and type replaces it while pending


class BroadcastIn(BaseModel):
    content: Content
    message_type: MessageType = MessageType.CHAT
    priority: MessagePriority = MessagePriority.NORMAL
    metadata: Optional[Dict[str, Any]] = None
    exclude_agents: Optional[List[str]] = None
    supersede: bool = False


class RegisterIn(BaseModel):
    agent_id: str
    description: Optional[str] = None
    capabilities: Optional[List[str]] = None
    metadata: Optional[Dict[str, Any]] = None


class GroupIn(BaseModel):
    group_name: str
    agent_ids: List[str]


class GroupSendIn(BaseModel):
    group_name: str
    content: Content
    message_type: MessageType = MessageType.CHAT
    priority: MessagePriority = MessagePriority.NORMAL
    metadata: Optional[Dict[str, Any]] = None
    supersede: bool = False


class TrimIn(BaseModel):
    max_messages: Optional[int] = None     # messages each agent keeps (None: no count limit)
    max_bytes: Optional[int] = None        # pending payload bytes each agent keeps, sum of pad32(len) (None: no limit)
    by_priority: bool = False              # drop the lowest priority first (oldest first within a level)
    agent_ids: Optional[List[str]] = None  # None: every agent


class MessageOut(BaseModel):
    id: str
    sender_id: str
    receiver_id: Optional[str]
    content: Content
    type: MessageType
    priority: MessagePriority
    timestamp: float
    status: MessageStatus
    metadata: Dict[str, Any]
    token_count: Optional[int] = None
    visible_to: List[str]

    @classmethod
    def of(cls, m: Message) -> "MessageOut":
        return cls(id=m.id, sender_id=m.sender_id, receiver_id=m.receiver_id, content=m.content, type=m.type,
                   priority=m.priority, timestamp=m.timestamp, status=m.status, metadata=m.metadata,
                   token_count=m.token_count, visible_to=m.visible_to)


class BroadcastOut(BaseModel):
    status: str
    message_id: str


class GroupSendOut(BaseModel):
    status: str
    message_ids: List[str]


class HealthOut(BaseModel):
    status: str
    version: str
    environment: str
    kafka_connected: bool          # name kept for clients of the reference: true when the device transport answers
    timestamp: float


class StatsOut(BaseModel):
    total_messages: int
    active_agents: int
    messages_by_type: Dict[str, int]
    messages_by_status: Dict[str, int]
    messages_by_agent: Dict[str, Dict[str, int]]
    last_save_time: float


class _RateLimiter:
    """Sliding one-minute window per client address (A:266-314: 300 requests / minute / IP by default)."""

    def __init__(self, per_minute: int) -> None:
        self.per_minute = per_minute
        self.hits: Dict[str, Deque[float]] = defaultdict(deque)

    def allow(self, client: str) -> bool:
        now = time.monotonic()
        q = self.hits[client]
        while q and now - q[0] > 60.0:
            q.popleft()
        if len(q) >= self.per_minute:
            return False
        q.append(now)
        return True


def create_app(db: Optional[SwarmsDB] = None, settings: Optional[Settings] = None) -> FastAPI:
    import jwt

    cfg = settings or Settings()
    if db is None:
        db = SwarmsDB(base_topic=f"{cfg.topic_prefix}messages", config=KafkaConfig(num_partitions=cfg.num_shards),
                      save_dir=cfg.history_dir, auto_save=True, save_interval=cfg.save_interval, gpu_config=GpuConfig())
    app = FastAPI(title="Agent Messaging System API (H100)", version=VERSION,
                  description="Agent communication and LLM load balancing over a GPU-resident message queue")
    app.state.db = db
    app.state.agent_metadata = {}
    app.add_middleware(CORSMiddleware, allow_origins=cfg.cors_origins, allow_credentials=True, allow_methods=["*"],
                       allow_headers=["*"])
    limiter = _RateLimiter(cfg.rate_limit_per_minute)

    @app.middleware("http")
    async def rate_limit(request: Request, call_next):
        client = request.client.host if request.client else "unknown"
        if not limiter.allow(client):
            return JSONResponse(status_code=http.HTTP_429_TOO_MANY_REQUESTS, content={"detail": "Rate limit exceeded"})
        return await call_next(request)

    bearer = HTTPBearer()

    def caller(cred: HTTPAuthorizationCredentials = Depends(bearer)) -> str:
        """The agent id inside a valid bearer token (A:337-362)."""
        denied = HTTPException(status_code=http.HTTP_401_UNAUTHORIZED, detail="Invalid authentication credentials",
                               headers={"WWW-Authenticate": "Bearer"})
        try:
            sub = jwt.decode(cred.credentials, cfg.jwt_secret, algorithms=[cfg.jwt_algorithm]).get("sub")
        except jwt.PyJWTError:
            raise denied
        if sub is None:
            raise denied
        return sub

    def admin(who: str = Depends(caller)) -> str:
        if who != "admin":
            raise HTTPException(status_code=http.HTTP_403_FORBIDDEN, detail="Admin privileges required")
        return who

    def guarded(what: str, fn):
        """Run one queue call: HTTP errors pass through untouched, anything else becomes a 500 naming the operation."""
        try:
            return fn()
        except HTTPException:
            raise
        except Exception as e:
            raise HTTPException(status_code=http.HTTP_500_INTERNAL_SERVER_ERROR, detail=f"Failed to {what}: {e}")

    # ---- auth -------------------------------------------------------------------------------------------------
    @app.post("/auth/token", response_model=TokenOut)
    def issue_token(c: Credentials):
        if not c.username or not c.password:       # like the reference, any non-empty pair is accepted (A:374-381)
            raise HTTPException(status_code=http.HTTP_401_UNAUTHORIZED, detail="Invalid username or password",
                                headers={"WWW-Authenticate": "Bearer"})
        exp = datetime.now(timezone.utc) + timedelta(minutes=cfg.token_minutes)
        return TokenOut(access_token=jwt.encode({"sub": c.username, "exp": exp}, cfg.jwt_secret, algorithm=cfg.jwt_algorithm),
                        token_type="bearer")

    # ---- registry ---------------------------------------------------------------------------------------------
    @app.post("/agents/register", status_code=http.HTTP_201_CREATED)
    def register(body: RegisterIn, who: str = Depends(caller)):
        if who not in (body.agent_id, "admin"):
            raise HTTPException(status_code=http.HTTP_403_FORBIDDEN,
                                detail="You can only register yourself or need admin privileges")
        guarded("register agent", lambda: db.register_agent(body.agent_id))
        if body.metadata or body.capabilities or body.description:
            app.state.agent_metadata[body.agent_id] = {"description": body.description, "capabilities": body.capabilities,
                                                       **(body.metadata or {})}
        return {"status": "success", "agent_id": body.agent_id}

    @app.delete("/agents/{agent_id}")
    def deregister(agent_id: str, who: str = Depends(caller)):
        if who not in (agent_id, "admin"):
            raise HTTPException(status_code=http.HTTP_403_FORBIDDEN,
                                detail="You can only deregister yourself or need admin privileges")
        guarded("deregister agent", lambda: db.deregister_agent(agent_id))
        app.state.agent_metadata.pop(agent_id, None)
        return {"status": "success", "agent_id": agent_id}

    # ---- send -------------------------------------------------------------------------------------------------
    # An Idempotency-Key header is the send's dedup_id (GpuConfig.dedup_entries): the route flushes, so that a retried
    # request whose first attempt was queued answers with the original message instead of queueing a second copy.
    def settled(mid: str, key: Optional[str]) -> str:
        if key is None:
            return mid
        db.flush()
        return db.original_id(mid) or mid

    @app.post("/messages", response_model=MessageOut)
    def send(body: SendIn, who: str = Depends(caller),
             idempotency_key: Optional[str] = Header(None, alias="Idempotency-Key")):
        def go():
            mid = db.send_message(sender_id=who, content=body.content, receiver_id=body.receiver_id,
                                  message_type=body.message_type, priority=body.priority, metadata=body.metadata,
                                  visible_to=body.visible_to, dedup_id=idempotency_key, supersede=body.supersede)
            return MessageOut.of(db.get_message(settled(mid, idempotency_key)))
        return guarded("send message", go)

    @app.post("/messages/broadcast", response_model=BroadcastOut)
    def broadcast(body: BroadcastIn, who: str = Depends(caller),
                  idempotency_key: Optional[str] = Header(None, alias="Idempotency-Key")):
        mid = guarded("broadcast message", lambda: settled(db.broadcast_message(
            sender_id=who, content=body.content, message_type=body.message_type, priority=body.priority,
            metadata=body.metadata, exclude_agents=body.exclude_agents, dedup_id=idempotency_key,
            supersede=body.supersede), idempotency_key))
        return BroadcastOut(status="success", message_id=mid)

    @app.post("/groups", status_code=http.HTTP_201_CREATED)
    def create_group(body: GroupIn, who: str = Depends(caller)):
        guarded("create agent group", lambda: db.add_agent_group(group_name=body.group_name, agent_ids=body.agent_ids))
        return {"status": "success", "group_name": body.group_name}

    @app.post("/groups/message", response_model=GroupSendOut)
    def send_group(body: GroupSendIn, who: str = Depends(caller),
                   idempotency_key: Optional[str] = Header(None, alias="Idempotency-Key")):
        def go():
            ids = db.send_to_group(sender_id=who, group_name=body.group_name, content=body.content,
                                   message_type=body.message_type, priority=body.priority, metadata=body.metadata,
                                   dedup_id=idempotency_key, supersede=body.supersede)
            return [settled(mid, idempotency_key) for mid in ids]
        return GroupSendOut(status="success", message_ids=guarded("send group message", go))

    # ---- read -------------------------------------------------------------------------------------------------
    @app.post("/agents/receive", response_model=List[MessageOut])
    def receive(max_messages: int = 100, timeout: float = 1.0, max_tokens: Optional[int] = Query(None, ge=1, lt=1 << 64),
                who: str = Depends(caller)):
        # max_tokens: as many pending messages as fit that many tokens of context (SwarmsDB.receive_messages)
        kw = {} if max_tokens is None else {"max_tokens": max_tokens}
        return [MessageOut.of(m) for m in guarded("receive messages", lambda: db.receive_messages(
            agent_id=who, max_messages=max_messages, timeout=timeout, **kw))]

    @app.get("/messages/{message_id}", response_model=MessageOut)
    def get_message(message_id: str, include_device: bool = False, who: str = Depends(caller)):
        # include_device: a message still queued on the device without a host record is found there too
        m = guarded("get message", lambda: db.get_message(message_id, include_device))
        if m is None:
            raise HTTPException(status_code=http.HTTP_404_NOT_FOUND, detail=f"Message {message_id} not found")
        may_see = who == "admin" or who in (m.sender_id, m.receiver_id) or not m.visible_to or who in m.visible_to   # A:554-562
        if not may_see:
            raise HTTPException(status_code=http.HTTP_403_FORBIDDEN, detail="You don't have permission to view this message")
        return MessageOut.of(m)

    @app.get("/messages", response_model=List[MessageOut])
    def query(sender_id: Optional[str] = None, receiver_id: Optional[str] = None, message_type: Optional[MessageType] = None,
              status_filter: Optional[MessageStatus] = Query(None, alias="status"), after_timestamp: Optional[float] = None,
              before_timestamp: Optional[float] = None, limit: int = 100, include_device: bool = False,
              who: str = Depends(caller)):
        if who != "admin" and sender_id and sender_id != who and receiver_id != who:
            raise HTTPException(status_code=http.HTTP_403_FORBIDDEN,
                                detail="You can only query messages you sent or received")
        if include_device and who != "admin" and receiver_id != who:
            # the device queues hold every agent's undelivered messages: a caller may read its own queue only
            raise HTTPException(status_code=http.HTTP_403_FORBIDDEN,
                                detail="include_device needs receiver_id set to yourself or admin privileges")
        found = guarded("query messages", lambda: db.query_messages(
            sender_id=sender_id, receiver_id=receiver_id, message_type=message_type, status=status_filter,
            after_timestamp=after_timestamp, before_timestamp=before_timestamp, limit=limit,
            include_device=include_device))                  # include_device: also the matching device-queued messages
        return [MessageOut.of(m) for m in found]

    @app.get("/agents/{agent_id}/messages", response_model=List[MessageOut])
    def agent_messages(agent_id: str, status_filter: Optional[MessageStatus] = Query(None, alias="status"),
                       limit: int = 100, skip: int = 0, who: str = Depends(caller)):
        if who not in (agent_id, "admin"):
            raise HTTPException(status_code=http.HTTP_403_FORBIDDEN, detail="You can only access your own messages")
        found = guarded("get agent messages", lambda: db.get_agent_messages(agent_id=agent_id, status=status_filter,
                                                                           limit=limit, skip=skip))
        return [MessageOut.of(m) for m in found]

    @app.put("/messages/{message_id}/status")
    def set_status(message_id: str, new_status: MessageStatus = Query(..., alias="status"), who: str = Depends(caller)):
        m = db.get_message(message_id)
        if m is None:
            raise HTTPException(status_code=http.HTTP_404_NOT_FOUND, detail=f"Message {message_id} not found")
        if who != "admin" and who != m.receiver_id:
            raise HTTPException(status_code=http.HTTP_403_FORBIDDEN,
                                detail="You can only update status of messages you received")
        if new_status == MessageStatus.PROCESSED:
            guarded("update message status", lambda: db.mark_message_as_processed(message_id))
        else:
            m.status = new_status
        return {"status": "success", "message_id": message_id}

    # ---- what the device knows (N3) ---------------------------------------------------------------------------
    @app.get("/agents/{agent_id}/load")
    def agent_load(agent_id: str, who: str = Depends(caller)):
        if who not in (agent_id, "admin"):
            raise HTTPException(status_code=http.HTTP_403_FORBIDDEN, detail="You can only access your own load")
        return guarded("read agent load", lambda: db.get_agent_queue_load(agent_id))

    @app.get("/queue")
    def queue(_: str = Depends(admin)):
        return guarded("read queue statistics", lambda: db.shard.queue_stats())

    # ---- operations -------------------------------------------------------------------------------------------
    @app.get("/health", response_model=HealthOut)
    def health():
        try:
            db.admin_client.list_topics(timeout=2)     # liveness of the device transport (A:798 probes the broker this way)
            alive = True
        except Exception:
            alive = False
        return HealthOut(status="ok", version=VERSION, environment=cfg.environment, kafka_connected=alive,
                         timestamp=time.time())

    @app.get("/stats", response_model=StatsOut)
    def stats(_: str = Depends(admin)):
        return guarded("get system stats", db.get_stats)

    @app.post("/admin/save")
    def save(_: str = Depends(admin)):
        guarded("save message history", db.save_message_history)
        return {"status": "success", "timestamp": time.time()}

    @app.post("/admin/flush")
    def flush_old(older_than: Optional[float] = None, include_device: bool = False, _: str = Depends(admin)):
        # include_device: also archive and expire the device-queued messages older than the cutoff
        return {"status": "success", "flushed_count": guarded("flush old messages",
                                                              lambda: db.flush_old_messages(older_than, include_device))}

    @app.post("/admin/trim")
    def trim(t: TrimIn, _: str = Depends(admin)):
        # bounded queues on demand: drop what takes each agent's device queue past the caps, without delivering it
        try:
            n = db.trim_queues(t.max_messages, t.max_bytes, t.agent_ids, t.by_priority)
        except ValueError as e:                   # limits outside what trim_queues accepts: the request is at fault
            raise HTTPException(status_code=422, detail=str(e))
        except Exception as e:
            raise HTTPException(status_code=http.HTTP_500_INTERNAL_SERVER_ERROR, detail=f"Failed to trim queues: {e}")
        return {"trimmed": n}

    @app.post("/admin/resend_failed")
    def resend_failed(_: str = Depends(admin)):
        ids = guarded("resend failed messages", db.resend_failed_messages)
        return {"status": "success", "resent_count": len(ids), "message_ids": ids}

    @app.post("/admin/scale_partitions")
    def scale(_: str = Depends(admin)):
        guarded("scale partitions", db.auto_scale_partitions)     # shards are the GPUs of the box: nothing to grow
        return {"status": "success", "timestamp": time.time()}

    @app.on_event("shutdown")
    def shutdown() -> None:
        try:
            db.close()
        except Exception as e:  # pragma: no cover
            print(f"Error closing messaging system: {e}")

    return app


def __getattr__(name: str):
    """`uvicorn swarmdb_b200.server:app` - the application is built on first access (it needs a GPU)."""
    if name == "app":
        global _app
        try:
            return _app
        except NameError:
            _app = create_app()
            return _app
    raise AttributeError(name)

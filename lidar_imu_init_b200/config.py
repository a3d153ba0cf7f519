"""The node's parameters: a reference YAML file as it ships (config/*.yaml) plus the launch-file <param>s, with the keys and defaults
of laserMapping.cpp:767-799, mapped onto LidarOdometry.

The YAML files are the nested maps of the reference; the parser reads that subset of YAML (maps by indentation, scalars, flow lists
[a, b, c], comments) and needs no YAML library.
"""
from __future__ import annotations

import ast
from dataclasses import dataclass, field, fields

LIDAR_NAMES = {1: "Livox (CustomMsg)", 2: "Velodyne", 3: "Ouster", 4: "L515", 5: "Pandar", 6: "Robosense"}


class ConfigError(ValueError):
    pass


@dataclass
class Config:
    """laserMapping.cpp:767-799: field = (parameter name, default)."""
    max_iteration: int = 4                  # max_iteration (launch <param>)
    point_filter_num: int = 2               # point_filter_num (launch <param>)
    cube_side_length: float = 200.0         # cube_side_length (launch <param>)
    lid_topic: str = "/livox/lidar"         # common/lid_topic
    imu_topic: str = "/livox/imu"           # common/imu_topic
    filter_size_surf: float = 0.5           # mapping/filter_size_surf
    filter_size_map: float = 0.5            # mapping/filter_size_map
    det_range: float = 300.0                # mapping/det_range
    gyr_cov: float = 0.1                    # mapping/gyr_cov
    acc_cov: float = 0.1                    # mapping/acc_cov
    grav_cov: float = 0.001                 # mapping/grav_cov
    b_gyr_cov: float = 0.0001               # mapping/b_gyr_cov
    b_acc_cov: float = 0.0001               # mapping/b_acc_cov
    blind: float = 1.0                      # preprocess/blind
    lidar_type: int = 1                     # preprocess/lidar_type (AVIA)
    scan_line: int = 16                     # preprocess/scan_line
    feature_extract_en: bool = False        # preprocess/feature_extract_en
    cut_frame: bool = True                  # initialization/cut_frame
    cut_frame_num: int = 1                  # initialization/cut_frame_num
    orig_odom_freq: int = 10                # initialization/orig_odom_freq
    online_refine_time: float = 20.0        # initialization/online_refine_time
    mean_acc_norm: float = 9.81             # initialization/mean_acc_norm
    data_accum_length: float = 300.0        # initialization/data_accum_length
    Rot_LI_cov: list = field(default_factory=list)     # initialization/Rot_LI_cov (no default: three values are required)
    Trans_LI_cov: list = field(default_factory=list)   # initialization/Trans_LI_cov
    path_en: bool = True                    # publish/path_en
    scan_publish_en: bool = True            # publish/scan_publish_en
    dense_publish_en: bool = True           # publish/dense_publish_en
    scan_bodyframe_pub_en: bool = True      # publish/scan_bodyframe_pub_en
    runtime_pos_log_enable: bool = False    # runtime_pos_log_enable
    pcd_save_en: bool = False               # pcd_save/pcd_save_en
    interval: int = -1                      # pcd_save/interval


# parameter name of the node -> Config field
PARAMS = {
    "max_iteration": "max_iteration", "point_filter_num": "point_filter_num", "cube_side_length": "cube_side_length",
    "common/lid_topic": "lid_topic", "common/imu_topic": "imu_topic",
    "mapping/filter_size_surf": "filter_size_surf", "mapping/filter_size_map": "filter_size_map", "mapping/det_range": "det_range",
    "mapping/gyr_cov": "gyr_cov", "mapping/acc_cov": "acc_cov", "mapping/grav_cov": "grav_cov", "mapping/b_gyr_cov": "b_gyr_cov",
    "mapping/b_acc_cov": "b_acc_cov",
    "preprocess/blind": "blind", "preprocess/lidar_type": "lidar_type", "preprocess/scan_line": "scan_line",
    "preprocess/feature_extract_en": "feature_extract_en",
    "initialization/cut_frame": "cut_frame", "initialization/cut_frame_num": "cut_frame_num", "initialization/orig_odom_freq": "orig_odom_freq",
    "initialization/online_refine_time": "online_refine_time", "initialization/mean_acc_norm": "mean_acc_norm",
    "initialization/data_accum_length": "data_accum_length", "initialization/Rot_LI_cov": "Rot_LI_cov",
    "initialization/Trans_LI_cov": "Trans_LI_cov",
    "publish/path_en": "path_en", "publish/scan_publish_en": "scan_publish_en", "publish/dense_publish_en": "dense_publish_en",
    "publish/scan_bodyframe_pub_en": "scan_bodyframe_pub_en", "runtime_pos_log_enable": "runtime_pos_log_enable",
    "pcd_save/pcd_save_en": "pcd_save_en", "pcd_save/interval": "interval",
}
_TYPES = {f.name: f.type for f in fields(Config)}


def _scalar(s: str):
    s = s.strip()
    if len(s) >= 2 and s[0] == s[-1] and s[0] in "\"'":
        return s[1:-1]
    low = s.lower()
    if low in ("true", "yes", "on"):
        return True
    if low in ("false", "no", "off"):
        return False
    if s.startswith("[") and s.endswith("]"):
        return [_scalar(x) for x in s[1:-1].split(",") if x.strip()]
    try:
        return ast.literal_eval(s)
    except (ValueError, SyntaxError):
        return s


def _strip_comment(line: str) -> str:
    q = None
    for i, ch in enumerate(line):
        if q:
            if ch == q:
                q = None
        elif ch in "\"'":
            q = ch
        elif ch == "#" and (i == 0 or line[i - 1] in " \t"):
            return line[:i]
    return line


def parse_yaml(text: str, where: str = "<yaml>") -> dict:
    """The nested maps of a reference config file, flattened to {"group/key": value}."""
    out, stack = {}, []   # stack of (indent, key)
    for no, raw in enumerate(text.splitlines(), 1):
        line = _strip_comment(raw).rstrip()
        if not line.strip():
            continue
        ind = len(line) - len(line.lstrip(" "))
        if "\t" in line[:ind + 1]:
            raise ConfigError(f"{where}:{no}: tab in indentation")
        key, sep, val = line.strip().partition(":")
        if not sep or not key:
            raise ConfigError(f"{where}:{no}: expected 'key: value', got {raw.strip()!r}")
        while stack and stack[-1][0] >= ind:
            stack.pop()
        name = "/".join([k for _, k in stack] + [key.strip()])
        if val.strip():
            out[name] = _scalar(val)
        else:
            stack.append((ind, key.strip()))
    return out


def _coerce(name: str, value, where: str):
    t = _TYPES[PARAMS[name]]
    try:
        if t == "bool":
            if isinstance(value, bool):
                return value
            if isinstance(value, int) and value in (0, 1):
                return bool(value)
            raise ValueError
        if t == "int":
            if isinstance(value, bool) or not float(value).is_integer():
                raise ValueError
            return int(value)
        if t == "float":
            if isinstance(value, bool):
                raise ValueError
            return float(value)
        if t == "str":
            return str(value)
        if t == "list":
            if not isinstance(value, list):
                raise ValueError
            return [float(v) for v in value]
    except (TypeError, ValueError):
        pass
    raise ConfigError(f"{where}: {name} = {value!r} is not a{'n' if t == 'int' else ''} {t}")


def parse_override(s: str):
    """'name=value' (a node parameter, e.g. max_iteration=5 or mapping/filter_size_map=0.2) -> (name, value)."""
    name, sep, val = s.partition("=")
    name = name.strip()
    if not sep or not name:
        raise ConfigError(f"--param {s!r}: expected name=value")
    if name not in PARAMS:
        raise ConfigError(f"--param {s!r}: unknown parameter {name!r}; known: {', '.join(sorted(PARAMS))}")
    return name, _scalar(val)


def load(path: str | None = None, overrides=()) -> Config:
    """A Config from a YAML file and 'name=value' overrides; parameters the file does not set keep the node's defaults. Keys the
    node does not read are ignored, as the node ignores them. Refuses what lies outside the ported scope."""
    cfg = Config()
    if path is not None:
        try:
            with open(path) as f:
                text = f.read()
        except OSError as e:
            raise ConfigError(f"{path}: {e.strerror}") from None
        for name, v in parse_yaml(text, path).items():
            if name in PARAMS:
                setattr(cfg, PARAMS[name], _coerce(name, v, path))
    for s in overrides:
        name, v = parse_override(s)
        setattr(cfg, PARAMS[name], _coerce(name, v, f"--param {s}"))
    check(cfg, path or "<defaults>")
    return cfg


def check(cfg: Config, where: str):
    """The run stops here for what the port does not cover (DESIGN §9) and for values the node would misread."""
    if not cfg.cut_frame:
        raise ConfigError(f"{where}: initialization/cut_frame: false is not supported; only the cut-frame preprocess is ported")
    if cfg.feature_extract_en:
        raise ConfigError(f"{where}: preprocess/feature_extract_en: true is not supported; feature extraction is not ported")
    if cfg.lidar_type == 4:
        raise ConfigError(f"{where}: preprocess/lidar_type 4 (L515) is not supported")
    if cfg.lidar_type not in LIDAR_NAMES:
        raise ConfigError(f"{where}: preprocess/lidar_type {cfg.lidar_type} is not a LiDAR type of the node (1, 2, 3, 5, 6)")
    for name in ("Rot_LI_cov", "Trans_LI_cov"):
        if len(getattr(cfg, name)) != 3:
            raise ConfigError(f"{where}: initialization/{name} must list three values, got {getattr(cfg, name)!r}")
    if cfg.cut_frame_num < 1 or cfg.orig_odom_freq < 1 or cfg.max_iteration < 1 or cfg.point_filter_num < 1:
        raise ConfigError(f"{where}: cut_frame_num, orig_odom_freq, max_iteration and point_filter_num must be positive")


def wanted_topics(cfg: Config, fmt: str) -> dict:
    """{topic: accepted message types} of the node's LiDAR and IMU subscriptions in a bag of format fmt (rosmsg.decoders)."""
    from . import rosmsg
    d = rosmsg.decoders(fmt, cfg.lidar_type)
    return {cfg.lid_topic: d.lidar_types, cfg.imu_topic: d.imu_types}


# the node's published clouds: LidarOdometry.published key -> topic (laserMapping.cpp:873-878)
CLOUD_TOPICS = {"registered": "/cloud_registered", "body": "/cloud_registered_body", "effect": "/cloud_effected"}
# every topic the node publishes a message on (:873-884; /Laser_map has none: publish_map has no caller)
RECORD_TOPICS = ("/cloud_registered", "/cloud_registered_body", "/cloud_effected", "/aft_mapped_to_init", "/tf", "/path")


def odometry_kwargs(cfg: Config, pcd_dir: str = "PCD", record_topics=None) -> dict:
    """LidarOdometry's constructor arguments (laserMapping.cpp:822-838). Without a recording there is no subscriber for the published
    clouds: only pcd_save's records are built, and only when pcd_save_en is set. record_topics (the topics a run records, see
    record_publish) builds the clouds those topics carry. (det_range and cube_side_length are read and checked but LidarOdometry does
    not segment the map by the field of view.)"""
    if record_topics is not None:
        publish = record_publish(cfg, record_topics, pcd_dir)
    else:
        publish = dict(scan_pub_en=False, pcd_save_en=True, interval=cfg.interval, pcd_dir=pcd_dir) if cfg.pcd_save_en else None
    return dict(filter_size_map=cfg.filter_size_map, max_iteration=cfg.max_iteration, gyr_cov=cfg.gyr_cov, acc_cov=cfg.acc_cov,
                orig_odom_freq=cfg.orig_odom_freq, cut_frame_num=cfg.cut_frame_num, data_accum_length=cfg.data_accum_length,
                filter_size_surf=cfg.filter_size_surf, rot_LI_cov=list(cfg.Rot_LI_cov), trans_LI_cov=list(cfg.Trans_LI_cov),
                b_gyr_cov=cfg.b_gyr_cov, b_acc_cov=cfg.b_acc_cov, mean_acc_norm=cfg.mean_acc_norm, publish=publish)


def record_publish(cfg: Config, topics, pcd_dir: str = "PCD") -> dict:
    """LidarOdometry's publish= for a run that records the topics `topics`: the node's publish/scan_publish_en, dense_publish_en and
    scan_bodyframe_pub_en and its pcd_save; a cloud whose topic is not recorded is not downloaded."""
    return dict(scan_pub_en=cfg.scan_publish_en, dense_pub_en=cfg.dense_publish_en, scan_body_pub_en=cfg.scan_bodyframe_pub_en,
                pcd_save_en=cfg.pcd_save_en, interval=cfg.interval, pcd_dir=pcd_dir,
                clouds=tuple(k for k, t in CLOUD_TOPICS.items() if t in topics))


def preprocess(cfg: Config) -> dict:
    """LidarOdometry.preprocess: the cut's sensor parameters (laserMapping.cpp:768,781-786)."""
    return dict(lidar_type=cfg.lidar_type, N_SCANS=cfg.scan_line, blind=cfg.blind, point_filter_num=cfg.point_filter_num)

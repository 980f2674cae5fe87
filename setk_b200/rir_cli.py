"""
setk_b200.rir_cli -- the image-method RIR command lines behind scripts/sptk/rir_generate_{1d,2d}.py.

One simulator serves both.  `geometry` ("1d" for a linear array, "2d" for a planar one) selects
what differs between the reference's two scripts: how the receivers are placed around the array's
centre (set_mic), the range of the sources' DoA (_place_spk), and the defaults of --array-rely,
--sound-speed and --source-distance, the form of --array-topo and the 1d-only --vertical-oriented.
Everything else -- the rooms, the retry loops, the random draws and their order, the batching of
the (room, source) pairs on the device and the rir.json schema -- is the same code for both.

Deviations from the reference:
  * _place_spk reads the module-global `args` there (so it only works as __main__); here self.args.
  * RoomGenerator.generate swaps the names of volume and surface in its minimum T60.  Kept: changing
    it would change which rooms the command draws.  A drawn T60 below the room's true Sabine minimum
    raises the reference's "cannot be calculated" ValueError, as rir-simulate fails there.
  * The room plot Room{r}.jpg is not drawn (matplotlib is not a dependency of this project).
"""
import argparse
import json
import random
from pathlib import Path

import numpy as np
import torch

from . import plan
from .libs.opts import str2tuple, strtobool
from .libs.sampler import UniformSampler
from .libs.utils import get_logger, write_wav

logger = get_logger(__name__)

# device memory for the responses of one batch of (room, source) pairs
BATCH_BYTES = 1 << 30


class Room(object):
    """
    Room instance
    """

    def __init__(self, l, w, h, rt60=None, refl=None):
        self.size = (l, w, h)
        self.beta = rt60 if rt60 is not None else [refl] * 6

    def set_mic(self, topo, center, geometry, vertical=False):
        """
        Place microphone array
        topo: tuple like (x1, x2, ...) for "1d", [(x1, y1), ...] for "2d"
        center: center 3D postion for microphone array
        """
        Mx, My, Mz = center
        if geometry == "2d":
            self.rpos = [(Mx + x, My + y, Mz) for (x, y) in topo]
        else:
            Mc = (topo[-1] - topo[0]) / 2
            if not vertical:
                self.rpos = [(Mx - Mc + x, My, Mz) for x in topo]
            else:
                self.rpos = [(Mx, My - Mc + x, Mz) for x in topo]
        self.topo = topo

    def conf(self):
        """
        Return configure of room (exclude sound sources)
        """
        Rf = lambda f: round(f, 3)  # noqa: E731
        return {
            "beta": [Rf(f) for f in self.beta] if isinstance(self.beta, list) else Rf(self.beta),
            "receiver_location": [tuple(Rf(n) for n in p) for p in self.rpos],
            "room_size": [Rf(n) for n in self.size],
            "receiver_geometric": self.topo
        }

    def problem(self, spos, v):
        """
        (room, beta, source, receivers) as rir-simulate receives them (rir_generate_1d.py:151-168,
        rir_generate_2d.py:146-163)
        """
        f3 = lambda p: [float("{:.3f}".format(f)) for f in p]  # noqa: E731
        room = f3(self.size)
        beta = f3(self.beta) if isinstance(self.beta, list) else round(self.beta, 3)
        return room, plan.rir_beta(room, beta, v), f3(spos), [f3(p) for p in self.rpos]


class RoomGenerator(object):
    """
    Room generator
    """

    def __init__(self, rt60_opt, absc_opt, room_dim):
        self.rt60_opt = rt60_opt
        if not rt60_opt:
            self.absc = UniformSampler(absc_opt)
        else:
            self.rt60 = UniformSampler(str2tuple(rt60_opt))
        dim_range = [str2tuple(t) for t in room_dim.split(";")]
        if len(dim_range) != 3:
            raise RuntimeError(f"Wrong format with --room-dim={room_dim}")
        self.dim_sampler = [UniformSampler(c) for c in dim_range]

    def generate(self, v=340):
        (l, w, h) = (s.sample() for s in self.dim_sampler)
        if self.rt60_opt:
            if self.rt60.max == 0:
                return Room(l, w, h, rt60=0)
            # the reference's names: S is the volume and V the surface here (kept, see the docstring)
            S, V = l * w * h, (l * w + l * h + w * h) * 2
            rt60_min = 24 * V * np.log(10) / (v * S)
            if rt60_min >= self.rt60.max:
                return None
            return Room(l, w, h, rt60=random.uniform(rt60_min, self.rt60.max))
        absc = self.absc.sample()
        return Room(l, w, h, refl=np.sqrt(1 - absc))


class RirSimulator(object):
    """
    RIR simulator of a linear ("1d") or planar ("2d") microphone array
    """

    def __init__(self, geometry, args):
        Path(args.dump_dir).mkdir(exist_ok=True, parents=True)
        self.rirs_cfg = []
        self.jobs = []
        self.room_generator = RoomGenerator(args.rt60, args.abs_range, args.room_dim)
        self.mx, self.my = args.array_relx, args.array_rely
        self.geometry = geometry
        if geometry == "2d":
            self.array_topo = [str2tuple(t) for t in args.array_topo.split(";")]
            self.vertical = False
        else:
            self.array_topo = args.array_topo
            self.vertical = args.vertical
        self.sr = args.sr
        self.args = args
        self.device = "cuda" if torch.cuda.is_available() else "cpu"

    def _place_mic(self, room):
        x, y, _ = room.size
        mx = random.uniform(*(x * v for v in self.mx))
        my = random.uniform(*(y * v for v in self.my))
        mz = random.uniform(*self.args.array_height)
        room.set_mic(self.array_topo, (mx, my, mz), self.geometry, vertical=self.vertical)
        return (mx, my), room

    def _max_src_dist(self, rpos_2d, room_size_2d):
        mx, my = rpos_2d
        rx, ry = room_size_2d
        bound = [(0, 0), (0, ry), (rx, 0), (rx, ry)]
        dist = [((mx - x)**2 + (my - y)**2)**0.5 for (x, y) in bound]
        return max(dist)

    def _place_spk(self, center, room):
        num_rirs = self.args.num_rirs
        done, ntry = 0, 0
        mx, my = center
        rx, ry, rz = room.size
        max_retry = self.args.retry * num_rirs
        stats = []
        min_src_dist, max_src_dist = self.args.src_dist
        max_src_dist = min(max_src_dist, self._max_src_dist((mx, my), (rx, ry)))
        Rf = lambda f: round(f, 3)  # noqa: E731
        while True:
            ntry += 1
            if ntry > max_retry:
                break
            sz = random.uniform(*self.args.speaker_height)
            if sz >= rz:
                continue
            dst = random.uniform(min_src_dist, max_src_dist)
            if self.geometry == "2d":
                # sample from 0-360
                doa = random.uniform(0, np.pi * 2)
            else:
                # sample from 0-180
                doa = random.uniform(0, np.pi)
            if not self.vertical:
                sx = mx + np.cos(doa) * dst
                sy = my + np.sin(doa) * dst
            else:
                sx = my - np.cos(doa) * dst
                sy = mx + np.sin(doa) * dst
            if 0 >= sx or sx >= rx or 0 >= sy or sy >= ry:
                continue
            done += 1
            stats.append({"pos": (Rf(sx), Rf(sy), Rf(sz)), "doa": Rf(doa * 180 / np.pi), "dst": Rf(dst)})
            if done == num_rirs:
                break
        logger.info(f"Put speaker point: try/done = {ntry}/{done}")
        return done == num_rirs, stats

    def run_for_instance(self, room_id):
        room = None
        while not room:
            room = self.room_generator.generate(v=self.args.speed)
        rpos, room = self._place_mic(room)
        succ, scfg = self._place_spk(rpos, room)
        if succ:
            rcfg = room.conf()
            for idx, cfg in enumerate(scfg):
                cfg["loc"] = f"{self.args.dump_dir}/Room{room_id}-{idx + 1}.wav"
                self.jobs.append((cfg["loc"], room.problem(cfg["pos"], self.args.speed)))
            rcfg["spk"] = scfg
            self.rirs_cfg.append(rcfg)
        return succ

    def simulate(self):
        """every (room, source) pair on the GPU, in batches of equal receiver counts"""
        L = int(self.sr * self.args.rir_dur)
        groups = {}
        for job in self.jobs:
            groups.setdefault(len(job[1][3]), []).append(job)
        for M, jobs in groups.items():
            step = max(1, BATCH_BYTES // (4 * M * max(L, 1)))
            for i in range(0, len(jobs), step):
                batch = jobs[i:i + step]
                room, beta, src, rcv = (np.array([job[1][k] for job in batch], dtype=np.float64) for k in range(4))
                rirs = plan.rir_image(room, beta, src, rcv, L, sr=self.sr, c=self.args.speed,
                                      device=self.device).cpu().numpy()
                for (fname, _), rir in zip(batch, rirs):
                    write_wav(fname, rir, sr=self.sr)

    def run(self):
        num_rooms = self.args.num_rooms
        max_retry = self.args.retry * num_rooms
        done, ntry = 0, 0
        while True:
            ntry += 1
            if ntry > max_retry:
                break
            succ = self.run_for_instance(done + 1)
            if succ:
                done += 1
            if done == num_rooms:
                break
        self.simulate()
        with open(Path(self.args.dump_dir) / "rir.json", "w") as f:
            json.dump(self.rirs_cfg, f, indent=2)
        logger.info(f"Generate {self.args.num_rirs * num_rooms:d} rirs, " +
                    f"{done:d} rooms done, try = {ntry}")


def _parser(geometry):
    linear = geometry == "1d"
    parser = argparse.ArgumentParser(
        description="Command to generate single/multi-channel RIRs "
        "(image method on the GPU). "
        "In this command, we will simulate several rirs for each room, which is "
        "configured using --num-rirs",
        formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("num_rooms", type=int, help="Total number of rooms to simulate")
    parser.add_argument("--num-rirs", type=int, default=40, help="Number of rirs to simulate for each room")
    parser.add_argument("--dump-cfg", type=strtobool, default=True,
                        help="If true, dump rir configures out in json format")
    parser.add_argument("--rir-dur", type=float, default=0.5, help="Duration of the simulated rir (s)")
    parser.add_argument("--sr", type=int, default=16000, help="Sample rate of simulated signal")
    parser.add_argument("--dump-dir", type=str, default="rir", help="Directory to dump generated rirs")
    parser.add_argument("--room-dim", type=str, default="7,10;7,10;3,4",
                        help="Constraint for room length/width/height, separated by semicolon")
    if linear:
        parser.add_argument("--vertical-oriented", type=strtobool, dest="vertical", default=False,
                            help="Orientation to place microphone array (vertical or horizontal)")
    parser.add_argument("--array-height", type=str2tuple, default=(1, 2), help="Range of array's height")
    parser.add_argument("--array-relx", type=str2tuple, default=(0.4, 0.6),
                        help="Area of room to place microphone array randomly"
                        "(relative values to room's length)")
    parser.add_argument("--array-rely", type=str2tuple, default=(0.05, 0.1) if linear else (0.4, 0.6),
                        help="Area of room to place microphone array randomly"
                        "(relative values to room's width)")
    parser.add_argument("--speaker-height", type=str2tuple, default=(1.6, 2), help="Range of speaker's height")
    if linear:
        parser.add_argument("--array-topo", type=str2tuple, default=(0, 0.1, 0.2, 0.3),
                            help="Linear topology for microphone arrays.")
    else:
        parser.add_argument("--array-topo", type=str, default="0,0.05;0.05,0;0,-0.05;-0.05,0",
                            help="Topology of the 2D microphone arrays.")
    parser.add_argument("--absorption-coefficient-range", type=str2tuple, dest="abs_range", default=(0.2, 0.8),
                        help="Range of absorption coefficient of the room material. Absorption coefficient "
                        "is located between 0 and 1, if a material offers no reflection, the absorption "
                        "coefficient is close to 1.")
    parser.add_argument("--rt60", type=str, default="0.2,0.7",
                        help="Range of RT60, this option has higher priority than "
                        "--absorption-coefficient-range")
    parser.add_argument("--sound-speed", type=float, dest="speed", default=340 if linear else 343,
                        help="Speed of sound")
    parser.add_argument("--retry", type=int, default=5,
                        help="Max number of times tried to generate rirs for a specific room (retry * num_rirs)")
    parser.add_argument("--source-distance", type=str2tuple, dest="src_dist", default=(1.5, 3) if linear else (1, 3),
                        help="Range of distance between microphone arrays and speakers")
    parser.add_argument("--gpu", type=strtobool, default=False,
                        help="Accepted for compatibility; every path runs on the GPU")
    return parser


def main(geometry, argv=None):
    """rir_generate_1d.py (geometry "1d") or rir_generate_2d.py ("2d") with the command line argv"""
    RirSimulator(geometry, _parser(geometry).parse_args(argv)).run()

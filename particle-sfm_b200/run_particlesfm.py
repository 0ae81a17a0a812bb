"""ParticleSfM's --assume_static pipeline as one command on the GPU, from the frames to the converted poses
(DESIGN.md §4.15).

    python -m particlesfm_b200.run_particlesfm --model raft-things.pth --assume_static
        (-i IMAGES -o OUT | --workspace_dir WS [--image_folder images] | --root_dir ROOT [--image_folder images])
        [--sample_ratio 2] [--traj_min_len 3] [--flow_check_thres 1.0] [--skip_path_consistency] [--skip_sfm]
        [--skip_exists] [--keep_intermediate]

Reference: run_particlesfm.py:99-178, its flags, defaults and three input modes.  The stages are those of
optical_flow, point_trajectory and sfm, joined in one process so that nothing passes through a file:

    flows + trajectories  the RAFT stage's batches go straight into one resident tracker on the same stream; a frame
                          advances as soon as its pairs are computed (FrameFeed), so the device holds one batch's
                          maps plus the few a later frame still needs, whatever the clip length
    track.npy             written from the device (psfm_tracker_track_npy) with --skip_sfm or --keep_intermediate
    sfm                   the finished tracker's track set goes into the database match table on the device
                          (psfm_tracker_matches), then verification, the global mapper and the conversion as in sfm

Deliberate differences from the reference:
  * Intermediates are not written unless asked for (OUT/optical_flows with --keep_intermediate, OUT/trajectories/
    track.npy with --skip_sfm or --keep_intermediate), and nothing is ever deleted: an intermediate an earlier run
    left stays where it is.
  * --traj_min_len reaches the tracker; the reference parses it and never passes it on.  The default, 3, is the
    reference's behaviour.
  * With --skip_exists an existing OUT/trajectories/track.npy skips the flows as well as the tracking.
  * --root_dir runs the sequences in child processes, one per visible GPU at a time.
  * Motion segmentation is not built: --assume_static is required.  Only --sfm_type global_theia is built.
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

from . import _lib, optical_flow, point_trajectory, sfm, tracker

PROG = "run_particlesfm"


# ----------------------------------------------------------------------------- the file plan

class Plan:
    """What a run does in OUT.  route: "fused" (frames -> flows -> track set on the device), "flow_dir" (the missing
    pairs of an existing OUT/optical_flows filled in, then the track set from that directory) or "track_npy" (an
    existing OUT/trajectories/track.npy, no flow and no tracking).  write_flows / write_track: whether files are
    written under OUT/optical_flows and to OUT/trajectories/track.npy; sfm: whether the SfM step runs."""

    def __init__(self, route, write_flows, write_track, sfm):
        self.route, self.write_flows, self.write_track, self.sfm = route, write_flows, write_track, sfm

    def stages(self):
        flows = {"fused": ["flows_trajectories"], "flow_dir": ["flows", "trajectories"], "track_npy": []}[self.route]
        return flows + (["sfm"] if self.sfm else [])


def workspace_paths(output_dir):
    """(flow directory, trajectory directory, track.npy) of a workspace, as the reference names them."""
    traj = os.path.join(output_dir, "trajectories")
    return os.path.join(output_dir, "optical_flows"), traj, os.path.join(traj, "track.npy")


def plan(output_dir, skip_sfm=False, skip_exists=False, keep_intermediate=False):
    flow_dir, _, track = workspace_paths(output_dir)
    if skip_exists and os.path.isfile(track):
        route = "track_npy"
    elif skip_exists and os.path.isdir(flow_dir):
        route = "flow_dir"
    else:
        route = "fused"
    return Plan(route, write_flows=route == "flow_dir" or (route == "fused" and keep_intermediate),
                write_track=route != "track_npy" and (skip_sfm or keep_intermediate), sfm=not skip_sfm)


# ----------------------------------------------------------------------------- flows -> tracker, frame by frame

class FrameFeed:
    """A sink for optical_flow._run (sink(batch, flows, images)) that advances a tracker as frames become ready.
    Frame t needs pair (t, 1) forward and backward, and with path consistency pair (t-1, 2) and the forward map of
    pair (t-1, 1) as well; optical_flow._pairs lists the pairs so that frames become ready in order.  After each batch
    every ready frame is advanced (advance(t, flow_f, flow_b, flow_prev, flow_f2, flow_b2)), and the maps a later
    frame still needs are copied out of the batch (keep) so that the batch can be freed: the maps held never exceed
    one batch's 2 n plus 3 (a frame's pending stride-2 pair and its predecessor's forward map)."""

    def __init__(self, num_frames, path_consistency, advance, keep=None):
        self.num_flows = num_frames - 1
        self.pc = path_consistency
        self.advance = advance
        self.keep = keep or (lambda m: m.clone())
        self.maps = {}                  # (t, stride) -> (forward, backward), pairs not consumed yet
        self.prev = None                # forward map of pair (next - 1, 1), with path consistency
        self.next = 0                   # the next frame to advance

    def _ready(self, t):
        return (t, 1) in self.maps and (not self.pc or t == 0 or (t - 1, 2) in self.maps)

    def held(self):
        """The maps this sink references between batches."""
        return 2 * len(self.maps) + (self.prev is not None)

    def __call__(self, batch, flows, images=None):
        n = len(batch)
        for j, p in enumerate(batch):
            self.maps[p] = (flows[j], flows[n + j])
        prev_pair = None
        while self.next < self.num_flows and self._ready(self.next):
            t = self.next
            f, b = self.maps.pop((t, 1))
            f2, b2 = self.maps.pop((t - 1, 2)) if self.pc and t >= 1 else (None, None)
            self.advance(t, f, b, self.prev, f2, b2)
            if self.pc:
                self.prev, prev_pair = f, (t, 1)
            self.next += 1
        here = set(batch)
        for p in [p for p in self.maps if p in here]:
            self.maps[p] = tuple(self.keep(m) for m in self.maps[p])
        if prev_pair in here:
            self.prev = self.keep(self.prev)

    def done(self):
        if self.next != self.num_flows or self.maps:
            raise RuntimeError("flows of %d of %d frames arrived; %d pairs left unused"
                               % (self.next, self.num_flows, len(self.maps)))
        self.prev = None


def raft_flow_source(state_dict):
    """The RAFT stage as a flow source: source(paths, h, w, pairs, sink) runs optical_flow._run."""
    def source(paths, h, w, pairs, sink):
        optical_flow._run(paths, h, w, state_dict, pairs, sink)
    return source


def array_flow_source(flows, pairs_per_batch=4):
    """A flow source of given maps: flows {(t, stride): (forward, backward)}, [h][w][2] float32 host arrays, handed
    to the sink in batches as optical_flow._run hands them (the maps uploaded, the flow images made on the device)."""
    def source(paths, h, w, pairs, sink):
        import torch
        for b0 in range(0, len(pairs), pairs_per_batch):
            batch = pairs[b0:b0 + pairs_per_batch]
            host = np.stack([flows[p][0] for p in batch] + [flows[p][1] for p in batch]).astype(np.float32, copy=False)
            maps = torch.from_numpy(host).cuda()
            sink(batch, maps, optical_flow.flow_to_image(maps[:len(batch)]))
    return source


# ----------------------------------------------------------------------------- one sequence

class RunReport:
    """stages: [(name, seconds)] in run order; plan: the Plan; sfm: main_global_sfm's MapperReport (None without
    the SfM step); success: False when the SfM step wrote no model."""

    def __init__(self, plan):
        self.plan, self.stages, self.sfm = plan, [], None

    @property
    def success(self):
        return self.sfm is None or self.sfm.success

    def add(self, name, t0):
        self.stages.append((name, time.perf_counter() - t0))

    def seconds(self, name):
        return sum(s for n, s in self.stages if n == name)


def check_inputs(image_dir, model=None, flow_source=None, with_sfm=True):
    """Everything a run reads, checked before anything is written or the device is touched -> (frame paths, h, w,
    flow source).  ValueError naming the directory or file: a missing image directory, frames optical_flow.frame_list
    refuses, weights optical_flow.load_weights refuses (when no flow source is given), and with the SfM step an image
    set that sfm.read_image_set refuses or that is not exactly the frames the flow step reads."""
    if not os.path.isdir(image_dir):
        raise ValueError("%s: the input image directory is not found" % image_dir)
    paths, h, w = optical_flow.frame_list(image_dir)
    if flow_source is None:
        if model is None:
            raise ValueError("--model: the RAFT weights file is required")
        flow_source = raft_flow_source(optical_flow.load_weights(model))
    if with_sfm:
        names = sfm.read_image_set(image_dir).names
        frames = [os.path.basename(p) for p in paths]
        if names != frames:
            odd = sorted(set(names) ^ set(frames)) or [a for a, b in zip(names, frames) if a != b]
            raise ValueError("%s: the flow step reads %d .png/.jpg frames and the SfM importer %d images; %s is read by "
                             "only one of them (frame ids and image ids would pair different images)"
                             % (image_dir, len(frames), len(names), os.path.join(image_dir, odd[0])))
    return paths, h, w, flow_source


def _fused(report, paths, h, w, source, output_dir, pc, sample_ratio, flow_check_thres, traj_min_len):
    """flows -> finished resident tracker, with the flow files and track.npy as the plan says."""
    flow_dir, traj_dir, npy = workspace_paths(output_dir)
    t0 = time.perf_counter()
    trk = tracker._ResidentTracker(h, w, sample_ratio, len(paths), path_consistency=pc)
    try:
        feed = FrameFeed(len(paths), pc, lambda t, f, b, prev, f2, b2: trk.advance(t, f, b, prev, f2, b2, flow_check_thres))
        pairs = optical_flow._pairs(len(paths), pc)
        if report.plan.write_flows:
            optical_flow.make_flow_dirs(flow_dir, pc)
            with optical_flow.FlowWriter(optical_flow.flow_files(paths, flow_dir)) as writer:

                def sink(batch, flows, images):
                    writer(batch, flows, images)
                    feed(batch, flows, images)
                source(paths, h, w, pairs, sink)
        else:
            source(paths, h, w, pairs, feed)
        feed.done()
        trk.finish(traj_min_len, result=False)         # returns once the set is assembled on the device
        report.add("flows_trajectories", t0)
        if report.plan.write_track:
            t0 = time.perf_counter()
            os.makedirs(traj_dir, exist_ok=True)
            with trk.track_npy_body() as body:
                point_trajectory.write_track_npy(npy, body.view())
            report.add("track_npy", t0)
        return trk
    except BaseException:
        trk.close()
        raise


def _from_flow_dir(report, paths, h, w, source, output_dir, pc, sample_ratio, flow_check_thres, traj_min_len):
    """--skip_exists with an existing OUT/optical_flows: its missing pairs written, then the track set from it."""
    flow_dir, traj_dir, npy = workspace_paths(output_dir)
    t0 = time.perf_counter()
    optical_flow.make_flow_dirs(flow_dir, pc)
    missing = optical_flow.missing_pairs(paths, flow_dir, pc)
    if missing:
        with optical_flow.FlowWriter(optical_flow.flow_files(paths, flow_dir)) as writer:
            source(paths, h, w, missing, writer)
    report.add("flows", t0)
    t0 = time.perf_counter()
    if report.plan.write_track:
        os.makedirs(traj_dir, exist_ok=True)
    arrays = point_trajectory.connect_point_trajectories(flow_dir, sample_ratio, flow_check_thres, traj_min_len, not pc,
                                                         npy if report.plan.write_track else None)
    report.add("trajectories", t0)
    return arrays


def particlesfm(image_dir, output_dir, model=None, flow_source=None, sample_ratio=2, flow_check_thres=1.0,
                traj_min_len=3, skip_path_consistency=False, skip_sfm=False, skip_exists=False, keep_intermediate=False,
                quiet=False):
    """run_particlesfm.py's particlesfm(args, image_dir, output_dir, ...) with --assume_static and --sfm_type
    global_theia, for one sequence.  flow_source(paths, h, w, pairs, sink) computes the flows of `pairs` and hands
    them to sink(batch, flows, images) in batches as optical_flow._run does; None: the RAFT stage with the weights
    `model`.  Returns a RunReport (its success False when the SfM step wrote no model).  Raises ValueError before
    anything is written or the device is touched (check_inputs), PsfmError without a device."""
    say = (lambda *a: None) if quiet else print
    p = plan(output_dir, skip_sfm, skip_exists, keep_intermediate)
    report = RunReport(p)
    pc = not skip_path_consistency
    paths, h, w, source = check_inputs(image_dir, model, flow_source, p.sfm)
    if not p.stages():
        return report
    optical_flow._require_device()
    os.makedirs(output_dir, exist_ok=True)
    _, traj_dir, _ = workspace_paths(output_dir)
    trajectories = traj_dir
    if p.route != "track_npy":
        # the reference's messages (run_particlesfm.py:32-40), "ParticleSFM" in the first as it prints it
        say("[ParticleSFM] Running pairwise optical flow inference......")
        if pc:
            say("[ParticleSfM] Running pairwise optical flow inference (stride 2)......")
        say("[ParticleSfM] Connecting (optimization {0}) point trajectories from optical flows......."
            .format("enabled" if pc else "disabled"))
        run = _fused if p.route == "fused" else _from_flow_dir
        trajectories = run(report, paths, h, w, source, output_dir, pc, sample_ratio, flow_check_thres, traj_min_len)
    try:
        if p.sfm:
            say("[ParticleSfM] Running global structure-from-motion with Theia........")
            t0 = time.perf_counter()
            report.sfm = sfm.main_global_sfm(os.path.join(output_dir, "sfm"), image_dir, trajectories, remove_dynamic=False,
                                             convert_path=os.path.join(output_dir, "colmap_outputs_converted"))
            report.add("sfm", t0)
    finally:
        if isinstance(trajectories, tracker._ResidentTracker):
            trajectories.close()
    return report


def print_report(report, out=print):
    for name, s in report.stages:
        out("%s: %-22s %9.1f ms" % (PROG, name, 1e3 * s))
    if report.sfm is not None:
        for name, s, _ in report.sfm.stages:
            out("%s: %-22s %9.1f ms" % (PROG, "sfm/" + name, 1e3 * s))


# ----------------------------------------------------------------------------- --root_dir

def visible_devices():
    """The devices this process may use, as CUDA_VISIBLE_DEVICES entries: its own list when set, else 0 .. n-1."""
    env = os.environ.get("CUDA_VISIBLE_DEVICES")
    if env is not None:
        return [d.strip() for d in env.split(",") if d.strip()]
    from . import device_count
    return [str(i) for i in range(max(0, device_count()))]


def schedule(names, devices, spawn, report, poll=0.05):
    """Run spawn(name, device) -> subprocess.Popen for every name, at most one running child per device, in order.
    report(name, device, returncode, seconds) is called as each child ends.  Returns {name: returncode}.  On any
    exception (a KeyboardInterrupt included) every running child is terminated and reaped before it propagates."""
    pending, free, running, codes = list(names), list(devices), {}, {}
    try:
        while pending or running:
            while pending and free:
                name, dev = pending.pop(0), free.pop(0)
                running[spawn(name, dev)] = (name, dev, time.perf_counter())
            for proc in list(running):
                rc = proc.poll()
                if rc is not None:
                    name, dev, t0 = running.pop(proc)
                    free.append(dev)
                    codes[name] = rc
                    report(name, dev, rc, time.perf_counter() - t0)
            if running:
                time.sleep(poll)
    except BaseException:
        for proc in running:
            proc.terminate()
        for proc in running:
            try:
                proc.wait(timeout=10)
            except subprocess.TimeoutExpired:
                proc.kill()
                proc.wait()
        raise
    return codes


def child_args(args, workspace_dir):
    """The command line of one --root_dir sequence: the parent's flags with --workspace_dir instead of --root_dir."""
    argv = ["--model", args.model, "--workspace_dir", workspace_dir, "--image_folder", args.image_folder,
            "--flow_check_thres", repr(args.flow_check_thres), "--sample_ratio", str(args.sample_ratio),
            "--traj_min_len", str(args.traj_min_len), "--window_size", str(args.window_size),
            "--traj_max_num", str(args.traj_max_num), "--sfm_type", args.sfm_type]
    for flag in ("skip_path_consistency", "assume_static", "skip_sfm", "skip_exists", "keep_intermediate"):
        if getattr(args, flag):
            argv.append("--" + flag)
    return argv


def root_sequences(root_dir, image_folder):
    """The sequences of --root_dir (sorted entries, as the reference lists them); ValueError naming the first entry
    without an image folder."""
    if not os.path.isdir(root_dir):
        raise ValueError("%s: the input folder is not found" % root_dir)
    names = sorted(os.listdir(root_dir))
    for n in names:
        if not os.path.isdir(os.path.join(root_dir, n, image_folder)):
            raise ValueError("%s: no image folder %r" % (os.path.join(root_dir, n), image_folder))
    return names


def run_root(args, devices=None, command=None, out=print):
    """--root_dir: every sequence in a child process of `command` (default: this command) with its own
    --workspace_dir, on one device of `devices` (default visible_devices()) at a time.  -> 0, or 1 when a sequence
    failed."""
    names = root_sequences(args.root_dir, args.image_folder)
    devices = visible_devices() if devices is None else list(devices)
    command = command or [sys.executable, "-m", "particlesfm_b200.run_particlesfm"]
    out("A total of {0} sequences found in {1}.".format(len(names), args.root_dir))

    def spawn(name, dev):
        env = dict(os.environ)
        if dev is not None:
            env["CUDA_VISIBLE_DEVICES"] = str(dev)
        return subprocess.Popen(command + child_args(args, os.path.join(args.root_dir, name)), env=env)

    def report(name, dev, rc, seconds):
        out("%s: %s: %s on device %s in %.1f s" % (PROG, name, "done" if rc == 0 else "failed with status %d" % rc,
                                                   dev, seconds))

    codes = schedule(names, devices or [None], spawn, report)
    failed = [n for n in names if codes[n] != 0]
    out("%s: %d of %d sequences done%s" % (PROG, len(names) - len(failed), len(names),
                                            "; failed: " + " ".join(failed) if failed else ""))
    return 1 if failed else 0


# ----------------------------------------------------------------------------- command line

def build_parser():
    p = argparse.ArgumentParser(PROG, description="Dense point trajectory based colmap reconstruction for videos, on "
                                                  "the GPU (--assume_static)")
    p.add_argument("--model", required=True, help="the RAFT weights file (raft-things.pth), as optical_flow takes it")
    # point trajectory
    p.add_argument("--flow_check_thres", type=float, default=1.0, help="the forward-backward flow consistency check threshold")
    p.add_argument("--sample_ratio", type=int, default=2, help="the sampling ratio for point trajectories")
    p.add_argument("--traj_min_len", type=int, default=3,
                   help="the minimum length for point trajectories; passed to the tracker (the reference parses it "
                        "and never passes it on, so its runs use the default, 3)")
    # motion segmentation: accepted and unused, as under --assume_static
    p.add_argument("--window_size", type=int, default=10, help="unused (motion segmentation is not built)")
    p.add_argument("--traj_max_num", type=int, default=100000, help="unused (motion segmentation is not built)")
    # sfm
    p.add_argument("--sfm_type", default="global_theia", help="sfm type; only global_theia is built")
    # pipeline control
    p.add_argument("--skip_path_consistency", action="store_true", help="whether to skip the path consistency optimization or not")
    p.add_argument("--assume_static", action="store_true", help="skip the motion segmentation (required)")
    p.add_argument("--skip_sfm", action="store_true", help="whether to skip structure-from-motion or not")
    p.add_argument("--skip_exists", action="store_true",
                   help="reuse OUT/trajectories/track.npy (no flows, no tracking), else fill in OUT/optical_flows")
    p.add_argument("--keep_intermediate", action="store_true",
                   help="write OUT/optical_flows and OUT/trajectories/track.npy (nothing is ever deleted)")
    # input modes
    p.add_argument("-i", "--image_dir", type=str, default="none", help="path to the sequence folder containing images")
    p.add_argument("-o", "--output_dir", type=str, default="none", help="workspace for output")
    p.add_argument("--workspace_dir", type=str, default="none", help="input workspace")
    p.add_argument("--image_folder", type=str, default="images", help="image folder")
    p.add_argument("--root_dir", type=str, default="none", help="path to the folder containing workspaces")
    return p


def refusal(args):
    """The message for flags this command does not run, or None."""
    if not args.assume_static:
        return ("--assume_static is required: motion segmentation (MiDaS and the trajectory network) is not built; "
                "run with --assume_static")
    if args.sfm_type != "global_theia":
        return "--sfm_type %s is not supported (only global_theia)" % args.sfm_type
    if not (args.image_dir != "none" and args.output_dir != "none") and args.workspace_dir == "none" \
            and args.root_dir == "none":
        return "no input: give -i/--image_dir with -o/--output_dir, --workspace_dir, or --root_dir"
    return None


def main(argv=None):
    args = build_parser().parse_args(sys.argv[1:] if argv is None else list(argv))
    why = refusal(args)
    if why:
        print("%s: %s" % (PROG, why), file=sys.stderr)
        return 2
    if args.image_dir != "none" and args.output_dir != "none":
        image_dir, output_dir = args.image_dir, args.output_dir
    elif args.workspace_dir != "none":
        image_dir, output_dir = os.path.join(args.workspace_dir, args.image_folder), args.workspace_dir
    else:
        try:
            return run_root(args)
        except ValueError as e:
            print("%s: %s" % (PROG, e), file=sys.stderr)
            return 2
    try:
        report = particlesfm(image_dir, output_dir, args.model, None, args.sample_ratio, args.flow_check_thres,
                             args.traj_min_len, args.skip_path_consistency, args.skip_sfm, args.skip_exists,
                             args.keep_intermediate)
    except ValueError as e:
        print("%s: %s" % (PROG, e), file=sys.stderr)
        return 2
    except (_lib.PsfmError, RuntimeError, OSError) as e:
        print("%s: %s" % (PROG, e), file=sys.stderr)
        return 1
    print_report(report)
    if not report.success:
        rep = report.sfm
        print("sfm: Could not reconstruct any model! (the %s stage failed: %s)" % (rep.failed_stage, rep.reason),
              file=sys.stderr)
        try:
            from . import convert
            convert.find_model(os.path.join(output_dir, "sfm"))
        except FileNotFoundError as e:
            print("sfm: %s" % e, file=sys.stderr)
        return 1
    if report.sfm is not None:
        print(report.sfm.stats)
    return 0


if __name__ == "__main__":
    sys.exit(main())

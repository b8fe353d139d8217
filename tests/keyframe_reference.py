"""NumPy restatement of Frontend::doWeNeedANewKeyframe (okvis_frontend/src/Frontend.cpp:295-369) and of the three
OpenCV routines it calls, in the arithmetic the device reproduces (okb_keyframe_overlap_batch):

  convex_hull      cv::convexHull(points, hull) on float points, clockwise = false: the points sorted by (x, y); Sklansky's
                   scan over the four quarter chains between the extreme points; coordinate differences in float, the
                   convexity test (ay*bx - ax*by) in double, a turn kept only when its sign is the chain's; duplicates
                   collapse, collinear points are not vertices, an all-equal set gives 1 vertex, an all-collinear set 2;
                   finally the cyclic shift that makes the vertex indices an ascending or descending run where one exists.
                   The sort breaks ties between equal points by index (std::sort leaves them in an unspecified order;
                   only the index of a duplicated vertex can depend on it).
  contour_area     cv::contourArea: |0.5 * sum (prev.x*q.y - prev.y*q.x)| in double, prev starting at the last vertex.
  point_polygon    cv::pointPolygonTest(contour, p, false) on a float contour: +1 inside, -1 outside, 0 on the boundary;
                   differences in float, the crossing test (dy*ex - dx*ey) in double.
  camera_overlap   one `im` of the reference's loop; keyframe_decision the maxima (std::max, NaN quirks included) and the
                   thresholds compared in double.

Products of two floats are exact in double, so a fused multiply-add on the device gives these results bit for bit.

extreme_filter is the device's Akl-Toussaint pre-filter: it drops the points that lie inside the octagon of the eight
extreme points by more than a margin far above float rounding; convex_hull(..., prefilter=True) runs the scan on the
survivors only and must give the same hull (tests/test_keyframe_reference.py checks it on every set)."""
import numpy as np

F32 = np.float32


def _sign(v):
    return int(v > 0) - int(v < 0)


def _sklansky(xs, ys, start, end, nsign, sign2):
    """Sklansky_ (OpenCV convhull.cpp) over sorted float coordinates; returns the stack (positions in the sorted list)."""
    incr = 1 if end > start else -1
    pprev, pcur, pnext = start, start + incr, start + 2 * incr
    if start == end or (xs[start] == xs[end] and ys[start] == ys[end]):
        return [start]
    stack = [pprev, pcur, pnext]
    end += incr
    while pnext != end:
        cury, nexty = ys[pcur], ys[pnext]
        by = F32(nexty - cury)
        if _sign(by) != nsign:
            ax = F32(xs[pcur] - xs[pprev])
            bx = F32(xs[pnext] - xs[pcur])
            ay = F32(cury - ys[pprev])
            convexity = float(ay) * float(bx) - float(ax) * float(by)
            if _sign(convexity) == sign2 and (ax != 0 or ay != 0):
                pprev, pcur = pcur, pnext
                pnext += incr
                stack.append(pnext)
            else:
                if pprev == start:
                    pcur = pnext
                    stack[1] = pcur
                    pnext += incr
                    stack[2] = pnext
                else:
                    stack[-2] = pnext
                    pcur = pprev
                    pprev = stack[-4]
                    stack.pop()
        else:
            pnext += incr
            stack[-1] = pnext
    return stack[:-1]


def extreme_filter(pts):
    """Mask of the points the device keeps: all but those inside the octagon of the extremes in x, y, x+y and x-y by
    more than 2^-12 of the bounding box's larger side (measured along each edge's normal, in the inf-norm of the edge)."""
    p = np.asarray(pts, np.float32).astype(np.float64)
    n = len(p)
    keep = np.ones(n, bool)
    if n < 4:
        return keep
    x, y = p[:, 0], p[:, 1]
    dirs = [x, x + y, y, y - x, -x, -x - y, -y, x - y]        # counter-clockwise (y up)
    V = np.array([p[int(np.argmax(d))] for d in dirs])         # first index of the maximum
    D = max(x.max() - x.min(), y.max() - y.min())
    inside = np.ones(n, bool)
    edges = 0
    for i in range(8):
        a, b = V[i], V[(i + 1) % 8]
        ex, ey = b[0] - a[0], b[1] - a[1]
        if ex == 0 and ey == 0:
            continue
        edges += 1
        cr = ex * (y - a[1]) - ey * (x - a[0])
        inside &= cr > 2.0 ** -12 * D * max(abs(ex), abs(ey))
    if edges == 0:
        return keep
    return ~inside


def convex_hull(pts, prefilter=False):
    """cv::convexHull(points, hull, false, true): returns the indices (into pts) of the hull vertices in cv2's order."""
    p = np.asarray(pts, np.float32).reshape(-1, 2) + F32(0.0)     # -0 compares equal to +0
    total = len(p)
    if total == 0:
        return np.zeros(0, np.int64)
    idx = np.arange(total)
    if prefilter:
        idx = idx[extreme_filter(p)]
    order = idx[np.lexsort((idx, p[idx, 1], p[idx, 0]))]        # by x, then y, then index
    xs = [F32(v) for v in p[order, 0]]
    ys = [F32(v) for v in p[order, 1]]
    m = len(order)
    miny = maxy = 0
    for i in range(1, m):
        if ys[miny] > ys[i]:
            miny = i
        if ys[maxy] < ys[i]:
            maxy = i
    hull = []
    if xs[0] == xs[m - 1] and ys[0] == ys[m - 1]:
        hull = [0]
    else:
        tl = _sklansky(xs, ys, 0, maxy, -1, 1)
        tr = _sklansky(xs, ys, m - 1, maxy, -1, -1)
        tl, tr = tr, tl                                          # clockwise = false
        hull += tl[:len(tl) - 1]
        hull += [tr[i] for i in range(len(tr) - 1, 0, -1)]
        stop = tr[1] if len(tr) > 2 else (tl[len(tl) - 2] if len(tl) > 2 else -1)
        bl = _sklansky(xs, ys, 0, miny, 1, -1)
        br = _sklansky(xs, ys, m - 1, miny, 1, 1)
        if stop >= 0:
            check = bl[1] if len(bl) > 2 else (br[2 - len(bl)] if len(bl) + len(br) > 2 else -1)
            if check == stop or (check >= 0 and xs[check] == xs[stop] and ys[check] == ys[stop]):
                bl, br = bl[:2], br[:2]                          # all points on one line
        hull += bl[:len(bl) - 1]
        hull += [br[i] for i in range(len(br) - 1, 0, -1)]
    hb = [int(order[h]) for h in hull]                          # original indices
    hb = _cyclic_shift(hb)
    return np.array(hb, np.int64)


def _cyclic_shift(hb):
    """The last step of cv::convexHull: rotate the index sequence so that it ascends or descends, where it can."""
    nout = len(hb)
    if nout < 3:
        return hb
    min_idx = max_idx = lt = 0
    for i in range(1, nout):
        v = hb[i]
        lt += hb[i - 1] < v
        if 1 < lt <= i - 2:
            break
        if v < hb[min_idx]:
            min_idx = i
        if v > hb[max_idx]:
            max_idx = i
    mmdist = abs(max_idx - min_idx)
    if (mmdist == 1 or mmdist == nout - 1) and (lt <= 1 or lt >= nout - 2):
        ascending = (max_idx + 1) % nout == min_idx
        i0 = min_idx if ascending else max_idx
        j = i0
        if i0 > 0:
            tmp = []
            i = 0
            while i < nout:
                cur = hb[j]
                tmp.append(cur)
                nj = j + 1 if j + 1 < nout else 0
                if i < nout - 1 and (ascending != (cur < hb[nj])):
                    break
                j = nj
                i += 1
            if i == nout:
                return tmp
    return hb


def contour_area(contour):
    """cv::contourArea(contour, false) on float points."""
    c = np.asarray(contour, np.float32).reshape(-1, 2)
    if len(c) == 0:
        return 0.0
    a = 0.0
    px, py = float(c[-1, 0]), float(c[-1, 1])
    for qx, qy in c.tolist():
        a += px * qy - py * qx
        px, py = qx, qy
    return abs(a * 0.5)


def point_polygon(contour, pts):
    """cv::pointPolygonTest(contour, p, false) for every p: int8 array of +1 / 0 / -1."""
    c = np.asarray(contour, np.float32).reshape(-1, 2)
    p = np.asarray(pts, np.float32).reshape(-1, 2)
    n = len(p)
    if len(c) == 0:
        return -np.ones(n, np.int8)
    px, py = p[:, 0], p[:, 1]
    zero = np.zeros(n, bool)
    counter = np.zeros(n, np.int64)
    vx, vy = c[-1, 0], c[-1, 1]
    for k in range(len(c)):
        v0x, v0y = vx, vy
        vx, vy = c[k, 0], c[k, 1]
        skip = ((v0y <= py) & (vy <= py)) | ((v0y > py) & (vy > py)) | ((v0x < px) & (vx < px))
        onb = skip & (py == vy) & ((px == vx) | ((py == v0y) & (((v0x <= px) & (px <= vx)) | ((vx <= px) & (px <= v0x)))))
        live = ~zero
        zero |= live & onb
        test = live & ~skip
        dist = (py - v0y).astype(np.float64) * np.float64(vx - v0x) - (px - v0x).astype(np.float64) * np.float64(vy - v0y)
        zero |= test & (dist == 0)
        if vy < v0y:
            dist = -dist
        counter += (test & (dist > 0) & ~zero).astype(np.int64)
    res = np.where(counter % 2 == 0, -1, 1).astype(np.int8)
    res[zero] = 0
    return res


def camera_overlap(kp, matched):
    """One camera of doWeNeedANewKeyframe.  kp: [n][2] keypoints (cast to float), matched: [n] bool (landmarkId != 0).
    Returns the values okb_keyframe_cam holds; a skipped camera has only its counts set."""
    kp = np.asarray(kp, np.float64).reshape(-1, 2).astype(np.float32)
    matched = np.asarray(matched, bool)
    n, nm = len(kp), int(matched.sum())
    r = dict(n_points=n, n_matched=nm, hull_all=0, hull_matched=0, inside=0, skipped=1, area_all=0.0, area_matched=0.0,
             overlap=0.0, ratio=0.0)
    if n < 3 or nm < 3:
        return r
    mk = kp[matched]
    ha, hm = convex_hull(kp), convex_hull(mk)
    aa, am = contour_area(kp[ha]), contour_area(mk[hm])
    inside = int((point_polygon(mk[hm], kp) > 0).sum()) if len(hm) > 2 else 0
    with np.errstate(divide="ignore", invalid="ignore"):
        overlap = float(np.float64(am) / np.float64(aa))
        ratio = float(np.float64(nm) / np.float64(inside))
    r.update(hull_all=len(ha), hull_matched=len(hm), inside=inside, skipped=0, area_all=aa, area_matched=am,
             overlap=overlap, ratio=ratio)
    return r


def std_max(a, b):
    """std::max(a, b) = (a < b) ? b : a."""
    return b if a < b else a


def keyframe_decision(cams, overlap_threshold=0.6, matching_ratio_threshold=0.2):
    """The maxima over cameras and the decision; the thresholds are floats (as keyframeInsertion*Threshold_) compared
    in double.  Returns (need_keyframe, overlap, ratio)."""
    overlap = ratio = 0.0
    for c in cams:
        if c["skipped"]:
            continue
        overlap = std_max(c["overlap"], overlap)
        ratio = std_max(c["ratio"], ratio)
    thr_o, thr_r = float(np.float32(overlap_threshold)), float(np.float32(matching_ratio_threshold))
    need = not (overlap > thr_o and ratio > thr_r)
    return need, overlap, ratio

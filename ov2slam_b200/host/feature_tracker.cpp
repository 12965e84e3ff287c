// FeatureTracker on the GPU: host shim over the C ABI (include/ov2b200.h).
// Behaviour mirrored: /root/reference/src/feature_tracker.cpp:35-137 (fbKltTracking), :216-221
// (inBorder).  No OpenCV calls on the hot path; no CPU fallback: a CUDA failure leaves every
// keypoint marked lost (status false) and prints the ABI error once, it never silently tracks on
// the CPU.
#include "feature_tracker.hpp"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/ov2b200.h"
#include "pyr_cache.hpp"

struct FeatureTracker::ThreadState {
    ov2_ctx* ctx = nullptr;
    // prev-left, cur-left, right + one spare: every image is uploaded (and its levels built) once, however many
    // fbKltTracking calls read it (pyr_cache.hpp)
    ov2shim::PyrCache<4> cache;
    ~ThreadState() {
        cache.clear();
        if (ctx) ov2_destroy(ctx);
    }
};

namespace {
std::mutex g_mu;
std::unordered_map<std::thread::id, FeatureTracker::ThreadState*>* g_states = nullptr;
int env_device() {
    // the reference's class takes no device: OV2_DEVICE names the GPU (default 0)
    const char* e = getenv("OV2_DEVICE");
    return e ? atoi(e) : 0;
}
}  // namespace

FeatureTracker::FeatureTracker(int nmax_iter, float fmax_px_precision, cv::Ptr<cv::CLAHE> pclahe)
    : klt_convg_crit_(cv::TermCriteria::COUNT + cv::TermCriteria::EPS, nmax_iter, fmax_px_precision), pclahe_(pclahe) {}

FeatureTracker::~FeatureTracker() {}

FeatureTracker::ThreadState* FeatureTracker::state() const {
    std::lock_guard<std::mutex> lk(g_mu);
    if (!g_states) g_states = new std::unordered_map<std::thread::id, ThreadState*>();
    auto it = g_states->find(std::this_thread::get_id());
    if (it != g_states->end()) return it->second;
    ThreadState* s = new ThreadState();
    if (ov2_create(env_device(), &s->ctx) != OV2_OK) {
        fprintf(stderr, "[ov2b200] FeatureTracker: no CUDA device - the GPU front-end has no CPU fallback\n");
        s->ctx = nullptr;
    }
    (*g_states)[std::this_thread::get_id()] = s;
    return s;
}

void FeatureTracker::fbKltTracking(const std::vector<cv::Mat> &vprevpyr, const std::vector<cv::Mat> &vcurpyr, int nwinsize,
        int nbpyrlvl, float ferr, float fmax_fbklt_dist, std::vector<cv::Point2f> &vkps,
        std::vector<cv::Point2f> &vpriorkps, std::vector<bool> &vkpstatus) const
{
    if (vkps.empty()) return;                               // feature_tracker.cpp:43-46
    const size_t nbkps = vkps.size();
    vkpstatus.reserve(vkpstatus.size() + nbkps);
    // the pyramid vector interleaves image / derivative Mats (2 per level); the 8-bit level 0 is all
    // the device path needs - the lower levels and the Scharr planes are recomputed on the GPU
    if ((int)vprevpyr.size() < 2 * (nbpyrlvl + 1)) nbpyrlvl = (int)vprevpyr.size() / 2 - 1;   // :50-52
    if (nbpyrlvl < 0) nbpyrlvl = 0;
    ThreadState* s = state();
    auto fail_all = [&]() { for (size_t i = 0; i < nbkps; ++i) vkpstatus.push_back(false); };
    if (!s->ctx || vprevpyr.empty() || vcurpyr.empty()) { fail_all(); return; }
    const cv::Mat& p0 = vprevpyr[0];
    const cv::Mat& c0 = vcurpyr[0];
    const int nlev_extra = (int)vprevpyr.size() / 2 - 1;
    ov2_pyr* dprev = s->cache.get(s->ctx, p0, nlev_extra);
    ov2_pyr* dcur = dprev ? s->cache.get(s->ctx, c0, nlev_extra) : nullptr;
    if (!dprev || !dcur) {
        fprintf(stderr, "[ov2b200] fbKltTracking: %s\n", ov2_last_error(s->ctx));
        fail_all();
        return;
    }
    ov2_klt_params prm;
    prm.win = nwinsize;
    prm.max_iter = klt_convg_crit_.maxCount;
    prm.eps = (float)klt_convg_crit_.epsilon;
    prm.ferr = ferr;
    prm.fb_dist = fmax_fbklt_dist;
    std::vector<uint8_t> status(nbkps, 0);
    static_assert(sizeof(cv::Point2f) == 2 * sizeof(float), "Point2f layout");
    ov2_status st = ov2_fb_klt(s->ctx, dprev, dcur, &prm, (int)nbkps, nullptr, 0, (int)nbkps, nullptr, nbpyrlvl,
                               reinterpret_cast<const float*>(vkps.data()), reinterpret_cast<float*>(vpriorkps.data()),
                               status.data());
    if (st != OV2_OK) {
        fprintf(stderr, "[ov2b200] fbKltTracking: %s\n", ov2_last_error(s->ctx));
        fail_all();
        return;
    }
    for (size_t i = 0; i < nbkps; ++i) vkpstatus.push_back(status[i] != 0);
}

// ---------------------------------------------------------------------------------------------------------------
// cv::getRectSubPix for 8-bit source and destination as OpenCV's own template evaluates it (imgproc/samplers.cpp,
// getRectSubPix_Cn_<uchar, uchar, int, scale_fixpt, cast_8u>): bilinear weights in 16-bit fixed point
// (cvRound(w * 65536)), result (sum + 2^15) >> 16, window centred on `center`, pixels outside the image replicated from
// the border.  (OpenCV builds WITH Intel IPP route this call to ippiCopySubpix, which differs from the template by one
// grey level on ~0.7 % of the pixels: the reference's result depends on how its OpenCV was built; the template is what
// distribution / ROS builds run.)
namespace {
inline int cv_round(float v) { return (int)lrintf(v); }
void get_rect_subpix_u8(const cv::Mat& src, int ww, int wh, float cx, float cy, std::vector<unsigned char>& dst) {
    dst.resize((size_t)ww * wh);
    cx -= (ww - 1) * 0.5f;
    cy -= (wh - 1) * 0.5f;
    const int ipx = (int)floorf(cx), ipy = (int)floorf(cy);
    const float a = cx - ipx, b = cy - ipy;
    const int a11 = cv_round((1.f - a) * (1.f - b) * 65536.f), a12 = cv_round(a * (1.f - b) * 65536.f);
    const int a21 = cv_round((1.f - a) * b * 65536.f), a22 = cv_round(a * b * 65536.f);
    auto px = [&](int x, int y) -> int {
        x = x < 0 ? 0 : (x >= src.cols ? src.cols - 1 : x);
        y = y < 0 ? 0 : (y >= src.rows ? src.rows - 1 : y);
        return src.ptr(y)[x];
    };
    for (int i = 0; i < wh; ++i)
        for (int j = 0; j < ww; ++j) {
            const int x = ipx + j, y = ipy + i;
            const int v = px(x, y) * a11 + px(x + 1, y) * a12 + px(x, y + 1) * a21 + px(x + 1, y + 1) * a22;
            dst[(size_t)i * ww + j] = (unsigned char)((v + (1 << 15)) >> 16);
        }
}
}  // namespace

// FeatureTracker::getLineMinSAD (/root/reference/src/feature_tracker.cpp:138-204), statement by statement: the window
// shrink near the borders (including its float-to-int arithmetic), the sub-pixel patch / target sampling, the scan from
// x downwards (bgoleft) or upwards in unit steps - so ties resolve to the same column - and the mean absolute
// difference in float.  Host code: it is the stereo prior of the `bdo_stereo_rect` configurations, one short line
// search per keypoint (SURVEY.md 8f-3).
void FeatureTracker::getLineMinSAD(const cv::Mat &iml, const cv::Mat &imr, const cv::Point2f &pt, const int nwinsize,
        float &xprior, float &l1err, bool bgoleft) const
{
    xprior = -1;
    if (nwinsize % 2 == 0) {
        fprintf(stderr, "\ngetLineMinSAD requires an odd window size\n");
        return;
    }
    const float x = pt.x;
    const float y = pt.y;
    int halfwin = nwinsize / 2;
    // (the reference's compound assignments convert int + float back to int by truncation)
    if (x - halfwin < 0) halfwin = (int)(halfwin + (x - halfwin));
    if (x + halfwin >= imr.cols) halfwin = (int)(halfwin + (x + halfwin - imr.cols - 1));
    if (y - halfwin < 0) halfwin = (int)(halfwin + (y - halfwin));
    if (y + halfwin >= imr.rows) halfwin = (int)(halfwin + (y + halfwin - imr.rows - 1));
    if (halfwin <= 0) return;
    const int ws = 2 * halfwin + 1;
    const int nbwinpx = ws * ws;
    float minsad = 255.f;
    std::vector<unsigned char> patch, target;
    get_rect_subpix_u8(iml, ws, ws, pt.x, pt.y, patch);
    auto sad_at = [&](float c) {
        get_rect_subpix_u8(imr, ws, ws, c, y, target);
        long s = 0;
        for (size_t k = 0; k < patch.size(); ++k) s += std::abs((int)patch[k] - (int)target[k]);
        float e = (float)(double)s;          // l1err = cv::norm(patch, target, NORM_L1)  (double -> float)
        e /= nbwinpx;
        return e;
    };
    if (bgoleft) {
        for (float c = x; c >= halfwin; c -= 1.f) {
            l1err = sad_at(c);
            if (l1err < minsad) { minsad = l1err; xprior = c; }
        }
    } else {
        for (float c = x; c < imr.cols - halfwin; c += 1.f) {
            l1err = sad_at(c);
            if (l1err < minsad) { minsad = l1err; xprior = c; }
        }
    }
    l1err = minsad;
}

// The same search for every point of a keyframe in ONE device call (csrc/frontend_sad.cu: one warp per point, identical
// arithmetic), on the cached device pyramids of the two images.
bool FeatureTracker::getLineMinSADBatch(const std::vector<cv::Mat> &vleftpyr, const std::vector<cv::Mat> &vrightpyr, int pyrlvl,
        const std::vector<cv::Point2f> &vpts, const int nwinsize, bool bgoleft, std::vector<float> &vxprior, std::vector<float> &vl1err) const
{
    vxprior.assign(vpts.size(), -1.f);
    vl1err.assign(vpts.size(), 255.f);
    if (vpts.empty()) return true;
    ThreadState* s = state();
    if (!s->ctx || vleftpyr.empty() || vrightpyr.empty()) return false;
    const int nlev_extra = (int)vleftpyr.size() / 2 - 1;
    if (pyrlvl < 0 || pyrlvl > nlev_extra || vrightpyr.size() != vleftpyr.size()) {
        fprintf(stderr, "[ov2b200] getLineMinSADBatch: pyramid level %d not in the pyramids\n", pyrlvl);
        return false;
    }
    ov2_pyr* dl = s->cache.get(s->ctx, vleftpyr[0], nlev_extra);
    ov2_pyr* dr = dl ? s->cache.get(s->ctx, vrightpyr[0], nlev_extra) : nullptr;
    ov2_status st = (dl && dr) ? OV2_OK : OV2_ERR_CUDA;
    if (st == OV2_OK)
        st = ov2_line_min_sad(s->ctx, dl, dr, pyrlvl, (int)vpts.size(), nullptr, 0, (int)vpts.size(),
                              reinterpret_cast<const float*>(vpts.data()), nwinsize, bgoleft ? 1 : 0, vxprior.data(), vl1err.data());
    if (st != OV2_OK) {
        fprintf(stderr, "[ov2b200] getLineMinSADBatch: %s\n", ov2_last_error(s->ctx));
        vxprior.assign(vpts.size(), -1.f);
        vl1err.assign(vpts.size(), 255.f);
        return false;
    }
    return true;
}

bool FeatureTracker::inBorder(const cv::Point2f &pt, const cv::Mat &im) const
{
    const float BORDER_SIZE = 1.f;
    return BORDER_SIZE <= pt.x && pt.x < im.cols - BORDER_SIZE && BORDER_SIZE <= pt.y && pt.y < im.rows - BORDER_SIZE;
}

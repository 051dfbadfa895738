/* TEST INFRASTRUCTURE ONLY -- the CPU oracle's orientation stage alone, on caller-given keypoints.
 *
 * oracle/sift_oracle.c keeps its orientation stage (orientation_one, a restatement of the reference's ori_par) static.
 * This file includes that translation unit unchanged and adds one entry point around it, so that the describe path's
 * PS_DESCRIBE_ORIENT results can be compared with the oracle on keypoints that did not come from its extrema stage.
 * Built by tests/orient_oracle.py with the oracle's own compiler flags (oracle/Makefile). */
#include "../oracle/sift_oracle.c"

/* num_ori_out[i] and ori4_out[4 i .. 4 i + 3] (unused angles 0) of n keypoints: kp3 = n x {x, y, sigma} (octave-local),
 * oct_lpos = n x {octave, lpos}, on the pyramid of a previous orc_run_* of ctx (a context of libsift_oracle.so, built
 * from the same source).  Returns -1 if an octave is out of range (that keypoint gets num_ori 0). */
int orc_orient(const orc_ctx* c, int n, const float* kp3, const int32_t* oct_lpos, int32_t* num_ori_out, float* ori4_out)
{
    int bad = 0;
    #pragma omp parallel for schedule(dynamic, 16) reduction(+:bad)
    for (int i = 0; i < n; i++) {
        iext_t ie;
        ext_t e;
        memset(&e, 0, sizeof(e));
        ie.x = kp3[3 * i]; ie.y = kp3[3 * i + 1]; ie.sigma = kp3[3 * i + 2];
        ie.octave = oct_lpos[2 * i]; ie.lpos = oct_lpos[2 * i + 1];
        if (ie.octave >= 0 && ie.octave < c->noct) orientation_one(c, &ie, &e);
        else bad++;
        num_ori_out[i] = e.num_ori;
        for (int k = 0; k < 4; k++) ori4_out[4 * i + k] = k < e.num_ori ? e.ori[k] : 0.0f;
    }
    return bad ? -1 : 0;
}

/* Plain-C use of the Player controls on a streaming session (include/rodio_b200.h): the block form of
 *     let player = rodio::Player::connect_new(&mixer);                 // src/player.rs:73-170
 *     player.append(intro.low_pass(2000));   player.append(song);      // a queue: the song starts where the intro ends
 *     player.set_volume(0.5);  ...  player.pause();  ...  player.play();
 * rodio wraps every appended sound in  speed -> pausable -> amplify(volume) -> ...  and lets the mixer convert the result
 * (src/player.rs:120-128), so the user's filter and the Player's volume sit IN FRONT of the conversion to the mixer's format.
 * Here: two slots of one session, declared held; the second follows the first (rb_session_follow); set_volume changes the
 * AMPLIFY in front of the conversion for every frame pulled from then on (rb_session_set_volume); while paused the shim pushes
 * silence behind the source's chain (rb_session_push_silence), like Pausable (src/source/pausable.rs:85-97): a fade or take at
 * the front of the chain stands still meanwhile.
 * Build:  gcc -std=c11 -Iinclude examples/live_player.c -Lrodio_b200 -l:librodio_b200.so -Wl,-rpath,$PWD/rodio_b200 -lm -o live_player
 * (needs a CUDA device at run time: rb_context_create fails loudly without one). */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "rodio_b200.h"

#define CHECK(call)                                                                          \
    do {                                                                                     \
        rb_status s_ = (call);                                                               \
        if (s_ != RB_OK) {                                                                   \
            fprintf(stderr, "%s: %s (%s)\n", #call, rb_status_string(s_), rb_last_error()); \
            return 1;                                                                        \
        }                                                                                    \
    } while (0)

enum { INTRO_RATE = 22050, SONG_RATE = 44100, MIX_RATE = 48000 };

int main(void) {
    rb_context* ctx = NULL;
    CHECK(rb_context_create(0, &ctx));

    /* intro: 22.05 kHz mono  .low_pass(2000)  -> Player's amplify -> mixer;   song: 44.1 kHz mono -> Player's amplify -> mixer */
    rb_effect intro_fx[3], song_fx[2];
    memset(intro_fx, 0, sizeof intro_fx), memset(song_fx, 0, sizeof song_fx);
    intro_fx[0].kind = RB_FX_LOW_PASS, intro_fx[0].u32[0] = 2000, intro_fx[0].f32[0] = 0.5f;
    intro_fx[1].kind = RB_FX_AMPLIFY, intro_fx[1].f32[0] = 1.0f;                 /* Player::volume, 1.0 until set_volume */
    intro_fx[2].kind = RB_FX_UNIFORM, intro_fx[2].u32[0] = 1, intro_fx[2].u32[1] = MIX_RATE;
    song_fx[0].kind = RB_FX_AMPLIFY, song_fx[0].f32[0] = 1.0f;
    song_fx[1].kind = RB_FX_UNIFORM, song_fx[1].u32[0] = 1, song_fx[1].u32[1] = MIX_RATE;
    rb_stream_desc descs[2];
    memset(descs, 0, sizeof descs);
    descs[0].sample_rate = INTRO_RATE, descs[0].channels = 1, descs[0].format = RB_FMT_F32, descs[0].n_effects = 3, descs[0].effects = intro_fx;
    descs[1].sample_rate = SONG_RATE, descs[1].channels = 1, descs[1].format = RB_FMT_F32, descs[1].n_effects = 2, descs[1].effects = song_fx;
    descs[0].mix_start = 0;                  /* the first sound plays at once */
    descs[1].mix_start = RB_SESSION_HELD;    /* the second one is queued behind it */

    rb_session* player = NULL;
    CHECK(rb_session_create(ctx, 1, MIX_RATE, descs, 2, /* fifo_frames */ 8192, /* max_block_frames */ 480, &player));
    CHECK(rb_session_follow(player, 1, 0));  /* Player::append(song) */

    const int intro_blocks = 20, song_blocks = 30;   /* 10 ms each */
    float pcm[441], out[480];
    uint64_t total = 0, silent = 0;
    double peak_loud = 0.0, peak_quiet = 0.0;
    int ended = 0, sent_intro = 0, sent_song = 0;
    for (int tick = 0; !ended; tick++) {
        const int paused = tick >= 25 && tick < 30;              /* player.pause() ... player.play() */
        if (tick == 35) {                                        /* player.set_volume(0.25) */
            CHECK(rb_session_set_volume(player, 0, 0.25f));
            CHECK(rb_session_set_volume(player, 1, 0.25f));
        }
        if (sent_intro < intro_blocks) {                         /* the decoder of the sound that is playing delivers 10 ms */
            for (int i = 0; i < 220; i++) pcm[i] = (float)(0.6 * sin(2 * M_PI * 330.0 * (sent_intro * 220 + i) / INTRO_RATE));
            sent_intro++;
            CHECK(rb_session_push(player, 0, pcm, 220, sent_intro == intro_blocks));
        } else if (paused) {
            CHECK(rb_session_push_silence(player, 1, 441));       /* Pausable: frames of zeros, the source is not pulled */
        } else if (sent_song < song_blocks) {
            for (int i = 0; i < 441; i++) pcm[i] = (float)(0.6 * sin(2 * M_PI * 440.0 * (sent_song * 441 + i) / SONG_RATE));
            sent_song++;
            CHECK(rb_session_push(player, 1, pcm, 441, sent_song == song_blocks));
        }
        for (;;) {
            uint64_t n = 0;
            CHECK(rb_session_render(player, out, 480, &n, &ended));
            for (uint64_t i = 0; i < n; i++) {
                const double a = fabs(out[i]);
                if (a == 0.0) silent++;
                if (tick < 25 && a > peak_loud) peak_loud = a;
                if (tick >= 40 && a > peak_quiet) peak_quiet = a;
            }
            total += n;
            if (n == 0 || ended) break;
        }
    }
    /* 0.2 s intro + 0.05 s pause + 0.3 s song at 48 kHz; the pause is silent; the tail plays at a quarter of the volume */
    printf("%llu frames, %llu silent, peak %.3f then %.3f\n", (unsigned long long)total, (unsigned long long)silent, peak_loud, peak_quiet);
    rb_session_destroy(player);
    rb_context_destroy(ctx);
    return 0;
}
